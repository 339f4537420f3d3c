"""Full Correlation Matrix Analysis (FCMA) — correlation-based voxel selection on H100.

Drop-in for ``brainiak.fcma.voxelselector.VoxelSelector`` (reference voxelselector.py:56-516):
same constructor arguments, same ``run(clf)`` result (``list[(voxel_id, accuracy)]`` sorted by
accuracy, descending), same private stage methods.  The three native stages of
``_voxel_scoring`` (voxelselector.py:467-516) run as sm_90a CUDA through libfcma_b200.so:

    corr GEMM (TMA + wgmma)  ->  Fisher-z + within-subject z-score  ->  per-voxel E x E kernel

The cross validation runs on the GPU for ``SVC(kernel='precomputed')`` on the kernel matrices and for
``SVC(kernel='linear' | 'rbf')`` on the normalised correlation vectors, ``SVC()``'s ``gamma='scale'`` included (see
``gpu_cv``); any other classifier is
cross-validated on the host by scikit-learn, exactly as in the reference (voxelselector.py:41-53).  Distribution: instead of the MPI master/worker farm (voxelselector.py:176-282) every
rank of ``torch.distributed`` owns a contiguous slice of voxel rows (work per row is uniform); the
per-voxel scores are gathered on ``master_rank``.  Without ``torch.distributed`` it runs on one GPU.
"""
import logging
import math
import multiprocessing
import time

import numpy as np
import sklearn
import sklearn.svm
from sklearn import model_selection

from .. import _lib
from . import engine

logger = logging.getLogger(__name__)

__all__ = ["VoxelSelector"]


def usable_cpu_count():
    """Reference utils/utils.py:701-717."""
    import os
    try:
        return len(os.sched_getaffinity(0))
    except AttributeError:
        return os.cpu_count()


def _cross_validation_for_one_voxel(clf, vid, num_folds, subject_data, labels):
    """Score classifier on data using cross validation (reference voxelselector.py:41-53)."""
    skf = model_selection.StratifiedKFold(n_splits=num_folds, shuffle=False)
    scores = model_selection.cross_val_score(clf, subject_data, y=labels, cv=skf, n_jobs=1)
    return (vid, scores.mean())


def _cv_chunk(clf, vids, num_folds, kernels, labels):
    return [_cross_validation_for_one_voxel(clf, int(v), num_folds, kernels[k], labels)
            for k, v in enumerate(vids)]


def _is_precomputed_svc(clf):
    return isinstance(clf, sklearn.svm.SVC) and clf.kernel == 'precomputed'


def held_out_keep(E, epochs_per_subj, subject):
    """The epochs left when ``subject`` is held out: ``[0, E)`` without ``[subject * eps, (subject + 1) * eps)``, in the
    original order (the reference example's ``subsampled_idx``, fcma_voxel_selection_cv.py:69-75)."""
    s0 = subject * epochs_per_subj
    return np.concatenate([np.arange(0, s0), np.arange(s0 + epochs_per_subj, E)]).astype(np.int64)


class _Case:
    """One cross validation of a kernel build: ``run()``'s over every epoch (``keep`` None), or that of a run without one
    held-out subject (``keep``: the epochs left), with that run's labels and fold count."""

    def __init__(self, E, labels, num_folds, keep=None):
        self.keep, self.labels, self.num_folds = keep, labels, num_folds
        self.E = E if keep is None else len(keep)

    def take(self, x, axes):
        """The host array ``x`` restricted to the kept epochs along ``axes`` (``x`` itself for every epoch)."""
        if self.keep is None:
            return x
        for ax in axes:
            x = np.take(x, self.keep, axis=ax)
        return x


def shrink_kernels_(kernels):
    """In-place decimal shrink of every ``[E, E]`` kernel (reference voxelselector.py:409-412):
    ``nd = len(str(int(K[i, 0, 0]))); if nd > 2: K[i] *= 10**(2 - nd)``."""
    for i in range(kernels.shape[0]):
        num_digits = len(str(int(kernels[i, 0, 0])))
        if num_digits > 2:
            proportion = 10 ** (2 - num_digits)
            kernels[i, :, :] *= proportion
    return kernels


class VoxelSelector:
    """Correlation-based voxel selection component of FCMA (H100 engine).

    Parameters (positional part identical to the reference, voxelselector.py:102-110)
    ----------
    labels, epochs_per_subj, num_folds, raw_data, raw_data2, voxel_unit, process_num, master_rank:
        as in ``brainiak.fcma.voxelselector.VoxelSelector``.  ``raw_data`` is a list of
        float32 ``[epoch length, nVoxels]`` arrays, already z-scored (voxelselector.py:72-76)
        unless ``normalize=True``.  ``voxel_unit`` keeps its meaning for the per-task stage
        methods; ``run`` processes ``block_rows`` rows per GPU pass.

    Keyword-only extensions
    -----------------------
    precision: 'fp32' (default: fp32-faithful correlations, |dr| <= 1e-6, via the 3-product split
        'fp16x3' for normalised data or 'tf32x3' otherwise), or explicitly 'fp16x3', 'tf32x3',
        'bf16x3' (|dr| ~ 1e-5), 'tf32' (1e-3), 'bf16' (8e-3)
    mask_self: zero the self-correlation column (rounding noise in the reference, see DESIGN.md)
    normalize: apply the per-epoch z-score of preprocessing.py:80-84 on the GPU while packing
    device: CUDA device (default: current / LOCAL_RANK)
    block_rows: voxel rows per GPU pass (default: sized to free HBM)
    symmetric: with a single mask (``raw_data2 is None``) use ``corr[i, e, j] == corr[j, e, i]``: only the
        blocks on and above the diagonal are contracted and each is used for its row and its column voxels
        (engine.voxel_kernels_sym; half the tensor work, same kernels up to fp32 summation order).  Over
        several GPUs the shards' partial kernel arrays are summed with one NCCL reduce-scatter (every rank keeps the
        rows it cross-validates).
    gpu_cv: run the voxelwise cross validation on the GPU (batched restatement of libsvm's SMO, with or without its
        shrinking heuristic as ``clf.shrinking`` says, with the same iterations and decisions as scikit-learn; more than
        two conditions one-vs-one with libsvm's vote, see engine.svm_cv_precomputed) for
        ``SVC(kernel='precomputed')`` on the kernel matrices (at most 256 epochs and 64 folds), and for ``SVC(kernel='linear')`` or ``SVC(kernel='rbf')``
        with ``gamma='auto'`` or a number on the normalised correlation vectors themselves: their fp64 kernel matrices
        are built on the GPU (engine.feature_kernels_f64, above 64 epochs engine.feature_kernels_f64_wide, without the
        decimal shrink, as scikit-learn sees the features) and cross-validated by engine.svm_cv_f64 (at most 256 epochs
        and 64 folds, no class weights, probability or tie
        breaking, and ``mask_self=False``, see engine.svc_feature_kind).  scikit-learn's default ``SVC()`` (rbf with
        ``gamma='scale'``, whose gamma depends on each fold's training features) runs there too under the same limits
        (engine.svc_scale_supported): G and D of the features and their per-sample moments are built once
        (engine.feature_gram_wide), then every fold gets its own gamma and kernels (engine.svm_cv_scale); a voxel whose
        exact variance NumPy's may miss by more than a few ulps is scored on the host.  ``False`` or any other
        classifier -> scikit-learn on the host, exactly as the reference (voxelselector.py:41-53)
    """

    def __init__(self, labels, epochs_per_subj, num_folds, raw_data, raw_data2=None,
                 voxel_unit=64, process_num=4, master_rank=0, *, precision="fp32",
                 mask_self=False, normalize=False, device=None, block_rows=None, gpu_cv=True,
                 symmetric=True):
        self.labels = labels
        self.epochs_per_subj = epochs_per_subj
        self.num_folds = num_folds
        self.raw_data = raw_data
        self.num_voxels = raw_data[0].shape[1]
        self.raw_data2 = raw_data2
        self.num_voxels2 = raw_data2[0].shape[1] if raw_data2 is not None else self.num_voxels
        self.voxel_unit = voxel_unit
        usable_cpus = usable_cpu_count()
        if process_num is None:
            self.process_num = usable_cpus
        else:
            self.process_num = np.min((process_num, usable_cpus))
        self.use_multiprocessing = self.process_num != 0
        self.master_rank = master_rank
        if self.raw_data2 is not None and len(self.raw_data) != len(self.raw_data2):
            raise ValueError('The raw data lists must have the same number '
                             'of elements for computing the correlations '
                             'element by element')
        if self.num_voxels == 0 or self.num_voxels2 == 0:
            raise ValueError('Zero processed voxels')
        # NOTE: the reference refuses a single MPI process (voxelselector.py:137-139) because its
        # master does no compute; here every rank computes, so one process is fine.
        if precision not in _lib.PREC_NAMES or precision == "f32simt":
            raise ValueError("unknown precision %r" % (precision,))
        self.precision = precision
        self.mask_self = bool(mask_self)
        if self.mask_self and (raw_data2 is not None
                               or not engine.fused_supported(len(raw_data), int(epochs_per_subj))):
            # the self column only exists with one mask, and it is zeroed inside the fused normalise+kernel kernels
            # (E <= 64, power-of-two epochs_per_subj): refuse loudly instead of returning unmasked results
            raise ValueError('mask_self=True needs a single mask (raw_data2 is None), at most 64 epochs and a '
                             'power-of-two epochs_per_subj')
        self.normalize = bool(normalize)
        self.device = device
        self.block_rows = block_rows
        self.gpu_cv = bool(gpu_cv)
        self.symmetric = bool(symmetric)
        self._rows_op = None
        self._cols_op = None
        self._work = None
        world = self._world()
        if self.master_rank >= world[1]:
            logger.warning('Master rank exceeds the number of launched processes, set to 0')
            self.master_rank = 0

    # ------------------------------------------------------------------ distribution helpers
    @staticmethod
    def _world():
        """(rank, world_size) of torch.distributed, or (0, 1)."""
        try:
            import torch.distributed as dist
            if dist.is_available() and dist.is_initialized():
                return dist.get_rank(), dist.get_world_size()
        except Exception:  # pragma: no cover
            pass
        return 0, 1

    @staticmethod
    def row_partition(num_voxels, world_size):
        """Static shard: rank r owns rows [r*ceil(V/W), min(V, (r+1)*ceil(V/W)))."""
        per = int(math.ceil(num_voxels / float(world_size)))
        return [(min(num_voxels, r * per), max(0, min(num_voxels, (r + 1) * per) - min(num_voxels, r * per)))
                for r in range(world_size)]

    # ------------------------------------------------------------------ device state
    def _torch_device(self):
        import os
        import torch
        if self.device is not None:
            return torch.device(self.device)
        if torch.distributed.is_available() and torch.distributed.is_initialized() \
                and "LOCAL_RANK" in os.environ:
            return torch.device("cuda", int(os.environ["LOCAL_RANK"]))
        return torch.device("cuda", torch.cuda.current_device())

    def _operands(self):
        """Upload + pack the epochs once (K-major, precision-split; HBM resident)."""
        if self._rows_op is None:
            _lib.load()
            _lib.require_device()
            dev = self._torch_device()
            rank, world = self._world()
            sharded = False
            if world > 1:
                import torch.distributed as dist
                sharded = dist.get_backend() == "nccl" and len(self.raw_data) >= world
            # several GPUs: every rank uploads its share of the epochs, NVLink all-gather (engine.upload_epochs_sharded)
            upload = (lambda rd: engine.upload_epochs_sharded(rd, dev)) if sharded else \
                (lambda rd: engine.stack_epochs(rd, dev))
            ep, T_e = upload(self.raw_data)
            prec = engine.resolve_precision(self.precision, ep, self.normalize)
            ep2 = None
            if self.raw_data2 is not None:
                ep2, T_e2 = upload(self.raw_data2)
                if T_e2 != T_e:
                    raise ValueError("raw_data and raw_data2 must have the same epoch lengths")
                if engine.resolve_precision(self.precision, ep2, self.normalize) != prec:
                    prec = "tf32x3"          # one of the two masks is outside the fp16-safe range
            self._rows_op = engine.pack_epochs(ep, T_e, prec, self.normalize)
            self._cols_op = engine.pack_epochs(ep2, T_e, prec, self.normalize) if ep2 is not None \
                else self._rows_op
        return self._rows_op, self._cols_op

    def _flags(self, fused):
        # __init__ guarantees that mask_self implies one mask and the fused path
        return _lib.FLAG_MASK_SELF if (self.mask_self and self.raw_data2 is None and fused) else 0

    # ------------------------------------------------------------------ public API
    def run(self, clf):
        """Run correlation-based voxel selection.

        Returns (on ``master_rank``; ``[]`` elsewhere, as voxelselector.py:149-174) the list of
        ``(voxel_id, accuracy)`` of all voxels in accuracy-descending order (stable: ties keep
        voxel order, the reference's tie order depends on message arrival)."""
        rank, world = self._world()
        start, n = self.row_partition(self.num_voxels, world)[rank]
        time1 = time.time()
        local = self._score_rows(start, n, clf) if n > 0 else []
        logger.info('rank %d scored rows [%d, %d) in %.2f s', rank, start, start + n,
                    time.time() - time1)
        results = self._gather(local, rank, world)
        if rank == self.master_rank:
            results.sort(key=lambda tup: tup[1], reverse=True)
            return results
        return []

    def held_out_cases(self, subjects=None, num_folds=None):
        """The leave-one-subject-out runs of ``run_held_out``: one ``_Case`` per subject of ``subjects`` (default: every
        subject), with ``labels_s`` and ``num_folds`` (default: subjects - 1).  Raises ValueError before any device is
        touched when E is not a whole number of subjects, there are fewer than 3 subjects, or ``subjects`` holds an index
        outside [0, S) or a duplicate."""
        E, eps = len(self.raw_data), int(self.epochs_per_subj)
        if eps < 1 or E % eps:
            raise ValueError('leave-one-subject-out needs whole subjects: %d epochs are not a multiple of '
                             'epochs_per_subj = %d' % (E, eps))
        S = E // eps
        if S < 3:
            raise ValueError('leave-one-subject-out needs at least 3 subjects, not %d' % S)
        subjects = list(range(S)) if subjects is None else [int(x) for x in subjects]
        if any(x < 0 or x >= S for x in subjects) or len(set(subjects)) != len(subjects):
            raise ValueError('subjects must be distinct indices in [0, %d): %r' % (S, subjects))
        num_folds = S - 1 if num_folds is None else int(num_folds)
        cases = []
        for x in subjects:
            keep = held_out_keep(E, eps, x)
            cases.append(_Case(E, [self.labels[i] for i in keep], num_folds, keep))
        return subjects, cases

    def run_held_out(self, clf, subjects=None, num_folds=None):
        """Leave-one-subject-out voxel selection from one kernel build.

        The reference's FCMA example (fcma_voxel_selection_cv.py) runs the whole selection once per held-out subject s:
        ``VoxelSelector(labels_s, eps, num_folds, raw_s, raw2_s, ...).run(clf)``, ``_s`` meaning the epochs
        ``[s * eps, (s + 1) * eps)`` removed.  The correlations, their within-subject z-scores and every kernel entry of
        the other subjects do not depend on subject s, so here every row block's kernels are built once over all E epochs,
        by the code ``run()`` uses, and each held-out run compacts them to its E - eps epochs on the device
        (engine.subset_kernels, with the decimal shrink counted on the compacted K00) before the cross validation
        ``run()`` would do with ``labels_s`` and ``svm_folds_for(labels_s, num_folds, E - eps)``.  The host routes
        take the same block with subject s's epochs sliced out.

        ``subjects``: the held-out subjects (default: all ``S = E // epochs_per_subj``); ``num_folds``: the inner fold
        count (default ``S - 1``, the example's ``num_subjs - 1``).  Returns ``{s: [(voxel_id, accuracy), ...]}``, each
        list sorted as ``run()`` sorts, on ``master_rank`` and ``{}`` elsewhere; equal to the per-subject ``run()``
        lists.  The precision is resolved once over all E epochs (``_operands``): when a subset alone would resolve to
        another split mode, the kernels agree within the fp32-faithful tolerance instead of bit for bit."""
        subjects, cases = self.held_out_cases(subjects, num_folds)
        rank, world = self._world()
        start, n = self.row_partition(self.num_voxels, world)[rank]
        time1 = time.time()
        local = self._score_cases(start, n, clf, cases) if n > 0 else [[] for _ in cases]
        logger.info('rank %d scored rows [%d, %d) for %d held-out subjects in %.2f s', rank, start, start + n,
                    len(cases), time.time() - time1)
        results = self._gather_held_out(local, rank, world)
        if rank != self.master_rank:
            return {}
        out = {}
        for x, res in zip(subjects, results):
            res.sort(key=lambda tup: tup[1], reverse=True)
            out[x] = res
        return out

    def _gather_held_out(self, local, rank, world):
        """Every rank's per-case lists of rows -> the per-case lists over all voxels on master_rank ([] elsewhere): one
        all-gather of the ``[cases, rows]`` accuracy matrix (on the device with NCCL, on the host with gloo)."""
        if world == 1:
            return [list(part) for part in local]
        import torch
        import torch.distributed as dist
        dev = self._torch_device() if dist.get_backend() == "nccl" else torch.device("cpu")
        parts = self.row_partition(self.num_voxels, world)
        per = max(n for _, n in parts)
        mine = torch.full((len(local), per), float("nan"), dtype=torch.float64)
        for i, part in enumerate(local):
            if part:
                mine[i, :len(part)] = torch.tensor([a for _, a in part], dtype=torch.float64)
        mine = mine.to(dev)
        allv = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(allv, mine)
        if rank != self.master_rank:
            return [[] for _ in local]
        host = torch.stack(allv).cpu().numpy()          # [world, cases, per]
        return [[(int(s0 + k), host[r, i, k]) for r, (s0, n) in enumerate(parts) for k in range(n)]
                for i in range(len(local))]

    def _gather(self, local, rank, world):
        if world == 1:
            return list(local)
        import torch
        import torch.distributed as dist
        if dist.get_backend() == "nccl":
            # NCCL moves tensors, not pickles: all-gather the (padded) per-shard accuracy vectors over
            # NVLink on this rank's own device (voxel ids are implied by the static row partition)
            dev = self._torch_device()
            parts = self.row_partition(self.num_voxels, world)
            per = max(n for _, n in parts)
            mine = torch.full((per,), float("nan"), dtype=torch.float64, device=dev)
            if local:
                mine[:len(local)] = torch.tensor([a for _, a in local], dtype=torch.float64, device=dev)
            allv = torch.empty((world, per), dtype=torch.float64, device=dev)
            dist.all_gather_into_tensor(allv, mine)
            if rank != self.master_rank:
                return []
            host = allv.cpu().numpy()
            out = []
            for r, (s0, n) in enumerate(parts):
                out += [(int(s0 + k), host[r, k]) for k in range(n)]
            return out
        gathered = [None] * world if rank == self.master_rank else None
        dist.gather_object(list(local), gathered, dst=self.master_rank)
        if rank != self.master_rank:
            return []
        out = []
        for part in gathered:      # rank order == voxel order
            out += part
        return out

    # ------------------------------------------------------------------ the hot loop
    def _symmetric_ok(self):
        """Symmetric self-correlation pipeline: one mask, fused normalise+kernel path, at least one 256-row
        tile per shard; over several ranks the partial kernels are summed with NCCL."""
        import os
        if not self.symmetric or self.raw_data2 is not None or os.environ.get("FCMA_NO_SYM") == "1":
            return False
        rank, world = self._world()
        if world > 1:
            import torch.distributed as dist
            if dist.get_backend() != "nccl":
                return False
        E = len(self.raw_data)
        return engine.sym_supported(E, self.epochs_per_subj) and self.num_voxels >= 512 * world

    def _precomputed_folds(self, clf, cases, E):
        """Per case: the GPU fold problems of its cross validation of ``SVC(kernel='precomputed')``, or None for the host."""
        return [engine.svm_folds_for(c.labels, c.num_folds, c.E)
                if self.gpu_cv and engine.svm_cv_supported(clf, c.labels, c.num_folds, c.E,
                                                           max_epochs=engine.SVM_WIDE_MAX_EPOCHS) else None
                for c in cases]

    def _cv_block(self, K, s, nb, clf, cases, folds):
        """a7 tail + a8 for the unshrunk device kernels ``K`` of rows [s, s+nb), once per case (``folds``:
        ``_precomputed_folds``).  Every epoch: shrunk in place; a held-out subject: compacted and shrunk out of place, so
        ``K`` stays the block's unshrunk kernels for the next case."""
        t0 = time.time()
        out, host = [], None
        for c, f in zip(cases, folds):
            if f is not None:
                # shrink + cross validation without leaving the device (SURVEY §8f rank 1)
                if c.keep is None:
                    engine.shrink_kernels_(K)
                    Kc = K
                else:
                    Kc = engine.subset_kernels(K, c.keep, shrink=True)
                acc = engine.svm_cv_precomputed(Kc, c.labels, c.num_folds, C=clf.C, tol=clf.tol,
                                                max_iter=clf.max_iter, folds=f, shrinking=bool(clf.shrinking))
                del Kc
                out.append([(int(s + k), acc[k]) for k in range(nb)])
                continue
            if host is None:
                host = K.cpu().numpy()
            kernels = c.take(host, (1, 2))
            shrink_kernels_(kernels)
            out.append(self._do_cross_validation(clf, kernels, (s, nb), c.labels, c.num_folds))
        logger.debug('rows [%d, %d): cv of %d cases %.3f s', s, s + nb, len(cases), time.time() - t0)
        return out

    def _score_rows_symmetric(self, start, n, clf, cases):
        """Single-mask path: this rank contracts its shard of the upper block triangle
        (engine.sym_row_partition), the [V, E, E] partial kernels are summed over the ranks, then every
        rank cross-validates rows [start, start+n), once per case."""
        import torch
        rank, world = self._world()
        op, _ = self._operands()
        E, V = op.E, self.num_voxels
        s0, n0 = engine.sym_row_partition(V, world)[rank]
        per = self.row_partition(V, world)[0][1]
        # this rank's partial sums for ALL rows (rows left of its shard stay zero), padded to world * per rows so that
        # one reduce-scatter hands every rank the summed kernels of exactly the rows it cross-validates
        K = torch.zeros((world * per, E, E), dtype=torch.float32, device=op.device)
        if n0 > 0:
            rows = self.block_rows or None
            if rows is None:
                free, _ = torch.cuda.mem_get_info(op.device)
                per_row = 2 * _lib.load().fcma_work_bytes_per_row(E, V - s0)
                rows = min(free // 2, 64 << 30) // per_row
            rows = max(256, min((n0 + 255) // 256 * 256, rows // 256 * 256, 4096 if not self.block_rows else 1 << 30))
            flags = self._flags(True)
            need = 256 <= _lib.load().fcma_sym_rows_per_pass(_lib.PREC[op.precision], E, self.epochs_per_subj, flags, V, s0,
                                                             self._work.buf.numel() if self._work is not None else 0)
            if not isinstance(self._work, engine.SymWorkspace) or not need or self._work.rows < rows:
                self._work = None       # release the old scratch first
                self._work = engine.SymWorkspace.for_operand(op, rows, self.epochs_per_subj, flags, start=s0)
            engine.voxel_kernels_sym(op, s0, n0, self.epochs_per_subj, flags=self._flags(True),
                                     work=self._work, out=K[:V])
        if world > 1:
            import torch.distributed as dist
            mine = torch.empty((per, E, E), dtype=torch.float32, device=op.device)
            dist.reduce_scatter_tensor(mine, K)      # NVLink; every rank keeps the rows [rank * per, ...) it scores
            del K
            K, k0 = mine, start
        else:
            k0 = 0
        folds = self._precomputed_folds(clf, cases, E)
        results = [[] for _ in cases]
        block = 8192
        for s in range(start, start + n, block):
            nb = min(block, start + n - s)
            for res, part in zip(results, self._cv_block(K[s - k0:s - k0 + nb], s, nb, clf, cases, folds)):
                res += part
        return results

    def _plain_block(self, n, fp64_outputs=False, fp64_matrices=2):
        """Rows per pass of the plain (row-block) pipeline, with its scratch allocated for them.  ``fp64_outputs``: the
        pass also holds ``fp64_matrices`` fp64 [E, E] matrices per row (engine.feature_block_rows)."""
        import torch
        rows_op, _ = self._operands()
        E = rows_op.E
        if self.block_rows or not fp64_outputs:
            block = self.block_rows or engine.Workspace.rows_for(E, self.num_voxels2, n, rows_op.device)
        else:
            free, _ = torch.cuda.mem_get_info(rows_op.device)
            block = engine.feature_block_rows(E, _lib.load().fcma_work_bytes_per_row(E, self.num_voxels2), n,
                                              min(free // 2, 32 << 30), matrices=fp64_matrices)
        block = max(1, min(block, n))
        if self._work is None or self._work.rows < block or isinstance(self._work, engine.SymWorkspace):
            self._work = None
            self._work = engine.Workspace(E, self.num_voxels2, block, rows_op.device)
        return block

    def _all_epochs(self):
        """``run()``'s one case: every epoch, the instance's labels and fold count."""
        return [_Case(len(self.raw_data), self.labels, self.num_folds)]

    def _feature_kind(self, clf, max_epochs=64, cases=None):
        """'linear' / 'rbf' when ``clf`` on the normalised correlation vectors is cross-validated on the GPU (fp64 kernel
        matrices + the fp64 solver) at up to ``max_epochs`` epochs for every case (default: ``run()``'s), else None.
        mask_self is not applied to the features by the host path, so that combination stays there."""
        if not self.gpu_cv or self.mask_self:
            return None
        kinds = {engine.svc_feature_kind(clf, c.labels, c.num_folds, c.E, max_epochs=max_epochs)
                 for c in (cases or self._all_epochs())}
        return kinds.pop() if len(kinds) == 1 else None

    def _scale_ok(self, clf, cases=None):
        """True when ``SVC(kernel='rbf', gamma='scale')`` on the normalised correlation vectors is cross-validated on the
        GPU with per-fold gammas (engine.svm_cv_scale) for every case, under the conditions of ``_feature_kind``."""
        if not self.gpu_cv or self.mask_self:
            return False
        return all(engine.svc_scale_supported(clf, c.labels, c.num_folds, c.E) for c in (cases or self._all_epochs()))

    def _score_rows_scale(self, start, n, clf, cases):
        """SVC(kernel='rbf', gamma='scale') on the features of rows [start, start+n): G, D and the per-sample moments of
        every row (engine.feature_gram_wide), then per case (compacted to its epochs) and fold the gamma of its training
        samples, its rbf kernels and the fp64 solver (engine.svm_cv_scale).  The voxels whose gamma may differ from
        scikit-learn's are scored on the host."""
        import torch
        rows_op, cols_op = self._operands()
        folds = [engine.svm_folds_for(c.labels, c.num_folds, c.E) for c in cases]
        held_out = any(c.keep is not None for c in cases)
        # a held-out case also holds its compacted G and D
        block = self._plain_block(n, fp64_outputs=True, fp64_matrices=6 if held_out else 4)
        results = [[] for _ in cases]
        for s in range(start, start + n, block):
            nb = min(block, start + n - s)
            G, D, moments = engine.feature_gram_wide(rows_op, cols_op, s, nb, self.epochs_per_subj, work=self._work)
            for c, f, res in zip(cases, folds, results):
                if c.keep is None:
                    Gc, Dc, mc = G, D, moments
                else:
                    Gc, Dc = engine.subset_kernels(G, c.keep), engine.subset_kernels(D, c.keep)
                    mc = moments.index_select(1, torch.as_tensor(c.keep, device=moments.device))
                acc, flagged = engine.svm_cv_scale(Gc, Dc, mc, self.num_voxels2, c.labels, c.num_folds, C=clf.C,
                                                   tol=clf.tol, max_iter=clf.max_iter, shrinking=bool(clf.shrinking),
                                                   folds=f)
                del Gc, Dc, mc
                part = [(int(s + k), acc[k]) for k in range(nb)]
                for k in np.flatnonzero(flagged):
                    task = (int(s + k), 1)
                    part[k] = (self._voxel_scoring(task, clf) if c.keep is None
                               else self._host_scoring(task, clf, [c])[0])[0]
                if flagged.any():
                    logger.info('rows [%d, %d): %d voxels scored on the host (gamma=\'scale\' variance check)', s,
                                s + nb, int(flagged.sum()))
                res += part
            del G, D, moments
        return results

    def _score_rows(self, start, n, clf):
        """GPU stages for rows [start, start+n) in HBM-sized blocks, then the cross validation (GPU or host)."""
        return self._score_cases(start, n, clf, self._all_epochs())[0]

    def _score_cases(self, start, n, clf, cases):
        """``_score_rows`` for every case of ``cases`` from one kernel build: one list of ``(voxel_id, accuracy)`` per
        case.  The build and its route are ``run()``'s over all E epochs; each case then cross-validates its epochs."""
        rows_op, cols_op = self._operands()
        E = rows_op.E
        results = [[] for _ in cases]
        held_out = any(c.keep is not None for c in cases)
        if _is_precomputed_svc(clf) and self._symmetric_ok():
            return self._score_rows_symmetric(start, n, clf, cases)
        kind = None if _is_precomputed_svc(clf) else self._feature_kind(clf, engine.SVM_WIDE_MAX_EPOCHS, cases)
        if kind is not None:
            # SVC(kernel='linear' | 'rbf') on the features: the fp64 kernels of the features give libsvm's iterations and
            # decisions (DESIGN.md §3.8); gamma='auto' is scikit-learn's 1 / n_features
            gamma = None if kind == 'linear' else (1.0 / self.num_voxels2 if clf.gamma == 'auto' else float(clf.gamma))
            wide = E > 64
            folds = [engine.svm_folds_for(c.labels, c.num_folds, c.E) for c in cases]
            feature_kernels = engine.feature_kernels_f64_wide if wide else engine.feature_kernels_f64
            # a held-out case also holds its compacted K_fit and K_pred
            block = self._plain_block(n, fp64_outputs=wide, fp64_matrices=4 if held_out else 2)
            for s in range(start, start + n, block):
                nb = min(block, start + n - s)
                K_fit, K_pred = feature_kernels(rows_op, cols_op, s, nb, self.epochs_per_subj, kind, gamma,
                                                work=self._work)
                for c, f, res in zip(cases, folds, results):
                    if c.keep is None:
                        Kf, Kp = K_fit, K_pred
                    else:
                        Kf = engine.subset_kernels(K_fit, c.keep)
                        Kp = Kf if K_pred is K_fit else engine.subset_kernels(K_pred, c.keep)
                    acc = engine.svm_cv_f64(Kf, Kp, c.labels, c.num_folds, C=clf.C, tol=clf.tol,
                                            max_iter=clf.max_iter, shrinking=bool(clf.shrinking), folds=f)
                    del Kf, Kp
                    res += [(int(s + k), acc[k]) for k in range(nb)]
                del K_fit, K_pred
        elif _is_precomputed_svc(clf):
            fused = engine.fused_supported(E, self.epochs_per_subj)
            block = self._plain_block(n)
            folds = self._precomputed_folds(clf, cases, E)
            for s in range(start, start + n, block):
                nb = min(block, start + n - s)
                K = engine.voxel_kernels(rows_op, cols_op, s, nb, self.epochs_per_subj,
                                         flags=self._flags(fused), work=self._work)
                for res, part in zip(results, self._cv_block(K, s, nb, clf, cases, folds)):
                    res += part
        elif self._scale_ok(clf, cases):
            results = self._score_rows_scale(start, n, clf, cases)
        else:
            unit = max(1, min(self.voxel_unit, n))
            for s in range(start, start + n, unit):
                nb = min(unit, start + n - s)
                for res, part in zip(results, self._host_scoring((s, nb), clf, cases)):
                    res += part
        return results

    # ------------------------------------------------------------------ reference stage methods
    def _correlation_computation(self, task):
        """a4 (voxelselector.py:284-329): corr ``[n, E, V2]`` float32 numpy for ``task = (start, n)``."""
        rows_op, cols_op = self._operands()
        corr = engine.corr_block(rows_op, cols_op, task[0], task[1], layout=0)
        return corr.cpu().numpy()

    def _correlation_normalization(self, corr):
        """Within-subject normalisation on the GPU; returns the normalised array like the reference's scipy path
        (voxelselector.py:331-369).  The arithmetic is that of the C++ normaliser the reference's hot loop actually
        calls (fcma_extension.cc:52-84): it differs from the scipy path in two documented corner cases -- |r| >= 1 is
        clamped (cc:68-72) instead of producing inf -> nan_to_num, and when the epoch count is not a multiple of
        ``epochs_per_subj`` the trailing partial subject is left untouched (cc:52), where the scipy path z-scores it."""
        import torch
        _lib.load()
        _lib.require_device()
        c = np.ascontiguousarray(corr, dtype=np.float32)
        if c.ndim != 3:
            raise RuntimeError("The multi-subject correlation data structure must be 3D")
        t = torch.from_numpy(c).to(self._torch_device())
        engine.within_subject_norm_(t, self.epochs_per_subj)
        out = np.nan_to_num(t.cpu().numpy())
        if isinstance(corr, np.ndarray) and corr.dtype == np.float32 and corr.flags.c_contiguous:
            corr[...] = out          # the reference normalises in place as well
        return out

    def _prepare_for_cross_validation(self, corr, clf):
        """a7 (voxelselector.py:371-421): kernel matrices for SVC(kernel='precomputed'), else corr."""
        import torch
        if _is_precomputed_svc(clf):
            z = torch.from_numpy(np.ascontiguousarray(corr, dtype=np.float32)).to(self._torch_device())
            kernels = engine.kernel_matrices(z).cpu().numpy()
            return shrink_kernels_(kernels)
        return corr

    def _do_cross_validation(self, clf, data, task, labels=None, num_folds=None):
        """a8 (voxelselector.py:423-465): voxelwise cross validation on the host, with ``labels`` and ``num_folds``
        (default: the instance's)."""
        time1 = time.time()
        labels = self.labels if labels is None else labels
        num_folds = self.num_folds if num_folds is None else num_folds
        n = task[1]
        if _is_precomputed_svc(clf) and self.use_multiprocessing and n > 1:
            nproc = int(self.process_num)
            chunk = max(1, int(math.ceil(n / float(nproc * 4))))
            inlist = [(clf, np.arange(c, min(n, c + chunk)) + task[0], num_folds,
                       data[c:min(n, c + chunk)], labels) for c in range(0, n, chunk)]
            with multiprocessing.Pool(nproc) as pool:
                parts = pool.starmap(_cv_chunk, inlist)
            results = [r for part in parts for r in part]
        else:
            results = [_cross_validation_for_one_voxel(clf, i + task[0], num_folds,
                                                       data[i, :, :], labels)
                       for i in range(n)]
        logger.debug('cross validation for %d voxels, takes %.2f s', n, time.time() - time1)
        return results

    def _voxel_scoring(self, task, clf):
        """One task ``(start, n)`` through the 3-stage pipeline of voxelselector.py:467-516."""
        return self._host_scoring(task, clf, self._all_epochs())[0]

    def _host_scoring(self, task, clf, cases):
        """``_voxel_scoring`` once per case: the task's kernels (shrunk per case on its epochs) or normalised
        correlations are computed once over all epochs, then each case cross-validates its epochs on the host."""
        time1 = time.time()
        rows_op, cols_op = self._operands()
        precomputed = _is_precomputed_svc(clf)
        if precomputed:
            fused = engine.fused_supported(rows_op.E, self.epochs_per_subj)
            K = engine.voxel_kernels(rows_op, cols_op, task[0], task[1], self.epochs_per_subj,
                                     flags=self._flags(fused))
            data = K.cpu().numpy()
        else:
            corr = engine.corr_block(rows_op, cols_op, task[0], task[1], layout=0)
            corr = corr.contiguous()
            engine.within_subject_norm_(corr, self.epochs_per_subj)
            data = corr.cpu().numpy()
        results = []
        for c in cases:
            d = c.take(data, (1, 2) if precomputed else (1,))
            if precomputed:
                shrink_kernels_(d)
            results.append(self._do_cross_validation(clf, d, task, c.labels, c.num_folds))
        logger.info('task %d takes %.2f s', int(task[0] / self.voxel_unit), time.time() - time1)
        return results
