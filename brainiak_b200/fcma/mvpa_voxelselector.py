"""Activity-based voxel selection (searchlight MVPA) on H100.

Drop-in for ``brainiak.fcma.mvpa_voxelselector.MVPAVoxelSelector`` (reference mvpa_voxelselector.py:52-136): every
searchlight centre of the mask is scored by the mean ``StratifiedKFold(num_folds, shuffle=False)`` cross-validation
accuracy of ``clf`` on the centre's features (the voxels of its cube inside both the mask and the searchlight shape,
in C order), and ``run(clf)`` returns ``(result_volume, results)`` as the reference does.

For ``SVC(kernel='linear')`` and ``SVC(kernel='rbf')`` with ``gamma='auto'`` or a number, both stages run on the
GPU for up to 256 epochs: k_searchlight_kernels (k_searchlight_kernels_tiled above 32 epochs) builds each centre's fp64
kernel matrices and the batched libsvm SMO restatement cross-validates them in fp64 (engine.svm_cv_f64, on
``engine.svm_folds_for`` folds: its wide form above 64 epochs).  libsvm keeps Q in float but QD and the decision values
in double, so fp64 kernels give the same iterations and predictions as scikit-learn on the features (DESIGN.md).
scikit-learn's default ``SVC()`` (rbf with ``gamma='scale'``, a gamma per centre and fold) runs there as well:
engine.searchlight_gram_wide gives each centre's G, D and per-sample moments once, and engine.svm_cv_scale derives every
fold's gamma and kernels from them; a centre whose exact variance NumPy's may miss by more than a few ulps is scored on
the host.  Any other classifier (poly, sigmoid, other estimators), float64 data, more than 256 epochs, folds the
solver cannot express or ``gpu_cv=False`` run the reference's per-centre ``cross_val_score`` on the host.
"""
import logging

import numpy as np
from sklearn import model_selection

from .. import _lib
from . import engine

logger = logging.getLogger(__name__)

__all__ = ["MVPAVoxelSelector"]


def _world():
    """(rank, world_size) of torch.distributed, or (0, 1)."""
    try:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            return dist.get_rank(), dist.get_world_size()
    except Exception:  # pragma: no cover
        pass
    return 0, 1


def _host_accuracy(clf, features, labels, num_folds):
    """The reference's per-centre score (_sfn, mvpa_voxelselector.py:34-49); ``features`` is [E, n_features]."""
    skf = model_selection.StratifiedKFold(n_splits=num_folds, shuffle=False)
    return np.mean(model_selection.cross_val_score(clf, features, y=labels, cv=skf, n_jobs=1))


class MVPAVoxelSelector:
    """Activity-based voxel selection component of FCMA (H100 engine).

    Parameters (positional part identical to the reference)
    ----------
    data: 4-D array ``[X, Y, Z, epochs]``, the epoch-averaged, normalised brain data
        (``preprocessing.prepare_searchlight_mvpa_data``)
    mask: 3-D array, the brain mask
    labels: 1-D array of the epochs' labels
    num_folds: number of cross-validation folds
    sl: searchlight parameters (``brainiak_b200.searchlight.Searchlight`` or ``brainiak.searchlight.Searchlight``); only
        ``sl_rad``, ``shape`` (the boolean ``(2r+1)^3`` mask) and ``min_active_voxels_proportion`` are read

    Keyword-only extensions
    -----------------------
    device: CUDA device (default: the current one)
    gpu_cv: score eligible SVC classifiers on the GPU (default; up to 256 epochs); ``False`` -> the reference's host
        loop
    batch_centres: centres per GPU batch (default: sized to free device memory; a centre's kernel matrices take
        8 E^2 bytes, twice that for rbf, four times for ``gamma='scale'``: G, D and one fold's two kernels)
    """

    def __init__(self, data, mask, labels, num_folds, sl, *, device=None, gpu_cv=True, batch_centres=None):
        self.data = data
        self.mask = mask.astype(bool)
        self.labels = labels
        self.num_folds = num_folds
        self.sl = sl
        self.device = device
        self.gpu_cv = bool(gpu_cv)
        if batch_centres is not None and int(batch_centres) <= 0:
            raise ValueError("batch_centres must be positive")
        self.batch_centres = batch_centres
        num_voxels = np.sum(self.mask)
        if num_voxels == 0:
            raise ValueError('Zero processed voxels')

    # ------------------------------------------------------------------ routing
    def _gpu_kind(self, clf):
        """'linear' / 'rbf' / 'scale' (rbf with gamma='scale') if ``clf`` and the data can be scored on the GPU, else
        None."""
        if not self.gpu_cv:
            return None
        E = self.data.shape[3]
        kind = engine.svc_feature_kind(clf, self.labels, self.num_folds, E, max_epochs=engine.SVM_WIDE_MAX_EPOCHS)
        if kind is None and engine.svc_scale_supported(clf, self.labels, self.num_folds, E):
            kind = 'scale'
        if kind is not None and np.asarray(self.data).dtype != np.float32:
            logger.info('MVPAVoxelSelector: data is %s, not float32: scoring on the host', np.asarray(self.data).dtype)
            return None
        return kind

    def _check_inputs(self):
        data = np.asarray(self.data)
        if data.ndim != 4:
            raise ValueError('data must be a 4-D array [X, Y, Z, epochs]')
        if self.mask.ndim != 3 or data.shape[:3] != self.mask.shape:
            raise ValueError('mask shape %s does not match the data volume %s' % (self.mask.shape, data.shape[:3]))
        if len(self.labels) != data.shape[3]:
            raise ValueError('%d labels for %d epochs' % (len(self.labels), data.shape[3]))
        r = int(self.sl.sl_rad)
        if np.asarray(self.sl.shape).shape != (2 * r + 1,) * 3:
            raise ValueError('the searchlight shape must be (2*sl_rad+1)^3')

    # ------------------------------------------------------------------ public
    def run(self, clf):
        """Run activity-based voxel selection: score every searchlight centre with ``clf``.

        Returns
        -------
        result_volume: object array of ``mask.shape``: the accuracy at every computed centre, None elsewhere
        results: list of ``(index among the mask's voxels in C order, accuracy)`` (None -> 0), sorted by accuracy,
            descending (stable); ``[]`` on ranks other than 0 of torch.distributed, whose volume is all None
        """
        rank, _ = _world()
        result_volume = np.empty(self.mask.shape, dtype=object)
        if rank != 0:
            return result_volume, []
        logger.info('running activity-based voxel selection via Searchlight')
        self._check_inputs()
        r = int(self.sl.sl_rad)
        shape = np.asarray(self.sl.shape).astype(bool)
        centres, nfeat = engine.searchlight_centres(self.mask, r, shape, self.sl.min_active_voxels_proportion)
        kind = self._gpu_kind(clf)
        if len(centres) == 0:
            acc = np.zeros(0)
        elif kind is None:
            acc = self._run_host(clf, centres, shape)
        else:
            acc = self._run_gpu(clf, kind, centres, nfeat, shape)
        flat = result_volume.reshape(-1)
        for c, a in zip(centres.tolist(), acc):
            flat[c] = a
        results = []
        for idx, value in enumerate(result_volume[self.mask]):
            if value is None:
                value = 0
            results.append((idx, value))
        results.sort(key=lambda tup: tup[1], reverse=True)
        logger.info('activity-based voxel selection via Searchlight is done')
        return result_volume, results

    # ------------------------------------------------------------------ host path (the reference's loop)
    def _features(self, c, shape):
        """The features ``[E, n_features]`` of centre ``c`` (a linear index into the mask), as the reference hands them to
        the classifier."""
        r = int(self.sl.sl_rad)
        ny, nz = self.mask.shape[1], self.mask.shape[2]
        x, y, z = c // (ny * nz), (c // nz) % ny, c % nz
        sl = np.s_[x - r:x + r + 1, y - r:y + r + 1, z - r:z + r + 1]
        m = self.mask[sl] * shape
        return np.asarray(self.data)[sl][m, :].T

    def _run_host(self, clf, centres, shape):
        return [_host_accuracy(clf, self._features(c, shape), self.labels, self.num_folds) for c in centres.tolist()]

    # ------------------------------------------------------------------ GPU path
    def _torch_device(self):
        import torch
        if self.device is not None:
            return torch.device(self.device)
        return torch.device("cuda", torch.cuda.current_device())

    def _run_gpu(self, clf, kind, centres, nfeat, shape):
        import torch
        _lib.load()
        _lib.require_device()
        if np.any(nfeat == 0):
            raise ValueError('a searchlight centre has no features (empty shape)')
        data = np.ascontiguousarray(self.data)
        r = int(self.sl.sl_rad)
        used = engine.searchlight_used_voxels(self.mask, centres, r, shape)
        if not np.isfinite(data[used]).all():
            raise ValueError('the data holds NaN or infinity in voxels the searchlight uses')
        dev = self._torch_device()
        E = data.shape[3]
        folds = engine.svm_folds_for(self.labels, self.num_folds, E)
        # both builders give the same bytes; the untiled one is faster up to 32 epochs, the tiled one from 64 on (DESIGN.md
        # §3.7), and only the tiled one goes past 64
        kernels = engine.searchlight_kernels_wide if E > 32 else engine.searchlight_kernels
        if kind == 'rbf':
            gamma = 1.0 / nfeat.astype(np.float64) if clf.gamma == 'auto' else np.full(len(centres), float(clf.gamma))
        with torch.cuda.device(dev):
            vol = torch.from_numpy(data).to(dev)
            mask_d = torch.from_numpy(self.mask.astype(np.uint8)).to(dev)
            shape_d = torch.from_numpy(shape.astype(np.uint8)).to(dev)
            per_centre = E * E * 8 * {'linear': 1, 'rbf': 2, 'scale': 4}[kind]
            if self.batch_centres:
                batch = int(self.batch_centres)
            else:
                free, _ = torch.cuda.mem_get_info(dev)
                batch = max(1, min(1 << 16, (free // 4) // per_centre))
            acc = []
            for b0 in range(0, len(centres), batch):
                cb = centres[b0:b0 + batch]
                if kind == 'scale':
                    G, D, moments = engine.searchlight_gram_wide(vol, mask_d, r, shape_d, cb)
                    a, flagged = engine.svm_cv_scale(G, D, moments, nfeat[b0:b0 + batch], self.labels, self.num_folds,
                                                     C=clf.C, tol=clf.tol, max_iter=clf.max_iter,
                                                     shrinking=clf.shrinking, folds=folds)
                    del G, D, moments
                    for k in np.flatnonzero(flagged):
                        a[k] = _host_accuracy(clf, self._features(int(cb[k]), shape), self.labels, self.num_folds)
                    if flagged.any():
                        logger.info('%d centres scored on the host (gamma=\'scale\' variance check)', int(flagged.sum()))
                    acc.append(a)
                    continue
                K_fit, K_pred = kernels(vol, mask_d, r, shape_d, cb, kind, gamma[b0:b0 + batch] if kind == 'rbf' else None)
                acc.append(engine.svm_cv_f64(K_fit, K_pred, self.labels, self.num_folds, C=clf.C, tol=clf.tol,
                                             max_iter=clf.max_iter, shrinking=clf.shrinking, folds=folds))
                del K_fit, K_pred
        return np.concatenate(acc)
