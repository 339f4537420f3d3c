"""Device-side plumbing of the FCMA correlation engine: torch tensors hold HBM, the kernels live in
libfcma_b200.so and are called through the C ABI (include/fcma_b200.h) with raw device pointers.

HBM layout
----------
* epochs          float32 ``[E, T, V]``        voxels contiguous (the reference's ``raw_data`` list,
                                               voxelselector.py:72-76, stacked; rows ``t >= T_e`` zero)
* packed operand  ``[planes, E, V, Kp]``       K-major (time contiguous per voxel), bf16 or tf32,
                                               hi/lo planes for the 3-product fp32-faithful modes
* corr block      float32 ``[nb, E, ld]``      ``ld = round_up(V2, 32)``; raw r or Fisher-z
* kernels         float32 ``[nb, E, E]``
"""
import ctypes

import numpy as np
import torch

from .. import _lib

_PREC_DEFAULT = "fp32"

# "fp32" (the default of the public classes) means fp32-faithful correlations (|dr| <= 1e-6 * |x_i| |x_j|) by
# the fastest 3-product split: fp16 hi/lo planes (pre-scaled by 2^6, bf16 tensor speed) when the data is in the
# normalised range the reference's contract guarantees (unit-norm voxels, voxelselector.py:72-76), tf32 hi/lo
# planes (any finite fp32 range) otherwise.  The fp16 split is faithful only while the low plane stays a normal
# fp16 number: an element below 2^-9 leaves it with an absolute quantum of 2^-31, i.e. an error of about
# 2^-30 * sqrt(T) / min(|x_i|, |x_j|) in r.  So the data must have |x| <= 8 (no overflow of x * 2^6 and its products)
# and every non-zero per-(epoch, voxel) L2 norm >= 1/8 (1.7e-7 at T = 500); all-zero voxels are exact either way.
_FP16_SAFE_AMAX = 8.0
_FP16_SAFE_MIN_NORM = 0.125
_FP16_SCALE = 64.0                  # FCMA_FP16_SCALE of the packer
_FP16_MAX = 65504.0


def resolve_precision(precision, epochs=None, normalize=False):
    """``"fp32"`` -> ``"fp16x3"`` where the fp16 split is fp32-faithful for ``epochs`` ([E, T, V]), else ``"tf32x3"``;
    any other precision is returned unchanged.  ``normalize=True``: the packer's output is unit-norm or zero."""
    if precision != "fp32":
        return precision
    if normalize or epochs is None:
        return "fp16x3"
    vmax = torch.linalg.vector_norm(epochs, float("inf"), dim=1)      # [E, V]
    norm = torch.linalg.vector_norm(epochs, 2, dim=1)
    # a non-zero voxel whose squares underflow has norm 0 < 1/8 and is caught as well
    unsafe = (vmax.max() > _FP16_SAFE_AMAX) | ((vmax > 0) & (norm < _FP16_SAFE_MIN_NORM)).any()
    return "tf32x3" if bool(unsafe) else "fp16x3"


def _stream_ptr():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def _prec_code(precision):
    try:
        return _lib.PREC[precision]
    except KeyError:
        raise ValueError("unknown precision %r (choose from %s)" % (precision, sorted(_lib.PREC)))


def stack_epochs(raw_data, device):
    """list of E float32 ``[T_e, V]`` host arrays (or a ``[E, T, V]`` tensor) -> (``[E, Tmax, V]``
    float32 CUDA tensor, list of T_e).  Copies go through pinned memory."""
    if isinstance(raw_data, torch.Tensor):
        t = raw_data.to(device=device, dtype=torch.float32).contiguous()
        if t.dim() != 3:
            raise ValueError("epoch tensor must be [E, T, V]")
        return t, [t.shape[1]] * t.shape[0]
    E = len(raw_data)
    if E == 0:
        raise ValueError("no epochs")
    V = raw_data[0].shape[1]
    T_e = [int(m.shape[0]) for m in raw_data]
    T = max(T_e)
    for m in raw_data:
        if m.ndim != 2 or m.shape[1] != V:
            raise ValueError("all epochs must be 2D with the same number of voxels")
    same = all(t == T for t in T_e)
    if all(isinstance(m, np.ndarray) and m.dtype == np.float32 and m.flags.c_contiguous for m in raw_data):
        # the reference's contract (C-contiguous float32): copy every epoch straight from the caller's array.  A pageable
        # source goes through the driver's staging buffers at ~10 GB/s -- 0.12 s for 1.28 GB, against 0.7 s for
        # allocating a pinned staging tensor first
        dev_t = (torch.empty if same else torch.zeros)((E, T, V), dtype=torch.float32, device=device)
        for e, m in enumerate(raw_data):
            dev_t[e, :T_e[e]].copy_(torch.from_numpy(m))
        return dev_t, T_e
    host = torch.empty((E, T, V), dtype=torch.float32, pin_memory=True) if same else \
        torch.zeros((E, T, V), dtype=torch.float32, pin_memory=True)
    hn = host.numpy()
    for e, m in enumerate(raw_data):
        hn[e, :T_e[e], :] = m          # numpy casts to float32 like Cython's float[:, ::1] would demand
    return host.to(device, non_blocking=True), T_e


def upload_epochs_sharded(raw_data, device, group=None, use_ipc=True):
    """Multi-GPU upload of the epochs when every rank can see the host data (the usual case after
    ``prepare_fcma_data``: all ranks hold ``raw_data``): each rank stages and uploads only ITS contiguous share of the
    epochs over its own PCIe link, then the shares are all-gathered over NVLink by the copy engines
    (``exchange.EpochExchange``; NCCL all-gather if CUDA IPC is unavailable).  Returns (``[E, Tmax, V]`` float32 CUDA
    tensor, list of T_e) like ``stack_epochs``.  Replaces W full uploads (or rank 0's upload + ``comm.bcast``,
    reference preprocessing.py:211-223) by 1/W of the bytes per link."""
    from .exchange import EpochExchange
    E = len(raw_data)
    if E == 0:
        raise ValueError("no epochs")
    V = raw_data[0].shape[1]
    T_e = [int(m.shape[0]) for m in raw_data]
    T = max(T_e)
    for m in raw_data:
        if m.ndim != 2 or m.shape[1] != V:
            raise ValueError("all epochs must be 2D with the same number of voxels")
    xch = EpochExchange(E, T, V, device, group=group, nbuf=1, use_ipc=use_ipc)
    e0, n = xch.share_of()
    same = all(t == T for t in T_e[e0:e0 + n])
    host = (torch.empty if same else torch.zeros)((max(n, 1), T, V), dtype=torch.float32, pin_memory=True)
    hn = host.numpy()
    for j in range(n):
        hn[j, :T_e[e0 + j], :] = raw_data[e0 + j]
    ep = xch.gather(0, host[:n])
    torch.cuda.current_stream(ep.device).synchronize()      # the peers' mappings of this buffer are closed below
    if torch.distributed.is_initialized() and xch.world > 1:
        torch.distributed.barrier(group=group, device_ids=[ep.device.index])
    xch.close()
    return ep, T_e


class PackedOperand:
    """K-major, precision-split copy of one set of epochs, ready for TMA."""

    def __init__(self, buf, E, T, V, precision, T_e):
        self.buf, self.E, self.T, self.V = buf, E, T, V
        self.precision, self.T_e = precision, T_e

    @property
    def device(self):
        return self.buf.device


def pack_epochs(epochs, T_e=None, precision=_PREC_DEFAULT, normalize=False, v_begin=0, out=None):
    """epochs: float32 CUDA ``[E, T, V]``.  normalize=True applies preprocessing.py:80-84 on the fly.

    ``v_begin``: pack only the voxels ``[v_begin, V)`` (into their places of the V-voxel operand): a shard of the
    symmetric pipeline that starts at row ``s`` never touches voxels below ``s``.  ``out``: a PackedOperand of the
    same shape / precision whose buffer is reused."""
    lib = _lib.load()
    _lib.require_device()
    if epochs.dtype != torch.float32 or not epochs.is_cuda or not epochs.is_contiguous():
        raise ValueError("epochs must be a contiguous float32 CUDA tensor [E, T, V]")
    E, T, V = epochs.shape
    if precision == "fp16x3" and not normalize:
        amax = float(torch.linalg.vector_norm(epochs, float("inf")))
        if amax * _FP16_SCALE > _FP16_MAX:
            raise ValueError("fp16x3 stores x * %g in fp16, which overflows for max |x| = %g (limit %g): use "
                             "'tf32x3' or 'fp32'" % (_FP16_SCALE, amax, _FP16_MAX / _FP16_SCALE))
    precision = resolve_precision(precision, epochs, normalize)
    code = _prec_code(precision)
    if code == _lib.PREC["f32simt"]:
        raise ValueError("f32simt works on unpacked epochs")
    nbytes = lib.fcma_operand_bytes(code, E, T, V)
    if out is not None:
        if (out.E, out.T, out.V, out.precision) != (E, T, V, precision) or out.buf.numel() < nbytes:
            raise ValueError("`out` operand does not match the epochs / precision")
        buf = out.buf
    else:
        buf = torch.empty(nbytes, dtype=torch.uint8, device=epochs.device)
    te = None
    if T_e is not None and any(t != T for t in T_e):
        te = (ctypes.c_int * E)(*T_e)
    with torch.cuda.device(epochs.device):
        _lib.check(lib.fcma_pack_operand_range(_ptr(epochs), E, T, V, V, te, int(bool(normalize)), code,
                                               int(v_begin), V, _ptr(buf), nbytes, _stream_ptr()))
    return PackedOperand(buf, E, T, V, precision, list(T_e) if T_e is not None else [T] * E)


def epoch_normalize_(epochs, T_e=None):
    lib = _lib.load()
    _lib.require_device()
    E, T, V = epochs.shape
    te = None
    if T_e is not None and any(t != T for t in T_e):
        te = (ctypes.c_int * E)(*T_e)
    with torch.cuda.device(epochs.device):
        _lib.check(lib.fcma_epoch_normalize(_ptr(epochs), E, T, V, V, te, _stream_ptr()))
    return epochs


def _check_pair(rows, cols):
    if rows.E != cols.E or rows.T != cols.T or rows.precision != cols.precision:
        raise ValueError("row/column operands must share epochs, epoch length and precision")


def corr_block(rows, cols, start, nb, layout=0, fisher_epochs=0, out=None, ld=None):
    """a4/a9 on tensor cores.  Returns ``[nb, E, V2]`` (layout 0) or ``[E, nb, V2]`` (layout 1)."""
    lib = _lib.load()
    _check_pair(rows, cols)
    E, V2 = rows.E, cols.V
    ld = V2 if ld is None else ld
    shape = (nb, E, ld) if layout == 0 else (E, nb, ld)
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=rows.device)
    si, se = (E * ld, ld) if layout == 0 else (ld, nb * ld)
    with torch.cuda.device(rows.device):
        _lib.check(lib.fcma_corr_block(_ptr(rows.buf), _ptr(cols.buf), _prec_code(rows.precision), E,
                                       rows.T, rows.V, V2, start, nb, _ptr(out), si, se,
                                       fisher_epochs, _stream_ptr()))
    return out[..., :V2] if ld != V2 else out


def corr_block_f32(epochs_r, epochs_c, start, nb, layout=0):
    """a4 with fp32 FFMA on the unpacked epochs (reference-order numerics)."""
    lib = _lib.load()
    _lib.require_device()
    E, T, V = epochs_r.shape
    V2 = epochs_c.shape[2]
    shape = (nb, E, V2) if layout == 0 else (E, nb, V2)
    out = torch.empty(shape, dtype=torch.float32, device=epochs_r.device)
    si, se = (E * V2, V2) if layout == 0 else (V2, nb * V2)
    with torch.cuda.device(epochs_r.device):
        _lib.check(lib.fcma_corr_block_f32(_ptr(epochs_r), V, _ptr(epochs_c), V2, E, T, V, V2, start,
                                           nb, _ptr(out), si, se, _stream_ptr()))
    return out


def within_subject_norm_(corr, eps):
    """a6 in place on a contiguous float32 CUDA ``[n0, E, n2]`` tensor."""
    lib = _lib.load()
    if corr.dim() != 3:
        raise RuntimeError("The multi-subject correlation data structure must be 3D")
    if corr.dtype != torch.float32 or not corr.is_contiguous():
        raise ValueError("corr must be contiguous float32")
    n0, E, n2 = corr.shape
    with torch.cuda.device(corr.device):
        _lib.check(lib.fcma_within_subject_norm(_ptr(corr), n0, E, n2, int(eps), _stream_ptr()))
    return corr


def kernel_matrices(z, beta=0.0, out=None, sum_over_rows=False):
    """a7/a11: ``K[i] = beta*K[i] + Z_i Z_i^T`` for ``z`` = ``[nb, E, n2]`` (last dim may be a view)."""
    lib = _lib.load()
    nb, E, n2 = z.shape
    if z.stride(2) != 1:
        raise ValueError("innermost dimension must be contiguous")
    if out is None:
        out = torch.zeros((E, E) if sum_over_rows else (nb, E, E), dtype=torch.float32,
                          device=z.device)
    with torch.cuda.device(z.device):
        _lib.check(lib.fcma_kernel_matrices(_ptr(z), nb, E, n2, z.stride(0), z.stride(1), float(beta),
                                            _ptr(out), int(sum_over_rows), _stream_ptr()))
    return out


def norm_kernel_matrices(corr, eps, fisher_done=False, self_col0=-1, beta=0.0, out=None,
                         sum_over_rows=False):
    """fused a6+a7 on a raw-correlation block ``[nb, E, n2]``."""
    lib = _lib.load()
    nb, E, n2 = corr.shape
    if out is None:
        out = torch.zeros((E, E) if sum_over_rows else (nb, E, E), dtype=torch.float32,
                          device=corr.device)
    with torch.cuda.device(corr.device):
        _lib.check(lib.fcma_norm_kernel_matrices(_ptr(corr), nb, E, n2, corr.stride(0), corr.stride(1),
                                                 int(eps), int(fisher_done), int(self_col0),
                                                 float(beta), _ptr(out), int(sum_over_rows),
                                                 _stream_ptr()))
    return out


def fused_supported(E, eps):
    return E <= 64 and eps >= 1 and (eps & (eps - 1)) == 0 and eps <= (32 if E <= 32 else 64)


class Workspace:
    """Scratch for the correlation block of the fused pipelines (never holds results)."""

    def __init__(self, E, V2, rows, device):
        lib = _lib.load()
        self.per_row = lib.fcma_work_bytes_per_row(E, V2)
        self.rows = rows
        self.buf = torch.empty(self.per_row * rows, dtype=torch.uint8, device=device)

    @staticmethod
    def rows_for(E, V2, nb, device, max_bytes=None):
        per_row = _lib.load().fcma_work_bytes_per_row(E, V2)
        if max_bytes is None:
            free, _ = torch.cuda.mem_get_info(device)
            max_bytes = min(free // 2, 32 << 30)
        rows = max(1, min(nb, max_bytes // per_row))
        if rows >= 256:
            rows = (rows // 256) * 256
        return rows


def voxel_kernels(rows, cols, start, nb, eps, flags=0, work=None, out=None):
    """a4 -> a6 -> a7 for voxel rows [start, start+nb): unshrunk kernels ``[nb, E, E]``."""
    lib = _lib.load()
    _check_pair(rows, cols)
    E, V2 = rows.E, cols.V
    if work is None:
        work = Workspace(E, V2, Workspace.rows_for(E, V2, nb, rows.device), rows.device)
    if out is None:
        out = torch.empty((nb, E, E), dtype=torch.float32, device=rows.device)
    with torch.cuda.device(rows.device):
        _lib.check(lib.fcma_voxel_kernels(_ptr(rows.buf), _ptr(cols.buf), _prec_code(rows.precision), E,
                                          rows.T, rows.V, V2, start, nb, int(eps), int(flags),
                                          _ptr(work.buf), work.buf.numel(), _ptr(out), _stream_ptr()))
    return out


def feature_kernels_f64(rows, cols, start, nb, eps, kind="linear", gamma=None, work=None):
    """a4 -> a6 -> fp64 kernel matrices of the normalised correlation vectors for voxel rows [start, start+nb)
    (fcma_voxel_feature_kernels, 1 <= E <= 64): z[i] is the ``[E, V2]`` block ``within_subject_norm_`` gives on the raw
    correlations, bit for bit.  ``kind='linear'``: returns ``(G, G)``, ``G_ab = sum_j z_aj z_bj``; ``kind='rbf'`` with a
    number ``gamma``: ``(K_fit, K_pred)``, the x_square form libsvm trains with and the difference form of its decisions.
    Both float64 CUDA ``[nb, E, E]``, ready for ``svm_cv_f64``; the result is that of ``SVC(kernel=kind)`` on the
    features."""
    return _feature_kernels(_lib.load().fcma_voxel_feature_kernels, rows, cols, start, nb, eps, kind, gamma, work)


def feature_kernels_f64_wide(rows, cols, start, nb, eps, kind="linear", gamma=None, work=None):
    """``feature_kernels_f64`` for 1 <= E <= 256 (fcma_voxel_feature_kernels_wide: the block normalised in place, then
    k_feature_gram_tiled): the same arguments and outputs.  D, and so the rbf ``K_pred``, equals ``feature_kernels_f64``'s
    bit for bit at E <= 64; G is summed in another order of its 4-column MMA steps."""
    return _feature_kernels(_lib.load().fcma_voxel_feature_kernels_wide, rows, cols, start, nb, eps, kind, gamma, work)


def feature_block_rows(E, per_row, n, budget, matrices=2):
    """Voxel rows per ``feature_kernels_f64_wide`` call: the workspace (``per_row`` bytes a row,
    ``fcma_work_bytes_per_row``) and the fp64 ``K_fit`` and ``K_pred`` (16 E^2 bytes a row) of at most ``n`` rows within
    ``budget`` bytes, whole 256-row GEMM blocks when there are more than 256; at least one row.  ``matrices``: the fp64
    ``[E, E]`` matrices a row holds (4 for ``feature_gram_wide``'s G and D plus one fold's ``K_fit`` and ``K_pred``)."""
    rows = max(1, min(n, budget // (per_row + 8 * matrices * E * E)))
    if rows >= 256:
        rows = (rows // 256) * 256
    return rows


def feature_gram_wide(rows, cols, start, nb, eps, work=None):
    """The fp64 sums behind ``SVC(kernel='rbf', gamma='scale')`` on the normalised correlation vectors of voxel rows
    [start, start+nb) (fcma_voxel_feature_gram_wide, 1 <= E <= 256): ``(G, D, moments)``, G and D float64 CUDA
    ``[nb, E, E]`` -- the entries ``feature_kernels_f64_wide(kind='rbf')`` exponentiates, bit for bit -- and ``moments``
    float64 ``[nb, E, 4]``: the double-double sums (s.hi, s.lo, q.hi, q.lo) of s_e = sum_j z_ej and q_e = sum_j z_ej^2."""
    lib = _lib.load()
    _check_pair(rows, cols)
    E, V2 = rows.E, cols.V
    if work is None:
        work = Workspace(E, V2, Workspace.rows_for(E, V2, nb, rows.device), rows.device)
    G = torch.empty((nb, E, E), dtype=torch.float64, device=rows.device)
    D = torch.empty_like(G)
    moments = torch.empty((nb, E, 4), dtype=torch.float64, device=rows.device)
    with torch.cuda.device(rows.device):
        _lib.check(lib.fcma_voxel_feature_gram_wide(_ptr(rows.buf), _ptr(cols.buf), _prec_code(rows.precision), E, rows.T,
                                                    rows.V, V2, start, nb, int(eps), _ptr(work.buf), work.buf.numel(),
                                                    _ptr(G), _ptr(D), _ptr(moments), _stream_ptr()))
    return G, D, moments


def _feature_kernels(entry, rows, cols, start, nb, eps, kind, gamma, work):
    """The body of feature_kernels_f64 and feature_kernels_f64_wide around one call of the C entry point ``entry``."""
    _check_pair(rows, cols)
    E, V2 = rows.E, cols.V
    if kind not in ("linear", "rbf"):
        raise ValueError("kind must be 'linear' or 'rbf', not %r" % (kind,))
    kcode = 0 if kind == "linear" else 1
    g = 0.0
    if kcode == 1:
        if gamma is None:
            raise ValueError("kind='rbf' needs gamma")
        g = float(gamma)
        if not (np.isfinite(g) and g >= 0):
            raise ValueError("gamma must be finite and non-negative")
    if work is None:
        work = Workspace(E, V2, Workspace.rows_for(E, V2, nb, rows.device), rows.device)
    K_fit = torch.empty((nb, E, E), dtype=torch.float64, device=rows.device)
    K_pred = K_fit if kcode == 0 else torch.empty_like(K_fit)
    with torch.cuda.device(rows.device):
        _lib.check(entry(_ptr(rows.buf), _ptr(cols.buf), _prec_code(rows.precision), E, rows.T, rows.V, V2, start, nb,
                         int(eps), kcode, g, _ptr(work.buf), work.buf.numel(), _ptr(K_fit),
                         _ptr(K_pred) if kcode else None, _stream_ptr()))
    return K_fit, K_pred


def sym_row_partition(num_voxels, world_size, align=256, pack_frac=0.01):
    """Shards of [0, V) for the symmetric pipeline.  Shard r contracts its rows with the columns at or to the right of
    its first row, so the work of rows [a, b) is the trapezoid area (1 - a/V)^2 - (1 - b/V)^2 of the upper triangle, plus
    the packing of the voxels [a, V) it touches (``pack_frac`` = time of packing ALL voxels as a fraction of a whole
    single-GPU step).  Cuts must be whole 256-row tiles (the last shard takes the
    ragged tail), so the shards are chosen as the min-max linear partition over those tiles (binary search on the
    bottleneck cost + greedy packing: optimal for contiguous shards).  Returns [(start, n)]."""
    V, W = int(num_voxels), int(world_size)
    if W <= 1:
        return [(0, V)]
    ntiles = (V + align - 1) // align
    edge = [min(k * align, V) for k in range(ntiles + 1)]

    def cost(a, b):                    # rows [a, b): kernel share + pack share of the whole step
        return ((1.0 - a / float(V)) ** 2 - (1.0 - b / float(V)) ** 2) + pack_frac * (1.0 - a / float(V))

    def greedy(limit):
        cuts, k = [0], 0
        for _ in range(W):
            k0 = k
            while k < ntiles and cost(edge[k0], edge[k + 1]) <= limit:
                k += 1
            if k == k0 and k < ntiles:
                return None                       # a single tile exceeds the limit
            cuts.append(edge[k])
        return cuts if k == ntiles else None

    lo, hi = 0.0, 1.0 + pack_frac
    for _ in range(50):
        mid = 0.5 * (lo + hi)
        if greedy(mid) is None:
            lo = mid
        else:
            hi = mid
    cuts = greedy(hi)
    return [(cuts[r], cuts[r + 1] - cuts[r]) for r in range(W)]


def sym_supported(E, eps, nb=None, start=0, V=None):
    """The symmetric self-correlation pipeline needs the fused normalise+kernel path and whole 256-row
    tiles (a ragged row count only when the rows end at V)."""
    ok = fused_supported(E, eps)
    if ok and nb is not None and V is not None:
        ok = nb >= 1 and (nb % 256 == 0 or start + nb == V) and (V - start) >= 256
    return ok


class SymWorkspace(Workspace):
    """Scratch of the symmetric pipeline sized for `rows` block rows WITH a transposed copy (E > 32);
    the column-pass variant (E <= 32) keeps only the block and takes twice as many rows per pass from the
    same buffer (fcma_sym_rows_per_pass)."""

    def __init__(self, E, V, rows, device, start=0, transposed_copy=True):
        lib = _lib.load()
        self.per_row = (2 if transposed_copy else 1) * lib.fcma_work_bytes_per_row(E, V - start)
        self.rows = max(256, (int(rows) + 255) // 256 * 256)
        self.buf = torch.empty(self.per_row * self.rows, dtype=torch.uint8, device=device)

    @classmethod
    def for_operand(cls, op, rows, eps, flags=0, start=0):
        """Scratch for exactly `rows` block rows per pass of fcma_voxel_kernels_sym on this operand: the block alone
        when the column pass applies (E <= 32), block + transposed copy otherwise."""
        cols = bool(_lib.load().fcma_sym_uses_column_pass(_prec_code(op.precision), op.E, int(eps), int(flags)))
        return cls(op.E, op.V, rows, op.device, start=start, transposed_copy=not cols)


def voxel_kernels_sym(op, start, nb, eps, flags=0, work=None, out=None):
    """Self-correlation a4 -> a6 -> a7 at half the tensor work (fcma_voxel_kernels_sym): rows
    [start, start+nb) against columns [start, V), every block used for its row AND its column voxels.
    ``out`` is the full ``[V, E, E]`` array and is accumulated into (zeros if not given)."""
    lib = _lib.load()
    E, V = op.E, op.V
    if work is None:
        free, _ = torch.cuda.mem_get_info(op.device)
        per_row = 2 * lib.fcma_work_bytes_per_row(E, V - start)
        rows = max(256, min((nb + 255) // 256 * 256, (min(free // 2, 64 << 30) // per_row) // 256 * 256, 4096))
        work = SymWorkspace.for_operand(op, rows, eps, flags, start)
    if out is None:
        out = torch.zeros((V, E, E), dtype=torch.float32, device=op.device)
    with torch.cuda.device(op.device):
        _lib.check(lib.fcma_voxel_kernels_sym(_ptr(op.buf), _prec_code(op.precision), E, op.T, V, start, nb,
                                              int(eps), int(flags), _ptr(work.buf), work.buf.numel(), _ptr(out),
                                              _stream_ptr()))
    return out


def voxel_kernels_sym_grouped(epochs, op, start, nb, eps, groups, events, flags=0, work=None, out=None, normalize=False):
    """``voxel_kernels_sym`` for epochs that are still arriving (``exchange.EpochExchange.gather_groups``): ``groups`` =
    ``[(e0, count)]`` contiguous epoch groups of ``epochs`` (float32 CUDA ``[E, T, V]``), ``events[g]`` a
    ``torch.cuda.Event`` (or None) that fires when group g is complete.  Packing (into ``op``, voxels ``[start, V)``) and
    the GEMMs of the first pass(es) follow the groups, the rest is the ordinary symmetric pipeline."""
    lib = _lib.load()
    E, T, V = epochs.shape
    if (op.E, op.T, op.V) != (E, T, V):
        raise ValueError("operand does not match the epochs")
    if work is None:
        work = SymWorkspace.for_operand(op, 2 * min(4096, (nb + 255) // 256 * 256), eps, flags, start)
    if out is None:
        out = torch.zeros((V, E, E), dtype=torch.float32, device=op.device)
    ng = len(groups)
    e0 = (ctypes.c_int * ng)(*[int(a) for a, _ in groups])
    cnt = (ctypes.c_int * ng)(*[int(c) for _, c in groups])
    evs = (ctypes.c_void_p * ng)(*[ctypes.c_void_p(ev.cuda_event) if ev is not None else None for ev in events])
    with torch.cuda.device(op.device):
        _lib.check(lib.fcma_voxel_kernels_sym_grouped(_ptr(epochs), None, int(bool(normalize)), _ptr(op.buf), op.buf.numel(),
                                                      _prec_code(op.precision), E, T, V, start, nb, int(eps), int(flags), ng,
                                                      e0, cnt, evs, _ptr(work.buf), work.buf.numel(), _ptr(out), _stream_ptr()))
    return out


def classifier_kernel(rows, cols, start, nb, eps, flags=0, work=None, out=None, symmetric=True):
    """a9 -> a10 -> a11: accumulates sum_i Z_i Z_i^T over rows [start, start+nb) into ``out`` [E, E].

    One mask, all rows at once and a fused-path eps: the symmetric pipeline's GEMM (z(i, :, j) == z(j, :, i), so only the
    blocks on/above the diagonal are contracted) followed by row passes only."""
    lib = _lib.load()
    _check_pair(rows, cols)
    E, V2 = rows.E, cols.V
    if (symmetric and rows is cols and start == 0 and nb == rows.V and eps > 1 and rows.V >= 512
            and sym_supported(E, eps) and not (flags & _lib.FLAG_FISHER_IN_PASS2)):
        # one mask: every voxel pair is contracted ONCE (symmetric GEMM) and summed by row passes only -- the diagonal
        # squares once, the blocks right of them twice (fcma_classifier_kernel_sym); no per-voxel kernels are formed
        if out is None:
            out = torch.zeros((E, E), dtype=torch.float32, device=rows.device)
        per_row = lib.fcma_work_bytes_per_row(E, V2)
        if work is None or work.buf.numel() < 256 * per_row:
            free, _ = torch.cuda.mem_get_info(rows.device)
            nrows = max(256, min((nb + 255) // 256 * 256, (min(free // 2, 64 << 30) // per_row) // 256 * 256, 4096))
            work = SymWorkspace(E, V2, nrows, rows.device, transposed_copy=False)
        with torch.cuda.device(rows.device):
            _lib.check(lib.fcma_classifier_kernel_sym(_ptr(rows.buf), _prec_code(rows.precision), E, rows.T, rows.V, int(eps),
                                                      int(flags), _ptr(work.buf), work.buf.numel(), _ptr(out), _stream_ptr()))
        return out
    if work is None:
        work = Workspace(E, V2, Workspace.rows_for(E, V2, nb, rows.device), rows.device)
    if out is None:
        out = torch.zeros((E, E), dtype=torch.float32, device=rows.device)
    with torch.cuda.device(rows.device):
        _lib.check(lib.fcma_classifier_kernel(_ptr(rows.buf), _ptr(cols.buf), _prec_code(rows.precision),
                                              E, rows.T, rows.V, V2, start, nb, int(eps), int(flags),
                                              _ptr(work.buf), work.buf.numel(), _ptr(out),
                                              _stream_ptr()))
    return out


def _check_rows(x, name):
    """The row kernels take float32 CUDA matrices with unit column stride and the row pitch ``stride(0)``."""
    if x.dtype != torch.float32 or not x.is_cuda or x.dim() != 2 or x.stride(1) != 1:
        raise ValueError("%s must be a 2-D float32 CUDA tensor with contiguous rows (stride(1) == 1)" % name)


def gemm_nt(a, b):
    """``a @ b.T`` in fp32 FFMA (a12/a15)."""
    lib = _lib.load()
    _check_rows(a, "a")
    _check_rows(b, "b")
    if a.shape[1] != b.shape[1] or a.device != b.device:
        raise ValueError("gemm_nt: a and b must share their inner dimension and device")
    M, K = a.shape
    N = b.shape[0]
    out = torch.empty((M, N), dtype=torch.float32, device=a.device)
    with torch.cuda.device(a.device):
        _lib.check(lib.fcma_gemm_nt(_ptr(a), _ptr(b), _ptr(out), M, N, K, a.stride(0), b.stride(0), N,
                                    _stream_ptr()))
    return out


def row_normalize_(x, nan_to_zero=True):
    lib = _lib.load()
    _check_rows(x, "x")
    R, D = x.shape
    with torch.cuda.device(x.device):
        _lib.check(lib.fcma_row_normalize(_ptr(x), R, D, x.stride(0), int(nan_to_zero), _stream_ptr()))
    return x


def host_voxel_kernels(raw_data, raw_data2, start, nb, eps, precision=_PREC_DEFAULT, normalize=False,
                       flags=0, device=None):
    """The C-ABI host entry point: numpy in, numpy out, all copies inside the call.  ``device`` defaults to the
    calling thread's current CUDA device (LOCAL_RANK's GPU in a rank process); the library restores the caller's
    current device before it returns."""
    lib = _lib.load()
    if device is None:
        device = torch.cuda.current_device() if torch.cuda.is_available() else 0
    E = len(raw_data)
    V = raw_data[0].shape[1]
    keep = [np.ascontiguousarray(m, dtype=np.float32) for m in raw_data]
    arr = (ctypes.POINTER(ctypes.c_float) * E)(*[m.ctypes.data_as(ctypes.POINTER(ctypes.c_float)) for m in keep])
    arr2, V2, keep2 = None, V, None
    if raw_data2 is not None:
        keep2 = [np.ascontiguousarray(m, dtype=np.float32) for m in raw_data2]
        V2 = keep2[0].shape[1]
        arr2 = (ctypes.POINTER(ctypes.c_float) * E)(
            *[m.ctypes.data_as(ctypes.POINTER(ctypes.c_float)) for m in keep2])
    te = (ctypes.c_int * E)(*[m.shape[0] for m in keep])
    K = np.empty((nb, E, E), np.float32)
    _lib.check(lib.fcma_host_voxel_kernels(arr, arr2, te, E, V, V2, start, nb, int(eps),
                                           _prec_code(precision), int(bool(normalize)), int(flags),
                                           int(device), K.ctypes.data_as(ctypes.c_void_p)))
    return K


def host_voxel_kernels_sym(raw_data, eps, precision="fp16x3", normalize=False, flags=0, device=None, rows_per_pass=0,
                           out=None):
    """The C-ABI host entry point of the single-mask worker loop (fcma_host_voxel_kernels_sym): E host arrays
    ``[T_e, V]`` (or one host tensor ``[E, T, V]``; pinned memory makes the copies asynchronous DMA) in, the unshrunk
    kernels ``[V, E, E]`` out (``out``: a host float32 tensor / array to fill, e.g. pinned).  H2D, packing, the symmetric
    pipeline and D2H all happen inside the call."""
    lib = _lib.load()
    if device is None:
        device = torch.cuda.current_device() if torch.cuda.is_available() else 0
    if isinstance(raw_data, torch.Tensor):
        if raw_data.is_cuda or raw_data.dtype != torch.float32 or not raw_data.is_contiguous() or raw_data.dim() != 3:
            raise ValueError("host epochs tensor must be contiguous float32 [E, T, V] in host memory")
        E, T, V = raw_data.shape
        ptrs = [raw_data.data_ptr() + e * T * V * 4 for e in range(E)]
        Ts, keep = [T] * E, raw_data
    else:
        keep = [np.ascontiguousarray(m, dtype=np.float32) for m in raw_data]
        E, V = len(keep), keep[0].shape[1]
        ptrs = [m.ctypes.data for m in keep]
        Ts = [m.shape[0] for m in keep]
    arr = (ctypes.POINTER(ctypes.c_float) * E)(*[ctypes.cast(p, ctypes.POINTER(ctypes.c_float)) for p in ptrs])
    te = (ctypes.c_int * E)(*Ts)
    if out is None:
        out = np.empty((V, E, E), np.float32)
    optr = out.data_ptr() if isinstance(out, torch.Tensor) else out.ctypes.data
    _lib.check(lib.fcma_host_voxel_kernels_sym(arr, te, E, V, int(eps), _prec_code(precision), int(bool(normalize)),
                                               int(flags), int(device), int(rows_per_pass), ctypes.c_void_p(optr)))
    del keep
    return out


# ------------------------------------------------------------------ a7 tail + a8 on the GPU
class _SvmFold(ctypes.Structure):
    _fields_ = [("n_train", ctypes.c_int), ("n_pos", ctypes.c_int), ("n_test", ctypes.c_int),
                ("pad", ctypes.c_int), ("train_idx", ctypes.c_int * 64), ("test_idx", ctypes.c_int * 64),
                ("test_pos", ctypes.c_ubyte * 64)]


class _SvmFoldWide(ctypes.Structure):
    """The fold problem of fcma_svm_cv_solve_wide: _SvmFold with room for 256 training and 256 held-out samples."""
    _fields_ = [("n_train", ctypes.c_int), ("n_pos", ctypes.c_int), ("n_test", ctypes.c_int),
                ("pad", ctypes.c_int), ("train_idx", ctypes.c_int * 256), ("test_idx", ctypes.c_int * 256),
                ("test_pos", ctypes.c_ubyte * 256)]


SVM_WIDE_MAX_EPOCHS = 256


def shrink_kernels_(K, return_digits=False):
    """In-place decimal shrink (voxelselector.py:409-412) of ``K`` = float32 CUDA ``[nv, E, E]``."""
    lib = _lib.load()
    nv, E, _ = K.shape
    digits = torch.empty(nv, dtype=torch.int32, device=K.device) if return_digits else None
    with torch.cuda.device(K.device):
        _lib.check(lib.fcma_shrink_kernels(_ptr(K), nv, E, _ptr(digits) if digits is not None else None,
                                           _stream_ptr()))
    return digits


def subset_kernels(K, keep, shrink=False, out=None, return_digits=False):
    """The kernels of the epochs ``keep`` (strictly increasing indices into [0, E), E <= 256):
    ``out[v] = K[v][keep][:, keep]`` for contiguous CUDA ``K`` ``[nv, E, E]``, float32 (fcma_subset_kernels) or float64
    (fcma_subset_kernels_f64), written out of place into ``out`` (``[nv, len(keep), len(keep)]`` of K's dtype,
    allocated if None) and returned.  ``shrink`` (float32 only): ``shrink_kernels_`` in the same pass, its digits counted
    on the compacted ``out[v, 0, 0]``; ``return_digits``: also those digit counts, int32 ``[nv]``."""
    lib = _lib.load()
    if K.dim() != 3 or K.shape[1] != K.shape[2] or not K.is_contiguous() or K.dtype not in (torch.float32, torch.float64):
        raise ValueError("K must be contiguous float32 or float64 [nv, E, E]")
    f64 = K.dtype == torch.float64
    if f64 and (shrink or return_digits):
        raise ValueError("the decimal shrink applies to float32 kernels only")
    keep_h = np.ascontiguousarray(keep, dtype=np.int32)
    if keep_h.ndim != 1:
        raise ValueError("keep must be a 1-D list of epoch indices")
    nv, E, _ = K.shape
    Ek = len(keep_h)
    if out is None:
        out = torch.empty((nv, Ek, Ek), dtype=K.dtype, device=K.device)
    elif out.shape != (nv, Ek, Ek) or out.dtype != K.dtype or out.device != K.device or not out.is_contiguous():
        raise ValueError("out must be contiguous [%d, %d, %d] of K's dtype and device" % (nv, Ek, Ek))
    digits = torch.empty(nv, dtype=torch.int32, device=K.device) if return_digits else None
    kp = keep_h.ctypes.data_as(ctypes.c_void_p)
    with torch.cuda.device(K.device):
        if f64:
            _lib.check(lib.fcma_subset_kernels_f64(_ptr(K), nv, E, kp, Ek, _ptr(out), _stream_ptr()))
        else:
            _lib.check(lib.fcma_subset_kernels(_ptr(K), nv, E, kp, Ek, _ptr(out), 1 if shrink else 0,
                                               _ptr(digits) if digits is not None else None, _stream_ptr()))
    return (out, digits) if return_digits else out


def svm_cv_supported(clf, labels, num_folds, E, allow_shrinking=True, max_epochs=64):
    """True if ``cross_val_score(clf, K, labels, cv=StratifiedKFold(num_folds))`` can run on the GPU:
    ``SVC(kernel='precomputed')`` without class weights / probability / tie breaking, E <= ``max_epochs`` (64, or up to
    ``SVM_WIDE_MAX_EPOCHS``, which ``svm_cv_precomputed`` solves with the wide solver above 64); two classes, or more
    (one-vs-one, as libsvm does) when every class is in the training part of every fold.

    The GPU solver restates libsvm's SMO with and without the shrinking heuristic (``clf.shrinking``; the reference's tests
    and examples use ``shrinking=False``, tests/fcma/test_voxel_selection.py:70; scikit-learn's default is ``True``).
    ``allow_shrinking=False`` sends ``shrinking=True`` classifiers to the host."""
    import sklearn.svm
    if not (isinstance(clf, sklearn.svm.SVC) and clf.kernel == 'precomputed'):
        return False
    if getattr(clf, 'shrinking', False) and not allow_shrinking:
        return False
    # scikit-learn >= 1.9 uses the string 'deprecated' as the default of `probability`
    if clf.class_weight is not None or getattr(clf, 'probability', False) is True or E > min(max_epochs, SVM_WIDE_MAX_EPOCHS) \
            or num_folds > 64:
        return False
    y = np.asarray(labels)
    classes = np.unique(y)
    if len(classes) == 2:
        return True
    if len(classes) < 2 or getattr(clf, 'break_ties', False):
        return False
    try:
        svm_folds_for(y, num_folds, E)
    except ValueError:
        return False
    return True


def svc_feature_kind(clf, labels, num_folds, E, max_epochs=64):
    """``'linear'`` / ``'rbf'`` if ``cross_val_score(clf, X, labels, cv=StratifiedKFold(num_folds))`` on float32
    features ``X`` (E samples) can be computed as ``svm_cv_f64`` on the fp64 kernel matrices of ``X``, else None:
    ``SVC(kernel='linear')`` or ``SVC(kernel='rbf')`` with ``gamma='auto'`` or a number >= 0, without class weights,
    probability or tie breaking, E <= ``max_epochs`` (64, or up to ``SVM_WIDE_MAX_EPOCHS``, solved with
    ``svm_folds_for`` folds), at most 64 folds that ``svm_folds_for`` accepts.  ``gamma='scale'`` depends on the variance
    of the training features and stays with scikit-learn."""
    import numbers
    import sklearn.svm
    if not isinstance(clf, sklearn.svm.SVC):
        return None
    if clf.kernel == 'linear':
        kind = 'linear'
    elif clf.kernel == 'rbf' and (clf.gamma == 'auto' or (isinstance(clf.gamma, numbers.Real)
                                                          and not isinstance(clf.gamma, bool) and clf.gamma >= 0)):
        kind = 'rbf'
    else:
        return None
    # scikit-learn >= 1.9 uses the string 'deprecated' as the default of `probability`
    if clf.class_weight is not None or getattr(clf, 'probability', False) is True or getattr(clf, 'break_ties', False):
        return None
    if E > min(max_epochs, SVM_WIDE_MAX_EPOCHS) or num_folds > 64:
        return None
    try:
        svm_folds_for(labels, num_folds, E)
    except ValueError:
        return None
    return kind


def svc_scale_supported(clf, labels, num_folds, E):
    """True if ``cross_val_score(clf, X, labels, cv=StratifiedKFold(num_folds))`` on float32 features ``X`` (E samples)
    can be computed by ``svm_cv_scale``: ``SVC(kernel='rbf', gamma='scale')`` -- scikit-learn's ``SVC()`` -- without class
    weights, probability or tie breaking, E <= ``SVM_WIDE_MAX_EPOCHS``, at most 64 folds that ``svm_folds_for``
    accepts.  The other rbf gammas and the linear kernel are ``svc_feature_kind``'s."""
    import sklearn.svm
    if not (isinstance(clf, sklearn.svm.SVC) and clf.kernel == 'rbf' and isinstance(clf.gamma, str)
            and clf.gamma == 'scale'):
        return False
    # scikit-learn >= 1.9 uses the string 'deprecated' as the default of `probability`
    if clf.class_weight is not None or getattr(clf, 'probability', False) is True or getattr(clf, 'break_ties', False):
        return False
    if E > SVM_WIDE_MAX_EPOCHS or num_folds > 64:
        return False
    try:
        svm_folds_for(labels, num_folds, E)
    except ValueError:
        return False
    return True


class SvmFolds:
    """Fold problems for the batched GPU solver: ``structs`` holds one _SvmFold per (fold, class pair) -- pair-major
    inside a fold, pairs in libsvm's order (0,1), (0,2), ..., (1,2), ... -- and everything the vote needs."""

    def __init__(self, structs, n_test, classes, pairs, test_labels):
        self.structs, self.n_test, self.classes, self.pairs, self.test_labels = structs, n_test, classes, pairs, test_labels
        self.num_folds = len(n_test)
        self.nproblems = len(structs)
        self.wide = structs._type_ is _SvmFoldWide     # for fcma_svm_cv_solve_wide

    def __iter__(self):          # (structs, n_test) unpacking of the two-class form
        return iter((self.structs, self.n_test))


def make_svm_folds(labels, num_folds):
    """Fold descriptions for fcma_svm_cv_precomputed / fcma_svm_cv_solve from sklearn's own splitter
    (StratifiedKFold(n_splits, shuffle=False), reference voxelselector.py:44-45).  With k > 2 classes each fold becomes
    k(k-1)/2 two-class problems (libsvm's one-vs-one: the pair (a, b), a < b, trains on the fold's samples of those two
    classes with class a as +1 and is evaluated on ALL held-out samples of the fold)."""
    return _build_svm_folds(labels, num_folds, _SvmFold, 64)


def make_svm_folds_wide(labels, num_folds):
    """``make_svm_folds`` for fcma_svm_cv_solve_wide: the same splits and problems, up to 256 training and 256 held-out
    samples per problem."""
    return _build_svm_folds(labels, num_folds, _SvmFoldWide, 256)


def svm_folds_for(labels, num_folds, E):
    """The fold problems ``svm_cv_precomputed`` solves E-epoch kernels with: ``make_svm_folds`` up to 64 epochs, else
    ``make_svm_folds_wide``."""
    return make_svm_folds(labels, num_folds) if E <= 64 else make_svm_folds_wide(labels, num_folds)


def fold_problems(folds, f):
    """The problems of fold ``f`` alone: an SvmFolds of one fold whose structs are the slice
    ``[f * npairs, (f + 1) * npairs)`` of ``folds.structs``, with that fold's ``n_test`` and ``test_labels``."""
    npairs = len(folds.pairs)
    struct = folds.structs._type_
    part = (struct * npairs)(*folds.structs[f * npairs:(f + 1) * npairs])
    return SvmFolds(part, folds.n_test[f:f + 1], folds.classes, folds.pairs, folds.test_labels[f:f + 1])


def fold_train_mask(folds, E):
    """uint8 ``[num_folds, E]``: 1 where epoch e is a training sample of fold f (every sample outside its held-out part)."""
    train = np.ones((folds.num_folds, E), dtype=np.uint8)
    npairs = len(folds.pairs)
    for f in range(folds.num_folds):
        fd = folds.structs[f * npairs]
        train[f, list(fd.test_idx[:fd.n_test])] = 0
    return train


def _build_svm_folds(labels, num_folds, struct, limit):
    from sklearn import model_selection
    y = np.asarray(labels)
    classes = np.unique(y)
    if len(classes) < 2:
        raise ValueError("GPU SVM cross-validation needs at least two classes")
    code = np.searchsorted(classes, y)
    k = len(classes)
    pairs = [(a, b) for a in range(k) for b in range(a + 1, k)]
    skf = model_selection.StratifiedKFold(n_splits=num_folds, shuffle=False)
    folds = (struct * (num_folds * len(pairs)))()
    n_test, test_labels = [], []
    for f, (tr, te) in enumerate(skf.split(np.zeros((len(y), 1)), y)):
        if len(te) > limit:
            raise ValueError("more than %d held-out samples in a fold" % limit)
        for q, (a, b) in enumerate(pairs):
            pos = [int(i) for i in tr if code[i] == a]     # smaller label first = class +1
            neg = [int(i) for i in tr if code[i] == b]
            if not pos or not neg:
                raise ValueError("a training fold misses a class")
            order = pos + neg
            if len(order) > limit:
                raise ValueError("more than %d training samples in a class pair" % limit)
            fd = folds[f * len(pairs) + q]
            fd.n_train, fd.n_pos, fd.n_test = len(order), len(pos), len(te)
            for j, i in enumerate(order):
                fd.train_idx[j] = i
            for j, i in enumerate(te):
                fd.test_idx[j] = int(i)
                fd.test_pos[j] = 1 if code[i] == a else 0
        n_test.append(len(te))
        test_labels.append(code[te].astype(np.int64))
    return SvmFolds(folds, np.asarray(n_test, dtype=np.float64), classes, pairs, test_labels)


def _ovo_vote(bits, folds):
    """libsvm's svm_predict vote on the device: ``bits`` int64 ``[nv, nproblems]``, or ``[nv, nproblems, words]`` (bit
    t % 64 of word t // 64 = held-out sample t on the side of the pair's first class) -> number of correctly predicted
    held-out samples per (voxel, fold).  Ties go to the smallest class index (the first maximum), as in libsvm."""
    if bits.dim() == 2:
        bits = bits[:, :, None]
    nv = bits.shape[0]
    k, npairs = len(folds.classes), len(folds.pairs)
    correct = torch.zeros((nv, folds.num_folds), dtype=torch.int32, device=bits.device)
    for f in range(folds.num_folds):
        nt = int(folds.n_test[f])
        t = torch.arange(nt, device=bits.device, dtype=torch.int64)
        word, shifts = t // 64, t % 64
        votes = torch.zeros((nv, nt, k), dtype=torch.int32, device=bits.device)
        for q, (a, b) in enumerate(folds.pairs):
            side = ((bits[:, f * npairs + q, word] >> shifts[None, :]) & 1).to(torch.int32)   # [nv, nt]
            votes[:, :, a] += side
            votes[:, :, b] += 1 - side
        # first maximum: argmax of votes * k + (k - 1 - class)
        key = votes * k + torch.arange(k - 1, -1, -1, device=bits.device, dtype=torch.int32)[None, None, :]
        pred = key.argmax(dim=2)
        truth = torch.as_tensor(folds.test_labels[f], device=bits.device)
        correct[:, f] = (pred == truth[None, :]).sum(dim=1).to(torch.int32)
    return correct


def _max_iter_arg(max_iter):
    """SVC(max_iter) for the solver: -1 (any negative value, or None) runs without a limit, 0 runs no iteration."""
    return -1 if max_iter is None or max_iter < 0 else int(max_iter)


def _svm_correct(solve, kernels, K, C, tol, max_iter, shrinking, folds, return_iters):
    """One call of the batched solver ``solve`` on the problems of ``folds`` (libsvm's one-vs-one vote for more than two
    classes): the int32 CUDA ``[nv, num_folds]`` counts of correctly predicted held-out samples, and the ``[nv,
    nproblems]`` iteration counts (or None)."""
    nv, E, _ = K.shape
    nprob = folds.nproblems
    two = len(folds.classes) == 2
    with torch.cuda.device(K.device):
        iters = torch.empty((nv, nprob), dtype=torch.int32, device=K.device) if return_iters else None
        correct = torch.empty((nv, nprob), dtype=torch.int32, device=K.device) if two else None
        bits = None if two else torch.empty((nv, nprob, 4) if folds.wide else (nv, nprob), dtype=torch.int64,
                                            device=K.device)
        _lib.check(solve(*kernels, nv, E, nprob, ctypes.cast(folds.structs, ctypes.c_void_p), float(C), float(tol),
                         _max_iter_arg(max_iter), 1 if shrinking else 0, _ptr(correct) if two else None,
                         _ptr(bits) if not two else None, _ptr(iters) if iters is not None else None, _stream_ptr()))
        if not two:
            correct = _ovo_vote(bits, folds)
    return correct, iters


def _svm_cv(solve, kernels, K, labels, num_folds, C, tol, max_iter, shrinking, folds, return_iters):
    """The body of svm_cv_precomputed and svm_cv_f64 around one call of the batched solver ``solve``
    (fcma_svm_cv_solve or fcma_svm_cv_solve_f64, whose leading arguments are the kernel pointers ``kernels``; ``K`` is
    one of those kernels): fold problems, outputs, libsvm's one-vs-one vote for more than two classes, and the mean
    accuracy per kernel."""
    if folds is None:
        folds = make_svm_folds(labels, num_folds)
    correct, iters = _svm_correct(solve, kernels, K, C, tol, max_iter, shrinking, folds, return_iters)
    scores = correct.cpu().numpy().astype(np.float64) / folds.n_test[None, :]   # accuracy_score per fold
    acc = scores.mean(axis=1)                                                   # cross_val_score(...).mean()
    return (acc, iters.cpu().numpy()) if return_iters else acc


def svm_cv_precomputed(K, labels, num_folds, C=1.0, tol=1e-3, max_iter=-1, folds=None, return_iters=False,
                       shrinking=False):
    """Mean cross-validation accuracy of ``SVC(kernel='precomputed', C, tol, shrinking)`` for every kernel of
    ``K`` (float32 CUDA ``[nv, E, E]``), computed by the batched GPU SMO solver.  Equivalent to
    ``cross_val_score(clf, K[v], y=labels, cv=StratifiedKFold(num_folds)).mean()`` per voxel; more than two classes are
    handled one-vs-one with libsvm's vote; ``shrinking`` selects the restatement of libsvm's shrinking heuristic.
    E <= 64 runs fcma_svm_cv_solve on ``make_svm_folds`` problems, 64 < E <= 256 fcma_svm_cv_solve_wide on
    ``make_svm_folds_wide`` problems (``folds``, when given, must be of that form)."""
    lib = _lib.load()
    E = K.shape[1]
    wide = E > 64
    if folds is None:
        folds = svm_folds_for(labels, num_folds, E)
    elif folds.wide != wide:
        raise ValueError("%d epochs need %s folds" % (E, "make_svm_folds_wide" if wide else "make_svm_folds"))
    solve = lib.fcma_svm_cv_solve_wide if wide else lib.fcma_svm_cv_solve
    return _svm_cv(solve, (_ptr(K),), K, labels, num_folds, C, tol, max_iter, shrinking, folds, return_iters)


def svm_cv_f64(K_fit, K_pred, labels, num_folds, C=1.0, tol=1e-3, max_iter=-1, shrinking=True, folds=None,
               return_iters=False):
    """``svm_cv_precomputed`` on fp64 kernels: ``K_fit`` / ``K_pred`` float64 CUDA ``[nv, E, E]`` (``K_pred`` may be
    ``K_fit``).  The solver keeps Q in float and QD, the gradient and the decisions in double with QD and the decisions
    read from the double kernels, which is what libsvm computes for ``SVC(kernel='linear' | 'rbf')`` on features whose
    fp64 kernel values these are (see k_searchlight_kernels).  The form of ``folds`` picks the solver:
    ``make_svm_folds`` problems (the default, at most 64 epochs) run fcma_svm_cv_solve_f64, ``make_svm_folds_wide`` /
    ``svm_folds_for`` problems fcma_svm_cv_solve_f64_wide (up to ``SVM_WIDE_MAX_EPOCHS``)."""
    lib = _lib.load()
    if K_fit.dtype != torch.float64 or K_pred.dtype != torch.float64 or K_fit.shape != K_pred.shape \
            or K_fit.dim() != 3 or K_fit.shape[1] != K_fit.shape[2]:
        raise ValueError("K_fit and K_pred must be float64 [nv, E, E] of the same shape")
    if not (K_fit.is_contiguous() and K_pred.is_contiguous()):
        raise ValueError("K_fit and K_pred must be contiguous")
    solve = lib.fcma_svm_cv_solve_f64_wide if folds is not None and folds.wide else lib.fcma_svm_cv_solve_f64
    return _svm_cv(solve, (_ptr(K_fit), _ptr(K_pred)), K_fit, labels, num_folds, C, tol, max_iter, shrinking, folds,
                   return_iters)


def _check_gd(G, D):
    if G.dtype != torch.float64 or D.dtype != torch.float64 or G.shape != D.shape or G.dim() != 3 \
            or G.shape[1] != G.shape[2] or not (G.is_contiguous() and D.is_contiguous()):
        raise ValueError("G and D must be contiguous float64 [n, E, E] of the same shape")


def fold_gammas(moments, train, nfeat):
    """scikit-learn's ``gamma='scale'`` per (item, fold) from per-sample moments (fcma_fold_gammas): ``moments`` float64
    CUDA ``[n, E, 4]`` (``feature_gram_wide`` / ``searchlight_gram_wide``), ``train`` uint8 ``[num_folds, E]``
    (``fold_train_mask``), ``nfeat`` the feature count: a number, or one per item.  Returns ``(gamma, flagged)``: float64
    and bool CUDA ``[n, num_folds]``; ``flagged`` marks where NumPy's two-pass variance may differ from the exact one by
    more than a few ulps (DESIGN.md §3.9)."""
    lib = _lib.load()
    if moments.dtype != torch.float64 or moments.dim() != 3 or moments.shape[2] != 4 or not moments.is_contiguous():
        raise ValueError("moments must be contiguous float64 [n, E, 4]")
    n, E, _ = moments.shape
    train = np.ascontiguousarray(train, dtype=np.uint8)
    if train.ndim != 2 or train.shape[1] != E:
        raise ValueError("train must be [num_folds, %d]" % E)
    nf = np.asarray(nfeat, dtype=np.int64)
    if nf.ndim > 1 or (nf.ndim == 1 and len(nf) != n) or (nf < 1).any():
        raise ValueError("nfeat must be a positive number or one per item (%d)" % n)
    nfeat_dev = torch.from_numpy(nf).to(moments.device) if nf.ndim == 1 else None
    nfolds = train.shape[0]
    gamma = torch.empty((n, nfolds), dtype=torch.float64, device=moments.device)
    flag = torch.empty((n, nfolds), dtype=torch.uint8, device=moments.device)
    with torch.cuda.device(moments.device):
        _lib.check(lib.fcma_fold_gammas(_ptr(moments), n, E, nfolds, train.ctypes.data_as(ctypes.c_void_p),
                                        _ptr(nfeat_dev) if nfeat_dev is not None else None,
                                        int(nf) if nf.ndim == 0 else 0, _ptr(gamma), _ptr(flag), _stream_ptr()))
    return gamma, flag.bool()


def rbf_fold_kernels(G, D, gamma, fold, out=None):
    """rbf kernels of fold ``fold`` (fcma_rbf_fold_kernels): ``K_fit = exp(-g ((G_aa + G_bb) - 2 G_ab))`` and
    ``K_pred = exp(-g D)`` with ``g = gamma[item, fold]`` (float64 CUDA ``[n, num_folds]``), written out of place into
    ``out = (K_fit, K_pred)`` (float64 ``[n, E, E]``, allocated if None) and returned.  The operations of
    ``feature_kernels_f64_wide``'s rbf epilogue: the same bits for the same gamma."""
    lib = _lib.load()
    _check_gd(G, D)
    n, E, _ = G.shape
    if gamma.dtype != torch.float64 or gamma.dim() != 2 or gamma.shape[0] != n or not gamma.is_contiguous():
        raise ValueError("gamma must be contiguous float64 [n, num_folds]")
    if out is None:
        out = (torch.empty_like(G), torch.empty_like(G))
    K_fit, K_pred = out
    _check_gd(K_fit, K_pred)
    if K_fit.shape != G.shape:
        raise ValueError("out must be two float64 [n, E, E] tensors")
    with torch.cuda.device(G.device):
        _lib.check(lib.fcma_rbf_fold_kernels(_ptr(G), _ptr(D), n, E, _ptr(gamma), gamma.shape[1], int(fold), _ptr(K_fit),
                                             _ptr(K_pred), _stream_ptr()))
    return K_fit, K_pred


def svm_cv_scale(G, D, moments, nfeat, labels, num_folds, C=1.0, tol=1e-3, max_iter=-1, shrinking=True, folds=None,
                 return_iters=False):
    """Mean cross-validation accuracy of ``SVC(kernel='rbf', gamma='scale', C, tol, shrinking)`` for every item of a
    block of ``feature_gram_wide`` / ``searchlight_gram_wide`` outputs (``nfeat`` features, a number or one per item):
    per fold f, the gamma of the fold's training samples (``fold_gammas``), that fold's kernels (``rbf_fold_kernels``, one
    ``[n, E, E]`` pair reused from fold to fold) and the fp64 solver on that fold's problems only; the ``[n, num_folds]``
    accuracies are averaged as ``cross_val_score(...).mean()``.  ``folds``: ``svm_folds_for`` problems (the default).
    Returns ``(acc, flagged)``: float64 ``[n]`` and the bool ``[n]`` mask of items whose gamma may differ from
    scikit-learn's (``fold_gammas``) -- score those on the host.  ``return_iters``: also the int32 ``[n, nproblems]``
    iteration counts."""
    lib = _lib.load()
    _check_gd(G, D)
    n, E, _ = G.shape
    if folds is None:
        folds = svm_folds_for(labels, num_folds, E)
    gamma, flag = fold_gammas(moments, fold_train_mask(folds, E), nfeat)
    solve = lib.fcma_svm_cv_solve_f64_wide if folds.wide else lib.fcma_svm_cv_solve_f64
    out = (torch.empty_like(G), torch.empty_like(G))
    correct, iters = [], []
    for f in range(folds.num_folds):
        K_fit, K_pred = rbf_fold_kernels(G, D, gamma, f, out=out)
        c, it = _svm_correct(solve, (_ptr(K_fit), _ptr(K_pred)), K_fit, C, tol, max_iter, shrinking,
                             fold_problems(folds, f), return_iters)
        correct.append(c)
        iters.append(it)
    scores = torch.cat(correct, dim=1).cpu().numpy().astype(np.float64) / folds.n_test[None, :]
    acc = scores.mean(axis=1)
    flagged = flag.any(dim=1).cpu().numpy()
    if return_iters:
        return acc, flagged, torch.cat(iters, dim=1).cpu().numpy()
    return acc, flagged


# ------------------------------------------------------------------ searchlight (MVPAVoxelSelector)
def searchlight_centres(mask, sl_rad, shape, min_active=0):
    """Centres of the reference's searchlight (searchlight.py:542-578) over a 3-D ``mask``: the mask voxels at least
    ``sl_rad`` from every face whose cube satisfies ``count(mask & shape) / cube.size > min_active`` (no test when
    ``min_active == 0``).  Returns ``(centres, n_features)``: int64 linear indices into ``mask`` in C order, and the
    number of features (voxels of ``mask & shape`` in the cube) of each."""
    from scipy import ndimage
    mask = np.asarray(mask).astype(bool)
    shape = np.asarray(shape).astype(bool)
    r = int(sl_rad)
    if mask.ndim != 3 or shape.shape != (2 * r + 1,) * 3:
        raise ValueError("mask must be 3-D and shape (2*sl_rad+1)^3")
    # counts[c] = sum_o mask[c - r + o] * shape[o]: an integer correlation centred on the cube
    counts = ndimage.correlate(mask.astype(np.int32), shape.astype(np.int32), mode="constant", cval=0)
    inner = np.zeros_like(mask)
    if all(n > 2 * r for n in mask.shape):
        inner[tuple(slice(r, n - r) for n in mask.shape)] = True
    sel = mask & inner
    if min_active != 0:
        sel &= (counts / shape.size) > min_active
    centres = np.flatnonzero(sel).astype(np.int64)
    return centres, counts.ravel()[centres].astype(np.int64)


def searchlight_used_voxels(mask, centres, sl_rad, shape):
    """Boolean volume of the voxels that are a feature of at least one of ``centres``."""
    from scipy import ndimage
    mask = np.asarray(mask).astype(bool)
    ind = np.zeros(mask.size, dtype=np.int32)
    ind[np.asarray(centres, dtype=np.int64)] = 1
    # used[v] = sum_o ind[v + r - o] * shape[o]  (v = c - r + o)
    cover = ndimage.convolve(ind.reshape(mask.shape), np.asarray(shape).astype(np.int32), mode="constant", cval=0)
    return mask & (cover > 0)


def searchlight_kernels(vol, mask, sl_rad, shape, centres, kind="linear", gamma=None):
    """fp64 kernel matrices of searchlight centres (k_searchlight_kernels): ``vol`` float32 CUDA ``[X, Y, Z, E]``,
    1 <= E <= 64, ``mask`` / ``shape`` uint8 (or bool) CUDA volumes, ``centres`` int64 host indices
    (``searchlight_centres``).  ``kind='linear'``: returns ``(G, G)``; ``kind='rbf'`` with one ``gamma`` per centre:
    ``(K_fit, K_pred)``, the x_square form libsvm trains with and the difference form its decisions use.  Both float64
    ``[M, E, E]``."""
    return _searchlight_kernels(_lib.load().fcma_searchlight_kernels, vol, mask, sl_rad, shape, centres, kind, gamma)


def searchlight_kernels_wide(vol, mask, sl_rad, shape, centres, kind="linear", gamma=None):
    """``searchlight_kernels`` for 1 <= E <= 256 (k_searchlight_kernels_tiled): the same arguments and outputs, and
    every entry the value ``searchlight_kernels`` gives for the same two epochs' features."""
    return _searchlight_kernels(_lib.load().fcma_searchlight_kernels_wide, vol, mask, sl_rad, shape, centres, kind,
                                gamma)


def _searchlight_kernels(entry, vol, mask, sl_rad, shape, centres, kind, gamma):
    """The body of searchlight_kernels and searchlight_kernels_wide around one call of the C entry point ``entry``."""
    if vol.dim() != 4 or vol.dtype != torch.float32 or not vol.is_contiguous():
        raise ValueError("vol must be a contiguous float32 [X, Y, Z, E] tensor")
    X, Y, Z, E = vol.shape
    if tuple(mask.shape) != (X, Y, Z):
        raise ValueError("mask shape %s does not match the volume %s" % (tuple(mask.shape), (X, Y, Z)))
    side = 2 * int(sl_rad) + 1
    if tuple(shape.shape) != (side, side, side):
        raise ValueError("shape must be (2*sl_rad+1)^3")
    mask = mask.to(device=vol.device, dtype=torch.uint8).contiguous()
    shape = shape.to(device=vol.device, dtype=torch.uint8).contiguous()
    c = np.ascontiguousarray(centres, dtype=np.int64)
    M = len(c)
    if kind not in ("linear", "rbf"):
        raise ValueError("kind must be 'linear' or 'rbf', not %r" % (kind,))
    kcode = 0 if kind == "linear" else 1
    g = None
    if kcode == 1:
        if gamma is None:
            raise ValueError("kind='rbf' needs gamma (a number or one per centre)")
        g = np.asarray(gamma, dtype=np.float64)
        if g.ndim > 1 or (g.ndim == 1 and len(g) != M):
            raise ValueError("gamma must be a number or one value per centre (%d)" % M)
        if not (np.isfinite(g).all() and (g >= 0).all()):
            raise ValueError("gamma must be finite and non-negative")
        g = np.ascontiguousarray(np.broadcast_to(g, (M,)))
    K_fit = torch.empty((M, E, E), dtype=torch.float64, device=vol.device)
    K_pred = K_fit if kcode == 0 else torch.empty_like(K_fit)
    with torch.cuda.device(vol.device):
        _lib.check(entry(_ptr(vol), X, Y, Z, E, _ptr(mask), int(sl_rad), _ptr(shape), c.ctypes.data_as(ctypes.c_void_p),
                         M, kcode, g.ctypes.data_as(ctypes.c_void_p) if g is not None else None, _ptr(K_fit),
                         _ptr(K_pred) if kcode == 1 else None, _stream_ptr()))
    return K_fit, K_pred


def searchlight_gram_wide(vol, mask, sl_rad, shape, centres):
    """The fp64 sums behind ``SVC(kernel='rbf', gamma='scale')`` on searchlight centres (fcma_searchlight_gram_wide, the
    arguments of ``searchlight_kernels_wide``, 1 <= E <= 256): ``(G, D, moments)``, G and D float64 ``[M, E, E]`` -- the
    entries ``searchlight_kernels_wide(kind='rbf')`` exponentiates, bit for bit -- and ``moments`` float64 ``[M, E, 4]``,
    the double-double sums (s.hi, s.lo, q.hi, q.lo) of each epoch's features and their squares in cube order."""
    if vol.dim() != 4 or vol.dtype != torch.float32 or not vol.is_contiguous():
        raise ValueError("vol must be a contiguous float32 [X, Y, Z, E] tensor")
    X, Y, Z, E = vol.shape
    if tuple(mask.shape) != (X, Y, Z):
        raise ValueError("mask shape %s does not match the volume %s" % (tuple(mask.shape), (X, Y, Z)))
    side = 2 * int(sl_rad) + 1
    if tuple(shape.shape) != (side, side, side):
        raise ValueError("shape must be (2*sl_rad+1)^3")
    mask = mask.to(device=vol.device, dtype=torch.uint8).contiguous()
    shape = shape.to(device=vol.device, dtype=torch.uint8).contiguous()
    c = np.ascontiguousarray(centres, dtype=np.int64)
    M = len(c)
    G = torch.empty((M, E, E), dtype=torch.float64, device=vol.device)
    D = torch.empty_like(G)
    moments = torch.empty((M, E, 4), dtype=torch.float64, device=vol.device)
    with torch.cuda.device(vol.device):
        _lib.check(_lib.load().fcma_searchlight_gram_wide(_ptr(vol), X, Y, Z, E, _ptr(mask), int(sl_rad), _ptr(shape),
                                                          c.ctypes.data_as(ctypes.c_void_p), M, _ptr(G), _ptr(D),
                                                          _ptr(moments), _stream_ptr()))
    return G, D, moments
