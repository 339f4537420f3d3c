"""TEST INFRASTRUCTURE — numpy/ctypes face of the CPU restatement in ``fcma_oracle.c``.

Every function cites the reference lines it restates (brainiak/brainiak @ 123f6e1, paths relative
to /root/reference).  Parity status: PINNED — see ``fcma_oracle.c`` and ``tests/test_oracle.py``.
"""
import ctypes
import math
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")
_lib = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("fcma_oracle.c", "svm_oracle.c")]
    if force or not os.path.exists(_LIB_PATH) or \
            os.path.getmtime(_LIB_PATH) < max(os.path.getmtime(f) for f in srcs):
        subprocess.check_call(["make", "-C", _HERE, "liboracle.so"],
                              stdout=subprocess.DEVNULL)
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(_LIB_PATH)
        _lib.oracle_num_threads.restype = ctypes.c_int
    return _lib


def _fptr(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def _ptr_array(mats):
    arr = (ctypes.POINTER(ctypes.c_float) * len(mats))()
    for k, m in enumerate(mats):
        arr[k] = _fptr(m)
    return arr


def _check_epochs(mats):
    out = []
    for m in mats:
        m = np.ascontiguousarray(m, dtype=np.float32)
        out.append(m)
    return out


def num_threads():
    return lib().oracle_num_threads()


def corr_block(raw, raw2, start, nb, layout=0, f64=False):
    """a4 — voxelselector.py:307-323 / classifier.py:166-178 (cython_blas.pyx:115-116, 477-478).

    Returns corr[nb, E, V2] (layout 0) or corr[E, nb, V2] (layout 1).
    """
    raw = _check_epochs(raw)
    raw2 = raw if raw2 is None else _check_epochs(raw2)
    E = len(raw)
    V = raw[0].shape[1]
    V2 = raw2[0].shape[1]
    T = (ctypes.c_int * E)(*[m.shape[0] for m in raw])
    shape = (nb, E, V2) if layout == 0 else (E, nb, V2)
    out = np.empty(shape, np.float64 if f64 else np.float32)
    fn = lib().oracle_corr_block_f64 if f64 else lib().oracle_corr_block
    fn(_ptr_array(raw), _ptr_array(raw2), T, ctypes.c_int(E), ctypes.c_long(V),
       ctypes.c_long(V2), ctypes.c_long(start), ctypes.c_long(nb), ctypes.c_int(layout),
       out.ctypes.data_as(ctypes.c_void_p))
    return out


def within_subject_norm(corr, eps):
    """a6 — fcma_extension.cc:29-86, in place on a C-contiguous float32 [n0, E, n2] array."""
    if corr.ndim != 3:
        raise RuntimeError("The multi-subject correlation data structure must be 3D")
    assert corr.dtype == np.float32 and corr.flags.c_contiguous
    n0, E, n2 = corr.shape
    lib().oracle_within_subject_norm(_fptr(corr), ctypes.c_long(n0), ctypes.c_int(E),
                                     ctypes.c_long(n2), ctypes.c_int(eps))
    return corr


def kernel_matrices(z, f64=False):
    """a7 — voxelselector.py:400-408 (cython_blas.pyx:197-207), WITHOUT the shrink."""
    assert z.dtype == np.float32 and z.flags.c_contiguous and z.ndim == 3
    nb, E, V2 = z.shape
    K = np.zeros((nb, E, E), np.float64 if f64 else np.float32)
    fn = lib().oracle_kernel_matrices_f64 if f64 else lib().oracle_kernel_matrices
    fn(_fptr(z), ctypes.c_long(nb), ctypes.c_int(E), ctypes.c_long(V2),
       K.ctypes.data_as(ctypes.c_void_p))
    return K


def kernel_matrix_accumulate(z2d, K, beta=1.0):
    """a11 — classifier.py:334-339: K = beta*K + Z Z^T with Z = [E, k]."""
    assert z2d.dtype == np.float32 and z2d.flags.c_contiguous and z2d.ndim == 2
    E, k = z2d.shape
    assert K.shape == (E, E) and K.dtype == np.float32 and K.flags.c_contiguous
    lib().oracle_kernel_matrix(_fptr(z2d), ctypes.c_int(E), ctypes.c_long(k),
                               ctypes.c_float(beta), _fptr(K))
    return K


def num_digits(k00):
    """voxelselector.py:409 / classifier.py:343: len(str(int(K[0, 0])))."""
    return len(str(int(k00)))


def shrink_(K):
    """voxelselector.py:409-412: in-place decimal shrink of ONE [E, E] float32 matrix."""
    nd = num_digits(K[0, 0])
    if nd > 2:
        K *= 10 ** (2 - nd)
    return nd


def epoch_normalize(mat):
    """a14 — preprocessing.py:80-84 on one [T, V] epoch; returns a new float32 array."""
    out = np.array(mat, dtype=np.float32, order="C", copy=True)
    T, V = out.shape
    lib().oracle_epoch_normalize(_fptr(out), ctypes.c_int(T), ctypes.c_long(V))
    return out


def epoch_normalize_numpy(mat):
    """a14 in plain numpy float32, mirroring scipy.stats.zscore(axis=0, ddof=0) + nan_to_num."""
    mat = np.asarray(mat, dtype=np.float32)
    mn = mat.mean(axis=0, keepdims=True)
    sd = mat.std(axis=0, ddof=0, keepdims=True)
    with np.errstate(invalid="ignore", divide="ignore"):
        z = (mat - mn) / sd
    z = np.nan_to_num(z)
    return (z / math.sqrt(mat.shape[0])).astype(np.float32)


def voxel_block(raw, raw2, start, nb, eps, shrink=True):
    """a4 -> a6 -> a7 for one task: returns (corr_raw, corr_norm, kernels[nb, E, E])."""
    r = corr_block(raw, raw2, start, nb, layout=0)
    z = within_subject_norm(r.copy(), eps)
    K = kernel_matrices(z)
    if shrink:
        for i in range(nb):
            shrink_(K[i])
    return r, z, K


def classifier_kernel(X1, X2, eps, num_processed_voxels, shrink=True):
    """a9 -> a10 -> a11 — classifier.py:279-348.  Returns (K[E, E], num_digits)."""
    E = len(X1)
    V1 = X1[0].shape[1]
    V2 = X2[0].shape[1]
    K = np.zeros((E, E), np.float32)
    sr = 0
    while sr < V1:
        rows = min(num_processed_voxels, V1 - sr)
        c = corr_block(X1, X2, sr, rows, layout=1)          # [E, rows, V2]
        if eps > 1:                                          # classifier.py:204
            within_subject_norm(c.reshape(1, E, rows * V2), eps)
        kernel_matrix_accumulate(c.reshape(E, rows * V2), K, beta=1.0)
        sr += rows
    nd = num_digits(K[0, 0])
    if shrink and nd > 2:
        K *= 10 ** (2 - nd)
    return K, nd


def compute_correlation(m1, m2, return_nans=False):
    """a15 — util.py:63-134 in float64 numpy (for tolerance checks, not bit parity)."""
    def norm(d):
        d = np.asarray(d, np.float32).astype(np.float64)
        mn = d.mean(axis=1, keepdims=True)
        sd = d.std(axis=1, keepdims=True)
        with np.errstate(invalid="ignore", divide="ignore"):
            z = (d - mn) / sd
        if not return_nans:
            z = np.nan_to_num(z)
        return z / math.sqrt(d.shape[1])
    return (norm(m1) @ norm(m2).T).astype(np.float32)


def svm_smo(K, train_idx, n_pos, C=1.0, tol=1e-3, max_iter=-1, shrinking=False):
    """One two-class C-SVC problem on the precomputed kernel ``K`` ([E, E] float32): training samples ``train_idx`` with the
    ``n_pos`` samples of class +1 first.  Restates scikit-learn's libsvm solver (svm_oracle.c; the reference reaches it through
    voxelselector.py:41-53).  Returns (alpha in the order of train_idx, rho, iterations)."""
    K = np.ascontiguousarray(K, dtype=np.float32)
    idx = np.ascontiguousarray(train_idx, dtype=np.int32)
    alpha = np.zeros(len(idx), np.float64)
    rho = ctypes.c_double(0)
    f = lib().oracle_svm_smo
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.POINTER(ctypes.c_float), ctypes.c_int, ctypes.POINTER(ctypes.c_int), ctypes.c_int, ctypes.c_int,
                  ctypes.c_double, ctypes.c_double, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_double),
                  ctypes.POINTER(ctypes.c_double)]
    it = f(_fptr(K), K.shape[0], idx.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), len(idx), int(n_pos), float(C), float(tol),
           int(max_iter), 1 if shrinking else 0, alpha.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), ctypes.byref(rho))
    if it < 0:
        raise ValueError("svm_smo: 2 <= n <= 64 training samples of both classes are required")
    return alpha, rho.value, it


def svm_last_stats():
    """(smallest active set, gradient reconstructions) of the last svm_smo call: whether the shrinking heuristic acted."""
    a, b = ctypes.c_int(0), ctypes.c_int(0)
    lib().oracle_svm_last_stats(ctypes.byref(a), ctypes.byref(b))
    return a.value, b.value


def svm_last_detail():
    """(reconstructions reading Q by rows, by columns, active set at the end) of the last svm_smo call: which loop orders
    of libsvm's reconstruct_gradient ran, and whether a max_iter cut left variables shrunk."""
    a, b, c = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_int(0)
    lib().oracle_svm_last_detail(ctypes.byref(a), ctypes.byref(b), ctypes.byref(c))
    return a.value, b.value, c.value


def svm_cv(K, labels, num_folds, C=1.0, tol=1e-3, shrinking=False):
    """cross_val_score(SVC(kernel='precomputed', C, tol, shrinking), K, labels, cv=StratifiedKFold(num_folds)) restated:
    scikit-learn's own splits, one-vs-one problems for more than two classes (pairs in libsvm's order, the smaller label is
    class +1), libsvm's vote (first maximum).  Returns (mean accuracy, iterations per (fold, pair))."""
    from sklearn import model_selection
    K = np.ascontiguousarray(K, dtype=np.float32)
    y = np.asarray(labels)
    classes = np.unique(y)
    code = np.searchsorted(classes, y)
    k = len(classes)
    pairs = [(a, b) for a in range(k) for b in range(a + 1, k)]
    skf = model_selection.StratifiedKFold(n_splits=num_folds, shuffle=False)
    scores, iters = [], []
    for tr, te in skf.split(np.zeros((len(y), 1)), y):
        votes = np.zeros((len(te), k), np.int64)
        for a, b in pairs:
            pos = [int(i) for i in tr if code[i] == a]
            neg = [int(i) for i in tr if code[i] == b]
            alpha, rho, it = svm_smo(K, pos + neg, len(pos), C, tol, -1, shrinking)
            iters.append(it)
            idx = np.asarray(pos + neg)
            coef = alpha * np.r_[np.ones(len(pos)), -np.ones(len(neg))]
            for t, i in enumerate(te):
                dec = 0.0
                for k in np.flatnonzero(alpha != 0):      # libsvm's svm_predict_values: training order, one by one
                    dec = dec + float(coef[k]) * float(K[i, idx[k]])
                dec -= rho
                votes[t, a if dec > 0 else b] += 1
        pred = np.argmax(votes, axis=1)          # first maximum, as libsvm
        scores.append(float(np.mean(pred == code[te])))
    return float(np.mean(scores)), iters
