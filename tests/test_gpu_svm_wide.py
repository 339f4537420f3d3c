"""Decision-by-decision tests of the wide batched SVM solver -- ``fcma_svm_cv_solve_wide``, ``k_svm_cv<float, SHRINK,
NS>`` with NS = 4 (no problem of the launch wider than 128) and NS = 8, Q read from the kernel in global memory --
against libsvm, as scikit-learn runs it, and of ``VoxelSelector`` above 64 epochs against its host path.

As in test_gpu_svm_solver.py nothing is compared under a tolerance: ``iters`` equals ``n_iter_`` of
``SVC(kernel='precomputed')`` fitted per problem on float64 copies of the float32 kernels, bit t of every problem equals
libsvm's side of held-out sample t (bit t % 64 of word t // 64), and ``correct`` counts the bits that match ``test_pos``.

| edge                                                                | covered by                                      |
|---------------------------------------------------------------------|-------------------------------------------------|
| n_train 2 .. 256 across the slot and word edges, n_pos 1, 31, 32, 33, 64, 65, n - 1; n_test 0, 1, 64, 65, 128, 129, 256; held-out indices that are training indices; NS = 4 and 8 | test_shapes_in_one_launch |
| long problems (several hundred iterations, asymmetric kernels; the CPU oracle that shows the shrinking acting stops at 64 samples), max_iter 0, 1, n, n + 1 | test_long_problems_and_max_iter |
| one-vs-one, 3 and 4 classes, held-out sets of 4 words               | test_multiclass_one_vs_one                      |
| decisions summed in training order at n_train > 64                  | test_order_rows; CPU: test_crafted_order_rows_are_order_sensitive |
| the wide entry point equals fcma_svm_cv_solve at E <= 64            | test_wide_equals_narrow                         |
| VoxelSelector, 65 .. 256 epochs, GPU against the host path          | test_voxel_selector_wide                        |
"""
import ctypes
import functools
import warnings

import numpy as np
import pytest
from sklearn import svm
from sklearn.exceptions import ConvergenceWarning

from brainiak_b200 import _lib
from brainiak_b200.fcma import engine


def _fold(pos, neg, test, truth=None, struct=engine._SvmFoldWide):
    fd = struct()
    order = [int(i) for i in pos] + [int(i) for i in neg]
    fd.n_train, fd.n_pos, fd.n_test = len(order), len(pos), len(test)
    for j, i in enumerate(order):
        fd.train_idx[j] = i
    for j, i in enumerate(test):
        fd.test_idx[j] = int(i)
        fd.test_pos[j] = int(truth[j]) if truth is not None else 0
    return fd


def _parts(fd):
    tr = [fd.train_idx[k] for k in range(fd.n_train)]
    te = [fd.test_idx[t] for t in range(fd.n_test)]
    y = np.r_[np.zeros(fd.n_pos, np.int64), np.ones(fd.n_train - fd.n_pos, np.int64)]
    return tr, te, y


def _fit(K, tr, y, C, tol, max_iter, shrinking, **kw):
    clf = svm.SVC(kernel="precomputed", C=C, tol=tol, shrinking=shrinking, max_iter=max_iter, **kw)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        clf.fit(np.asarray(K, np.float64)[np.ix_(tr, tr)], y)
    return clf


def _libsvm(K, fd, C, tol, max_iter, shrinking):
    tr, te, y = _parts(fd)
    clf = _fit(K, tr, y, C, tol, max_iter, shrinking)
    bits = 0
    if te:
        first = clf.predict(np.asarray(K, np.float64)[np.ix_(te, tr)]) == 0
        bits = sum(1 << t for t in range(len(te)) if first[t])
    return int(clf.n_iter_[0]), bits


def _solve(K, folds, C=1.0, tol=1e-3, max_iter=-1, shrinking=False, wide=True):
    """One launch of fcma_svm_cv_solve_wide (or fcma_svm_cv_solve) on float32 [nv, E, E]: (bits as Python ints,
    iters, correct), each [nv][nproblems]."""
    import torch
    lib = _lib.load()
    dev = torch.device("cuda:0")
    nv, E, _ = K.shape
    nprob = len(folds)
    struct = engine._SvmFoldWide if wide else engine._SvmFold
    arr = (struct * nprob)(*folds)
    words = 4 if wide else 1
    bits = torch.full((nv, nprob, words), -1, dtype=torch.int64, device=dev)
    iters = torch.full((nv, nprob), -7, dtype=torch.int32, device=dev)
    correct = torch.full((nv, nprob), -7, dtype=torch.int32, device=dev)
    Kd = torch.from_numpy(np.ascontiguousarray(K, np.float32)).to(dev)
    solve = lib.fcma_svm_cv_solve_wide if wide else lib.fcma_svm_cv_solve
    _lib.check(solve(Kd.data_ptr(), nv, E, nprob, ctypes.cast(arr, ctypes.c_void_p), float(C), float(tol), int(max_iter),
                     int(shrinking), correct.data_ptr(), bits.data_ptr(), iters.data_ptr(), None))
    torch.cuda.synchronize()
    b = bits.cpu().numpy().view(np.uint64)
    out = [[sum(int(b[v, p, w]) << (64 * w) for w in range(words)) for p in range(nprob)] for v in range(nv)]
    return out, iters.cpu().numpy(), correct.cpu().numpy()


def _check(K, folds, C=1.0, tol=1e-3, max_iter=-1, shrinking=False):
    K = np.asarray(K, np.float32)
    bits, iters, correct = _solve(K, folds, C, tol, max_iter, shrinking)
    bad = []
    for v in range(K.shape[0]):
        for p, fd in enumerate(folds):
            it, ref = _libsvm(K[v], fd, C, tol, max_iter, shrinking)
            truth = sum(1 << t for t in range(fd.n_test) if fd.test_pos[t])
            ok = fd.n_test - bin((bits[v][p] ^ truth) & ((1 << fd.n_test) - 1)).count("1")
            if iters[v, p] != it or bits[v][p] != ref or correct[v, p] != ok:
                bad.append((v, p, fd.n_train, fd.n_pos, fd.n_test, int(iters[v, p]), it, hex(bits[v][p] ^ ref),
                            int(correct[v, p]), ok))
    assert not bad, "%d of %d problems differ from libsvm (v, p, n, n_pos, n_test, iters, n_iter_, bits ^ libsvm, " \
                    "correct, expected): %s" % (len(bad), K.shape[0] * len(folds), bad[:8])
    return iters


def _kernels(rng, nv, E, signal, dims=(3, 10, 40)):
    Ks = []
    for _ in range(nv):
        X = rng.randn(E, int(rng.choice(dims)))
        X[:, 0] += signal
        Xf = X.astype(np.float32).astype(np.float64)
        Ks.append((Xf @ Xf.T).astype(np.float32))
    return np.array(Ks)


# ------------------------------------------------------------------------------------------- shapes
N_TRAIN = (2, 33, 64, 65, 96, 127, 128, 129, 224, 255, 256)
N_POS = (1, 31, 32, 33, 64, 65)
N_TEST = (0, 1, 64, 65, 128, 129, 256)


def _shape_folds(rng, E, signal, limit):
    folds = []
    for n in (n for n in N_TRAIN if n <= limit):
        for n_pos in sorted({p for p in N_POS + (n - 1,) if 1 <= p <= n - 1}):
            for n_test in (t for t in N_TEST if t <= limit):
                pref = np.argsort(-signal + 0.8 * rng.randn(E), kind="stable")
                tr = [int(i) for i in (pref[:n] if rng.rand() < 0.5 else rng.permutation(E)[:n])]
                pos = sorted(tr[:n_pos]) if rng.rand() < 0.5 else tr[:n_pos]
                te = rng.choice(E, n_test, replace=False)        # overlaps the training samples
                folds.append(_fold(pos, tr[n_pos:], te, [1 if signal[i] > 0 else 0 for i in te]))
    return folds


@pytest.mark.gpu
@pytest.mark.parametrize("shrinking", [False, True])
@pytest.mark.parametrize("limit", [128, 256], ids=["NS4", "NS8"])
def test_shapes_in_one_launch(shrinking, limit):
    """Every shape up to ``limit`` samples in one launch of 2 kernels: warps of a block on different shapes, a partial
    last block; limit 128 runs the 4-slot instantiation, 256 the 8-slot one."""
    rng = np.random.RandomState(13 + 2 * shrinking + limit)
    E = 256
    signal = rng.choice([-0.7, 0.7], size=E)
    K = _kernels(rng, 2, E, signal)
    folds = _shape_folds(rng, E, signal, limit)
    if len(folds) % 2 == 0:
        folds.append(folds[-1])
    iters = _check(K, folds, shrinking=shrinking)
    assert iters.min() >= 1


# ------------------------------------------------------------------------------------------- long problems, max_iter
@functools.lru_cache(maxsize=None)
def _long_problems():
    """Overlapping classes, C = 1, 200 training samples: several hundred iterations; kernels 2 and 3 are kernels 0 and 1
    with an asymmetric perturbation, which tells the two loop orders of reconstruct_gradient apart.  Held out: the 56
    others and 24 training samples."""
    rng = np.random.RandomState(7)
    E, n, n_pos = 256, 200, 97
    signal = np.r_[np.full(n_pos, 0.6), np.full(n - n_pos, -0.6), np.zeros(E - n)]
    K = _kernels(rng, 2, E, signal, dims=(20, 40))
    K = np.concatenate([K, (K + 0.05 * rng.randn(*K.shape)).astype(np.float32)])
    te = list(range(n, E)) + list(range(0, 12)) + list(range(n_pos, n_pos + 12))
    truth = [1 if i < n_pos else 0 for i in te]
    return K, _fold(range(n_pos), range(n_pos, n), te, truth)


@pytest.mark.gpu
@pytest.mark.parametrize("shrinking", [False, True])
def test_long_problems_and_max_iter(shrinking):
    """Several hundred iterations to convergence, and cut at max_iter 0, 1, n and n + 1 (the first do_shrinking)."""
    K, fold = _long_problems()
    iters = _check(K, [fold] * 3, shrinking=shrinking)
    assert iters.max() >= 300
    for cut in (0, 1, 200, 201):
        iters = _check(K, [fold], max_iter=cut, shrinking=shrinking)
        assert np.all(iters <= cut)


# ------------------------------------------------------------------------------------------- one-vs-one
@pytest.mark.gpu
@pytest.mark.parametrize("shrinking", [False, True])
@pytest.mark.parametrize("nclass", [3, 4])
def test_multiclass_one_vs_one(shrinking, nclass):
    """One problem per class pair, evaluated on all 256 samples (4 words), bits against the sign of libsvm's per-pair
    decision, iterations against n_iter_ per pair."""
    rng = np.random.RandomState(43 + nclass + 2 * shrinking)
    E = 256
    lab = rng.permutation(np.arange(E) % nclass)
    K = _kernels(rng, 2, E, signal=0.8 * lab - 0.8)
    pairs = [(a, b) for a in range(nclass) for b in range(a + 1, nclass)]
    tr = np.sort(rng.permutation(E)[:200])
    te = np.arange(E)
    folds = [_fold([i for i in tr if lab[i] == a], [i for i in tr if lab[i] == b], te,
                   [1 if lab[i] == a else 0 for i in te]) for a, b in pairs]
    bits, iters, _ = _solve(K, folds, C=0.7, shrinking=shrinking)
    for v in range(len(K)):
        clf = _fit(K[v], tr, lab[tr], 0.7, 1e-3, -1, shrinking, decision_function_shape="ovo")
        dec = clf.decision_function(np.asarray(K[v], np.float64)[np.ix_(te, tr)])
        assert np.array_equal(iters[v], clf.n_iter_), (v, iters[v], clf.n_iter_)
        for q in range(len(pairs)):
            ref = sum(1 << t for t in range(len(te)) if dec[t, q] > 0)
            assert bits[v][q] == ref, (v, pairs[q], hex(bits[v][q] ^ ref))


# ------------------------------------------------------------------------------------------- crafted near-tie rows
def _coef(clf, n):
    c = np.zeros(n)
    c[clf.support_] = -clf.dual_coef_[0]
    return c


def _seq_sum(coef, row):
    s = 0.0
    for c, k in zip(coef, row):
        if c != 0.0:
            s = s + float(c) * float(k)
    return s


def _slot_sum(coef, row, ns=8):
    """The same terms in a warp's lane-slot order: lane l adds its slots l + 32 s, then a __shfl_xor butterfly."""
    t = np.zeros(32 * ns)
    for k in range(len(coef)):
        if coef[k] != 0.0:
            t[k] = float(coef[k]) * float(row[k])
    part = []
    for lane in range(32):
        acc = 0.0
        for s in range(ns):
            acc = acc + t[lane + 32 * s]
        part.append(acc)
    for off in (16, 8, 4, 2, 1):
        part = [part[lane] + part[lane ^ off] for lane in range(32)]
    return part[0]


@functools.lru_cache(maxsize=None)
def _order_case(shrinking):
    """Problems of 160 training samples whose held-out rows 160 .. 191 are crafted as in test_gpu_svm_solver.py: two
    bound support vectors of opposite sign with the same value ~2^40 .. 2^60 and a free one whose term is of the order
    of rho, kept where libsvm's sequential sum and the lane-slot order give different sides."""
    rng = np.random.RandomState(99 + shrinking)
    E, n, n_pos = 192, 160, 80
    signal = np.r_[np.full(n_pos, 0.5), np.full(n - n_pos, -0.5), np.zeros(E - n)]
    fold = _fold(range(n_pos), range(n_pos, n), range(n, E), [1] * 16 + [0] * 16)
    tr, _, y = _parts(fold)
    Ks, crafted = [], []
    while len(Ks) < 3:
        K = _kernels(rng, 1, E, signal, dims=(4, 8))[0].copy()
        clf = _fit(K, tr, y, 1.0, 1e-3, -1, shrinking)
        coef = _coef(clf, n)
        rho = float(clf.intercept_[0])
        up, dn = np.flatnonzero(coef == 1.0), np.flatnonzero(coef == -1.0)
        free = np.flatnonzero((coef != 0) & (np.abs(coef) < 1.0))
        if not (len(up) and len(dn) and len(free)) or rho == 0.0:
            continue
        rows = []
        for t in range(n, E):
            for _ in range(400):
                p, q, r = int(rng.choice(up)), int(rng.choice(dn)), int(rng.choice(free))
                row = np.zeros(n, np.float32)
                row[p] = row[q] = np.float32(2.0 ** rng.randint(40, 61) * (1 + rng.randint(0, 1 << 23) / 2 ** 23))
                row[r] = np.float32(rho * (1 + rng.uniform(-1, 1) * 2.0 ** -rng.randint(1, 30)) / coef[r])
                if (_seq_sum(coef, row) - rho > 0) != (_slot_sum(coef, row) - rho > 0):
                    break
            else:
                continue
            rows.append(t)
            K[t, :] = np.r_[row, np.zeros(E - n, np.float32)]      # a held-out row: training never reads it
        if len(rows) < 16:
            continue
        crafted.append(rows)
        Ks.append(K)
    return np.array(Ks, np.float32), fold, crafted


@pytest.mark.parametrize("shrinking", [False, True])
def test_crafted_order_rows_are_order_sensitive(shrinking):
    """Every crafted row: its emulated sequential sum gives scikit-learn's side, the lane-slot order the other."""
    K, fold, crafted = _order_case(shrinking)
    tr, te, y = _parts(fold)
    for v in range(len(K)):
        clf = _fit(K[v], tr, y, 1.0, 1e-3, -1, shrinking)
        coef, rho = _coef(clf, len(tr)), float(clf.intercept_[0])
        pred = clf.predict(np.asarray(K[v], np.float64)[np.ix_(te, tr)])
        for j, t in enumerate(te):
            if t in crafted[v]:
                row = np.asarray(K[v][t, tr], np.float64)
                assert (pred[j] == 0) == (_seq_sum(coef, row) - rho > 0), (v, t)
                assert (_seq_sum(coef, row) - rho > 0) != (_slot_sum(coef, row) - rho > 0), (v, t)


@pytest.mark.gpu
@pytest.mark.parametrize("shrinking", [False, True])
def test_order_rows(shrinking):
    """The decisions summed sequentially in training order at n_train = 160: the crafted rows land on libsvm's side."""
    K, fold, _ = _order_case(shrinking)
    _check(K, [fold], shrinking=shrinking)


# ------------------------------------------------------------------------------------------- wide against narrow
@pytest.mark.gpu
@pytest.mark.parametrize("shrinking", [False, True])
def test_wide_equals_narrow(shrinking):
    """At E <= 64 the wide entry point (4 slots, Q from global memory) gives the narrow solver's bits, iterations and
    counts on the same problems."""
    rng = np.random.RandomState(61 + shrinking)
    E = 64
    signal = rng.choice([-0.7, 0.7], size=E)
    K = _kernels(rng, 5, E, signal)
    K = np.concatenate([K, (K[:2] + 0.05 * rng.randn(2, E, E)).astype(np.float32)])
    narrow, wide = [], []
    for n in (2, 3, 31, 32, 33, 63, 64):
        for n_test in (0, 1, 33, 64):
            n_pos = int(rng.randint(1, n))
            tr = [int(i) for i in rng.permutation(E)[:n]]
            te = rng.choice(E, n_test, replace=False)
            truth = [1 if signal[i] > 0 else 0 for i in te]
            narrow.append(_fold(tr[:n_pos], tr[n_pos:], te, truth, engine._SvmFold))
            wide.append(_fold(tr[:n_pos], tr[n_pos:], te, truth))
    for C, max_iter in ((1.0, -1), (1e3, 500), (0.01, -1)):
        a = _solve(K, narrow, C=C, max_iter=max_iter, shrinking=shrinking, wide=False)
        b = _solve(K, wide, C=C, max_iter=max_iter, shrinking=shrinking)
        assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


# ------------------------------------------------------------------------------------------- VoxelSelector
def _planted(V, T, E, nclass, seed, informative=48):
    """E epochs [T, V]: voxels < informative share a per-epoch component whose amplitude follows the condition."""
    rng = np.random.RandomState(seed)
    labels = [e % nclass for e in range(E)]
    raw = []
    for e in range(E):
        x = rng.randn(T, V).astype(np.float32)
        x[:, :informative] += (0.5 * (labels[e] + 1) * rng.randn(T, 1)).astype(np.float32)
        raw.append(x)
    return raw, labels


@pytest.mark.gpu
@pytest.mark.parametrize("E,eps,folds,nclass,two_masks,shrinking", [
    (140, 20, 7, 2, False, False),      # the reference script's shape
    (140, 20, 7, 2, False, True),
    (140, 20, 7, 3, False, False),
    (140, 20, 7, 2, True, True),
    (65, 13, 5, 2, False, True),
    (256, 16, 16, 2, False, False),
])
def test_voxel_selector_wide(E, eps, folds, nclass, two_masks, shrinking):
    """VoxelSelector.run with gpu_cv=True equals gpu_cv=False as lists above 64 epochs (T = 15, 432 voxels with a
    planted signal)."""
    from brainiak_b200.fcma.voxelselector import VoxelSelector
    raw, labels = _planted(432, 15, E, nclass, seed=E + nclass + 10 * two_masks)
    raw2 = _planted(300, 15, E, nclass, seed=E + 5)[0] if two_masks else None
    clf = svm.SVC(kernel="precomputed", shrinking=shrinking, C=1)
    assert engine.svm_cv_supported(clf, labels, folds, E, max_epochs=256)
    a = VoxelSelector(labels, eps, folds, raw, raw2, voxel_unit=64, process_num=0, gpu_cv=True).run(clf)
    b = VoxelSelector(labels, eps, folds, raw, raw2, voxel_unit=64, process_num=0, gpu_cv=False).run(clf)
    assert a == b
    assert max(acc for _, acc in a) > 1.0 / nclass + 0.1      # the planted voxels stand out from chance
