"""Decision-by-decision tests of the batched SVM solver -- ``k_svm_cv`` without and with shrinking, each on float and
on double kernels -- against libsvm itself, as scikit-learn runs it.

References and bounds
---------------------
* The reference is ``sklearn.svm.SVC(kernel='precomputed', C, tol, shrinking, max_iter)`` fitted per problem on float64
  copies of the same arrays.  Float path (``fcma_svm_cv_solve``): it fits on ``K[train][:, train]`` and predicts
  ``K[test][:, train]``.  Double path (``fcma_svm_cv_solve_f64``): it fits on ``K_fit[train][:, train]`` and predicts
  ``K_pred[test][:, train]``.  The solver restates libsvm's arithmetic, so nothing is compared under a tolerance:
  - ``iters`` of every problem **equals** ``n_iter_``;
  - bit t of ``bits`` of every problem **equals** libsvm's side of held-out sample t, taken from ``predict`` (the
    first class = the pair's class +1 = libsvm's decision > 0; scikit-learn negates the binary ``decision_function``,
    so its sign is not used).  One-vs-one: bit t of the problem of pair (a, b) equals the sign of column (a, b) of
    ``decision_function_shape='ovo'``, whose convention is pinned against ``predict`` by libsvm's vote;
  - ``correct`` equals the number of held-out samples whose bit matches ``test_pos``.
* The problems are built here as ``_SvmFold`` structs, including what ``make_svm_folds`` never produces: n_train = 64,
  n_test = 0 and 64, and held-out indices that are training indices too.
* Crafted held-out rows.  Training reads only ``K[train, train]``, so a held-out row can be set freely: the alphas stay
  the same and only that decision moves.  scikit-learn is given the same rows.
  - rho rows (double path): C a power of two, the row zero except at one bound support vector (``alpha y = +-C``), so
    libsvm's decision sum is exactly rho (``intercept_``) in one row and ``nextafter(rho, inf)`` in the other: libsvm
    puts the first on the second class and the second on the first.  A rho that differs from libsvm's in its last bit
    flips one of the two.
  - order rows (both paths): two bound support vectors of opposite sign with the same K value ~2^40 to 2^60 (exact in
    float32), and one free support vector whose term is of the order of rho.  The rows are picked so that the sign of
    libsvm's sum -- added sequentially in training order, then rho subtracted -- differs from the sign of the same terms
    added in the lane-slot butterfly order of a warp (slot k and k + 32 per lane, then ``__shfl_xor`` 16 ... 1).
  CPU tests (no ``gpu`` mark) check every crafted row against scikit-learn's ``predict`` and the emulated orders, so
  the GPU cases cannot silently stop being near-ties.

Coverage
--------
| instantiation / edge                         | covered by                                                          |
|----------------------------------------------|---------------------------------------------------------------------|
| ``k_svm_cv<float, false>`` / ``<double, false>`` | every GPU test at ``shrinking`` False                             |
| ``k_svm_cv<float, true>`` / ``<double, true>``   | every GPU test at ``shrinking`` True                              |
| n_train 2, 3, 31, 32, 33, 63, 64; n_pos 1, 31, 32, 33, n_train - 1; n_test 0, 1, 31, 32, 33, 64 (bit 63) | test_shapes_in_one_launch |
| warps of a block on different shapes, partial last block (nv nproblems = 3 mod 4) | test_shapes_in_one_launch, test_degenerate_kernels |
| held-out indices that are training indices  | test_shapes_in_one_launch                                          |
| duplicate samples in one class / across the classes (quad = 0: TAU), all-zero, rank-one, indefinite (quad < 0), entries over 1e-12 .. 1e12 of scale | test_degenerate_kernels |
| C 1e-4 (every alpha at the bound: rho from the (ub + lb) / 2 midpoint), 1, 1e4; tol 1e-1, 1e-3, 1e-6 | test_degenerate_kernels |
| several hundred iterations, variables shrunk, ``reconstruct`` by rows and by columns | test_long_problems; CPU: test_long_problems_exercise_shrinking |
| max_iter 0, 1, n, n + 1 (the first do_shrinking), cuts while variables are shrunk | test_max_iter_cuts; CPU: test_oracle_max_iter_cuts_match_sklearn |
| one-vs-one, 3 and 4 classes                  | test_multiclass_one_vs_one                                          |
| rho summed in libsvm's order                  | test_rho_rows (double path); CPU: test_crafted_rho_rows_are_ties    |
| decisions summed in libsvm's order            | test_order_rows; CPU: test_crafted_order_rows_are_order_sensitive   |
| ``max_iter=0`` is 0 iterations in scikit-learn | CPU: test_sklearn_max_iter_zero_runs_no_iteration                   |
"""
import ctypes
import functools
import math
import warnings

import numpy as np
import pytest
from sklearn import svm
from sklearn.exceptions import ConvergenceWarning

from brainiak_b200 import _lib
from brainiak_b200.fcma import engine
from oracle import fcma_oracle as orc

VARIANTS = [("float", False), ("float", True), ("double", False), ("double", True)]
VIDS = ["float", "float-shrink", "double", "double-shrink"]


# ------------------------------------------------------------------------------------------- problems and references
def _fold(pos, neg, test, truth=None):
    """One _SvmFold: training samples ``pos`` (class +1) then ``neg``, held-out samples ``test``; ``truth[t]`` = 1 where
    held-out sample t belongs to class +1 (read only by the ``correct`` output)."""
    fd = engine._SvmFold()
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


def _fit(K_fit, tr, y, C, tol, max_iter, shrinking, **kw):
    clf = svm.SVC(kernel="precomputed", C=C, tol=tol, shrinking=shrinking, max_iter=max_iter, **kw)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        clf.fit(np.asarray(K_fit, np.float64)[np.ix_(tr, tr)], y)
    return clf


def _libsvm(K_fit, K_pred, fd, C=1.0, tol=1e-3, max_iter=-1, shrinking=False):
    """libsvm on one problem: (n_iter_, bits) -- bit t set where held-out sample t is predicted as the first class."""
    tr, te, y = _parts(fd)
    clf = _fit(K_fit, tr, y, C, tol, max_iter, shrinking)
    bits = 0
    if te:
        first = clf.predict(np.asarray(K_pred, np.float64)[np.ix_(te, tr)]) == 0
        bits = sum(1 << t for t in range(len(te)) if first[t])
    return int(clf.n_iter_[0]), bits


def _solve(kt, K_fit, K_pred, folds, C=1.0, tol=1e-3, max_iter=-1, shrinking=False):
    """The solver through its C entry point on [nv, E, E] kernels (float: K_fit only).  Returns (bits as Python ints,
    iters, correct), each [nv][nproblems]."""
    import torch
    lib = _lib.load()
    dev = torch.device("cuda:0")
    nv, E, _ = K_fit.shape
    nprob = len(folds)
    arr = (engine._SvmFold * nprob)(*folds)
    bits = torch.zeros((nv, nprob), dtype=torch.int64, device=dev)
    iters = torch.full((nv, nprob), -7, dtype=torch.int32, device=dev)
    correct = torch.full((nv, nprob), -7, dtype=torch.int32, device=dev)
    if kt == "float":
        Kf = torch.from_numpy(np.ascontiguousarray(K_fit, np.float32)).to(dev)
        rc = lib.fcma_svm_cv_solve(Kf.data_ptr(), nv, E, nprob, ctypes.cast(arr, ctypes.c_void_p), float(C), float(tol),
                                   int(max_iter), int(shrinking), correct.data_ptr(), bits.data_ptr(), iters.data_ptr(),
                                   None)
    else:
        Kf = torch.from_numpy(np.ascontiguousarray(K_fit, np.float64)).to(dev)
        Kp = torch.from_numpy(np.ascontiguousarray(K_pred, np.float64)).to(dev)
        rc = lib.fcma_svm_cv_solve_f64(Kf.data_ptr(), Kp.data_ptr(), nv, E, nprob, ctypes.cast(arr, ctypes.c_void_p),
                                       float(C), float(tol), int(max_iter), int(shrinking), correct.data_ptr(),
                                       bits.data_ptr(), iters.data_ptr(), None)
    _lib.check(rc)
    torch.cuda.synchronize()
    b = bits.cpu().numpy().view(np.uint64)
    return [[int(x) for x in row] for row in b], iters.cpu().numpy(), correct.cpu().numpy()


def _check(kt, K_fit, K_pred, folds, C=1.0, tol=1e-3, max_iter=-1, shrinking=False):
    """GPU against libsvm on every (kernel, problem): iterations, the bit of every held-out sample, and ``correct``."""
    if kt == "float":
        K_fit = np.asarray(K_fit, np.float32)
        K_pred = K_fit
    bits, iters, correct = _solve(kt, K_fit, K_pred, folds, C, tol, max_iter, shrinking)
    bad = []
    for v in range(K_fit.shape[0]):
        for p, fd in enumerate(folds):
            it, ref = _libsvm(K_fit[v], K_pred[v], fd, C, tol, max_iter, shrinking)
            truth = sum(1 << t for t in range(fd.n_test) if fd.test_pos[t])
            mask = (1 << fd.n_test) - 1
            ok = fd.n_test - bin((bits[v][p] ^ truth) & mask).count("1")
            if iters[v, p] != it or bits[v][p] != ref or correct[v, p] != ok:
                bad.append((v, p, fd.n_train, fd.n_pos, fd.n_test, int(iters[v, p]), it,
                            hex(bits[v][p] ^ ref), int(correct[v, p]), ok))
    assert not bad, "%d of %d problems differ from libsvm (v, p, n, n_pos, n_test, iters, n_iter_, bits ^ libsvm, " \
                    "correct, expected): %s" % (len(bad), K_fit.shape[0] * len(folds), bad[:8])
    return iters


def _random_kernels(rng, kt, nv, E, signal=None, dims=(3, 10, 40)):
    """nv kernels of random features (with an optional class signal per sample).  float: the float32 Gram matrix (K_pred
    is K_fit); double: libsvm's two rbf forms as MVPAVoxelSelector builds them -- the x_square form for training, the
    difference form for the decisions."""
    Kf, Kp = [], []
    for _ in range(nv):
        d = int(rng.choice(dims))
        X = rng.randn(E, d)
        if signal is not None:
            X[:, 0] += signal
        if kt == "float":
            Xf = X.astype(np.float32)
            K = (Xf.astype(np.float64) @ Xf.astype(np.float64).T).astype(np.float32)
            Kf.append(K)
            Kp.append(K)
        else:
            g = 1.0 / d
            G = X @ X.T
            dg = np.diag(G)
            Kf.append(np.exp(-g * ((dg[:, None] + dg[None, :]) - 2 * G)))
            Kp.append(np.exp(-g * ((X[:, None, :] - X[None, :, :]) ** 2).sum(-1)))
    dt = np.float32 if kt == "float" else np.float64
    return np.array(Kf, dt), np.array(Kp, dt)


# ------------------------------------------------------------------------------------------- shapes, degenerate kernels
N_TRAIN = (2, 3, 31, 32, 33, 63, 64)
N_TEST = (0, 1, 31, 32, 33, 64)


def _shape_folds(rng, E, signal):
    """Every (n_train, n_pos) of the matrix, each with every n_test: 121 problems (one more with a held-out set equal to
    the training set), training samples of class +1 drawn preferably from signal > 0."""
    folds = []
    for n in N_TRAIN:
        for n_pos in sorted({p for p in (1, 31, 32, 33, n - 1) if 1 <= p <= n - 1}):
            for n_test in N_TEST:
                pref = np.argsort(-signal + 0.8 * rng.randn(E), kind="stable")
                tr = pref[:n] if rng.rand() < 0.5 else rng.permutation(E)[:n]
                tr = [int(i) for i in tr]
                pos = sorted(tr[:n_pos]) if rng.rand() < 0.5 else tr[:n_pos]
                neg = tr[n_pos:]
                te = rng.choice(E, n_test, replace=False)
                truth = [1 if signal[i] > 0 else 0 for i in te]
                folds.append(_fold(pos, neg, te, truth))
    tr = rng.permutation(E)[:40]
    folds.append(_fold(tr[:17], tr[17:], tr, [1] * 17 + [0] * 23))
    return folds


@pytest.mark.gpu
@pytest.mark.parametrize("kt,shrinking", VARIANTS, ids=VIDS)
def test_shapes_in_one_launch(kt, shrinking):
    """Every shape of the matrix in one launch: the four warps of a block solve problems of different sizes, and 3
    kernels x 121 problems leave the last block with three warps."""
    rng = np.random.RandomState(11 + 2 * shrinking + (kt == "double"))
    E = 64
    signal = rng.choice([-0.7, 0.7], size=E)
    Kf, Kp = _random_kernels(rng, kt, 3, E, signal)
    folds = _shape_folds(rng, E, signal)
    assert len(folds) == 121 and (3 * len(folds)) % 4 == 3
    iters = _check(kt, Kf, Kp, folds, C=1.0, tol=1e-3, shrinking=shrinking)
    assert iters.min() >= 1


def _degenerate_kernels(kt, E, rng):
    """[dup, zero, rank-one, indefinite, wide] kernels.  dup: sample 1 repeats sample 0 and sample 3 repeats sample 2
    (the folds put 0, 1, 2 in class +1 and 3 in class -1: duplicates in one class, and across the classes)."""
    X = rng.randn(E, 6)
    src = np.arange(E)
    src[1], src[3] = 0, 2
    G = X @ X.T
    dup = G[np.ix_(src, src)]
    zero = np.zeros((E, E))
    u = rng.randn(E) * 2
    rank1 = np.outer(u, u)
    A = rng.randn(E, E)
    indef = (A + A.T) / 2
    s = 10.0 ** rng.uniform(-6, 6, size=E)
    Y = rng.randn(E, 8)
    wide = s[:, None] * (Y @ Y.T) * s[None, :]
    Ks = np.array([dup, zero, rank1, indef, wide])
    if kt == "float":
        Ks = Ks.astype(np.float32)              # duplicates stay exact: equal fp64 values round alike
        return Ks, Ks
    return Ks, Ks.copy()


DEGENERATE_MAX_ITER = 20000


@pytest.mark.gpu
@pytest.mark.parametrize("kt,shrinking", VARIANTS, ids=VIDS)
def test_degenerate_kernels(kt, shrinking):
    """Duplicates within and across the classes, all-zero, rank-one, indefinite and wide-range kernels, at every C and
    tol of the matrix; 5 kernels x 3 problems per launch.  At C = 1e4 several of these problems take millions of
    iterations in libsvm too, so every run is cut at DEGENERATE_MAX_ITER (the same cut for both)."""
    rng = np.random.RandomState(23 + 2 * shrinking + (kt == "double"))
    E = 48
    Kf, Kp = _degenerate_kernels(kt, E, rng)
    rest = rng.permutation(np.arange(4, E))
    folds = [_fold([0, 1, 2] + list(rest[:15]), [3] + list(rest[15:33]), list(rest[33:]) + [0, 3]),
             _fold(rest[:7], rest[7:20], np.arange(E)),
             _fold([0, 2, 1], [3, 5], [1, 3, 4])]
    for C in (1e-4, 1.0, 1e4):
        for tol in (1e-1, 1e-3, 1e-6):
            _check(kt, Kf, Kp, folds, C=C, tol=tol, max_iter=DEGENERATE_MAX_ITER, shrinking=shrinking)


# ------------------------------------------------------------------------------------------- long problems, max_iter
LONG_N, LONG_NPOS, LONG_E = 60, 29, 64


@functools.lru_cache(maxsize=None)
def _long_problems():
    """Float32 kernels (exact in fp64, so the oracle serves the double path too) whose problems need several hundred
    iterations: overlapping classes, C = 1.  Kernels 4 .. 7 are kernels 0 .. 3 with an asymmetric perturbation: the two
    loop orders of reconstruct_gradient read opposite triangles of Q, which only an asymmetric kernel tells apart (the C
    entry points, like libsvm, read K[i][j] as given).  One fold: 60 training samples; held out, the 4 others and 12
    training samples."""
    rng = np.random.RandomState(5)
    E = LONG_E
    signal = np.r_[np.full(LONG_NPOS, 0.8), np.full(LONG_N - LONG_NPOS, -0.8), np.zeros(E - LONG_N)]
    Kf, _ = _random_kernels(rng, "float", 4, E, signal, dims=(20, 40))
    asym = (Kf + 0.05 * rng.randn(*Kf.shape)).astype(np.float32)
    Kf = np.concatenate([Kf, asym])
    truth = [1] * 2 + [0] * 2 + [1] * 6 + [0] * 6
    te = list(range(LONG_N, E)) + list(range(0, 6)) + list(range(LONG_NPOS, LONG_NPOS + 6))
    fold = _fold(range(LONG_NPOS), range(LONG_NPOS, LONG_N), te, truth)
    return Kf, fold


LONG_C = 1.0


def _oracle_run(K, max_iter=-1, shrinking=True):
    it = orc.svm_smo(K, list(range(LONG_N)), LONG_NPOS, LONG_C, 1e-3, max_iter, shrinking)[2]
    return it, orc.svm_last_stats(), orc.svm_last_detail()


def test_long_problems_exercise_shrinking():
    """The long problems make the shrinking heuristic act (variables shrunk, gradients reconstructed, both loop orders
    of reconstruct_gradient), need several hundred iterations, and the oracle's iterations equal scikit-learn's."""
    Kf, fold = _long_problems()
    tr, _, y = _parts(fold)
    by_rows = by_cols = shrunk = 0
    longest = 0
    for v, K in enumerate(Kf):
        it, (min_active, reconstructs), (r, c, _) = _oracle_run(K)
        assert it == int(_fit(K, tr, y, LONG_C, 1e-3, -1, True).n_iter_[0])
        longest = max(longest, it)
        shrunk += min_active < LONG_N and reconstructs > 0
        if v >= 4:                       # the asymmetric kernels
            by_rows += r
            by_cols += c
    assert not np.array_equal(Kf[4], Kf[4].T)
    assert longest >= 300 and shrunk >= 4 and by_rows >= 1 and by_cols >= 1, (longest, shrunk, by_rows, by_cols)


@functools.lru_cache(maxsize=None)
def _mid_cuts():
    """max_iter values that stop the shrinking solver while variables are shrunk (oracle: active set below n at the end)."""
    Kf, _ = _long_problems()
    cuts = []
    for K in Kf:
        n_it = _oracle_run(K)[0]
        for cut in range(max(LONG_N + 2, n_it // 2), n_it, 7):
            if _oracle_run(K, cut)[2][2] < LONG_N:
                cuts.append(cut)
                break
    return sorted(set(cuts))[:3]


def test_oracle_max_iter_cuts_match_sklearn():
    """scikit-learn's max_iter (0 = no iteration, -1 = no limit) and the oracle agree on every cut used on the GPU: the
    iteration count, rho and the dual coefficients; some cuts stop the solver while variables are shrunk."""
    Kf, fold = _long_problems()
    tr, _, y = _parts(fold)
    mids = _mid_cuts()
    assert len(mids) >= 2
    for K in Kf[::2]:
        for shrinking in (False, True):
            for cut in (0, 1, LONG_N, LONG_N + 1) + tuple(mids):
                alpha, rho, it = orc.svm_smo(K, tr, LONG_NPOS, LONG_C, 1e-3, cut, shrinking)
                clf = _fit(K, tr, y, LONG_C, 1e-3, cut, shrinking)
                assert it == int(clf.n_iter_[0]) and rho == clf.intercept_[0], (cut, shrinking, it, clf.n_iter_)
                coef = alpha * np.where(np.arange(LONG_N) < LONG_NPOS, 1.0, -1.0)
                ref = np.zeros(LONG_N)
                ref[clf.support_] = -clf.dual_coef_[0]
                assert np.array_equal(coef, ref)


def test_sklearn_max_iter_zero_runs_no_iteration():
    """scikit-learn's SVC(max_iter=0) runs no SMO iteration: every alpha is 0, rho is the midpoint of -1 and 1, and every
    decision is 0 -- the second class; -1 runs to convergence."""
    Kf, fold = _long_problems()
    tr, te, y = _parts(fold)
    clf = _fit(Kf[0], tr, y, LONG_C, 1e-3, 0, False)
    assert list(clf.n_iter_) == [0] and clf.intercept_[0] == 0.0 and len(clf.support_) == 0
    assert np.all(clf.predict(Kf[0].astype(np.float64)[np.ix_(te, tr)]) == 1)
    assert orc.svm_smo(Kf[0], tr, LONG_NPOS, LONG_C, 1e-3, 0, False)[2] == 0
    assert _fit(Kf[0], tr, y, LONG_C, 1e-3, -1, False).n_iter_[0] > 100


@pytest.mark.gpu
@pytest.mark.parametrize("kt", ["float", "double"])
def test_long_problems(kt):
    """Several hundred iterations with the shrinking heuristic acting (see test_long_problems_exercise_shrinking)."""
    Kf, fold = _long_problems()
    Kd = Kf.astype(np.float64) if kt == "double" else Kf
    iters = _check(kt, Kd, Kd, [fold] * 3, C=LONG_C, shrinking=True)
    assert iters.max() >= 300


@pytest.mark.gpu
@pytest.mark.parametrize("kt,shrinking", VARIANTS, ids=VIDS)
def test_max_iter_cuts(kt, shrinking):
    """max_iter 0 (no iteration: every sample on the second class), 1, n, n + 1 (the first do_shrinking) and cuts while
    variables are shrunk; -1 runs to convergence."""
    Kf, fold = _long_problems()
    Kd = Kf.astype(np.float64) if kt == "double" else Kf
    for cut in (0, 1, LONG_N, LONG_N + 1) + tuple(_mid_cuts()) + (-1,):
        iters = _check(kt, Kd, Kd, [fold], C=LONG_C, max_iter=cut, shrinking=shrinking)
        if cut >= 0:
            assert np.all(iters <= cut)


@pytest.mark.gpu
@pytest.mark.parametrize("kt", ["float", "double"])
def test_max_iter_public_api(kt):
    """svm_cv_precomputed / svm_cv_f64 pass max_iter=0 through as no iteration, as scikit-learn does."""
    import torch
    Kf, _ = _long_problems()
    labels = (np.arange(LONG_E) >= LONG_E // 2).astype(int)
    dev = torch.device("cuda:0")
    if kt == "float":
        acc, iters = engine.svm_cv_precomputed(torch.from_numpy(Kf).to(dev), labels, 4, C=LONG_C, max_iter=0,
                                               return_iters=True)
    else:
        Kd = torch.from_numpy(Kf.astype(np.float64)).to(dev)
        acc, iters = engine.svm_cv_f64(Kd, Kd, labels, 4, C=LONG_C, max_iter=0, return_iters=True)
    assert np.all(iters == 0)
    assert np.all(acc == 0.5)             # every held-out sample on the second class, half of each fold


# ------------------------------------------------------------------------------------------- one-vs-one
@pytest.mark.gpu
@pytest.mark.parametrize("kt,shrinking", VARIANTS, ids=VIDS)
@pytest.mark.parametrize("nclass", [3, 4])
def test_multiclass_one_vs_one(kt, shrinking, nclass):
    """One problem per class pair, bits against the sign of libsvm's per-pair decision (decision_function_shape='ovo',
    its sign pinned by libsvm's vote against predict), iterations against n_iter_ per pair."""
    rng = np.random.RandomState(41 + nclass + 2 * shrinking + (kt == "double"))
    E = 60
    lab = rng.permutation(np.arange(E) % nclass)
    Kf, Kp = _random_kernels(rng, kt, 3, E, signal=0.8 * lab - 0.8)
    pairs = [(a, b) for a in range(nclass) for b in range(a + 1, nclass)]
    tr = np.sort(rng.permutation(E)[:44])
    te = np.arange(E)
    folds = []
    for a, b in pairs:
        pos = [int(i) for i in tr if lab[i] == a]
        neg = [int(i) for i in tr if lab[i] == b]
        folds.append(_fold(pos, neg, te, [1 if lab[i] == a else 0 for i in te]))
    bits, iters, _ = _solve(kt, Kf, Kp, folds, C=0.7, tol=1e-3, shrinking=shrinking)
    for v in range(len(Kf)):
        clf = _fit(Kf[v], tr, lab[tr], 0.7, 1e-3, -1, shrinking, decision_function_shape="ovo")
        dec = clf.decision_function(np.asarray(Kp[v], np.float64)[np.ix_(te, tr)])
        votes = np.zeros((len(te), nclass), np.int64)
        for q, (a, b) in enumerate(pairs):
            votes[:, a] += dec[:, q] > 0
            votes[:, b] += dec[:, q] <= 0
        assert np.array_equal(np.argmax(votes, axis=1), clf.predict(np.asarray(Kp[v], np.float64)[np.ix_(te, tr)]))
        assert np.array_equal(iters[v], clf.n_iter_), (v, iters[v], clf.n_iter_)
        for q in range(len(pairs)):
            ref = sum(1 << t for t in range(len(te)) if dec[t, q] > 0)
            assert bits[v][q] == ref, (v, pairs[q], hex(bits[v][q] ^ ref))


# ------------------------------------------------------------------------------------------- crafted near-tie rows
def _coef(clf, n):
    """libsvm's alpha_k y_k by training index (scikit-learn stores the binary model negated)."""
    c = np.zeros(n)
    c[clf.support_] = -clf.dual_coef_[0]
    return c


def _seq_sum(coef, row):
    """libsvm's svm_predict_values: support vectors added sequentially in training order, products rounded on their own."""
    s = 0.0
    for c, k in zip(coef, row):
        if c != 0.0:
            s = s + float(c) * float(k)
    return s


def _butterfly_sum(coef, row):
    """The same terms in a warp's lane-slot order: lane l adds slots l and l + 32, then a __shfl_xor butterfly 16 ... 1."""
    t = np.zeros(64)
    for k in range(len(coef)):
        if coef[k] != 0.0:
            t[k] = float(coef[k]) * float(row[k])
    part = [(0.0 + t[l]) + t[l + 32] for l in range(32)]
    for off in (16, 8, 4, 2, 1):
        part = [part[l] + part[l ^ off] for l in range(32)]
    return part[0]


RHO_C = 0.5          # a power of two: alpha y = +-C and rho / C are exact


@functools.lru_cache(maxsize=None)
def _rho_case(shrinking):
    """Double-path problems with at least 2 free variables; held-out rows 40 and 41 of K_pred are zero except at one bound
    support vector, where the decision sum is exactly rho and nextafter(rho, inf).  Returns (K_fit, K_pred, fold, rho)."""
    rng = np.random.RandomState(71 + shrinking)
    E, n, n_pos = 48, 40, 20
    signal = np.r_[np.full(n_pos, 0.6), np.full(n - n_pos, -0.6), np.zeros(E - n)]
    fold = _fold(range(n_pos), range(n_pos, n), [40, 41], [0, 1])
    tr, _, y = _parts(fold)
    Kfs, Kps, rhos = [], [], []
    while len(Kfs) < 24:
        Kf, Kp = _random_kernels(rng, "double", 1, E, signal, dims=(4, 8))
        clf = _fit(Kf[0], tr, y, RHO_C, 1e-3, -1, shrinking)
        coef = _coef(clf, n)
        free = np.flatnonzero((coef != 0) & (np.abs(coef) < RHO_C))
        bound = np.flatnonzero(np.abs(coef) == RHO_C)
        rho = float(clf.intercept_[0])
        if len(free) < 2 or len(bound) == 0 or rho == 0.0:
            continue
        s = int(bound[rng.randint(len(bound))])
        Kp = Kp[0].copy()
        Kp[40, :] = 0.0
        Kp[41, :] = 0.0
        Kp[40, s] = rho / coef[s]
        Kp[41, s] = math.nextafter(rho, math.inf) / coef[s]
        Kfs.append(Kf[0])
        Kps.append(Kp)
        rhos.append(rho)
    return np.array(Kfs), np.array(Kps), fold, rhos


@pytest.mark.parametrize("shrinking", [False, True])
def test_crafted_rho_rows_are_ties(shrinking):
    """Every rho row: libsvm's decision sum is exactly rho (row 40: the second class) or its successor (row 41: the first
    class); scikit-learn's predict agrees, and the problem has at least 2 free variables."""
    Kf, Kp, fold, rhos = _rho_case(shrinking)
    tr, te, y = _parts(fold)
    assert len(Kf) >= 20
    for v in range(len(Kf)):
        clf = _fit(Kf[v], tr, y, RHO_C, 1e-3, -1, shrinking)
        coef = _coef(clf, len(tr))
        assert ((coef != 0) & (np.abs(coef) < RHO_C)).sum() >= 2
        assert _seq_sum(coef, Kp[v][40, tr]) == rhos[v]
        assert _seq_sum(coef, Kp[v][41, tr]) == math.nextafter(rhos[v], math.inf)
        assert list(clf.predict(Kp[v][np.ix_(te, tr)])) == [1, 0]


@pytest.mark.gpu
@pytest.mark.parametrize("shrinking", [False, True])
def test_rho_rows(shrinking):
    """rho summed in libsvm's order: any last-bit difference puts one of the two rows on the other side."""
    Kf, Kp, fold, _ = _rho_case(shrinking)
    _check("double", Kf, Kp, [fold], C=RHO_C, shrinking=shrinking)


ORDER_C = 1.0


@functools.lru_cache(maxsize=None)
def _order_case(kt, shrinking):
    """Problems of 40 training samples whose held-out rows 40 .. 63 are crafted: two bound support vectors of opposite
    sign with the same K value A ~ 2^40 .. 2^60 and one free support vector whose term is rho (1 + small), every value
    exact in float32, kept where libsvm's sequential sum and the butterfly order put the sample on different sides.
    Returns (K_fit, K_pred, fold, the crafted rows of each kernel)."""
    rng = np.random.RandomState(97 + 2 * shrinking + (kt == "double"))
    E, n, n_pos = 64, 40, 20
    signal = np.r_[np.full(n_pos, 0.5), np.full(n - n_pos, -0.5), np.zeros(E - n)]
    fold = _fold(range(n_pos), range(n_pos, n), range(n, E), [1] * 12 + [0] * 12)
    tr, _, y = _parts(fold)
    Kfs, Kps, crafted = [], [], []
    while len(Kfs) < 6:
        Kf, Kp = _random_kernels(rng, kt, 1, E, signal, dims=(4, 8))
        Kf, Kp = Kf[0].copy(), Kp[0].copy()
        clf = _fit(Kf, tr, y, ORDER_C, 1e-3, -1, shrinking)
        coef = _coef(clf, n)
        rho = float(clf.intercept_[0])
        up = np.flatnonzero(coef == ORDER_C)
        dn = np.flatnonzero(coef == -ORDER_C)
        free = np.flatnonzero((coef != 0) & (np.abs(coef) < ORDER_C))
        if not (len(up) and len(dn) and len(free)) or rho == 0.0:
            continue
        rows = []
        for t in range(n, E):
            for _ in range(400):
                p, q, r = int(rng.choice(up)), int(rng.choice(dn)), int(rng.choice(free))
                row = np.zeros(n, np.float32)
                row[p] = row[q] = np.float32(2.0 ** rng.randint(40, 61) * (1 + rng.randint(0, 1 << 23) / 2 ** 23))
                row[r] = np.float32(rho * (1 + rng.uniform(-1, 1) * 2.0 ** -rng.randint(1, 30)) / coef[r])
                d_seq = _seq_sum(coef, row) - rho
                if (d_seq > 0) != (_butterfly_sum(coef, row) - rho > 0):
                    break
            else:
                continue
            rows.append(t)
            full = np.zeros(E)
            full[:n] = row
            if kt == "float":
                Kf[t, :] = full                 # a held-out row: training never reads it
            else:
                Kp[t, :] = full
        if len(rows) < 12:
            continue
        crafted.append(rows)
        Kfs.append(Kf)
        Kps.append(Kf if kt == "float" else Kp)
    dt = np.float32 if kt == "float" else np.float64
    return np.array(Kfs, dt), np.array(Kps, dt), fold, crafted


@pytest.mark.parametrize("kt,shrinking", VARIANTS, ids=VIDS)
def test_crafted_order_rows_are_order_sensitive(kt, shrinking):
    """Every crafted row: exact in float32, its emulated sequential sum gives scikit-learn's predicted side, and the
    butterfly order of the same terms gives the other side."""
    Kf, Kp, fold, crafted = _order_case(kt, shrinking)
    tr, te, y = _parts(fold)
    assert sum(len(r) for r in crafted) >= 72
    for v in range(len(Kf)):
        clf = _fit(Kf[v], tr, y, ORDER_C, 1e-3, -1, shrinking)
        coef = _coef(clf, len(tr))
        rho = float(clf.intercept_[0])
        pred = clf.predict(np.asarray(Kp[v], np.float64)[np.ix_(te, tr)])
        for j, t in enumerate(te):
            if t not in crafted[v]:
                continue
            row = np.asarray(Kp[v][t, tr], np.float64)
            assert np.array_equal(row.astype(np.float32).astype(np.float64), row)
            d_seq = _seq_sum(coef, row) - rho
            assert (pred[j] == 0) == (d_seq > 0), (v, t)
            assert (d_seq > 0) != (_butterfly_sum(coef, row) - rho > 0), (v, t)


@pytest.mark.gpu
@pytest.mark.parametrize("kt,shrinking", VARIANTS, ids=VIDS)
def test_order_rows(kt, shrinking):
    """The decisions summed sequentially in training order: the crafted near-tie rows land on libsvm's side."""
    Kf, Kp, fold, _ = _order_case(kt, shrinking)
    _check(kt, Kf, Kp, [fold], C=ORDER_C, shrinking=shrinking)
