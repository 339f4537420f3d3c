"""The activity-based searchlight selector above 64 epochs on the GPU: k_searchlight_kernels_tiled, the fp64 wide SMO
(fcma_svm_cv_solve_f64_wide) and MVPAVoxelSelector.run up to 256 epochs.

References and bounds
---------------------
* ``searchlight_kernels_wide`` element by element against ``math.fsum`` with the bounds of
  test_gpu_mvpa.py::test_searchlight_kernels_elementwise, at tile edges and partial last tiles; both matrices exactly
  symmetric and ``K_fit_aa`` exactly 1.
* Tile independence: an entry is summed from the two epochs' features only, so the entries of any 64-epoch subset S equal
  ``searchlight_kernels`` (the untiled kernel) on the volume of those epochs, bit for bit.
* ``fcma_svm_cv_solve_f64_wide`` against ``SVC(kernel='precomputed')`` fitted per problem on the same fp64 arrays: every
  ``n_iter_`` and every held-out decision bit.  At E <= 64 the wide and narrow solvers agree bit for bit.
* ``MVPAVoxelSelector.run`` against the unmodified reference (mvpa_w1: the example's call at 216 epochs; mvpa_w2), and
  against its own host path at 65, 140, 216 and 256 epochs.
"""
import ctypes
import math

import numpy as np
import pytest
import torch
from sklearn import model_selection, svm

from brainiak_b200 import _lib
from brainiak_b200 import searchlight as slm
from brainiak_b200.fcma import engine
from brainiak_b200.fcma.mvpa_voxelselector import MVPAVoxelSelector
from test_gpu_mvpa import SHAPES, U, _case, _features, _fp64_kernels
from test_mvpa_cpu import assert_matches_fixture, load_fixture

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


# every radius 0-3 and every shape (cube / diamond / ball by (E + r) % 3) with the tile edges and partial last tiles
@pytest.mark.parametrize("E, r", [(E, i % 4) for i, E in enumerate([1, 63, 64, 65, 127, 128, 129, 140, 216, 256])])
def test_searchlight_kernels_wide_elementwise(E, r):
    shape = SHAPES[(E + r) % 3](r).mask_
    vol, mask, centres = _case(E, r, 1000 * E + r + 7)
    vt, mt, st = torch.from_numpy(vol).to(DEV), torch.from_numpy(mask).to(DEV), torch.from_numpy(shape).to(DEV)
    all_c, all_n = engine.searchlight_centres(mask, r, shape, 0)
    nf = all_n[np.searchsorted(all_c, centres)]
    assert nf[0] == 1                                     # the isolated inner corner: one feature
    gamma = 1.0 / nf
    G, G2 = engine.searchlight_kernels_wide(vt, mt, r, st, centres, "linear")
    assert G2 is G
    Kf, Kp = engine.searchlight_kernels_wide(vt, mt, r, st, centres, "rbf", gamma)
    G, Kf, Kp = G.cpu().numpy(), Kf.cpu().numpy(), Kp.cpu().numpy()
    for m, c in enumerate(centres):
        X = _features(vol, mask, shape, r, c)
        n = X.shape[1]
        assert n == nf[m]
        gn = n * U / (1 - n * U)
        for M in (G[m], Kf[m], Kp[m]):
            assert np.array_equal(M, M.T)
        assert np.all(np.diag(Kf[m]) == 1.0)
        sq = X * X
        ssq = sq.sum(axis=1)
        for a in range(E):
            P = X[a] * X[a:]                               # [E - a, n], exact in fp64
            gx = np.array([math.fsum(p) for p in P])
            sab = np.abs(P).sum(axis=1)
            assert np.all(np.abs(G[m, a, a:] - gx) <= gn * sab + U * np.abs(gx)), (m, a)
            s = np.array([math.fsum(np.concatenate([sq[a], sq[b], -2.0 * P[b - a]])) for b in range(a, E)])
            s = np.maximum(s, 0.0)
            k_ref = np.exp(-gamma[m] * s)
            e_s = 1.01 * (gn * (ssq[a] + ssq[a:] + 2 * sab) + 2 * U * (ssq[a] + ssq[a:] + s))
            tol_fit = k_ref * (gamma[m] * e_s + 2 * U * gamma[m] * s) + 4 * U * 2 * k_ref + 1e-300
            assert np.all(np.abs(Kf[m, a, a + 1:] - k_ref[1:]) <= tol_fit[1:]), (m, a)
            e_d = 1.01 * (gn + 3 * U) * s
            tol_pred = k_ref * (gamma[m] * e_d + 2 * U * gamma[m] * s) + 4 * U * 2 * k_ref + 1e-300
            assert np.all(np.abs(Kp[m, a, a:] - k_ref) <= tol_pred), (m, a)


@pytest.mark.parametrize("E", [140, 256])
@pytest.mark.parametrize("r", [1, 2])
def test_searchlight_kernels_wide_tile_independence(E, r):
    shape = SHAPES[r](r).mask_
    vol, mask, centres = _case(E, r, 77 * E + r)
    rng = np.random.RandomState(E + r)
    vt, mt, st = torch.from_numpy(vol).to(DEV), torch.from_numpy(mask).to(DEV), torch.from_numpy(shape).to(DEV)
    gamma = rng.uniform(0.01, 0.5, size=len(centres))
    wide = [engine.searchlight_kernels_wide(vt, mt, r, st, centres, "linear")[0].cpu().numpy()]
    wide += [k.cpu().numpy() for k in engine.searchlight_kernels_wide(vt, mt, r, st, centres, "rbf", gamma)]
    # subsets across the tile edges at 64 and 128, the last 64 epochs, and a scattered subset
    subsets = [np.arange(32, 96), np.arange(100, 164) % E, np.arange(E - 64, E),
               np.sort(rng.choice(E, size=64, replace=False))]
    for S in subsets:
        vs = torch.from_numpy(np.ascontiguousarray(vol[..., S])).to(DEV)
        narrow = [engine.searchlight_kernels(vs, mt, r, st, centres, "linear")[0].cpu().numpy()]
        narrow += [k.cpu().numpy() for k in engine.searchlight_kernels(vs, mt, r, st, centres, "rbf", gamma)]
        for w, k in zip(wide, narrow):
            assert np.array_equal(w[:, S[:, None], S[None, :]], k), S[:4]


def _solve_wide(Kf_d, Kp_d, folds, C, shrinking, wide):
    """fcma_svm_cv_solve_f64(_wide) called directly: (bits [nv, nproblems, words], iters, correct) for two classes."""
    lib = _lib.load()
    nv, E, _ = Kf_d.shape
    nprob = folds.nproblems
    bits = torch.zeros((nv, nprob, 4 if wide else 1), dtype=torch.int64, device=DEV)
    iters = torch.empty((nv, nprob), dtype=torch.int32, device=DEV)
    correct = torch.empty((nv, nprob), dtype=torch.int32, device=DEV)
    solve = lib.fcma_svm_cv_solve_f64_wide if wide else lib.fcma_svm_cv_solve_f64
    _lib.check(solve(ctypes.c_void_p(Kf_d.data_ptr()), ctypes.c_void_p(Kp_d.data_ptr()), nv, E, nprob,
                     ctypes.cast(folds.structs, ctypes.c_void_p), float(C), 1e-3, -1, int(shrinking),
                     ctypes.c_void_p(correct.data_ptr()), ctypes.c_void_p(bits.data_ptr()),
                     ctypes.c_void_p(iters.data_ptr()), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return bits.cpu().numpy().view(np.uint64), iters.cpu().numpy(), correct.cpu().numpy()


@pytest.mark.parametrize("kernel", ["linear", "rbf"])
@pytest.mark.parametrize("shrinking", [False, True])
@pytest.mark.parametrize("nclass", [2, 3, 4])
@pytest.mark.parametrize("E, nfolds", [(140, 7), (216, 4)])
def test_svm_cv_f64_wide_matches_sklearn_problem_by_problem(kernel, shrinking, nclass, E, nfolds):
    rng = np.random.RandomState(E + 31 * nclass + 2 * shrinking + (kernel == "rbf"))
    for C in (0.02, 1.0, 100.0):
        y, Kf, Kp = _fp64_kernels(rng, 2, E, nclass, kernel)
        Kf_d = torch.from_numpy(Kf).to(DEV)
        Kp_d = Kf_d if kernel == "linear" else torch.from_numpy(Kp).to(DEV)
        folds = engine.make_svm_folds_wide(y, nfolds)
        bits, iters, _ = _solve_wide(Kf_d, Kp_d, folds, C, shrinking, True)
        for p, fd in enumerate(folds.structs):
            tr = list(fd.train_idx[:fd.n_train])
            te = list(fd.test_idx[:fd.n_test])
            lab = np.r_[np.zeros(fd.n_pos, int), np.ones(fd.n_train - fd.n_pos, int)]
            order = np.argsort(tr, kind="stable")              # the samples in their original order, as libsvm sees them
            tr_o, lab_o = np.asarray(tr)[order], lab[order]
            for v in range(len(Kf)):
                clf = svm.SVC(kernel="precomputed", C=C, shrinking=shrinking).fit(Kf[v][np.ix_(tr_o, tr_o)], lab_o)
                assert clf.n_iter_[0] == iters[v, p], (C, v, p)
                side = clf.predict(Kp[v][np.ix_(te, tr_o)]) == 0
                want = np.zeros(4, dtype=np.uint64)
                for t in np.flatnonzero(side):
                    want[t // 64] |= np.uint64(1) << np.uint64(t % 64)
                assert np.array_equal(bits[v, p], want), (C, v, p)
        assert (max(fd.n_train for fd in folds.structs) > 128) == (E == 216 and nclass == 2)
        acc = engine.svm_cv_f64(Kf_d, Kp_d, y, nfolds, C=C, shrinking=shrinking, folds=folds)
        acc_sk = []
        skf = model_selection.StratifiedKFold(n_splits=nfolds, shuffle=False)
        for v in range(len(Kf)):
            sc = []
            for tr, te in skf.split(np.zeros((E, 1)), y):
                clf = svm.SVC(kernel="precomputed", C=C, shrinking=shrinking).fit(Kf[v][np.ix_(tr, tr)], y[tr])
                sc.append(np.mean(clf.predict(Kp[v][np.ix_(te, tr)]) == y[te]))
            acc_sk.append(np.mean(sc))
        assert np.array_equal(acc, np.array(acc_sk)), C


@pytest.mark.parametrize("kernel", ["linear", "rbf"])
@pytest.mark.parametrize("shrinking", [False, True])
def test_svm_cv_f64_wide_equals_narrow_up_to_64_epochs(kernel, shrinking):
    rng = np.random.RandomState(9 + shrinking)
    for E, nclass in ((24, 2), (64, 2), (64, 3)):
        y, Kf, Kp = _fp64_kernels(rng, 5, E, nclass, kernel)
        Kf_d = torch.from_numpy(Kf).to(DEV)
        Kp_d = Kf_d if kernel == "linear" else torch.from_numpy(Kp).to(DEV)
        for C in (0.05, 1.0, 30.0):
            nb, ni, nc = _solve_wide(Kf_d, Kp_d, engine.make_svm_folds(y, 4), C, shrinking, False)
            wb, wi, wc = _solve_wide(Kf_d, Kp_d, engine.make_svm_folds_wide(y, 4), C, shrinking, True)
            assert np.array_equal(wb[:, :, 0], nb[:, :, 0]) and not wb[:, :, 1:].any()
            assert np.array_equal(wi, ni) and np.array_equal(wc, nc)
            a_n = engine.svm_cv_f64(Kf_d, Kp_d, y, 4, C=C, shrinking=shrinking)
            a_w = engine.svm_cv_f64(Kf_d, Kp_d, y, 4, C=C, shrinking=shrinking, folds=engine.make_svm_folds_wide(y, 4))
            assert np.array_equal(a_n, a_w)


@pytest.mark.parametrize("name", ["w1", "w2"])
def test_run_matches_reference_fixture_wide(golden, name):
    z, sl, clf = load_fixture(golden, name)
    mvs = MVPAVoxelSelector(z["data"], z["mask"], z["labels"], int(z["num_folds"]), sl)
    assert z["data"].shape[3] > 64 and mvs._gpu_kind(clf) is not None
    before = _lib.load().fcma_launch_count()
    volume, results = mvs.run(clf)
    assert _lib.load().fcma_launch_count() >= before + 2         # kernel matrices + solver ran on the device
    assert_matches_fixture(z, volume, results)


@pytest.mark.parametrize("batch", [1, 7, None])
@pytest.mark.parametrize("name", ["w1", "w2"])
def test_run_is_independent_of_batching_wide(golden, name, batch):
    z, sl, clf = load_fixture(golden, name)
    mvs = MVPAVoxelSelector(z["data"], z["mask"], z["labels"], int(z["num_folds"]), sl, batch_centres=batch)
    assert_matches_fixture(z, *mvs.run(clf))


@pytest.mark.parametrize("E, nclass, clf", [
    (65, 2, svm.SVC(kernel="linear", C=0.3, shrinking=True)),
    (140, 3, svm.SVC(kernel="rbf", gamma="auto", C=2.0, shrinking=False)),
    (140, 3, svm.SVC(kernel="linear", C=1.0, shrinking=False)),
    (216, 2, svm.SVC(kernel="linear", C=1.0, shrinking=False)),
    (216, 2, svm.SVC(kernel="rbf", gamma="auto", C=10.0, shrinking=True)),
    (256, 3, svm.SVC(kernel="rbf", gamma=0.05, C=1.0, shrinking=True)),
], ids=["65-linear-shrinking", "140-rbf-auto", "140-linear", "216-linear", "216-rbf-auto-shrinking", "256-rbf-gamma"])
def test_gpu_and_host_paths_agree_wide(E, nclass, clf):
    rng = np.random.RandomState(E + nclass)
    dims = (10, 9, 9)
    data = rng.randn(*dims, E).astype(np.float32)
    labels = np.arange(E) % nclass
    data[3:7, 3:7, 3:6] += (0.4 * labels).astype(np.float32)
    mask = rng.rand(*dims) > 0.2
    sl = slm.Searchlight(sl_rad=1, shape=slm.Cube)
    centres, _ = engine.searchlight_centres(mask, 1, sl.shape, 0)
    assert len(centres) > 200
    gpu = MVPAVoxelSelector(data, mask, labels, 4, sl).run(clf)
    host = MVPAVoxelSelector(data, mask, labels, 4, sl, gpu_cv=False).run(clf)
    assert gpu[1] == host[1]
    assert all((a is None and b is None) or a == b for a, b in zip(gpu[0].ravel(), host[0].ravel()))


def test_rejections_wide():
    mask = torch.ones((3, 3, 3), dtype=torch.uint8, device=DEV)
    st = torch.from_numpy(slm.Cube(1).mask_).to(DEV)
    big = torch.zeros((3, 3, 3, 257), dtype=torch.float32, device=DEV)
    with pytest.raises(ValueError, match="E = 257"):
        engine.searchlight_kernels_wide(big, mask, 1, st, np.array([13]), "linear")
    K = torch.zeros((2, 257, 257), dtype=torch.float64, device=DEV)
    y = np.arange(257) % 2
    with pytest.raises(ValueError):
        engine.svm_cv_f64(K, K, y, 2, folds=engine.make_svm_folds_wide(y, 2))
