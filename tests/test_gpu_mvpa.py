"""The activity-based searchlight selector on the GPU: k_searchlight_kernels, the fp64 SMO solver and
MVPAVoxelSelector.run.

References and bounds
---------------------
* ``k_searchlight_kernels``, element by element, against G computed here with ``math.fsum`` over the exact fp64
  products of the float32 features (correctly rounded).  The kernel adds the n products of a pair sequentially, so
  ``|G - G_exact| <= gamma_n sum_f |x_a x_b| + u |G_exact|`` with ``gamma_n = n u / (1 - n u)``, ``u = 2^-53`` (the last
  term is the rounding of the reference itself).  rbf: ``s = (G_aa + G_bb) - 2 G_ab`` carries the three Gram errors plus
  two roundings, and ``exp(-gamma s)`` turns an absolute error e of s into a relative ``gamma e`` of K; CUDA's and
  numpy's ``exp`` add an ulp each.  The difference form ``D = sum_f (x_a - x_b)^2`` is off by ``(gamma_n + 3u) D``.
  Both matrices are exactly symmetric, and ``K_fit_aa`` is exactly 1.
* ``svm_cv_f64`` against ``SVC(kernel='precomputed')`` fitted on the same fp64 arrays (``K_fit`` for training,
  ``K_pred`` rows for the decisions): the same semantics, so every problem's ``n_iter_`` and every accuracy are identical.
* ``MVPAVoxelSelector.run`` against the unmodified reference's output (tests/golden/make_golden_mvpa.py): identical
  None positions, accuracies and lists; the GPU path against the host path on about 2 000 centres; across batch sizes.
"""
import math

import numpy as np
import pytest
import torch
from sklearn import model_selection, svm

from brainiak_b200 import _lib
from brainiak_b200 import searchlight as slm
from brainiak_b200.fcma import engine
from brainiak_b200.fcma.mvpa_voxelselector import MVPAVoxelSelector
from test_mvpa_cpu import assert_matches_fixture, load_fixture

pytestmark = pytest.mark.gpu
U = 2.0 ** -53
SHAPES = [slm.Cube, slm.Diamond, slm.Ball]


def _case(E, r, seed):
    """Volume with mask holes, and centres: an inner corner whose neighbourhood is the centre alone, the opposite inner
    corner, and random interior mask voxels."""
    rng = np.random.RandomState(seed)
    dims = (2 * r + 4, 2 * r + 5, 2 * r + 3)
    vol = (rng.randn(*dims, E) * rng.choice([0.01, 1.0, 30.0], size=dims + (1,))).astype(np.float32)
    mask = rng.rand(*dims) > 0.3
    mask[0:2 * r + 1, 0:2 * r + 1, 0:2 * r + 1] = False
    mask[r, r, r] = True
    far = (dims[0] - 1 - r, dims[1] - 1 - r, dims[2] - 1 - r)
    mask[far] = True
    inner = np.zeros(dims, dtype=bool)
    inner[r:dims[0] - r, r:dims[1] - r, r:dims[2] - r] = True
    cand = np.flatnonzero((mask & inner).ravel())
    extra = rng.choice(cand, size=min(4, len(cand)), replace=False)
    centres = np.unique(np.concatenate([[np.ravel_multi_index((r, r, r), dims), np.ravel_multi_index(far, dims)],
                                        extra])).astype(np.int64)
    return vol, mask, centres


def _features(vol, mask, shape, r, c):
    x, y, z = np.unravel_index(c, mask.shape)
    sl = np.s_[x - r:x + r + 1, y - r:y + r + 1, z - r:z + r + 1]
    return vol[sl][mask[sl] & shape, :].T.astype(np.float64)          # [E, n], C order of the cube


@pytest.mark.parametrize("E", [1, 2, 7, 16, 33, 64])
@pytest.mark.parametrize("r", [0, 1, 2, 3])
def test_searchlight_kernels_elementwise(E, r):
    shape = SHAPES[(E + r) % 3](r).mask_
    vol, mask, centres = _case(E, r, 1000 * E + r)
    dev = torch.device("cuda")
    vt, mt, st = torch.from_numpy(vol).to(dev), torch.from_numpy(mask).to(dev), torch.from_numpy(shape).to(dev)
    all_c, all_n = engine.searchlight_centres(mask, r, shape, 0)
    nf = all_n[np.searchsorted(all_c, centres)]
    assert nf[0] == 1                                     # the isolated inner corner: one feature
    gamma = 1.0 / nf
    G, G2 = engine.searchlight_kernels(vt, mt, r, st, centres, "linear")
    assert G2 is G                                        # linear: the decisions use G as well
    Kf, Kp = engine.searchlight_kernels(vt, mt, r, st, centres, "rbf", gamma)
    G, Kf, Kp = G.cpu().numpy(), Kf.cpu().numpy(), Kp.cpu().numpy()
    for m, c in enumerate(centres):
        X = _features(vol, mask, shape, r, c)
        n = X.shape[1]
        assert n == nf[m]
        gn = n * U / (1 - n * U)
        for M in (G[m], Kf[m], Kp[m]):
            assert np.array_equal(M, M.T)
        assert np.all(np.diag(Kf[m]) == 1.0)
        for a in range(E):
            for b in range(a, E):
                pab = X[a] * X[b]                          # exact in fp64
                gx = math.fsum(pab)
                sab = float(np.abs(pab).sum())
                assert abs(G[m, a, b] - gx) <= gn * sab + U * abs(gx), (m, a, b)
                saa, sbb = float((X[a] * X[a]).sum()), float((X[b] * X[b]).sum())
                s = math.fsum(np.concatenate([X[a] * X[a], X[b] * X[b], -2.0 * pab]))   # = sum (x_a - x_b)^2
                s = max(s, 0.0)
                k_ref = math.exp(-gamma[m] * s)
                e_s = 1.01 * (gn * (saa + sbb + 2 * sab) + 2 * U * (saa + sbb + s))
                tol_fit = k_ref * (gamma[m] * e_s + 2 * U * gamma[m] * s) + 4 * U * 2 * k_ref + 1e-300
                if a != b:
                    assert abs(Kf[m, a, b] - k_ref) <= tol_fit, (m, a, b, Kf[m, a, b], k_ref)
                e_d = 1.01 * (gn + 3 * U) * s
                tol_pred = k_ref * (gamma[m] * e_d + 2 * U * gamma[m] * s) + 4 * U * 2 * k_ref + 1e-300
                assert abs(Kp[m, a, b] - k_ref) <= tol_pred, (m, a, b, Kp[m, a, b], k_ref)


def _fp64_kernels(rng, nv, E, nclass, kernel):
    y = np.arange(E) % nclass
    Kf, Kp = [], []
    for v in range(nv):
        n = int(rng.choice([5, 19, 33]))
        X = rng.randn(E, n)
        X[:, : max(1, n // 4)] += 0.4 * y[:, None]
        G = X @ X.T
        if kernel == "linear":
            Kf.append(G)
            Kp.append(G)
        else:
            g = 1.0 / n
            dg = np.diag(G)
            Kf.append(np.exp(-g * ((dg[:, None] + dg[None, :]) - 2 * G)))
            Kp.append(np.exp(-g * ((X[:, None, :] - X[None, :, :]) ** 2).sum(-1)))
    return y, np.array(Kf), np.array(Kp)


@pytest.mark.parametrize("kernel", ["linear", "rbf"])
@pytest.mark.parametrize("shrinking", [False, True])
@pytest.mark.parametrize("nclass", [2, 3, 4])
def test_svm_cv_f64_matches_sklearn_problem_by_problem(kernel, shrinking, nclass):
    rng = np.random.RandomState(31 * nclass + 2 * shrinking + (kernel == "rbf"))
    E, folds = 40, 4
    for C in (0.02, 0.5, 3.0, 100.0):
        y, Kf, Kp = _fp64_kernels(rng, 6, E, nclass, kernel)
        dev = torch.device("cuda")
        Kf_d = torch.from_numpy(Kf).to(dev)
        Kp_d = Kf_d if kernel == "linear" else torch.from_numpy(Kp).to(dev)
        acc, iters = engine.svm_cv_f64(Kf_d, Kp_d, y, folds, C=C, shrinking=shrinking, return_iters=True)
        npairs = nclass * (nclass - 1) // 2
        skf = model_selection.StratifiedKFold(n_splits=folds, shuffle=False)
        for v in range(len(Kf)):
            scores = []
            for f, (tr, te) in enumerate(skf.split(np.zeros((E, 1)), y)):
                clf = svm.SVC(kernel="precomputed", C=C, shrinking=shrinking).fit(Kf[v][np.ix_(tr, tr)], y[tr])
                assert np.array_equal(iters[v, f * npairs:(f + 1) * npairs], clf.n_iter_), (C, v, f)
                scores.append(np.mean(clf.predict(Kp[v][np.ix_(te, tr)]) == y[te]))
            assert acc[v] == np.mean(scores), (C, v)


@pytest.mark.parametrize("name", ["a", "b1", "b2", "b3", "b4"])
def test_run_matches_reference_fixture(golden, name):
    z, sl, clf = load_fixture(golden, name)
    mvs = MVPAVoxelSelector(z["data"], z["mask"], z["labels"], int(z["num_folds"]), sl)
    assert mvs._gpu_kind(clf) is not None
    before = _lib.load().fcma_launch_count()
    volume, results = mvs.run(clf)
    assert _lib.load().fcma_launch_count() >= before + 2         # kernel matrices + solver ran on the device
    assert_matches_fixture(z, volume, results)


@pytest.mark.parametrize("batch", [1, 7, 100, 100000])
def test_run_is_independent_of_batching(golden, batch):
    z, sl, clf = load_fixture(golden, "b1")
    mvs = MVPAVoxelSelector(z["data"], z["mask"], z["labels"], int(z["num_folds"]), sl, batch_centres=batch)
    assert_matches_fixture(z, *mvs.run(clf))


@pytest.mark.parametrize("clf", [svm.SVC(kernel="rbf", gamma="auto", C=2.0),
                                 svm.SVC(kernel="linear", C=0.3, shrinking=True),
                                 svm.SVC(kernel="rbf", gamma=0.05, C=1.0, shrinking=False)],
                         ids=["rbf-auto", "linear-shrinking", "rbf-gamma"])
def test_gpu_and_host_paths_agree(clf):
    rng = np.random.RandomState(5)
    dims, E = (16, 16, 14), 24
    data = rng.randn(*dims, E).astype(np.float32)
    labels = np.arange(E) % 3 if clf.kernel == "linear" else np.arange(E) % 2
    data[6:10, 6:10, 5:9] += (0.5 * labels).astype(np.float32)
    mask = rng.rand(*dims) > 0.2
    sl = slm.Searchlight(sl_rad=1, shape=slm.Cube)
    centres, _ = engine.searchlight_centres(mask, 1, sl.shape, 0)
    assert len(centres) > 1800
    gpu = MVPAVoxelSelector(data, mask, labels, 3, sl).run(clf)
    host = MVPAVoxelSelector(data, mask, labels, 3, sl, gpu_cv=False).run(clf)
    assert gpu[1] == host[1]
    assert all((a is None and b is None) or a == b for a, b in zip(gpu[0].ravel(), host[0].ravel()))


def test_rejections():
    rng = np.random.RandomState(2)
    data = rng.randn(6, 6, 6, 8).astype(np.float32)
    mask = np.ones((6, 6, 6), dtype=bool)
    labels = [0, 1] * 4
    sl = slm.Searchlight(sl_rad=1)
    clf = svm.SVC(kernel="linear")
    with pytest.raises(ValueError, match="mask shape"):
        MVPAVoxelSelector(data[:5], mask, labels, 2, sl).run(clf)
    bad = data.copy()
    bad[3, 3, 3, 2] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        MVPAVoxelSelector(bad, mask, labels, 2, sl).run(clf)
    outside = data.copy()
    outside[0, 0, 0, 1] = np.inf                 # a corner voxel no centre's cube reaches with this mask
    m2 = mask.copy()
    m2[0, 0, 0] = False
    MVPAVoxelSelector(outside, m2, labels, 2, sl).run(clf)
    dev = torch.device("cuda")
    K = torch.zeros((2, 65, 65), dtype=torch.float64, device=dev)
    with pytest.raises(ValueError):
        engine.svm_cv_f64(K, K, np.arange(65) % 2, 2)
    vt = torch.from_numpy(data).to(dev)
    mt = torch.from_numpy(mask).to(dev)
    st = torch.from_numpy(sl.shape).to(dev)
    with pytest.raises(ValueError, match="face"):
        engine.searchlight_kernels(vt, mt, 1, st, np.array([0]), "linear")
    with pytest.raises(ValueError, match="outside"):
        engine.searchlight_kernels(vt, mt, 1, st, np.array([6 * 6 * 6]), "linear")
    with pytest.raises(ValueError, match="gamma"):
        engine.searchlight_kernels(vt, mt, 1, st, np.array([43]), "rbf")
    with pytest.raises(ValueError, match="gamma"):
        engine.searchlight_kernels(vt, mt, 1, st, np.array([43, 44]), "rbf", np.array([0.1, 0.2, 0.3]))
    big = torch.zeros((3, 3, 3, 65), dtype=torch.float32, device=dev)
    with pytest.raises(ValueError, match="E = 65"):
        engine.searchlight_kernels(big, torch.ones((3, 3, 3), dtype=torch.uint8, device=dev), 1, st,
                                   np.array([13]), "linear")
