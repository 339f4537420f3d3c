"""SVC(kernel='rbf', gamma='scale') cross-validated on the GPU: per-fold gammas from per-sample moments.

* engine.feature_gram_wide / searchlight_gram_wide: G and D bit-identical to the existing builders' linear G and to the
  sums their rbf forms exponentiate; the moments (double-double) against ``math.fsum`` of the features: hi is within an ulp
  of the correctly rounded sum, hi + lo within 2^-100 sum |x| of the exact one.  Rows at E in {1, 16, 63, 64, 65, 140, 256}
  and V2 in {1, 33, 257, 4129}, one and two masks, tiled and strided blocks, trailing raw epochs; centres at sl_rad 0-3,
  cube, diamond and ball, one-feature centres.
* engine.fold_gammas against ``SVC().fit(X_train)._gamma`` for every (item, fold) with 2, 3 and 4 classes (within 4 ulps,
  the bound test_svc_scale_cpu.py checks for the exact-variance gamma); all-zero features give exactly 1.0; constant
  nonzero and large-mean features are flagged and scored as on the host, features just below the flag bound are not.
* engine.rbf_fold_kernels bit-identical to feature_kernels_f64_wide / searchlight_kernels_wide called with that gamma.
* engine.svm_cv_scale: the iteration count of every problem equals ``SVC().fit`` on the fold's training features, for
  rows and for searchlight centres.
* ``VoxelSelector.run`` and ``MVPAVoxelSelector.run`` with ``gpu_cv=True`` return the lists ``gpu_cv=False`` returns;
  two runs are bit-identical; items flagged for the host (forced) are scored there, and the lists are unchanged.
* Both selectors, with ``SVC()`` and ``SVC(C=10, shrinking=False)``, reproduce the unmodified reference's lists on the
  fixtures of tests/golden/make_golden_scale.py, on the GPU path and on the host path.
"""
import math

import numpy as np
import pytest
import torch
from sklearn import model_selection, svm

from brainiak_b200 import searchlight as slm
from brainiak_b200.fcma import engine, synthetic
from brainiak_b200.fcma.mvpa_voxelselector import MVPAVoxelSelector
from brainiak_b200.fcma.voxelselector import VoxelSelector
from test_gpu_feature_svc import _operands, dev  # noqa: F401  (dev: fixture)
from test_gpu_mvpa import _case, _features
from test_gpu_parity import _probe_matches
from test_svc_scale_cpu import assert_matches_scale_fixture

pytestmark = pytest.mark.gpu
SHAPES = [slm.Cube, slm.Diamond, slm.Ball]


def _check_moments(x, mom, name):
    """x: float64 [n, E, F] features; mom: [n, E, 4]."""
    n, E, _ = x.shape
    for i in range(n):
        for e in range(E):
            for k, vals in ((0, x[i, e]), (2, x[i, e] * x[i, e])):
                hi, lo = mom[i, e, k], mom[i, e, k + 1]
                rounded = math.fsum(vals)
                assert abs(hi - rounded) <= np.spacing(abs(rounded)), (name, i, e, k, hi, rounded)
                resid = math.fsum(list(vals) + [-hi, -lo])
                assert abs(resid) <= 2.0 ** -100 * np.abs(vals).sum() + 1e-300, (name, i, e, k, resid)


def _z(op, op2, start, nb, eps):
    r = engine.corr_block(op, op2, start, nb, layout=0).contiguous()
    return engine.within_subject_norm_(r, eps).cpu().numpy()


# name, V, V2 (None: one mask), T, E, eps, start, nb, ragged
ROW_CASES = [
    ("E1_V33", 300, 33, 40, 1, 1, 0, 3, False),
    ("E16_V1", 300, 1, 40, 16, 4, 5, 2, False),
    ("E63_V257", 300, 257, 40, 63, 3, 5, 2, False),
    ("E64_V4129", 300, 4129, 40, 64, 16, 250, 2, False),
    ("E65_self", 300, None, 40, 65, 20, 7, 2, True),
    ("E140_V4129", 300, 4129, 40, 140, 20, 3, 1, True),
    ("E256_V257", 300, 257, 40, 256, 16, 40, 1, False),
]


@pytest.mark.parametrize("layout", ["strided", "tiled"])
@pytest.mark.parametrize("name,V,V2,T,E,eps,start,nb,ragged", ROW_CASES, ids=[c[0] for c in ROW_CASES])
def test_feature_gram_and_moments(dev, name, V, V2, T, E, eps, start, nb, ragged, layout):
    op, op2 = _operands(V, V2, T, E, dev, seed=E * 31 + (V2 or 0), ragged=ragged)
    n2 = op2.V
    work = engine.Workspace(E, n2, 2 if layout == "strided" else 256, dev)
    G, D, mom = engine.feature_gram_wide(op, op2, start, nb, eps, work=work)
    Gl, _ = engine.feature_kernels_f64_wide(op, op2, start, nb, eps, "linear", work=work)
    assert torch.equal(G, Gl)
    gamma = 0.37 / n2
    Kf, Kp = engine.feature_kernels_f64_wide(op, op2, start, nb, eps, "rbf", gamma, work=work)
    g = torch.full((nb, 3), gamma, dtype=torch.float64, device=dev)
    g[:, 0] = 2 * gamma
    Ff, Fp = engine.rbf_fold_kernels(G, D, g, 1)
    assert torch.equal(Ff, Kf) and torch.equal(Fp, Kp)
    assert torch.all(torch.diagonal(Ff, dim1=1, dim2=2) == 1) and torch.all(torch.diagonal(Fp, dim1=1, dim2=2) == 1)
    _check_moments(_z(op, op2, start, nb, eps).astype(np.float64), mom.cpu().numpy(), name)


@pytest.mark.parametrize("E, r", [(E, i % 4) for i, E in enumerate([1, 16, 63, 64, 65, 140, 216, 256])])
def test_searchlight_gram_and_moments(E, r):
    dev = torch.device("cuda")
    shape = SHAPES[(E + r) % 3](r).mask_
    vol, mask, centres = _case(E, r, 500 * E + r)
    vt, mt, st = torch.from_numpy(vol).to(dev), torch.from_numpy(mask).to(dev), torch.from_numpy(shape).to(dev)
    G, D, mom = engine.searchlight_gram_wide(vt, mt, r, st, centres)
    Gl, _ = engine.searchlight_kernels_wide(vt, mt, r, st, centres, "linear")
    assert torch.equal(G, Gl)
    gam = np.linspace(0.01, 0.5, len(centres))
    Kf, Kp = engine.searchlight_kernels_wide(vt, mt, r, st, centres, "rbf", gam)
    g = torch.from_numpy(np.stack([gam * 3, gam], axis=1)).to(dev).contiguous()
    Ff, Fp = engine.rbf_fold_kernels(G, D, g, 1)
    assert torch.equal(Ff, Kf) and torch.equal(Fp, Kp)
    x = [_features(vol, mask, shape, r, int(c)) for c in centres]
    assert min(f.shape[1] for f in x) == 1                    # the corner centre has one feature
    mom = mom.cpu().numpy()
    for m, f in enumerate(x):
        _check_moments(f[None], mom[m:m + 1], "E%d_r%d_c%d" % (E, r, m))


def _sk_gammas(X, y, folds):
    skf = model_selection.StratifiedKFold(folds)
    return [svm.SVC().fit(X[tr], y[tr])._gamma for tr, _ in skf.split(X, y)]


def _ulps(a, b):
    return np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b)))


@pytest.mark.parametrize("ncls,E,eps,folds", [(2, 16, 4, 4), (3, 65, 13, 5), (4, 140, 20, 7)])
def test_fold_gammas_and_iterations_rows(dev, ncls, E, eps, folds):
    op, op2 = _operands(300, 257, 40, E, dev, seed=E + ncls)
    nb = 6
    G, D, mom = engine.feature_gram_wide(op, op2, 20, nb, eps)
    y = np.arange(E) % ncls
    fl = engine.svm_folds_for(y, folds, E)
    gamma, flag = engine.fold_gammas(mom, engine.fold_train_mask(fl, E), 257)
    assert not flag.any()
    gamma = gamma.cpu().numpy()
    z = _z(op, op2, 20, nb, eps)
    for C, shrinking in ((1.0, True), (10.0, False)):
        acc, flagged, iters = engine.svm_cv_scale(G, D, mom, 257, y, folds, C=C, shrinking=shrinking, folds=fl,
                                                  return_iters=True)
        assert not flagged.any()
        for i in range(nb):
            X = z[i]
            assert np.all(_ulps(gamma[i], np.array(_sk_gammas(X, y, folds))) <= 4), i
            want_iters = []
            for tr, _ in model_selection.StratifiedKFold(folds).split(X, y):
                want_iters += list(np.atleast_1d(svm.SVC(C=C, shrinking=shrinking).fit(X[tr], y[tr]).n_iter_))
            assert list(iters[i]) == want_iters, i
            want = model_selection.cross_val_score(svm.SVC(C=C, shrinking=shrinking), X, y,
                                                   cv=model_selection.StratifiedKFold(folds)).mean()
            assert acc[i] == want, i


def test_fold_gammas_searchlight_zero_constant_large_mean_and_below_bound():
    """All-zero features: gamma exactly 1, not flagged.  Constant nonzero and |mean| / sigma = 2^23 features: flagged.
    |mean| / sigma = 2^17, just below the 2^18 bound: not flagged, and within 4 ulps of scikit-learn's gamma in every
    fold.  run() with the flagged centres scored on the host equals the host path."""
    dev = torch.device("cuda")
    rng = np.random.RandomState(3)
    E, r = 24, 1
    dims = (15, 5, 5)
    vol = rng.randn(*dims, E).astype(np.float32)
    sub = (3,) + dims[1:] + (E,)
    vol[0:3] = 0.0                                          # centre x = 1: all features zero
    vol[3:6] = 3.0                                          # centre x = 4: constant nonzero
    vol[6:9] = (2.0 ** 24 + rng.choice([-2.0, 2.0], size=sub)).astype(np.float32)    # x = 7: mean / sd = 2^23
    vol[12:15] = (2.0 ** 17 + rng.choice([-1.0, 1.0], size=sub)).astype(np.float32)  # x = 13: mean / sd = 2^17
    mask = np.ones(dims, dtype=bool)
    shape = slm.Cube(r).mask_
    centres = np.array([np.ravel_multi_index((x, 2, 2), dims) for x in (1, 4, 7, 10, 13)])
    G, D, mom = engine.searchlight_gram_wide(torch.from_numpy(vol).to(dev), torch.from_numpy(mask).to(dev), r,
                                             torch.from_numpy(shape).to(dev), centres)
    y = np.arange(E) % 2
    fl = engine.svm_folds_for(y, 4, E)
    gamma, flag = engine.fold_gammas(mom, engine.fold_train_mask(fl, E), 27)
    gamma, flag = gamma.cpu().numpy(), flag.cpu().numpy()
    assert np.all(gamma[0] == 1.0) and not flag[0].any()
    assert flag[1].all() and flag[2].all() and not flag[3].any() and not flag[4].any()
    for k in (3, 4):
        X = _features(vol, mask, shape, r, int(centres[k]))
        assert np.all(_ulps(gamma[k], np.array(_sk_gammas(X, y, 4))) <= 4), k
    sl = slm.Searchlight(sl_rad=r, shape=slm.Cube)
    gpu = MVPAVoxelSelector(vol, mask, y, 4, sl).run(svm.SVC())
    host = MVPAVoxelSelector(vol, mask, y, 4, sl, gpu_cv=False).run(svm.SVC())
    assert gpu[1] == host[1]


@pytest.mark.parametrize("ncls,E,folds", [(2, 24, 4), (3, 48, 4), (4, 64, 8), (3, 140, 7)])
def test_fold_gammas_and_iterations_searchlight(ncls, E, folds):
    """Every centre's gamma per fold against SVC().fit(X_train)._gamma, every problem's iteration count against
    scikit-learn's n_iter_, and the accuracies against cross_val_score, with 2, 3 and 4 classes."""
    dev = torch.device("cuda")
    r = 1
    shape = slm.Ball(r).mask_
    vol, mask, centres = _case(E, r, 900 + E + ncls)
    vt, mt, st = torch.from_numpy(vol).to(dev), torch.from_numpy(mask).to(dev), torch.from_numpy(shape).to(dev)
    G, D, mom = engine.searchlight_gram_wide(vt, mt, r, st, centres)
    x = [_features(vol, mask, shape, r, int(c)).astype(np.float32) for c in centres]
    nfeat = np.array([f.shape[1] for f in x])
    y = np.arange(E) % ncls
    fl = engine.svm_folds_for(y, folds, E)
    gamma, flag = engine.fold_gammas(mom, engine.fold_train_mask(fl, E), nfeat)
    gamma = gamma.cpu().numpy()
    assert not flag.any()
    acc, flagged, iters = engine.svm_cv_scale(G, D, mom, nfeat, y, folds, folds=fl, return_iters=True)
    assert not flagged.any()
    skf = model_selection.StratifiedKFold(folds)
    for m, X in enumerate(x):
        assert np.all(_ulps(gamma[m], np.array(_sk_gammas(X, y, folds))) <= 4), m
        want_iters = []
        for tr, _ in skf.split(X, y):
            want_iters += list(np.atleast_1d(svm.SVC().fit(X[tr], y[tr]).n_iter_))
        assert list(iters[m]) == want_iters, m
        assert acc[m] == model_selection.cross_val_score(svm.SVC(), X, y, cv=skf).mean(), m


def _flag_every_third(monkeypatch):
    """engine.fold_gammas flags the items 0, 3, 6, ... in one fold, whatever their variance: the selectors' host
    fallback for flagged items is taken."""
    orig = engine.fold_gammas

    def flagged(moments, train, nfeat):
        gamma, flag = orig(moments, train, nfeat)
        flag[0::3, -1] = True
        return gamma, flag
    monkeypatch.setattr(engine, "fold_gammas", flagged)


def test_voxel_selector_host_fallback_for_flagged_voxels(dev, monkeypatch):
    raw, _ = synthetic.make_epochs(70, 48, 32, seed=123)
    labels = [e % 3 for e in range(32)]
    host = VoxelSelector(labels, 8, 4, raw, device=dev, gpu_cv=False, process_num=0).run(svm.SVC())
    _flag_every_third(monkeypatch)
    vs = VoxelSelector(labels, 8, 4, raw, device=dev, block_rows=32)
    calls = []
    orig = vs._voxel_scoring

    def spy(task, clf):
        out = orig(task, clf)
        calls.append((task, out))
        return out
    vs._voxel_scoring = spy
    got = vs.run(svm.SVC())
    # blocks of 32 rows: items 0, 3, ... of each block
    want_rows = [s + k for s in range(0, 70, 32) for k in range(0, min(32, 70 - s), 3)]
    assert [t for t, _ in calls] == [(v, 1) for v in want_rows]
    assert all(len(out) == 1 and out[0][0] == t[0] for t, out in calls)
    assert got == host


def test_mvpa_host_fallback_for_flagged_centres(monkeypatch):
    rng = np.random.RandomState(8)
    dims, E = (8, 8, 7), 24
    data = rng.randn(*dims, E).astype(np.float32)
    labels = np.arange(E) % 2
    mask = rng.rand(*dims) > 0.2
    sl = slm.Searchlight(sl_rad=1, shape=slm.Cube)
    host = MVPAVoxelSelector(data, mask, labels, 4, sl, gpu_cv=False).run(svm.SVC())
    _flag_every_third(monkeypatch)
    import brainiak_b200.fcma.mvpa_voxelselector as mv
    calls = []
    orig = mv._host_accuracy
    monkeypatch.setattr(mv, "_host_accuracy", lambda *a: calls.append(1) or orig(*a))
    gpu = MVPAVoxelSelector(data, mask, labels, 4, sl, batch_centres=40).run(svm.SVC())
    ncentres = len(engine.searchlight_centres(mask, 1, sl.shape, sl.min_active_voxels_proportion)[0])
    assert len(calls) == sum(len(range(0, min(40, ncentres - b), 3)) for b in range(0, ncentres, 40))
    assert gpu[1] == host[1]
    assert all((a is None and b is None) or a == b for a, b in zip(gpu[0].ravel(), host[0].ravel()))


# the fixtures of tests/golden/make_golden_scale.py: the unmodified reference's lists for SVC() and
# SVC(C=10, shrinking=False); the inputs are regenerated from the generator's seeds
SCALE_CLFS = {"default": svm.SVC(), "c10": svm.SVC(C=10, shrinking=False)}


def _vs_scale_inputs(name):
    if name == "s1":
        raw, labels = synthetic.make_dyadic_epochs(48, 20, 140, seed=6161, informative=8)
        return raw, None, labels
    raw, _ = synthetic.make_dyadic_epochs(24, 16, 48, seed=7171, informative=6)
    raw2, _ = synthetic.make_dyadic_epochs(40, 16, 48, seed=8181, informative=10)
    return raw, raw2, [e % 3 for e in range(48)]


@pytest.mark.parametrize("gpu_cv", [True, False])
@pytest.mark.parametrize("name", ["s1", "s2"])
def test_voxel_selector_matches_reference_fixture(dev, golden, name, gpu_cv):
    """s1: E = 140, eps 20, 7 folds, one mask of 48 voxels, two classes; s2: E = 48, eps 12, 4 folds, three classes,
    two masks (24 x 40 voxels).  Dyadic inputs: the features are exact, so every accuracy is pinned."""
    g = golden("vs_scale_" + name)
    raw, raw2, labels = _vs_scale_inputs(name)
    assert _probe_matches(raw, g["probe"])
    if raw2 is not None:
        assert _probe_matches(raw2, g["probe2"])
    assert labels == [int(v) for v in g["labels"]]
    for key, clf in SCALE_CLFS.items():
        vs = VoxelSelector(labels, int(g["eps"]), int(g["num_folds"]), raw, raw2, device=dev, gpu_cv=gpu_cv,
                           process_num=0)
        assert vs._scale_ok(clf) == gpu_cv
        got = vs.run(clf)
        assert [v for v, _ in got] == g["vids_" + key].tolist(), key
        assert [a for _, a in got] == g["accs_" + key].tolist(), key


@pytest.mark.parametrize("batch", [None, 1, 7])
@pytest.mark.parametrize("name", ["s1", "s2"])
def test_mvpa_matches_reference_fixture(golden, name, batch):
    """s1: E = 32, 4 folds, two classes; s2: E = 216, 18 folds, three classes; sl_rad 1 cube."""
    z = golden("mvpa_scale_" + name)
    sl = slm.Searchlight(sl_rad=1, shape=slm.Cube)
    for key, clf in SCALE_CLFS.items():
        mvs = MVPAVoxelSelector(z["data"], z["mask"], z["labels"], int(z["num_folds"]), sl, batch_centres=batch)
        assert mvs._gpu_kind(clf) == "scale"
        assert_matches_scale_fixture(z, key, *mvs.run(clf))


VS_CASES = [
    # E, eps, folds, V, two masks, classes
    (12, 3, 3, 200, False, 2),
    (12, 3, 3, 160, True, 3),
    (32, 8, 4, 200, False, 3),
    (65, 13, 5, 120, True, 2),
    (140, 20, 7, 100, False, 2),
    (140, 20, 7, 90, True, 3),
    (256, 16, 16, 64, False, 3),
]


@pytest.mark.parametrize("E,eps,folds,V,two,ncls", VS_CASES)
def test_voxel_selector_run_matches_host(dev, E, eps, folds, V, two, ncls):
    raw, _ = synthetic.make_epochs(V, 48, E, seed=E * 17 + V)
    raw2 = synthetic.make_epochs(V - 23, 48, E, seed=E * 17 + V + 1)[0] if two else None
    labels = [e % ncls for e in range(E)]
    for clf in (svm.SVC(), svm.SVC(C=10, shrinking=False)):
        gpu = VoxelSelector(labels, eps, folds, raw, raw2, device=dev, gpu_cv=True)
        assert gpu._scale_ok(clf)
        host = VoxelSelector(labels, eps, folds, raw, raw2, device=dev, gpu_cv=False, process_num=0)
        got, want = gpu.run(clf), host.run(clf)
        assert got == want, (clf, [(g, w) for g, w in zip(got, want) if g != w][:5])


def test_voxel_selector_two_runs_bit_identical(dev):
    raw, _ = synthetic.make_epochs(300, 40, 140, seed=9)
    labels = [e % 2 for e in range(140)]
    vs = VoxelSelector(labels, 20, 7, raw, device=dev)
    a, b = vs.run(svm.SVC()), vs.run(svm.SVC())
    assert a == b
    op, _ = vs._operands()
    x = engine.feature_gram_wide(op, op, 0, 300, 20)
    y = engine.feature_gram_wide(op, op, 0, 300, 20)
    assert all(torch.equal(p, q) for p, q in zip(x, y))


@pytest.mark.parametrize("E,ncls,batch", [(16, 2, None), (16, 3, 37), (64, 2, None), (64, 4, 100), (216, 2, None),
                                          (216, 3, 250)])
def test_mvpa_run_matches_host(E, ncls, batch):
    rng = np.random.RandomState(E + ncls)
    dims = (10, 9, 9)
    data = rng.randn(*dims, E).astype(np.float32)
    labels = np.arange(E) % ncls
    data[3:7, 3:7, 3:6] += (0.4 * labels).astype(np.float32)
    mask = rng.rand(*dims) > 0.2
    sl = slm.Searchlight(sl_rad=1, shape=slm.Cube)
    for clf in (svm.SVC(), svm.SVC(C=10, shrinking=False)):
        mvs = MVPAVoxelSelector(data, mask, labels, 4, sl, batch_centres=batch)
        assert mvs._gpu_kind(clf) == "scale"
        gpu = mvs.run(clf)
        host = MVPAVoxelSelector(data, mask, labels, 4, sl, gpu_cv=False).run(clf)
        assert gpu[1] == host[1]
        assert all((a is None and b is None) or a == b for a, b in zip(gpu[0].ravel(), host[0].ravel()))


def test_entry_points_reject_bad_arguments(dev):
    op, _ = _operands(300, None, 40, 8, dev, seed=5)
    G, D, mom = engine.feature_gram_wide(op, op, 0, 4, 4)
    with pytest.raises(ValueError):
        engine.fold_gammas(mom, np.ones((2, 7), np.uint8), 300)           # wrong E
    with pytest.raises(ValueError):
        engine.fold_gammas(mom, np.zeros((2, 8), np.uint8), 300)          # a fold without training samples
    with pytest.raises(ValueError):
        engine.fold_gammas(mom, np.ones((2, 8), np.uint8), 0)
    g = torch.ones((4, 2), dtype=torch.float64, device=dev)
    with pytest.raises(ValueError):
        engine.rbf_fold_kernels(G, D, g, 2)
    with pytest.raises(ValueError):
        engine.rbf_fold_kernels(G, D.float(), g, 0)
