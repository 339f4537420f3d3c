"""SVC(kernel='rbf', gamma='scale') on the GPU, the parts that need no device.

* The routing table of engine.svc_scale_supported, VoxelSelector._scale_ok and MVPAVoxelSelector._gpu_kind; the existing
  routes keep their meaning (svc_feature_kind(SVC()) is None).
* The gamma of fcma_fold_gammas restated with exact rational sums -- var = Q / N - (S / N)^2 rounded once, then
  scikit-learn's 1 / (F var) -- against ``SVC().fit(X)._gamma``, and its flag rule ``mean^2 > 2^36 var`` on both sides of
  the bound (DESIGN.md §3.9).
* engine.fold_problems and engine.fold_train_mask: the problems of one fold, for two and more classes.
"""
from fractions import Fraction

import numpy as np
import pytest
from sklearn import model_selection, svm

from brainiak_b200 import searchlight as slm
from brainiak_b200.fcma import engine
from brainiak_b200.fcma.mvpa_voxelselector import MVPAVoxelSelector
from brainiak_b200.fcma.voxelselector import VoxelSelector

FLAG_BOUND = 2.0 ** 36


def _labels(E, k):
    return [e % k for e in range(E)]


@pytest.mark.parametrize("clf,E,folds,k,want", [
    (svm.SVC(), 32, 4, 2, True),
    (svm.SVC(C=10), 140, 7, 2, True),
    (svm.SVC(kernel="rbf"), 256, 16, 3, True),
    (svm.SVC(shrinking=False, tol=1e-4), 12, 3, 3, True),
    (svm.SVC(gamma="auto"), 32, 4, 2, False),
    (svm.SVC(gamma=0.1), 32, 4, 2, False),
    (svm.SVC(kernel="linear"), 32, 4, 2, False),
    (svm.SVC(kernel="poly"), 32, 4, 2, False),
    (svm.SVC(kernel="sigmoid"), 32, 4, 2, False),
    (svm.SVC(kernel="precomputed"), 32, 4, 2, False),
    (svm.SVC(class_weight="balanced"), 32, 4, 2, False),
    (svm.SVC(probability=True), 32, 4, 2, False),
    (svm.SVC(break_ties=True, decision_function_shape="ovr"), 32, 4, 3, False),
    (svm.SVC(), 257, 4, 2, False),
    (svm.SVC(), 260, 65, 2, False),
    (svm.SVC(), 6, 4, 2, False),                 # 3 samples per class cannot make 4 stratified folds
    (svm.LinearSVC(), 32, 4, 2, False),
])
def test_routing_table(clf, E, folds, k, want):
    assert engine.svc_scale_supported(clf, _labels(E, k), folds, E) is want


def test_existing_routes_unchanged():
    y = _labels(32, 2)
    assert engine.svc_feature_kind(svm.SVC(), y, 4, 32) is None
    assert engine.svc_feature_kind(svm.SVC(kernel="rbf"), y, 4, 32, max_epochs=256) is None
    assert engine.svc_feature_kind(svm.SVC(gamma="auto"), y, 4, 32) == "rbf"
    assert engine.svc_feature_kind(svm.SVC(kernel="poly"), y, 4, 32) is None
    assert engine.svc_feature_kind(svm.SVC(kernel="sigmoid"), y, 4, 32) is None


def test_selector_routing():
    rng = np.random.RandomState(0)
    raw = [rng.randn(20, 30).astype(np.float32) for _ in range(16)]
    y = _labels(16, 2)
    vs = VoxelSelector(y, 4, 4, raw)
    assert vs._scale_ok(svm.SVC()) and vs._scale_ok(svm.SVC(C=10))
    assert vs._feature_kind(svm.SVC(), max_epochs=256) is None
    assert not vs._scale_ok(svm.SVC(gamma="auto")) and not vs._scale_ok(svm.SVC(kernel="precomputed"))
    assert not VoxelSelector(y, 4, 4, raw, gpu_cv=False)._scale_ok(svm.SVC())
    assert not VoxelSelector(y, 4, 4, raw, mask_self=True)._scale_ok(svm.SVC())
    data = rng.randn(5, 5, 5, 16).astype(np.float32)
    sl = slm.Searchlight(sl_rad=1, shape=slm.Cube)
    mask = np.ones((5, 5, 5), dtype=bool)
    assert MVPAVoxelSelector(data, mask, y, 4, sl)._gpu_kind(svm.SVC()) == "scale"
    assert MVPAVoxelSelector(data, mask, y, 4, sl)._gpu_kind(svm.SVC(gamma="auto")) == "rbf"
    assert MVPAVoxelSelector(data.astype(np.float64), mask, y, 4, sl)._gpu_kind(svm.SVC()) is None
    assert MVPAVoxelSelector(data, mask, y, 4, sl, gpu_cv=False)._gpu_kind(svm.SVC()) is None


def exact_gamma(X):
    """fcma_fold_gammas restated: exact S, Q and N; var rounded once; scikit-learn's roundings; the flag."""
    X = np.asarray(X, dtype=np.float64)
    n, F = X.shape
    N = n * F
    S = sum(Fraction(float(x)) for x in X.ravel())
    Q = sum(Fraction(float(x)) ** 2 for x in X.ravel())
    var = float(Q / N - (S / N) ** 2)
    mean = float(S / N)
    gamma = 1.0 / (F * var) if var != 0 else 1.0
    return gamma, mean * mean > FLAG_BOUND * var


def _ulps(a, b):
    return abs(a - b) / np.spacing(max(abs(a), abs(b)))


@pytest.mark.parametrize("n,F,loc,seed", [(12, 27, 0.0, 0), (20, 300, 0.3, 1), (60, 33, -2.0, 2), (200, 257, 0.0, 3),
                                          (36, 5000, 1.0, 4), (140, 40, 100.0, 5), (17, 1, 0.0, 6), (99, 129, 1e3, 7)])
def test_exact_variance_gamma_matches_sklearn(n, F, loc, seed):
    rng = np.random.RandomState(seed)
    X = (loc + rng.randn(n, F)).astype(np.float32)
    y = np.arange(n) % 2
    want = svm.SVC().fit(X, y)._gamma
    got, flagged = exact_gamma(X)
    assert not flagged
    assert _ulps(got, want) <= 4, (got, want)


def test_all_zero_features_give_one():
    X = np.zeros((10, 7), dtype=np.float32)
    assert exact_gamma(X) == (1.0, False)
    assert svm.SVC().fit(X, np.arange(10) % 2)._gamma == 1.0


@pytest.mark.parametrize("c", [3.0, 0.1, -7.25, 1e-3])
def test_constant_nonzero_features_are_flagged(c):
    X = np.full((30, 11), c, dtype=np.float32)
    gamma, flagged = exact_gamma(X)
    assert flagged and gamma == 1.0


def test_flag_bound_both_sides():
    """|mean| / sigma just below 2^18 is kept and matches scikit-learn; above it the item is flagged.  The bound is a
    sufficient condition: on float32 features NumPy's sums are usually exact, so a flagged item often has the same
    gamma on both sides -- it is scored on the host all the same."""
    rng = np.random.RandomState(11)
    noise = rng.choice([-1.0, 1.0], size=(24, 16))          # sigma = 1 exactly
    below = np.float32(2.0 ** 17) + noise.astype(np.float32)
    g, flagged = exact_gamma(below)
    assert not flagged
    assert _ulps(g, svm.SVC().fit(below, np.arange(24) % 2)._gamma) <= 4
    above = np.float32(2.0 ** 19) + (noise * 2.0 ** -4).astype(np.float32)   # |mean| / sigma = 2^23
    assert np.all(above.astype(np.float64) - 2.0 ** 19 == noise * 2.0 ** -4)
    _, flagged = exact_gamma(above)
    assert flagged
    far = (2.0 ** 40 + noise * 2.0 ** 17).astype(np.float64)   # |mean| / sigma = 2^23, exact in float32 too
    far32 = far.astype(np.float32)
    assert np.array_equal(far32.astype(np.float64), far)
    _, flagged = exact_gamma(far32)
    assert flagged


# the MVPAVoxelSelector fixtures of tests/golden/make_golden_scale.py (the unmodified reference's volumes and lists for
# SVC() and SVC(C=10, shrinking=False)); the host path needs no GPU
SCALE_CLFS = {"default": svm.SVC(), "c10": svm.SVC(C=10, shrinking=False)}


def assert_matches_scale_fixture(z, key, volume, results):
    ref = z["volume_" + key]
    none = np.array([v is None for v in volume.ravel()]).reshape(volume.shape)
    assert np.array_equal(none, np.isnan(ref))
    got = np.array([np.nan if v is None else v for v in volume.ravel()], dtype=np.float64).reshape(volume.shape)
    assert np.array_equal(got[~none], ref[~none])
    assert [t[0] for t in results] == z["ids_" + key].tolist()
    assert np.array_equal(np.array([t[1] for t in results], dtype=np.float64), z["acc_" + key])


@pytest.mark.parametrize("key", list(SCALE_CLFS))
@pytest.mark.parametrize("name", ["s1", "s2"])
def test_mvpa_host_path_matches_reference_fixture(golden, name, key):
    z = golden("mvpa_scale_" + name)
    sl = slm.Searchlight(sl_rad=1, shape=slm.Cube)
    mvs = MVPAVoxelSelector(z["data"], z["mask"], z["labels"], int(z["num_folds"]), sl, gpu_cv=False)
    assert_matches_scale_fixture(z, key, *mvs.run(SCALE_CLFS[key]))


@pytest.mark.parametrize("k,E,folds", [(2, 16, 4), (3, 24, 4), (4, 140, 7), (2, 256, 16)])
def test_fold_problems_and_train_mask(k, E, folds):
    y = np.asarray(_labels(E, k))
    full = engine.svm_folds_for(y, folds, E)
    npairs = len(full.pairs)
    assert npairs == k * (k - 1) // 2
    skf = list(model_selection.StratifiedKFold(folds).split(np.zeros((E, 1)), y))
    train = engine.fold_train_mask(full, E)
    assert train.shape == (folds, E) and train.dtype == np.uint8
    for f, (tr, te) in enumerate(skf):
        want = np.zeros(E, dtype=np.uint8)
        want[tr] = 1
        assert np.array_equal(train[f], want)
        part = engine.fold_problems(full, f)
        assert part.num_folds == 1 and part.nproblems == npairs and part.wide == full.wide
        assert part.pairs == full.pairs and np.array_equal(part.classes, full.classes)
        assert np.array_equal(part.n_test, [len(te)]) and np.array_equal(part.test_labels[0], full.test_labels[f])
        for q in range(npairs):
            assert bytes(part.structs[q]) == bytes(full.structs[f * npairs + q])


def test_feature_block_rows_counts_four_matrices():
    E, per_row = 140, 1 << 20
    budget = 1 << 30
    two = engine.feature_block_rows(E, per_row, 1 << 20, budget)
    four = engine.feature_block_rows(E, per_row, 1 << 20, budget, matrices=4)
    assert two == engine.feature_block_rows(E, per_row, 1 << 20, budget, matrices=2)
    assert four <= two and four * (per_row + 32 * E * E) <= budget
