"""MVPAVoxelSelector above 64 epochs, the host-side pieces (no GPU needed).

* ``engine.svc_feature_kind`` with ``max_epochs``: the default keeps the 64-epoch limit, ``SVM_WIDE_MAX_EPOCHS`` accepts
  up to 256 epochs with ``svm_folds_for`` folds; ``MVPAVoxelSelector._gpu_kind`` asks for the wide limit.
* The host path reproduces the unmodified reference on the fixtures above 64 epochs
  (tests/golden/make_golden_mvpa_wide.py): the example's call at 216 epochs, and a three-class rbf case at 140 epochs.
* The exactness argument of the GPU path at 140 and 216 epochs: ``SVC(kernel='linear' | 'rbf')`` on float32 features
  and ``SVC(kernel='precomputed')`` on the fp64 kernels summed sequentially in feature order give identical iteration
  counts, support sets and predictions.
"""
import numpy as np
import pytest
from sklearn import model_selection, svm

from brainiak_b200 import searchlight as slm
from brainiak_b200.fcma import engine
from brainiak_b200.fcma.mvpa_voxelselector import MVPAVoxelSelector
from test_mvpa_cpu import _seq_dist, _seq_gram, assert_matches_fixture, load_fixture


@pytest.mark.parametrize("E, default, wide", [(64, "linear", "linear"), (65, None, "linear"), (256, None, "linear"),
                                              (257, None, None)])
def test_svc_feature_kind_max_epochs(E, default, wide):
    labels = np.arange(E) % 2
    clf = svm.SVC(kernel="linear")
    assert engine.svc_feature_kind(clf, labels, 4, E) == default
    assert engine.svc_feature_kind(clf, labels, 4, E, max_epochs=engine.SVM_WIDE_MAX_EPOCHS) == wide
    rbf = svm.SVC(kernel="rbf", gamma="auto")
    assert engine.svc_feature_kind(rbf, labels, 4, E, max_epochs=256) == (wide and "rbf")


def test_svc_feature_kind_wide_limits():
    labels = np.arange(200) % 2
    assert engine.svc_feature_kind(svm.SVC(kernel="linear"), labels, 64, 200, max_epochs=256) == "linear"
    assert engine.svc_feature_kind(svm.SVC(kernel="linear"), labels, 65, 200, max_epochs=256) is None
    assert engine.svc_feature_kind(svm.SVC(kernel="rbf", gamma="scale"), labels, 4, 200, max_epochs=256) is None
    # a class missing from a training fold: svm_folds_for refuses the folds
    odd = np.zeros(200, dtype=int)
    odd[:2] = [1, 2]
    assert engine.svc_feature_kind(svm.SVC(kernel="linear"), odd, 2, 200, max_epochs=256) is None


def test_gpu_kind_routes_up_to_256_epochs():
    sl = slm.Searchlight(sl_rad=1)
    mask = np.ones((4, 4, 4), dtype=bool)
    clf = svm.SVC(kernel="linear", shrinking=False, C=1)
    for E, dtype, want in ((216, np.float32, "linear"), (257, np.float32, None), (216, np.float64, None)):
        data = np.zeros((4, 4, 4, E), dtype=dtype)
        assert MVPAVoxelSelector(data, mask, np.arange(E) % 2, 18, sl)._gpu_kind(clf) == want, (E, dtype)


@pytest.mark.parametrize("name", ["w1", "w2"])
def test_host_path_matches_reference_wide(golden, name):
    z, sl, clf = load_fixture(golden, name)
    assert z["data"].shape[3] > 64
    mvs = MVPAVoxelSelector(z["data"], z["mask"], z["labels"], int(z["num_folds"]), sl, gpu_cv=False)
    assert_matches_fixture(z, *mvs.run(clf))


@pytest.mark.parametrize("kernel", ["linear", "rbf"])
@pytest.mark.parametrize("shrinking", [False, True])
@pytest.mark.parametrize("E", [140, 216])
def test_fp64_kernels_reproduce_svc_on_features_wide(kernel, shrinking, E):
    rng = np.random.RandomState(E + 2 * shrinking + (kernel == "rbf"))
    problems = 0
    for trial in range(3):
        nclass = 2 + trial % 2
        n = int(rng.choice([7, 27, 33]))
        C = float(rng.choice([0.1, 1.0, 10.0]))
        y = np.arange(E) % nclass
        X = rng.randn(E, n).astype(np.float32)
        X[:, : max(1, n // 4)] += (np.float32(0.3) * y[:, None]).astype(np.float32)
        G = _seq_gram(X)
        if kernel == "linear":
            Kfit = Kpred = G
        else:
            g = 1.0 / n
            dg = np.diag(G)
            Kfit = np.exp(-g * ((dg[:, None] + dg[None, :]) - 2 * G))
            Kpred = np.exp(-g * _seq_dist(X))
        skf = model_selection.StratifiedKFold(n_splits=int(rng.choice([4, 7])), shuffle=False)
        for tr, te in skf.split(X, y):
            a = svm.SVC(kernel=kernel, C=C, gamma="auto", shrinking=shrinking).fit(X[tr], y[tr])
            b = svm.SVC(kernel="precomputed", C=C, shrinking=shrinking).fit(Kfit[np.ix_(tr, tr)], y[tr])
            assert np.array_equal(a.n_iter_, b.n_iter_)
            assert np.array_equal(a.support_, b.support_)
            assert np.array_equal(a.predict(X[te]), b.predict(Kpred[np.ix_(te, tr)]))
            problems += 1
    assert problems >= 12
