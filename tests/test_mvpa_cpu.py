"""Host-side pieces of the activity-based searchlight selector (MVPAVoxelSelector), no GPU needed.

* The searchlight shapes equal the reference definitions (cube; cityblock / euclidean distance <= r, computed here with
  scipy as the reference does).
* ``engine.searchlight_centres`` equals a direct loop written like the reference's ``_singlenode_searchlight``
  (searchlight.py:542-578): interior mask voxels, the proportion test with its strict ``>`` and ``p = 0`` = no test.
* The exactness argument the GPU path rests on, pinned against scikit-learn: ``SVC(kernel='linear' | 'rbf')`` fitted on
  float32 features and ``SVC(kernel='precomputed')`` fitted on the fp64 kernels k_searchlight_kernels computes (G summed
  in fp64 in feature order; rbf: x_square form for training, difference form for the decisions) give identical
  iteration counts, support sets and predictions.
* ``generate_epochs_info``, ``prepare_mvpa_data`` and ``prepare_searchlight_mvpa_data`` reproduce the unmodified
  reference bit for bit on its two test subjects (and agree with its own expected files) and on a synthetic case with
  unequal epoch lengths, a subject with one epoch of a condition, a constant voxel and the reproducible voxel shuffle.
* The host path of ``MVPAVoxelSelector`` (any classifier the GPU does not take, or ``gpu_cv=False``) reproduces the
  unmodified reference's volumes and lists on every fixture of tests/golden/make_golden_mvpa.py.
"""
import numpy as np
import pytest
from scipy.spatial.distance import cityblock, euclidean
from sklearn import model_selection, svm
from sklearn.linear_model import LogisticRegression

from brainiak_b200 import searchlight as slm
from brainiak_b200.fcma import engine, preprocessing
from brainiak_b200.fcma.mvpa_voxelselector import MVPAVoxelSelector

FIXTURES = ["a", "b1", "b2", "b3", "b4", "c"]


@pytest.mark.parametrize("rad", [0, 1, 2, 3, 4])
def test_shapes_match_reference_definitions(rad):
    side = 2 * rad + 1
    cube = np.ones((side,) * 3, dtype=bool)
    diamond = np.zeros((side,) * 3, dtype=bool)
    ball = np.zeros((side,) * 3, dtype=bool)
    for i in range(side):
        for j in range(side):
            for k in range(side):
                diamond[i, j, k] = cityblock((i, j, k), (rad, rad, rad)) <= rad
                ball[i, j, k] = euclidean((i, j, k), (rad, rad, rad)) <= rad
    assert np.array_equal(slm.Cube(rad).mask_, cube)
    assert np.array_equal(slm.Diamond(rad).mask_, diamond)
    assert np.array_equal(slm.Ball(rad).mask_, ball)
    sl = slm.Searchlight(sl_rad=rad, shape=slm.Ball)
    assert sl.sl_rad == rad and np.array_equal(sl.shape, ball)


def _loop_centres(mask, r, shape, p):
    """Centres as _singlenode_searchlight visits them on the whole volume."""
    out, nf = [], []
    X, Y, Z = mask.shape
    for i in range(r, X - r):
        for j in range(r, Y - r):
            for k in range(r, Z - r):
                if not mask[i, j, k]:
                    continue
                m = mask[i - r:i + r + 1, j - r:j + r + 1, k - r:k + r + 1] * shape
                if p == 0 or np.count_nonzero(m) / m.size > p:
                    out.append(np.ravel_multi_index((i, j, k), mask.shape))
                    nf.append(np.count_nonzero(m))
    return np.array(out, dtype=np.int64), np.array(nf, dtype=np.int64)


@pytest.mark.parametrize("shape_cls", [slm.Cube, slm.Diamond, slm.Ball])
@pytest.mark.parametrize("r", [0, 1, 2, 3])
@pytest.mark.parametrize("p", [0, 0.2, 0.5, 0.7])
def test_centre_selection_matches_searchlight_loop(shape_cls, r, p):
    rng = np.random.RandomState(100 * r + int(10 * p))
    mask = rng.rand(9, 8, 10) > 0.35
    mask[0] = True                       # a face fully in the mask: never a centre (r > 0)
    shape = shape_cls(r).mask_
    c, n = engine.searchlight_centres(mask, r, shape, p)
    c_ref, n_ref = _loop_centres(mask, r, shape, p)
    assert np.array_equal(c, c_ref) and np.array_equal(n, n_ref)


def test_centre_selection_strict_threshold_and_small_volume():
    mask = np.ones((3, 3, 3), dtype=bool)
    shape = slm.Cube(1).mask_
    mask[0, 0, 0] = False                # 26 / 27 active
    assert len(engine.searchlight_centres(mask, 1, shape, 26 / 27)[0]) == 0
    assert len(engine.searchlight_centres(mask, 1, shape, 25.9 / 27)[0]) == 1
    assert len(engine.searchlight_centres(mask, 2, slm.Cube(2).mask_, 0)[0]) == 0   # volume smaller than a cube


def _seq_gram(X):
    """fp64 Gram matrix summed sequentially over the features (k_searchlight_kernels' order)."""
    X = X.astype(np.float64)
    G = np.zeros((len(X), len(X)))
    for f in range(X.shape[1]):
        G = G + X[:, f, None] * X[None, :, f]
    return G


def _seq_dist(X):
    X = X.astype(np.float64)
    D = np.zeros((len(X), len(X)))
    for f in range(X.shape[1]):
        d = X[:, f, None] - X[None, :, f]
        D = D + d * d
    return D


@pytest.mark.parametrize("kernel", ["linear", "rbf"])
@pytest.mark.parametrize("shrinking", [False, True])
@pytest.mark.parametrize("nclass", [2, 3, 4])
def test_fp64_kernels_reproduce_svc_on_features(kernel, shrinking, nclass):
    rng = np.random.RandomState(7 * nclass + (kernel == "rbf") + 2 * shrinking)
    problems = 0
    for trial in range(6):
        E = int(rng.choice([16, 24, 40, 64]))
        n = int(rng.choice([7, 19, 27, 33]))
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
        skf = model_selection.StratifiedKFold(n_splits=int(rng.choice([2, 4])), shuffle=False)
        for tr, te in skf.split(X, y):
            a = svm.SVC(kernel=kernel, C=C, gamma="auto", shrinking=shrinking).fit(X[tr], y[tr])
            b = svm.SVC(kernel="precomputed", C=C, shrinking=shrinking).fit(Kfit[np.ix_(tr, tr)], y[tr])
            assert np.array_equal(a.n_iter_, b.n_iter_)
            assert np.array_equal(a.support_, b.support_)
            assert np.array_equal(a.predict(X[te]), b.predict(Kpred[np.ix_(te, tr)]))
            problems += 1
    assert problems >= 12


def load_fixture(golden, name):
    z = golden("mvpa_" + name)
    shape_cls = {"Cube": slm.Cube, "Ball": slm.Ball, "Diamond": slm.Diamond}[str(z["shape"])]
    sl = slm.Searchlight(sl_rad=int(z["sl_rad"]), shape=shape_cls, min_active_voxels_proportion=float(z["min_active"]))
    spec = str(z["clf"])
    if spec == "logistic":
        clf = LogisticRegression()
    elif spec.startswith("rbf"):
        clf = svm.SVC(kernel="rbf", C=10, gamma="auto")
    else:
        clf = svm.SVC(kernel="linear", shrinking=False, C=1)
    return z, sl, clf


def assert_matches_fixture(z, volume, results):
    assert volume.shape == z["mask"].shape and volume.dtype == object
    ref = z["volume"]
    none = np.array([v is None for v in volume.ravel()]).reshape(volume.shape)
    assert np.array_equal(none, np.isnan(ref))
    got = np.array([np.nan if v is None else v for v in volume.ravel()], dtype=np.float64).reshape(volume.shape)
    assert np.array_equal(got[~none], ref[~none])
    assert [t[0] for t in results] == z["ids"].tolist()
    assert np.array_equal(np.array([t[1] for t in results], dtype=np.float64), z["acc"])


@pytest.mark.parametrize("name", FIXTURES)
def test_host_path_matches_reference(golden, name):
    z, sl, clf = load_fixture(golden, name)
    mvs = MVPAVoxelSelector(z["data"], z["mask"], z["labels"], int(z["num_folds"]), sl, gpu_cv=False)
    volume, results = mvs.run(clf)
    assert_matches_fixture(z, volume, results)


def test_zero_voxels_and_shape_mismatch_raise():
    sl = slm.Searchlight(sl_rad=1)
    with pytest.raises(ValueError, match="Zero processed voxels"):
        MVPAVoxelSelector(np.zeros((4, 4, 4, 8), np.float32), np.zeros((4, 4, 4)), [0, 1] * 4, 2, sl)
    mvs = MVPAVoxelSelector(np.zeros((4, 4, 5, 8), np.float32), np.ones((4, 4, 4)), [0, 1] * 4, 2, sl, gpu_cv=False)
    with pytest.raises(ValueError, match="mask shape"):
        mvs.run(LogisticRegression())


class _Image:
    def __init__(self, data):
        self.data = data

    def get_fdata(self):
        return self.data

    def get_filename(self):
        return "image"


def test_generate_epochs_info_matches_reference(golden):
    z = golden("mvpa_preproc")
    for ep, info in ((z["epochs"], z["info"]), (z["ep"], z["syn_info"])):
        got = preprocessing.generate_epochs_info(list(ep))
        assert [tuple(int(v) for v in t) for t in got] == [tuple(t) for t in info.tolist()]


@pytest.mark.parametrize("as_array", [False, True])
def test_prepare_mvpa_data_matches_reference(golden, as_array):
    z = golden("mvpa_preproc")
    wrap = (lambda v: v) if as_array else _Image
    pd, labels = preprocessing.prepare_mvpa_data([wrap(v) for v in z["subj"]], list(z["epochs"]), z["mask"])
    assert pd.dtype == z["pd"].dtype and np.array_equal(pd, z["pd"]) and np.allclose(pd, z["expected"])
    assert np.array_equal(labels, z["labels"])
    pd, labels = preprocessing.prepare_mvpa_data([wrap(v) for v in z["vols"]], list(z["ep"]), z["smask"])
    assert np.array_equal(pd, z["syn_pd"]) and np.array_equal(labels, z["syn_labels"])


@pytest.mark.parametrize("as_array", [False, True])
def test_prepare_searchlight_mvpa_data_matches_reference(golden, as_array):
    z = golden("mvpa_preproc")
    wrap = (lambda v: v) if as_array else _Image
    sd, labels = preprocessing.prepare_searchlight_mvpa_data([wrap(v) for v in z["subj"]], list(z["epochs"]))
    assert sd.dtype == np.float32 and np.array_equal(sd, z["sd"]) and np.allclose(sd, z["expected_sl"])
    assert np.array_equal(labels, z["sl_labels"])
    sd, _ = preprocessing.prepare_searchlight_mvpa_data([wrap(v) for v in z["vols"]], list(z["ep"]))
    assert np.array_equal(sd, z["syn_sd"])
    assert np.all(sd[2, 3, 1, :] == 0)                   # the constant voxel: sigma 0 -> nan -> 0
    sd, _ = preprocessing.prepare_searchlight_mvpa_data([wrap(v) for v in z["vols"]], list(z["ep"]),
                                                        random=preprocessing.RandomType.REPRODUCIBLE)
    assert np.array_equal(sd, z["syn_sd_rand"])
