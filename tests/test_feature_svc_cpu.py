"""VoxelSelector with SVC(kernel='linear' | 'rbf') on the GPU, the parts that need no GPU.

* The exactness argument of the feature path (DESIGN.md §3.8), at FCMA scale: libsvm keeps Q in float and QD and the
  decisions in double, so ``SVC(kernel=k)`` fitted on float32 features gives the same iterations, support vectors, dual
  coefficients and predictions as ``SVC(kernel='precomputed')`` on fp64 kernel matrices of those features whose sums are
  taken in another order -- here 64-column blocks through BLAS, as k_norm_gram_f64 sums in its own order.
* The routing table: which classifiers and options VoxelSelector cross-validates on the GPU.
"""
import numpy as np
import pytest
from sklearn import model_selection, svm
from sklearn.linear_model import LogisticRegression

from brainiak_b200.fcma import engine
from brainiak_b200.fcma.voxelselector import VoxelSelector


def _features(E, V2, nclass, eps, seed):
    """float32 within-subject z-scored correlation vectors of one voxel with a weak class signal, and their labels."""
    rng = np.random.default_rng(seed)
    y = np.arange(E) % nclass
    r = np.tanh(rng.normal(0.0, 0.25, (E, V2)) + 0.04 * rng.normal(size=(nclass, V2))[y]).astype(np.float32)
    z = 0.5 * np.log((1 + r) / (1 - r))
    z = z.reshape(E // eps, eps, V2)
    z = (z - z.mean(axis=1, keepdims=True)) / z.std(axis=1, keepdims=True)
    return z.reshape(E, V2).astype(np.float32), y


def _blocked_kernels(X, kind, gamma):
    """fp64 G (and D) summed over 64-column blocks, then libsvm's rbf forms: (K_fit, K_pred)."""
    X = X.astype(np.float64)
    E, V2 = X.shape
    G = np.zeros((E, E))
    D = np.zeros((E, E))
    for j in range(0, V2, 64):
        b = X[:, j:j + 64]
        G += b @ b.T
        if kind == 'rbf':
            D += ((b[:, None, :] - b[None, :, :]) ** 2).sum(axis=2)
    if kind == 'linear':
        return G, G
    d = np.diag(G)
    return np.exp(-gamma * ((d[:, None] + d[None, :]) - 2 * G)), np.exp(-gamma * D)


CASES = [
    # E, V2, classes, eps, kind, gamma, shrinking, C
    (16, 4099, 2, 8, 'linear', None, False, 1.0),
    (16, 50000, 2, 4, 'rbf', 'auto', True, 100.0),
    (32, 50000, 2, 8, 'linear', None, True, 0.02),
    (30, 50000, 3, 6, 'rbf', 'auto', False, 1.0),
    (32, 4099, 4, 8, 'rbf', 0.5, True, 10.0),
    (32, 50000, 4, 8, 'linear', None, False, 100.0),
    (64, 50000, 2, 16, 'rbf', 1e-4, True, 1.0),
    (64, 50000, 3, 8, 'linear', None, True, 1.0),
    (64, 4099, 2, 4, 'rbf', 'auto', False, 0.02),
]


@pytest.mark.parametrize("E,V2,nclass,eps,kind,gamma,shrinking,C", CASES)
def test_feature_svc_equals_precomputed_fp64_kernels(E, V2, nclass, eps, kind, gamma, shrinking, C):
    X, y = _features(E, V2, nclass, eps, seed=E * 7 + V2 + nclass)
    g = (1.0 / V2 if gamma == 'auto' else gamma) if kind == 'rbf' else None
    K_fit, K_pred = _blocked_kernels(X, kind, g)
    kw = dict(C=C, shrinking=shrinking)
    for tr, te in model_selection.StratifiedKFold(n_splits=4, shuffle=False).split(X, y):
        a = svm.SVC(kernel=kind, gamma=gamma, **kw) if kind == 'rbf' else svm.SVC(kernel=kind, **kw)
        a.fit(X[tr], y[tr])
        b = svm.SVC(kernel='precomputed', **kw).fit(K_fit[np.ix_(tr, tr)], y[tr])
        assert np.array_equal(a.n_iter_, b.n_iter_)
        assert np.array_equal(a.support_, b.support_)
        # QD (the kernel diagonal) enters each alpha step in double, so a different order of the sums moves the dual
        # coefficients in their last bits -- never enough to change a working-set choice, the support or a prediction
        np.testing.assert_allclose(a.dual_coef_, b.dual_coef_, rtol=1e-9, atol=0)
        assert np.array_equal(a.predict(X[te]), b.predict(K_pred[np.ix_(te, tr)]))


def test_routing_table():
    """engine.svc_feature_kind: the classifiers whose cross-validation on features runs as the fp64 GPU solver."""
    y2, y3 = [0, 1] * 8, [0, 1, 2] * 4
    kind = engine.svc_feature_kind
    assert kind(svm.SVC(kernel='linear'), y2, 4, 16) == 'linear'
    assert kind(svm.SVC(kernel='linear', shrinking=False, C=0.1), y3, 2, 12) == 'linear'
    assert kind(svm.SVC(kernel='rbf', gamma='auto'), y2, 4, 16) == 'rbf'
    assert kind(svm.SVC(kernel='rbf', gamma=0.25), y2, 4, 16) == 'rbf'
    assert kind(svm.SVC(kernel='rbf', gamma=0), y2, 4, 16) == 'rbf'
    assert kind(svm.SVC(kernel='rbf'), y2, 4, 16) is None                          # gamma='scale'
    assert kind(svm.SVC(kernel='rbf', gamma=-1.0), y2, 4, 16) is None
    assert kind(svm.SVC(kernel='rbf', gamma=True), y2, 4, 16) is None
    assert kind(svm.SVC(kernel='poly'), y2, 4, 16) is None
    assert kind(svm.SVC(kernel='sigmoid'), y2, 4, 16) is None
    assert kind(svm.SVC(kernel='precomputed'), y2, 4, 16) is None
    assert kind(svm.SVC(kernel='linear', class_weight='balanced'), y2, 4, 16) is None
    assert kind(svm.SVC(kernel='linear', probability=True), y2, 4, 16) is None
    assert kind(svm.SVC(kernel='linear', break_ties=True, decision_function_shape='ovr'), y3, 2, 12) is None
    assert kind(LogisticRegression(), y2, 4, 16) is None
    assert kind(svm.SVC(kernel='linear'), [0, 1] * 40, 4, 80) is None             # E > 64
    assert kind(svm.SVC(kernel='linear'), [0, 1] * 40, 65, 64) is None            # more than 64 folds
    assert kind(svm.SVC(kernel='linear'), [0] * 16, 4, 16) is None                # one class
    # the precomputed-kernel test is a different question and keeps its answer
    assert not engine.svm_cv_supported(svm.SVC(kernel='linear'), y2, 4, 16)


def test_voxel_selector_routing():
    """VoxelSelector._feature_kind: gpu_cv and mask_self are honoured on top of the classifier test."""
    rng = np.random.default_rng(0)
    raw = [rng.normal(size=(20, 40)).astype(np.float32) for _ in range(16)]
    labels = [0, 1] * 8

    def vs(**kw):
        return VoxelSelector(labels, 4, 4, raw, **kw)

    assert vs()._feature_kind(svm.SVC(kernel='linear')) == 'linear'
    assert vs()._feature_kind(svm.SVC(kernel='rbf', gamma='auto')) == 'rbf'
    assert vs(gpu_cv=False)._feature_kind(svm.SVC(kernel='linear')) is None
    assert vs(mask_self=True)._feature_kind(svm.SVC(kernel='linear')) is None
    assert vs()._feature_kind(svm.SVC(kernel='rbf')) is None
    assert vs()._feature_kind(LogisticRegression()) is None
    raw65 = [rng.normal(size=(20, 40)).astype(np.float32) for _ in range(66)]
    assert VoxelSelector([0, 1] * 33, 2, 4, raw65)._feature_kind(svm.SVC(kernel='linear')) is None
