"""VoxelSelector with SVC(kernel='linear' | 'rbf') on the GPU above 64 epochs, the parts that need no GPU.

* The exactness argument of the feature path (DESIGN.md §3.8) at 96 to 256 epochs, on the splits of
  ``engine.svm_folds_for``: ``SVC(kernel=k)`` on float32 features gives the iterations, support vectors, dual
  coefficients and predictions of ``SVC(kernel='precomputed')`` on fp64 kernel matrices of those features summed in
  another order.
* The routing: ``VoxelSelector._feature_kind(clf, max_epochs=256)`` accepts up to 256 epochs, the default keeps 64.
* ``engine.feature_block_rows``: the workspace and the fp64 outputs of one pass stay within the budget.
"""
import numpy as np
import pytest
from sklearn import model_selection, svm
from sklearn.linear_model import LogisticRegression

from brainiak_b200.fcma import engine
from brainiak_b200.fcma.voxelselector import VoxelSelector
from test_feature_svc_cpu import _blocked_kernels, _features

CASES = [
    # E, V2, classes, eps, folds, kind, gamma, shrinking, C
    (96, 50000, 2, 8, 4, 'linear', None, False, 1.0),
    (140, 50000, 2, 20, 7, 'rbf', 'auto', True, 100.0),
    (140, 4099, 3, 20, 7, 'linear', None, True, 0.02),
    (216, 2049, 4, 12, 18, 'rbf', 1e-4, False, 10.0),
    (216, 4099, 3, 12, 6, 'rbf', 'auto', True, 0.02),
    (256, 1000, 3, 16, 16, 'linear', None, False, 100.0),
    (256, 4099, 2, 16, 16, 'rbf', 'auto', False, 1.0),
    (256, 2049, 4, 16, 8, 'linear', None, True, 10.0),
]


@pytest.mark.parametrize("E,V2,nclass,eps,folds,kind,gamma,shrinking,C", CASES)
def test_feature_svc_equals_precomputed_fp64_kernels_wide(E, V2, nclass, eps, folds, kind, gamma, shrinking, C):
    X, y = _features(E, V2, nclass, eps, seed=E * 7 + V2 + nclass)
    assert engine.svm_folds_for(y, folds, E).wide
    g = (1.0 / V2 if gamma == 'auto' else gamma) if kind == 'rbf' else None
    K_fit, K_pred = _blocked_kernels(X, kind, g)
    kw = dict(C=C, shrinking=shrinking)
    for tr, te in model_selection.StratifiedKFold(n_splits=folds, shuffle=False).split(X, y):
        a = svm.SVC(kernel=kind, gamma=gamma, **kw) if kind == 'rbf' else svm.SVC(kernel=kind, **kw)
        a.fit(X[tr], y[tr])
        b = svm.SVC(kernel='precomputed', **kw).fit(K_fit[np.ix_(tr, tr)], y[tr])
        assert np.array_equal(a.n_iter_, b.n_iter_)
        assert np.array_equal(a.support_, b.support_)
        np.testing.assert_allclose(a.dual_coef_, b.dual_coef_, rtol=1e-9, atol=0)
        assert np.array_equal(a.predict(X[te]), b.predict(K_pred[np.ix_(te, tr)]))


def _vs(E, eps=None, folds=4, nclass=2, **kw):
    rng = np.random.default_rng(E)
    raw = [rng.normal(size=(12, 24)).astype(np.float32) for _ in range(E)]
    return VoxelSelector(list(np.arange(E) % nclass), eps or E // 5 or 1, folds, raw, **kw)


@pytest.mark.parametrize("E", [65, 140, 256])
def test_voxel_selector_routing_wide(E):
    lin, rbf = svm.SVC(kernel='linear'), svm.SVC(kernel='rbf', gamma='auto')
    vs = _vs(E)
    assert vs._feature_kind(lin, max_epochs=256) == 'linear'
    assert vs._feature_kind(rbf, max_epochs=256) == 'rbf'
    assert vs._feature_kind(svm.SVC(kernel='rbf', gamma=0.5), max_epochs=256) == 'rbf'
    assert vs._feature_kind(lin) is None                          # the default keeps the 64-epoch limit
    assert vs._feature_kind(rbf) is None
    assert _vs(E, gpu_cv=False)._feature_kind(lin, max_epochs=256) is None
    assert vs._feature_kind(svm.SVC(kernel='rbf'), max_epochs=256) is None            # gamma='scale'
    assert vs._feature_kind(LogisticRegression(), max_epochs=256) is None
    assert _vs(E, folds=65)._feature_kind(lin, max_epochs=256) is None                # more than 64 folds
    # mask_self is not applied to the features: refused above 64 epochs, and host-side below
    with pytest.raises(ValueError):
        _vs(E, eps=1, mask_self=True)
    assert _vs(64, eps=16, mask_self=True)._feature_kind(lin, max_epochs=256) is None


def test_voxel_selector_routing_above_256():
    assert _vs(257)._feature_kind(svm.SVC(kernel='linear'), max_epochs=256) is None
    assert _vs(257)._feature_kind(svm.SVC(kernel='linear'), max_epochs=1000) is None


def _per_row(E, V2):
    """fcma_work_bytes_per_row: the tiled block holds E x ceil(V2 / 256) x 256 float32 per row."""
    return E * (-(-V2 // 256) * 256) * 4


@pytest.mark.parametrize("budget", [32 << 30, 6 << 30, 1 << 30])
def test_feature_block_rows_within_budget(budget):
    for E in (65, 100, 140, 200, 256):
        for V2 in (1, 255, 1000, 4129, 20000, 50000):
            per_row = _per_row(E, V2)
            for n in (1, 255, 1000, 50000):
                cost = per_row + 16 * E * E
                rows = engine.feature_block_rows(E, per_row, n, budget)
                assert 1 <= rows <= n
                assert rows * cost <= budget, (E, V2, n, rows)
                if rows > 256:
                    assert rows % 256 == 0
                # when the budget is what limits the pass: as many rows as fit (whole 256-row blocks above 256)
                if budget // cost < n:
                    assert (rows + (256 if rows >= 256 else 1)) * cost > budget


def test_feature_block_rows_counts_outputs():
    # 50 000 row voxels against a 1 000-voxel second mask at 256 epochs: the workspace alone would take 32 768 rows (32 GB),
    # and their K_fit + K_pred another 32 GB
    per_row = _per_row(256, 1000)
    assert (32 << 30) // per_row >= 32768
    rows = engine.feature_block_rows(256, per_row, 50000, 32 << 30)
    assert rows == 16384
    assert rows * (per_row + 16 * 256 * 256) <= 32 << 30
