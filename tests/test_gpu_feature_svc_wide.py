"""VoxelSelector's GPU path for SVC(kernel='linear' | 'rbf') on the normalised correlation vectors above 64 epochs.

* engine.feature_kernels_f64_wide (the block normalised in place, then k_feature_gram_tiled) element by element against
  exact sums of the fp64 products of the z that ``within_subject_norm_`` gives on the same raw correlations, with the
  bounds of test_gpu_feature_svc.py, at 64-epoch tile edges, with trailing raw epochs, one and two masks, tiled and
  strided blocks.
* Both matrices exactly symmetric, rbf diagonals exactly 1; entries of the same epoch pair bit-identical in every tile.
* At E <= 64: D and the rbf K_pred bit-identical to feature_kernels_f64, and the same cross-validation.
* Two runs bit-identical; the entry point's argument checks.
* ``VoxelSelector.run(clf)`` with ``gpu_cv=True`` returns the list ``gpu_cv=False`` returns at 65, 140 and 256 epochs,
  and the unmodified reference's list on the fixtures of tests/golden/make_golden_feature_wide.py.
"""
import ctypes

import numpy as np
import pytest
import torch
from sklearn import svm

from brainiak_b200 import _lib
from brainiak_b200.fcma import engine, synthetic
from brainiak_b200.fcma.voxelselector import VoxelSelector
from test_gpu_feature_svc import U, _exact_sums, _gamma_n, _operands, dev  # noqa: F401  (dev: fixture)
from test_gpu_parity import _probe_matches

pytestmark = pytest.mark.gpu


def _check_against_exact(op, op2, start, nb, eps, G, Kf, Kp, gamma, name):
    n2 = op2.V
    r = engine.corr_block(op, op2, start, nb, layout=0).contiguous()
    z = engine.within_subject_norm_(r, eps).cpu().numpy()
    G_ex, A, D_ex = _exact_sums(z, rbf=True)
    bound = _gamma_n(n2 + 16) * A + U * np.abs(G_ex)
    assert np.all(np.abs(G - G_ex) <= bound), (name, np.max(np.abs(G - G_ex) - bound))
    assert np.array_equal(G, np.swapaxes(G, 1, 2))
    d = np.diagonal(G, axis1=1, axis2=2)
    want = np.exp(-gamma * ((d[:, :, None] + d[:, None, :]) - 2.0 * G))
    assert np.all(np.abs(Kf - want) <= 2 * np.spacing(want)), name
    assert np.array_equal(Kf, np.swapaxes(Kf, 1, 2))
    assert np.all(np.diagonal(Kf, axis1=1, axis2=2) == 1.0)
    bd = _gamma_n(n2 + 1) * D_ex + U * D_ex
    lo, hi = np.exp(-gamma * (D_ex + bd)), np.exp(-gamma * np.maximum(D_ex - bd, 0))
    assert np.all((Kp >= lo - 2 * np.spacing(lo)) & (Kp <= hi + 2 * np.spacing(hi))), name
    assert np.array_equal(Kp, np.swapaxes(Kp, 1, 2))
    assert np.all(np.diagonal(Kp, axis1=1, axis2=2) == 1.0)


# name, V (rows), V2 (two masks) or None (one mask: V2 = V), T, E, eps, start, nb, ragged
CASES = [
    ("E1_eps1", 300, 33, 40, 1, 1, 0, 3, False),
    ("E63_eps3", 300, 257, 40, 63, 3, 5, 2, False),
    ("E64_eps16", 300, 4129, 40, 64, 16, 250, 2, False),
    ("E65_eps20", 300, 255, 40, 65, 20, 7, 2, True),
    ("E127_eps16", 300, 1, 40, 127, 16, 299, 1, False),
    ("E128_eps16", 300, None, 40, 128, 16, 17, 2, False),
    ("E129_eps3", 300, 257, 40, 129, 3, 100, 2, False),
    ("E140_eps20", 300, 4129, 40, 140, 20, 3, 1, True),
    ("E200_eps16", 300, 33, 40, 200, 16, 11, 2, False),
    ("E256_eps256", 300, 255, 40, 256, 256, 0, 2, False),
    ("E256_eps1", 300, 257, 40, 256, 1, 40, 1, True),
]


@pytest.mark.parametrize("layout", ["strided", "tiled"])
@pytest.mark.parametrize("name,V,V2,T,E,eps,start,nb,ragged", CASES, ids=[c[0] for c in CASES])
def test_feature_kernels_wide_element_by_element(dev, name, V, V2, T, E, eps, start, nb, ragged, layout):
    op, op2 = _operands(V, V2, T, E, dev, seed=E * 101 + (V2 or 0), ragged=ragged)
    n2 = op2.V
    # fewer than 256 rows of scratch: strided [nb][E][ld] block; 256: tiled block
    work = engine.Workspace(E, n2, 2 if layout == "strided" else 256, dev)
    G, G2 = engine.feature_kernels_f64_wide(op, op2, start, nb, eps, "linear", work=work)
    assert G is G2
    gamma = 0.37 / max(n2, 1)
    Kf, Kp = engine.feature_kernels_f64_wide(op, op2, start, nb, eps, "rbf", gamma, work=work)
    G = G.cpu().numpy()
    _check_against_exact(op, op2, start, nb, eps, G, Kf.cpu().numpy(), Kp.cpu().numpy(), gamma, name)


def test_tiles_are_independent(dev):
    """One 64-epoch pattern of whole subjects (eps 16) repeated four times: the entries of the same epoch pair sit in
    different tiles (diagonal and off-diagonal, above and below the diagonal) at the same position mod 8 and must be
    bit-identical."""
    V, T = 300, 40
    raw, _ = synthetic.make_epochs(V, T, 64, seed=3)
    raw2, _ = synthetic.make_epochs(517, T, 64, seed=4)
    raw, raw2 = raw * 4, raw2 * 4
    ep, T_e = engine.stack_epochs(raw, dev)
    ep2, _ = engine.stack_epochs(raw2, dev)
    op, op2 = engine.pack_epochs(ep, T_e, "tf32x3"), engine.pack_epochs(ep2, T_e, "tf32x3")
    for layout_rows in (2, 256):
        work = engine.Workspace(256, 517, layout_rows, dev)
        for kind, gamma in (("linear", None), ("rbf", 1e-3)):
            Kf, Kp = engine.feature_kernels_f64_wide(op, op2, 9, 3, 16, kind, gamma, work=work)
            for K in (Kf, Kp):
                K = K.cpu().numpy()
                base = K[:, :64, :64]
                for p in range(4):
                    for q in range(4):
                        assert np.array_equal(K[:, 64 * p:64 * p + 64, 64 * q:64 * q + 64], base), (kind, p, q)


@pytest.mark.parametrize("E,eps,V2,ncls", [(1, 1, 33, 1), (16, 4, 4129, 2), (33, 3, 257, 3), (64, 16, 1000, 2)])
def test_wide_matches_narrow_up_to_64_epochs(dev, E, eps, V2, ncls):
    op, op2 = _operands(300, V2, 40, E, dev, seed=E * 7 + V2)
    work = engine.Workspace(E, V2, 256, dev)
    nb, start = 40, 13
    gamma = 0.5 / V2
    Gn, _ = engine.feature_kernels_f64(op, op2, start, nb, eps, "linear", work=work)
    Gw, _ = engine.feature_kernels_f64_wide(op, op2, start, nb, eps, "linear", work=work)
    Fn, Pn = engine.feature_kernels_f64(op, op2, start, nb, eps, "rbf", gamma, work=work)
    Fw, Pw = engine.feature_kernels_f64_wide(op, op2, start, nb, eps, "rbf", gamma, work=work)
    assert torch.equal(Pn, Pw)            # D, then the same rbf_pred
    _check_against_exact(op, op2, start, 2, eps, Gw[:2].cpu().numpy(), Fw[:2].cpu().numpy(), Pw[:2].cpu().numpy(),
                         gamma, "E%d" % E)
    if ncls < 2:
        return
    labels = [e % ncls for e in range(E)]
    folds = 4 if E >= 16 else 2
    for Kn, Kw, Pn_, Pw_ in ((Gn, Gw, Gn, Gw), (Fn, Fw, Pn, Pw)):
        for shrinking in (False, True):
            an, itn = engine.svm_cv_f64(Kn, Pn_, labels, folds, C=1.0, shrinking=shrinking, return_iters=True)
            aw, itw = engine.svm_cv_f64(Kw, Pw_, labels, folds, C=1.0, shrinking=shrinking, return_iters=True)
            assert np.array_equal(an, aw) and np.array_equal(itn, itw)


def test_two_runs_bit_identical(dev):
    op, op2 = _operands(600, 700, 40, 140, dev, seed=77)
    work = engine.Workspace(140, 700, 256, dev)
    a = engine.feature_kernels_f64_wide(op, op2, 0, 600, 20, "rbf", 1e-3, work=work)
    b = engine.feature_kernels_f64_wide(op, op2, 0, 600, 20, "rbf", 1e-3, work=work)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_entry_point_rejects_bad_arguments(dev):
    E = 8
    op, _ = _operands(300, None, 40, E, dev, seed=5)
    lib = _lib.load()
    work = engine.Workspace(E, 300, 4, dev)
    K = torch.empty((4, E, E), dtype=torch.float64, device=dev)

    def call(E_=E, eps=4, kind=1, gamma=0.1, K_fit=K, K_pred=K):
        return lib.fcma_voxel_feature_kernels_wide(
            op.buf.data_ptr(), op.buf.data_ptr(), _lib.PREC[op.precision], E_, op.T, op.V, op.V, 0, 4, eps, kind,
            gamma, work.buf.data_ptr(), work.buf.numel(), K_fit.data_ptr() if K_fit is not None else None,
            K_pred.data_ptr() if K_pred is not None else None, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))

    assert call() == 0
    torch.cuda.synchronize()
    for kw in (dict(E_=0), dict(E_=257), dict(kind=2), dict(kind=-1), dict(gamma=-1.0), dict(gamma=float("inf")),
               dict(gamma=float("nan")), dict(eps=0), dict(eps=-3), dict(K_fit=None), dict(K_pred=None)):
        assert call(**kw) != 0, kw
    assert call(kind=0, K_pred=None) == 0
    torch.cuda.synchronize()
    with pytest.raises(ValueError):
        engine.feature_kernels_f64_wide(op, op, 0, 4, 4, "poly")
    with pytest.raises(ValueError):
        engine.feature_kernels_f64_wide(op, op, 0, 4, 4, "rbf", -1.0)
    with pytest.raises(ValueError):
        engine.feature_kernels_f64_wide(op, op, 0, 4, 0, "linear")


RUN_CASES = [
    # E, eps, folds, V, two masks, classes
    (65, 13, 5, 120, False, 3),
    (140, 20, 7, 100, True, 2),
    (256, 16, 16, 64, False, 3),
    (256, 16, 16, 64, True, 2),
]
CLFS = [
    svm.SVC(kernel="linear", shrinking=False),
    svm.SVC(kernel="linear", C=0.05),
    svm.SVC(kernel="rbf", gamma="auto", shrinking=False),
    svm.SVC(kernel="rbf", gamma=2e-3, C=10.0),
]


@pytest.mark.parametrize("E,eps,folds,V,two,ncls", RUN_CASES)
def test_run_matches_host_path_wide(dev, E, eps, folds, V, two, ncls):
    raw, _ = synthetic.make_epochs(V, 48, E, seed=E * 13 + V)
    raw2 = synthetic.make_epochs(V - 17, 48, E, seed=E * 13 + V + 1)[0] if two else None
    labels = [e % ncls for e in range(E)]
    for clf in CLFS:
        gpu = VoxelSelector(labels, eps, folds, raw, raw2, device=dev, gpu_cv=True)
        assert gpu._feature_kind(clf, max_epochs=engine.SVM_WIDE_MAX_EPOCHS) is not None
        host = VoxelSelector(labels, eps, folds, raw, raw2, device=dev, gpu_cv=False, process_num=0)
        got, want = gpu.run(clf), host.run(clf)
        assert got == want, (clf, [(g, w) for g, w in zip(got, want) if g != w][:5])


# the inputs of tests/golden/make_golden_feature_wide.py, regenerated from their seeds, and the classifiers
FIXTURES = {
    "w1": (lambda: (synthetic.make_dyadic_epochs(48, 20, 140, seed=4242, informative=8)[0], None),
           svm.SVC(kernel="linear", shrinking=False, C=1)),
    "w2": (lambda: tuple(synthetic.make_two_masks(24, 40, 16, 256, seed=5151)[:2]),
           svm.SVC(kernel="rbf", gamma="auto", C=10)),
}


@pytest.mark.parametrize("gpu_cv", [True, False])
@pytest.mark.parametrize("name", ["w1", "w2"])
def test_run_matches_reference_fixture(dev, golden, name, gpu_cv):
    """The unmodified reference's voxel list and accuracies: w1 E = 140, eps 20, 7 folds, linear, one mask; w2 E = 256,
    eps 16, 16 folds, three classes, two masks, rbf gamma='auto' C=10.  gpu_cv=False is the host path on the same GPU
    correlations."""
    g = golden("vs_feat_" + name)
    make, clf = FIXTURES[name]
    raw, raw2 = make()
    assert _probe_matches(raw, g["probe"])
    if raw2 is not None:
        assert _probe_matches(raw2, g["probe2"])
    labels = [int(x) for x in g["labels"]]
    vs = VoxelSelector(labels, int(g["eps"]), int(g["num_folds"]), raw, raw2, device=dev, gpu_cv=gpu_cv,
                       process_num=0)
    assert (vs._feature_kind(clf, max_epochs=engine.SVM_WIDE_MAX_EPOCHS) is not None) == gpu_cv
    got = vs.run(clf)
    want = [(int(v), float(a)) for v, a in zip(g["vids"], g["accs"])]
    assert [v for v, _ in got] == [v for v, _ in want]
    assert [a for _, a in got] == [a for _, a in want]
