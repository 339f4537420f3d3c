"""VoxelSelector's GPU path for SVC(kernel='linear' | 'rbf') on the normalised correlation vectors.

* engine.feature_kernels_f64 (k_norm_gram_f64) element by element against exact sums of the fp64 products of the z that
  ``within_subject_norm_`` gives on the same raw correlations (an error-free cascaded sum: TwoSum on every addition,
  TwoProduct for the squared differences).  Bound: ``|G - G_exact| <= gamma_n sum|z_a z_b| + u |G_exact|``, the same
  for D.  At small V2 that bound is below one fp32 ulp of a single z, so these cases also pin the kernel's z to the host
  normaliser's bit for bit.
* Two runs are bit-identical.
* ``VoxelSelector.run(clf)`` with ``gpu_cv=True`` returns the list ``gpu_cv=False`` returns (scikit-learn on the host, on
  the same GPU correlations).
"""
import numpy as np
import pytest
import torch
from sklearn import svm

from brainiak_b200 import _lib
from brainiak_b200.fcma import engine, synthetic
from brainiak_b200.fcma.voxelselector import VoxelSelector

pytestmark = pytest.mark.gpu
U = 2.0 ** -53


@pytest.fixture(scope="module")
def dev():
    assert _lib.device_count() > 0, "no sm_90 device"
    return torch.device("cuda:0")


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _split(a):
    c = 134217729.0 * a          # 2^27 + 1 (Veltkamp)
    hi = c - (c - a)
    return hi, a - hi


def _two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _exact_sums(z, rbf):
    """z: float32 [n, E, V2] -> fp64 (G, sum|z_a z_b|, D) [n, E, E], each sum correctly rounded up to a
    relative 2u (the products of fp32 values are exact in fp64; fl(z_a - z_b) is what the kernel squares as well)."""
    z = z.astype(np.float64)
    n, E, V2 = z.shape
    sg, cg, ag = (np.zeros((n, E, E)) for _ in range(3))
    sd, cd = np.zeros((n, E, E)), np.zeros((n, E, E))
    for j in range(V2):
        col = z[:, :, j]
        p = col[:, :, None] * col[:, None, :]
        sg, e = _two_sum(sg, p)
        cg += e
        ag += np.abs(p)
        if rbf:
            df = col[:, :, None] - col[:, None, :]
            hi, lo = _two_prod(df, df)
            sd, e = _two_sum(sd, hi)
            cd += e + lo
    return sg + cg, ag, sd + cd


def _gamma_n(n):
    return n * U / (1 - n * U)


def _operands(V, V2, T, E, dev, seed, ragged=False):
    raw, _ = synthetic.make_epochs(V, T, E, seed=seed)
    raw2 = synthetic.make_epochs(V2, T, E, seed=seed + 1)[0] if V2 else None
    if ragged:
        raw = [m[:T - 7 * (e % 4)] for e, m in enumerate(raw)]
        raw2 = [m[:T - 7 * (e % 4)] for e, m in enumerate(raw2)] if raw2 is not None else None
    ep, T_e = engine.stack_epochs(raw, dev)
    op = engine.pack_epochs(ep, T_e, "tf32x3")
    op2 = op
    if raw2 is not None:
        ep2, _ = engine.stack_epochs(raw2, dev)
        op2 = engine.pack_epochs(ep2, T_e, "tf32x3")
    return op, op2


# name, V (rows), V2 (two masks) or None (one mask: V2 = V), T, E, eps, start, nb, ragged
CASES = [
    ("E1", 300, 33, 40, 1, 2, 0, 5, False),
    ("E2_eps1", 300, 31, 40, 2, 1, 7, 5, False),
    ("E3_eps3", 300, 257, 40, 3, 3, 100, 4, False),
    ("E12_eps5", 300, 255, 40, 12, 5, 3, 4, False),
    ("E12_eps12", 300, 3, 40, 12, 12, 0, 4, True),
    ("E16_eps4_V2_1", 300, 1, 40, 16, 4, 299, 1, False),
    ("E31_eps3", 300, None, 40, 31, 3, 17, 3, False),
    ("E32_eps8", 300, 4129, 40, 32, 8, 11, 3, False),
    ("E33_eps3", 300, 257, 40, 33, 3, 5, 3, True),
    ("E64_eps12", 300, 33, 40, 64, 12, 0, 3, False),
    ("E64_eps16", 300, 4129, 40, 64, 16, 250, 2, False),
]


@pytest.mark.parametrize("layout", ["strided", "tiled"])
@pytest.mark.parametrize("name,V,V2,T,E,eps,start,nb,ragged", CASES, ids=[c[0] for c in CASES])
def test_feature_kernels_element_by_element(dev, name, V, V2, T, E, eps, start, nb, ragged, layout):
    op, op2 = _operands(V, V2, T, E, dev, seed=E * 101 + (V2 or 0), ragged=ragged)
    n2 = op2.V
    # fewer than 256 rows of scratch: strided [nb][E][ld] block; 256: tiled block
    work = engine.Workspace(E, n2, 2 if layout == "strided" else 256, dev)
    r = engine.corr_block(op, op2, start, nb, layout=0).contiguous()
    z = engine.within_subject_norm_(r, eps).cpu().numpy()
    G_ex, A, D_ex = _exact_sums(z, rbf=True)
    bound = _gamma_n(n2 + 16) * A + U * np.abs(G_ex)
    G, G2 = engine.feature_kernels_f64(op, op2, start, nb, eps, "linear", work=work)
    assert G is G2
    G = G.cpu().numpy()
    assert np.all(np.abs(G - G_ex) <= bound), (name, np.max(np.abs(G - G_ex) - bound))
    assert np.array_equal(G, np.swapaxes(G, 1, 2))
    gamma = 0.37 / max(n2, 1)
    Kf, Kp = engine.feature_kernels_f64(op, op2, start, nb, eps, "rbf", gamma, work=work)
    Kf, Kp = Kf.cpu().numpy(), Kp.cpu().numpy()
    # the x_square form is computed from the kernel's own G, through exp: within an ulp or two of numpy's
    d = np.diagonal(G, axis1=1, axis2=2)
    want = np.exp(-gamma * ((d[:, :, None] + d[:, None, :]) - 2.0 * G))
    assert np.all(np.abs(Kf - want) <= 2 * np.spacing(want)), name
    assert np.all(np.diagonal(Kf, axis1=1, axis2=2) == 1.0)
    # the difference form: D within the summation bound, then exp (one more ulp)
    bd = _gamma_n(n2 + 1) * D_ex + U * D_ex
    lo, hi = np.exp(-gamma * (D_ex + bd)), np.exp(-gamma * np.maximum(D_ex - bd, 0))
    assert np.all((Kp >= lo - 2 * np.spacing(lo)) & (Kp <= hi + 2 * np.spacing(hi))), name
    assert np.array_equal(Kp, np.swapaxes(Kp, 1, 2))
    assert np.all(np.diagonal(Kp, axis1=1, axis2=2) == 1.0)


def test_feature_kernels_two_runs_bit_identical(dev):
    op, _ = _operands(1000, None, 60, 32, dev, seed=77)
    work = engine.Workspace(32, 1000, 512, dev)
    a = engine.feature_kernels_f64(op, op, 0, 1000, 8, "rbf", 1e-3, work=work)
    b = engine.feature_kernels_f64(op, op, 0, 1000, 8, "rbf", 1e-3, work=work)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_feature_kernels_rejects_bad_arguments(dev):
    op, _ = _operands(300, None, 40, 8, dev, seed=5)
    with pytest.raises(ValueError):
        engine.feature_kernels_f64(op, op, 0, 4, 4, "poly")
    with pytest.raises(ValueError):
        engine.feature_kernels_f64(op, op, 0, 4, 4, "rbf", -1.0)
    with pytest.raises(ValueError):
        engine.feature_kernels_f64(op, op, 0, 4, 0, "linear")


RUN_CASES = [
    # E, eps, V, two masks, classes
    (12, 3, 300, False, 2),
    (12, 3, 257, True, 3),
    (32, 8, 300, False, 3),
    (32, 8, 260, True, 2),
]
CLFS = [
    svm.SVC(kernel="linear", shrinking=False),
    svm.SVC(kernel="linear", C=0.05),
    svm.SVC(kernel="rbf", gamma="auto", shrinking=False),
    svm.SVC(kernel="rbf", gamma=2e-3, C=10.0),
]


@pytest.mark.parametrize("E,eps,V,two,ncls", RUN_CASES)
def test_run_matches_host_path(dev, E, eps, V, two, ncls):
    raw, _ = synthetic.make_epochs(V, 48, E, seed=E * 13 + V)
    raw2 = synthetic.make_epochs(V - 40, 48, E, seed=E * 13 + V + 1)[0] if two else None
    labels = [e % ncls for e in range(E)]
    for clf in CLFS:
        gpu = VoxelSelector(labels, eps, 3 if E == 12 else 4, raw, raw2, device=dev, gpu_cv=True)
        assert gpu._feature_kind(clf) is not None
        host = VoxelSelector(labels, eps, 3 if E == 12 else 4, raw, raw2, device=dev, gpu_cv=False, process_num=0)
        got, want = gpu.run(clf), host.run(clf)
        assert got == want, (clf, [(g, w) for g, w in zip(got, want) if g != w][:5])
