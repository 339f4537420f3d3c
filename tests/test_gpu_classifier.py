"""Element-wise tests of the Classifier's routes (brainiak_b200/fcma/classifier.py): its kernel builds, its test-vs-train
similarities and its feature path, at multi-tile shapes, through ``fit`` / ``predict`` / ``decision_function``.  Every
case records the C entry points it reached (``Spy``) and asserts its route, so a change of the dispatch conditions in
``engine.classifier_kernel`` cannot move a case to another route unnoticed.

| route | code path |
|---|---|
| R1 small mask | corr_block layout 1 -> within_subject_norm_ over [1, E, V1 V2] -> kernel_matrices(sum_over_rows) (tf32 SYRK, E > 64 k_syrk_simt) |
| R2 portion, one mask >= 512, E <= 64, power-of-two eps >= 2 | fcma_classifier_kernel_sym |
| R3 portion, fused, two masks or one mask < 512 | fcma_classifier_kernel -> run_pipeline(sum_over_rows=1) |
| R4 portion, generic | E > 64 or non-power-of-two eps, eps in {0, 1} (no normalisation) |
| P1 predict(X) after a small-mask fit | corr + normalise over n_test (n_test = 1: none) -> gemm_nt -> x float32(10**(2 - num_digits_)) |
| P2 predict(X) after a portion fit | _streamed_similarity |
| P3 fit-time test samples | test_data_ = K[n_train:, :n_train] |
| F1 LogisticRegression | features = corr + normalise (train: eps, test: n_test) |

Coverage (route x edge -> test):

| route | edge | test |
|---|---|---|
| R1 + P1 | masks 40 x 257 passed smaller-first, E = 33, eps 5, n_test 2, fp16x3, tf32 SYRK | test_small_mask[s1] |
| R1 + P1 | one mask V1 = 255, E = 65 (k_syrk_simt), eps 12, n_test 1 | test_small_mask[s2] |
| R1 + P1 | ragged T_e, one voxel x 2^-4 (tf32x3), E = 17, eps 8, n_test 50 > 64 - 17 | test_small_mask[s3] |
| R1 + P1 | precision 'bf16' (r to R_TOL), eps 2 | test_small_mask[s4] |
| R1 + P1 | one mask of 7 voxels, eps 0: num_digits_ <= 2 | test_small_mask[s5] |
| R1 + P1 | masks 300 x 700 smaller-first, E = 30 + 10, eps 5: the reference's outputs | test_reference_w2 |
| R2 + P3 | V1 = 512, E = 64, eps 16, num_processed_voxels 1; R2 == R3 on the same data | test_portion[p1] |
| R2 + P3 + P2 | V1 = 640, E = 32, eps 8, num_processed_voxels 200; the reference's outputs; predict(X[24:]) == the reference's fit-time test_data_ | test_reference_w1 |
| R3 + P3 + P2 | masks 511 x 300, E = 64, eps 4; streamed 3 rows a portion | test_portion[p2] |
| R3 + P3 | masks 257 x 100, one voxel x 2^-4 (tf32x3), E = 16, eps 4 | test_portion[p3] |
| R4 + P3 + P2 | E = 300 (E^2 % 4096 != 0), eps 8, n_train 290 (n_train % eps = 2); streamed 1 row a portion, Es = 301 | test_portion[p4] |
| R4 + P3 + P2 | masks 257 x 40, ragged T_e, E = 33, eps 5, n_train 23 (% eps = 3); streamed 3 rows a portion, ragged last | test_portion[p5] |
| R4 + P3 + P2 | one mask 300, E = 140, eps 0, n_test 1; default portions 299 + 1 | test_portion[p6] |
| R4 + P3 | E = 17, eps 1 | test_portion[p7] |
| R4 + P3 + P2 | E = 65, eps = E, n_train 50 (the whole fit is one subject) | test_portion[p8] |
| R4 + P3 | masks 120 x 90, E = 100, eps 12 (4 trailing): the reference's outputs | test_reference_w3 |
| F1 | LogisticRegression, masks 40 x 30, E = 16 + 8, eps 4: the reference's outputs | test_reference_w4 |
| errors | RuntimeError, ValueError, AssertionError as the reference; 800 samples (fit, and Es of a streamed prediction) | test_errors_and_sample_limit |

Reference: r is the fp64 contraction of the float32 samples (``orc.corr_block(f64=True)``), with one mask the self
entries against the sequential fp32 chain the GEMM's fix-up stores; z is ``wsc_ref`` (test_generic_pipeline_cpu.py) of
the GPU's own r, ill-conditioned subjects exempt by its rule, trailing epochs of a partial subject bit-identical to r.

Bounds:
* r: ``tol_r`` of test_gpu_corr_gemm.py, Fisher-z (fused routes) to its bound there; bf16 to ``R_TOL``.
* K of R1, R4 and P2: the z the SYRK read is recomputed (or captured) bit for bit, ``check_summed`` of
  test_gpu_generic_pipeline.py element by element.
* K of R2 and R3: fp64 sum z z^T of the fp64-normalised r within the parity table's kernel-matrix bound
  ``(5e-4 sqrt(256 / n2) + 2e-6) max|K|``, n2 = V1 V2; R2 against R3 on the same operands within the same bound.
  ``num_digits_`` equals the fp64 digit count unless K00 lies within the bound of a power of ten.
* P1: ``test_data_`` bit-identical to the sequential fp32 FMA chain of the GPU's test features against
  ``training_data_`` times the shrink factor; P3: bit-identical to the shrunk kernel's block.
* P2: the similarity against fp64 z_test z_train^T, z_train rows [0, n_train) of the fit's normalisation of the fit
  samples: ``sum_j (Dt |zf| + |zt| Df + Dt Df) + c sum_j |zt zf|``, D the normaliser bound of wsc_ref for an r off by
  tol_r (ill-conditioned elements: the GPU's own deviation), c = 2^-10 + 50u for the tf32 SYRK (two operands rounded to
  tf32), n2 u for k_syrk_simt, plus u per portion (atomics) and u |sim| for the shrink.
* the reference's fixtures (tests/golden/make_golden_clf_wide.py): ``predict`` and ``num_digits_`` exactly,
  ``decision_function`` and ``test_data_`` within 2e-3, the shrunk kernel within the kernel-matrix bound.

Measured on one H100 80GB HBM3 (700 W power limit), largest fraction of each bound used: r 0.24 (fp16x3), 0.21
(tf32x3), 0.32 (bf16); normaliser 0.20; R2 / R3 kernels against fp64 0.25, R2 against R3 0.064; the streamed similarity
against fp64 0.32; the reference's shrunk kernels 0.24.  Without the fix of ``_streamed_similarity`` the cases with
n_train % eps != 0 (p4, p5, p8) fail there by 0.57 to 1.4 in the columns of the cut subject (bounds 0.001 to 0.13).  The
file runs in about 20 s there.
"""
import functools
import inspect
import math

import numpy as np
import pytest
import torch
from sklearn import svm
from sklearn.linear_model import LogisticRegression

from brainiak_b200 import _lib
from brainiak_b200.fcma import classifier as clf_mod
from brainiak_b200.fcma import engine, synthetic
from brainiak_b200.fcma.classifier import Classifier
from oracle import fcma_oracle as orc
from test_generic_pipeline_cpu import digits, near_power_of_ten, wsc_ref
from test_gpu_corr_gemm import FAITHFUL, R_TOL, check_values
from test_gpu_generic_pipeline import check_summed, per_row_z

pytestmark = pytest.mark.gpu

STATS = {}
SCALE = 2.0 ** -4             # on one voxel: moves the 'fp32' precision from fp16x3 to tf32x3 (a voxel norm below 1/8)


@pytest.fixture(scope="module")
def dev():
    assert _lib.device_count() > 0, "no sm_90 device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    for k, v in sorted(STATS.items()):
        print("classifier %s: %.3g of the bound" % (k, v))


def record(key, frac):
    STATS[key] = max(STATS.get(key, 0.0), float(frac))


def svc():
    return svm.SVC(kernel="precomputed", shrinking=False, C=1)


# ------------------------------------------------------------------------------- route recording
class Spy:
    """Within the block, records every call of the engine stages the Classifier uses (arguments, the input of an
    in-place normalisation, clones of the results) and the names of the C entry points reached."""
    ENGINE = ("corr_block", "within_subject_norm_", "kernel_matrices", "classifier_kernel", "gemm_nt")
    LIB = ("fcma_classifier_kernel_sym", "fcma_classifier_kernel", "fcma_kernel_matrices", "fcma_within_subject_norm",
           "fcma_gemm_nt", "fcma_corr_block")

    def __init__(self):
        self.calls, self.entries = [], []

    def __enter__(self):
        self._saved = []
        for name in self.ENGINE:
            fn = getattr(engine, name)
            self._saved.append((engine, name, fn))
            setattr(engine, name, self._engine(name, fn))
        lib = _lib.load()
        for name in self.LIB:
            fn = getattr(lib, name)
            self._saved.append((lib, name, fn))
            setattr(lib, name, self._entry(name, fn))
        return self

    def __exit__(self, *exc):
        for owner, name, fn in reversed(self._saved):
            setattr(owner, name, fn)

    def _engine(self, name, fn):
        sig = inspect.signature(fn)

        @functools.wraps(fn)
        def call(*args, **kw):
            b = sig.bind(*args, **kw)
            b.apply_defaults()
            rec = dict(b.arguments)
            if name == "within_subject_norm_":
                rec["before"] = rec["corr"].clone()
            if name == "kernel_matrices":
                rec["zin"] = rec["z"].clone()
            res = fn(*args, **kw)
            rec["res"] = res.clone()
            self.calls.append((name, rec))
            return res
        return call

    def _entry(self, name, fn):
        def call(*args):
            self.entries.append(name)
            return fn(*args)
        return call

    def of(self, name):
        return [rec for n, rec in self.calls if n == name]


def route(spy, expect):
    """The C entry points of one Classifier operation, checked against route ``expect``."""
    got = set(spy.entries)
    if expect == "R2":
        assert "fcma_classifier_kernel_sym" in got and "fcma_classifier_kernel" not in got, got
    elif expect in ("R3", "R4"):
        assert "fcma_classifier_kernel" in got and "fcma_classifier_kernel_sym" not in got, got
        k = spy.of("classifier_kernel")[0]
        fused = k["eps"] > 1 and engine.fused_supported(k["rows"].E, k["eps"])
        assert fused == (expect == "R3"), (expect, k["rows"].E, k["eps"])
    elif expect in ("R1", "P2"):
        assert "fcma_kernel_matrices" in got and not got & {"fcma_classifier_kernel", "fcma_classifier_kernel_sym",
                                                             "fcma_gemm_nt"}, got
    elif expect == "P1":
        assert "fcma_gemm_nt" in got and "fcma_kernel_matrices" not in got, got
    elif expect == "F1":
        assert not got & {"fcma_kernel_matrices", "fcma_classifier_kernel", "fcma_classifier_kernel_sym",
                          "fcma_gemm_nt"}, got


# ------------------------------------------------------------------------------- inputs
def make_mask(V, E, T, seed, lens=None, scale=1.0, dyadic=False):
    """E float32 epochs [T_e, V]: normalised Gaussian (synthetic.make_epochs' recipe, ``lens`` = per-epoch lengths) or
    dyadic (exact r in any order), voxel 0 times ``scale``."""
    if dyadic:
        raw = synthetic.make_dyadic_epochs(V, T, E, seed=seed)[0]
    else:
        lens = lens or [T] * E
        raw = [synthetic.normalize_epoch(synthetic.raw_epoch(e, lens[e], V, seed=seed)) for e in range(E)]
    if scale != 1.0:
        for m in raw:
            m[:, 0] *= np.float32(scale)
    return raw


def make_samples(c):
    """(X, labels) of case ``c``: pairs in the order given to the Classifier (smaller mask first where c['swap'])."""
    E, T = c["E"], c.get("T", 20)
    lens = None
    if c.get("ragged"):
        rng = np.random.RandomState(c["seed"])
        lens = [int(t) for t in rng.randint(T // 2, T + 1, size=E)]
        lens[0] = T
    a = make_mask(c["V1"], E, T, c["seed"], lens, c.get("scale", 1.0), c.get("dyadic", False))
    if c.get("V2") is None:
        X = list(zip(a, a))
    else:
        b = make_mask(c["V2"], E, T, c["seed"] + 7919, lens, 1.0, c.get("dyadic", False))
        X = list(zip(b, a)) if c.get("swap") else list(zip(a, b))
    return X, [e % 2 for e in range(E)]


def masks(X):
    """(rows, cols or None) in the Classifier's order: the larger mask first, None for one mask."""
    A, B = [x for x, _ in X], [y for _, y in X]
    if all(x is y for x, y in X):
        return A, None
    return (B, A) if A[0].shape[1] < B[0].shape[1] else (A, B)


def shrink_factor(nd):
    return 10 ** (2 - nd) if nd > 2 else None


def shrunk(K, nd):
    """The Classifier's shrink of a float32 [E, E] numpy kernel (classifier.py:343-347)."""
    K = np.array(K, dtype=np.float32)
    if nd > 2:
        K *= 10 ** (2 - nd)
    return K


def kbound(K64, n2):
    """The parity table's kernel-matrix bound (DESIGN.md §5)."""
    return (5e-4 * math.sqrt(256.0 / n2) + 2e-6) * float(K64.abs().max())


# ------------------------------------------------------------------------------- stage checks
def r_tol(rows, r64, chain):
    return max(1e-6, 2.0 * float(np.max(np.abs(chain - r64)))) if rows.precision in FAITHFUL else R_TOL[rows.precision]


def check_r(rows, cols, A, B, what, fisher=0):
    """r (and Fisher-z of the first ``fisher`` epochs) of the whole block [V1, E, V2] of the operands against the fp64
    contraction of the samples; one mask: self entries against the sequential fp32 chain."""
    V1 = rows.V
    got = engine.corr_block(rows, cols, 0, V1, fisher_epochs=fisher).cpu().numpy()
    r64 = orc.corr_block(A, B, 0, V1, f64=True)
    chain = orc.corr_block(A, B, 0, V1, f64=False)
    E = r64.shape[1]
    tol = r_tol(rows, r64, chain)
    self_j = np.arange(V1) if B is None else None
    chain_self = chain[np.arange(V1), :, np.arange(V1)] if B is None else None
    st = check_values(got, r64, [e < fisher for e in range(E)], tol, self_j, chain_self, what=what)
    record("r %s" % rows.precision, st["raw"] / tol)
    return r64, chain


def check_z(before, after, eps, what):
    """A within_subject_norm_ result ([n0, E, n2] CUDA) against wsc_ref of its own input."""
    z64, delta, ill = wsc_ref(before.double(), eps)
    S = (before.shape[1] // eps) * eps
    assert torch.equal(after[:, S:], before[:, S:]), what + ": trailing epochs differ from r"
    err = (after.double() - z64).abs()
    bad = (err > delta) & ~ill
    assert not bad.any(), "%s: %d normalised values outside the bound, e.g. %s" % (what, int(bad.sum()),
                                                                                   bad.nonzero()[:3].tolist())
    assert float(ill.double().mean()) <= 0.15, what
    ok = ~ill & (delta > 0)
    if ok.any():
        record("normaliser", (err[ok] / delta[ok]).max())


def z64_of(r64, eps, dev, self_chain=None):
    """fp64-normalised r ([V1, E, V2] numpy -> CUDA fp64), self entries from the fp32 chain for one mask."""
    r = torch.from_numpy(r64).to(dev)
    if self_chain is not None:
        i = torch.arange(r.shape[0], device=dev)
        r[i, :, i] = torch.from_numpy(self_chain.astype(np.float64)).to(dev)
    return wsc_ref(r, eps)[0] if eps > 1 else r


def check_fp64_kernel(K, z64, nd, what):
    """An unshrunk [E, E] kernel against sum_i z64_i z64_i^T; the digit count."""
    K64 = torch.einsum("iaj,ibj->ab", z64, z64)
    n2 = z64.shape[0] * z64.shape[2]
    lim = kbound(K64, n2)
    err = float((K.double().to(K64.device) - K64).abs().max())
    assert torch.isfinite(K).all() and err <= lim, "%s: max |K - K64| %.3g > %.3g" % (what, err, lim)
    record("kernel fp64", err / lim)
    k00 = float(K64[0, 0])
    if not near_power_of_ten(k00, lim):
        assert nd == digits(k00), "%s: num_digits_ %d, fp64 %d" % (what, nd, digits(k00))
    return K64, lim


# ------------------------------------------------------------------------------- R1 + P1: small mask
SMALL = {
    "s1": dict(V1=257, V2=40, swap=True, E=35, n_fit=33, eps=5, T=24, seed=101, prec="fp16x3"),
    "s2": dict(V1=255, E=66, n_fit=65, eps=12, seed=102, prec="fp16x3"),
    "s3": dict(V1=30, V2=20, E=67, n_fit=17, eps=8, T=24, ragged=True, scale=SCALE, seed=103, prec="tf32x3"),
    "s4": dict(V1=64, V2=48, E=18, n_fit=16, eps=2, seed=104, precision="bf16", prec="bf16"),
    "s5": dict(V1=7, E=18, n_fit=16, eps=0, seed=105, prec="fp16x3"),
}


def fit_small(c, X, labels, dev):
    """fit + predict on the rest, with every stage of R1 and P1 checked; returns (classifier, fit spy, predict spy)."""
    n, eps = c["n_fit"], c["eps"]
    clf = Classifier(svc(), epochs_per_subj=eps, precision=c.get("precision", "fp32"), device=dev)
    with Spy() as sf:
        clf.fit(X[:n], labels[:n])
    route(sf, "R1")
    A, B = masks(X[:n])
    cb = sf.of("corr_block")[0]
    assert cb["rows"].precision == c["prec"], cb["rows"].precision
    r64, chain = check_r(cb["rows"], cb["cols"], A, B, "fit r")
    km = sf.of("kernel_matrices")
    assert len(km) == 1 and km[0]["sum_over_rows"]
    z = km[0]["zin"]
    norm = sf.of("within_subject_norm_")
    if eps > 1:
        assert len(norm) == 1 and norm[0]["eps"] == eps
        check_z(norm[0]["before"], norm[0]["res"], eps, "fit z")
        assert torch.equal(norm[0]["res"], z)
    else:
        assert not norm
        assert torch.equal(cb["res"].reshape(z.shape), z)
    K = km[0]["res"]
    E = z.shape[1]
    check_summed(K, z, E, "R1 %s" % c)
    assert clf.num_digits_ == digits(float(K[0, 0]))
    assert np.array_equal(clf.training_data_, z[0].cpu().numpy())
    # P1
    test = X[n:]
    with Spy() as sp:
        conf = clf.decision_function(test)
    route(sp, "P1")
    nt = len(test)
    At, Bt = masks(test)
    ct = sp.of("corr_block")[0]
    check_r(ct["rows"], ct["cols"], At, Bt, "test r")
    norm = sp.of("within_subject_norm_")
    if nt > 1:
        assert len(norm) == 1 and norm[0]["eps"] == nt
        check_z(norm[0]["before"], norm[0]["res"], nt, "test z")
    else:
        assert not norm
    g = sp.of("gemm_nt")[0]
    a, b = g["a"].cpu().numpy(), g["b"].cpu().numpy()
    assert np.array_equal(b, clf.training_data_)
    if nt > 1:
        assert np.array_equal(a, norm[0]["res"][0].cpu().numpy())
    want = orc.corr_block([np.ascontiguousarray(a.T)], [np.ascontiguousarray(b.T)], 0, nt, f64=False)[:, 0, :]
    p = shrink_factor(clf.num_digits_)
    if p is not None:
        want *= p
    assert np.array_equal(clf.test_data_, want), "P1: test_data_ differs from the fp32 chain"
    assert np.array_equal(conf, clf.clf.decision_function(want))
    return clf, sf, sp


@pytest.mark.parametrize("name", sorted(SMALL))
def test_small_mask(dev, name):
    """R1 + P1: the small-mask fit (features kept as training_data_) and predict on new samples, stage by stage."""
    c = SMALL[name]
    X, labels = make_samples(c)
    clf, _, _ = fit_small(c, X, labels, dev)
    if name == "s5":
        assert clf.num_digits_ <= 2
    else:
        assert clf.num_digits_ > 2
    assert np.array_equal(clf.predict(X[c["n_fit"]:]), clf.clf.predict(clf.test_data_))


# ------------------------------------------------------------------------------- R2 / R3 / R4 + P3 + P2: portions
PORTION = {
    "p1": dict(V1=512, E=64, eps=16, npv=1, n_train=60, T=24, dyadic=True, seed=201, route="R2"),
    "p2": dict(V1=511, V2=300, E=67, n_fit=64, eps=4, npv=100, n_train=40, seed=202, route="R3", rows=3),
    "p3": dict(V1=257, V2=100, E=16, eps=4, npv=256, n_train=10, scale=SCALE, seed=203, route="R3", prec="tf32x3"),
    "p4": dict(V1=60, V2=33, E=305, n_fit=300, eps=8, npv=20, n_train=290, seed=204, route="R4", rows=1),
    "p5": dict(V1=257, V2=40, E=35, n_fit=33, eps=5, npv=64, n_train=23, ragged=True, T=24, seed=205, route="R4",
               rows=3),
    "p6": dict(V1=300, E=141, n_fit=140, eps=0, npv=299, n_train=130, dyadic=True, seed=206, route="R4", rows=0),
    "p7": dict(V1=33, V2=20, E=17, eps=1, npv=5, n_train=16, seed=207, route="R4"),
    "p8": dict(V1=70, V2=65, E=67, n_fit=65, eps=65, npv=10, n_train=50, seed=208, route="R4", rows=0),
}


def fit_portion(c, X, labels, dev):
    """Portion-mode fit with the route's checks and P3; returns (classifier, the unshrunk kernel, spy record)."""
    n_fit, eps, n_train = len(X), c["eps"], c["n_train"]
    clf = Classifier(svc(), num_processed_voxels=c["npv"], epochs_per_subj=eps, device=dev)
    with Spy() as sf:
        clf.fit(X, labels, num_training_samples=n_train)
    route(sf, c["route"])
    k = sf.of("classifier_kernel")
    assert len(k) == 1
    k = k[0]
    rows, cols = k["rows"], k["cols"]
    assert rows.precision == c.get("prec", rows.precision)
    if not c.get("dyadic") and "prec" not in c:
        assert rows.precision == "fp16x3"
    K = k["res"]
    A, B = masks(X)
    E = n_fit
    fused = c["route"] in ("R2", "R3")
    S = (E // eps) * eps if eps > 1 else 0
    r64, chain = check_r(rows, cols, A, B, "fit r", fisher=S if fused else 0)
    what = "%s %s" % (c["route"], c)
    if fused:
        self_chain = chain[np.arange(rows.V), :, np.arange(rows.V)] if B is None else None
        z64 = z64_of(r64, eps, dev, self_chain)
        K64, lim = check_fp64_kernel(K, z64, clf.num_digits_, what)
        if c["route"] == "R2":
            K3 = engine.classifier_kernel(rows, cols, 0, rows.V, eps, symmetric=False)
            err = float((K3.double() - K.double()).abs().max())
            assert err <= lim, "R2 vs R3: %.3g > %.3g" % (err, lim)
            record("R2 vs R3", err / lim)
    else:
        z = per_row_z(rows, cols, 0, rows.V, eps)
        if eps > 1:
            check_z(engine.corr_block(rows, cols, 0, rows.V), z, eps, "fit z")
        check_summed(K, z, E, what)
    assert clf.num_digits_ == digits(float(K[0, 0]))
    # P3
    Ks = shrunk(K.cpu().numpy(), clf.num_digits_)
    assert np.array_equal(clf.test_data_, Ks[n_train:, :n_train])
    assert clf.training_data_ is None
    return clf, K


def n2_of(X, V1):
    """V2 of the samples X (the smaller mask; V1 for one mask)."""
    B = masks(X)[1]
    return V1 if B is None else B[0].shape[1]


def z64_bound(X, V1, eps, zg, dev):
    """(z64, D): the fp64-normalised r of the samples X ([V1, E, V2] CUDA), and the bound of |z_gpu - z64| (wsc_ref's
    normaliser bound for an r off by tol_r; where wsc_ref has none, the GPU's own deviation ``|zg - z64|``)."""
    A, B = masks(X)
    r64 = orc.corr_block(A, B, 0, V1, f64=True)
    tol = max(1e-6, 2.0 * float(np.max(np.abs(orc.corr_block(A, B, 0, V1, f64=False) - r64))))
    r = torch.from_numpy(r64).to(dev)
    if eps > 1:
        z, D, ill = wsc_ref(r, eps, torch.full_like(r, tol))
    else:
        z, D, ill = r, torch.full_like(r, tol), torch.zeros(r.shape, dtype=torch.bool, device=dev)
    n = zg.shape[1]
    z, D, ill = z[:, :n], D[:, :n], ill[:, :n]
    assert float(ill.double().mean()) <= 0.15
    return z, torch.where(ill, (zg - z).abs(), D)


def check_streamed(c, clf, X_fit, X_new, dev):
    """P2: predict(X_new) after the portion fit, stage by stage and against the fp64 similarity."""
    eps, n_train = c["eps"], c["n_train"]
    nt = len(X_new)
    Es = len(clf._train_raw_[0]) + nt
    if c.get("rows"):
        V2 = n2_of(X_new, c["V1"])
        clf._streamed_similarity = functools.partial(Classifier._streamed_similarity, clf,
                                                     max_bytes=c["rows"] * Es * V2 * 4)
    with Spy() as sp:
        conf = clf.decision_function(X_new)
    route(sp, "P2")
    km = sp.of("kernel_matrices")
    V1 = c["V1"]
    rows = c.get("rows") or min(c["npv"], V1)
    assert len(km) == -(-V1 // rows), (len(km), rows)
    zs = [r["zin"] for r in km]
    span = Es - nt                 # the training samples the similarity was formed with
    n2 = max(z.shape[2] for z in zs)
    zpad = torch.zeros((len(zs), Es, n2), dtype=torch.float32, device=dev)
    for i, z in enumerate(zs):
        zpad[i, :, :z.shape[2]] = z[0]
    K = km[-1]["res"]
    check_summed(K, zpad, Es, "P2 %s" % c)
    for rec in sp.of("within_subject_norm_"):
        check_z(rec["before"], rec["res"], rec["eps"], "P2 z")
    p = shrink_factor(clf.num_digits_)
    want = K.cpu().numpy()[span:, :n_train]
    if p is not None:
        want *= p
    assert np.array_equal(clf.test_data_, want)
    assert np.array_equal(conf, clf.clf.decision_function(want))
    # fp64: the training rows of the fit's normalisation of all fit samples and the test rows, against the GPU's z
    # (the portions' z side by side) within the normaliser bound; ill-conditioned elements: their own deviation
    V2 = n2_of(X_new, V1)
    zg = torch.cat([z[0].view(Es, -1, V2) for z in zs], dim=1).transpose(0, 1).double()        # [V1, Es, V2]
    zf, Df = z64_bound(X_fit, V1, eps, zg[:, :span], dev)
    zt, Dt = z64_bound(X_new, V1, nt, zg[:, span:], dev)
    zf, Df = zf[:, :n_train], Df[:, :n_train]
    sim = torch.einsum("iaj,ibj->ab", zt, zf)
    at, af = zt.abs(), zf.abs()
    c_acc = (2.0 ** -10 + 50 * 2.0 ** -24) if Es <= 64 else zs[0].shape[2] * 2.0 ** -24
    lim = (torch.einsum("iaj,ibj->ab", Dt, af) + torch.einsum("iaj,ibj->ab", at, Df) + torch.einsum("iaj,ibj->ab", Dt, Df)
           + (c_acc + len(km) * 2.0 ** -24) * torch.einsum("iaj,ibj->ab", at, af))
    got = torch.from_numpy(clf.test_data_).double().to(dev)
    if p is not None:
        sim, lim = sim * p, lim * p
    lim = lim + 2.0 ** -24 * sim.abs()
    err = (got - sim).abs()
    bad = err > lim
    assert not bad.any(), "P2: %d similarities off the fp64 value, columns %s (worst %.3g over a bound of %.3g)" % (
        int(bad.sum()), sorted(set(bad.nonzero()[:, 1].tolist()))[:10], float(err.max()), float(lim.min()))
    record("streamed fp64", float((err / lim).max()))


@pytest.mark.parametrize("name", sorted(PORTION))
def test_portion(dev, name):
    """R2 / R3 / R4 + P3: a portion-mode fit, its kernel and its fit-time test block; P2: predict on new samples."""
    c = PORTION[name]
    X, labels = make_samples(c)
    n_fit = c.get("n_fit", c["E"])
    clf, _ = fit_portion(c, X[:n_fit], labels[:n_fit], dev)
    if n_fit < len(X):
        check_streamed(c, clf, X[:n_fit], X[n_fit:], dev)
    eps, n_train = c["eps"], c["n_train"]
    assert len(clf._train_raw_[0]) == (n_train if eps <= 1 else min(n_fit, -(-n_train // eps) * eps))


# ------------------------------------------------------------------------------- the reference's fixtures
def golden_inputs(g, name):
    import make_golden_clf_wide as mk
    X, labels, eps, npv, split = mk.clf_inputs(name)
    assert np.array_equal(mk.input_probe([x for x, _ in X]), g["probe"])
    assert np.array_equal(mk.input_probe([y for _, y in X]), g["probe2"])
    assert list(g["labels"]) == labels and int(g["eps"]) == eps
    return X, labels, eps, npv, split


def check_golden_kernel(Ks, g, n2, what):
    ref = g["kernel"].astype(np.float64)
    lim = (5e-4 * math.sqrt(256.0 / n2) + 2e-6) * np.abs(ref).max()
    err = np.abs(Ks.astype(np.float64) - ref).max()
    assert err <= lim, "%s: shrunk kernel off the reference's by %.3g > %.3g" % (what, err, lim)
    record("reference kernel", err / lim)


@pytest.fixture(scope="module")
def golden_path():
    import os
    import sys
    d = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    if d not in sys.path:
        sys.path.insert(0, d)


def test_reference_w1(dev, golden, golden_path):
    """R2 + P3: one mask of 640 voxels in portions of 200, E = 32, eps 8, 24 training samples; the anchor of P2: the
    fit-time test samples are one subject, so predict on them after the portion fit gives the reference's test_data_."""
    g = golden("clf_w1")
    X, labels, eps, npv, split = golden_inputs(g, "w1")
    c = dict(V1=640, E=32, eps=eps, npv=npv, n_train=split, dyadic=True, route="R2")
    clf, K = fit_portion(c, X, labels, dev)
    assert clf.num_digits_ == int(g["num_digits"])
    check_golden_kernel(shrunk(K.cpu().numpy(), clf.num_digits_), g, 640 * 640, "w1")
    assert np.max(np.abs(clf.test_data_ - g["test_data"])) <= 2e-3
    assert np.max(np.abs(clf.decision_function() - g["decision"])) <= 2e-3
    assert np.array_equal(clf.predict(), g["predict"])
    assert clf.score(None, labels[split:]) == float(g["score"])
    clf.decision_function(X[split:])                   # new data: the streamed similarity of the same samples
    assert np.max(np.abs(clf.test_data_ - g["test_data"])) <= 2e-3
    assert np.array_equal(clf.predict(X[split:]), g["predict"])


def test_reference_w2(dev, golden, golden_path):
    """R1 + P1: masks of 300 and 700 voxels passed smaller-first, fit on 30 samples (eps 5), predict the other 10."""
    g = golden("clf_w2")
    X, labels, eps, npv, split = golden_inputs(g, "w2")
    clf = Classifier(svc(), num_processed_voxels=npv, epochs_per_subj=eps, device=dev)
    with Spy() as sf:
        clf.fit(X[:split], labels[:split])
    route(sf, "R1")
    K = sf.of("kernel_matrices")[0]["res"]
    assert clf.num_digits_ == int(g["num_digits"])
    check_golden_kernel(shrunk(K.cpu().numpy(), clf.num_digits_), g, 700 * 300, "w2")
    test = X[split:]
    assert np.max(np.abs(clf.decision_function(test) - g["decision"])) <= 2e-3
    assert np.max(np.abs(clf.test_data_ - g["test_data"])) <= 2e-3
    assert np.array_equal(clf.predict(test), g["predict"])
    assert clf.score(test, labels[split:]) == float(g["score"])


def test_reference_w3(dev, golden, golden_path):
    """R4 + P3: masks of 120 and 90 voxels, E = 100, eps 12 (4 trailing epochs), 84 training samples."""
    g = golden("clf_w3")
    X, labels, eps, npv, split = golden_inputs(g, "w3")
    c = dict(V1=120, V2=90, E=100, eps=eps, npv=npv, n_train=split, dyadic=True, route="R4")
    clf, K = fit_portion(c, X, labels, dev)
    assert clf.num_digits_ == int(g["num_digits"])
    check_golden_kernel(shrunk(K.cpu().numpy(), clf.num_digits_), g, 120 * 90, "w3")
    assert np.max(np.abs(clf.test_data_ - g["test_data"])) <= 2e-3
    assert np.max(np.abs(clf.decision_function() - g["decision"])) <= 2e-3
    assert np.array_equal(clf.predict(), g["predict"])
    assert clf.score(None, labels[split:]) == float(g["score"])


def test_reference_w4(dev, golden, golden_path):
    """F1: LogisticRegression on the normalised correlations (train: eps 4, test: over the 8 test samples)."""
    g = golden("clf_w4")
    X, labels, eps, npv, split = golden_inputs(g, "w4")
    clf = Classifier(LogisticRegression(), epochs_per_subj=eps, device=dev)
    with Spy() as sf:
        clf.fit(X[:split], labels[:split])
    route(sf, "F1")
    (nf,) = sf.of("within_subject_norm_")
    assert nf["eps"] == eps
    check_z(nf["before"], nf["res"], eps, "F1 train z")
    test = X[split:]
    with Spy() as sp:
        conf = clf.decision_function(test)
    route(sp, "F1")
    (nt,) = sp.of("within_subject_norm_")
    assert nt["eps"] == len(test)
    check_z(nt["before"], nt["res"], len(test), "F1 test z")
    assert np.array_equal(clf.test_data_, nt["res"][0].cpu().numpy())
    assert np.max(np.abs(conf - g["decision"])) <= 2e-3
    assert np.array_equal(clf.predict(test), g["predict"])
    assert clf.score(test, labels[split:]) == float(g["score"])


# ------------------------------------------------------------------------------- errors and the sample limit
def test_errors_and_sample_limit(dev):
    """The reference's exceptions (RuntimeError: portions without num_training_samples; ValueError: num_training_samples
    >= the samples; AssertionError: feature count at predict, TR counts of X1 and X2), and the 799-sample limit of the
    kernel matrix: 800 samples in fit, and 800 in a streamed prediction (training span + test), raise ValueError
    naming it; 799 in a streamed prediction run."""
    X, labels = make_samples(dict(V1=6, V2=4, E=16, eps=4, seed=301))
    with pytest.raises(RuntimeError, match="num_training_samples"):
        Classifier(svc(), num_processed_voxels=2, epochs_per_subj=4, device=dev).fit(X, labels)
    with pytest.raises(ValueError, match="smaller than"):
        Classifier(svc(), num_processed_voxels=2, epochs_per_subj=4, device=dev).fit(X, labels, num_training_samples=16)
    clf = Classifier(svc(), epochs_per_subj=4, device=dev).fit(X[:12], labels[:12])
    Y, _ = make_samples(dict(V1=6, V2=5, E=4, seed=302))
    with pytest.raises(AssertionError, match="number of features"):
        clf.predict(Y)
    bad = [(a, b[:-1]) for a, b in X]
    with pytest.raises(AssertionError, match="TRs"):
        Classifier(svc(), epochs_per_subj=4, device=dev).fit(bad[:12], labels[:12])
    # the sample limit
    assert clf_mod.MAX_KERNEL_SAMPLES == 799
    big, lab = make_samples(dict(V1=3, V2=2, E=800, T=8, seed=303))
    with pytest.raises(ValueError, match="limited to 799"):
        Classifier(svc(), device=dev).fit(big, lab)
    clf = Classifier(svc(), num_processed_voxels=1, epochs_per_subj=0, device=dev)
    clf.fit(big[:70], lab[:70], num_training_samples=60)
    with pytest.raises(ValueError, match="limited to 799"):
        clf.predict(big[60:800])
    with Spy() as sp:
        clf.decision_function(big[61:800])                # Es = 799: the largest k_syrk_simt takes
    route(sp, "P2")
    assert clf.test_data_.shape == (739, 60) and np.isfinite(clf.test_data_).all()
