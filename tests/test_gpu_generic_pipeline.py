"""Element-wise tests of the generic kernel-matrix pipeline: more than 64 epochs, or an epochs_per_subj that is not a
power of two, where neither fused normalise + SYRK kernel applies.  ``run_pipeline`` (fcma_b200.cu) then has the
correlation GEMM write raw r into a strided ``[n][E][ld]`` block (ld = round_up(V2, 32)), normalises it in place
(``k_within_subject_norm``: ``within_subject_column`` per subject and column) and forms the kernels with ``k_syrk_simt``
(E > 64) or the tf32 plain SYRK ``k_norm_syrk<EPS = 0>`` (E <= 64).  ``kernel_matrices`` runs the last stage alone,
``classifier_kernel`` and the Classifier's small-mask path sum it over rows (fp32 atomics).

Reference: fp64 sums of the exact fp32 values each stage reads -- the z the SYRK consumed (read back from the workspace),
the r the normaliser read (``engine.corr_block`` of the same rows, bit-identical to the GEMM's strided block).

Bounds, element by element, u = 2^-24:
* dyadic inputs (z = k/8, |k| <= 8): every product is a multiple of 2^-6 of magnitude <= 1, every partial sum of fewer
  than 2^18 terms (and every sum over nb rows of such, nb n2 < 2^18) is exact in fp32, whatever the summation order,
  pair blocking or atomic order; beta K_old with dyadic K_old (multiples of 2^-6, beta = 0.5 or -1) is exact too.  So K
  must equal the fp64 sum bit for bit: no tolerance at all.
* ``k_syrk_simt`` on Gaussian inputs (``chain_bound``): a sequential fp32 FMA chain over n2 terms errs by at most
  ``n2 u sum_j |z_aj z_bj|``; beta: ``+ 2u (|beta K_old| + |K|)``; sum_over_rows (fp32 atomics, any order):
  ``+ nb u sum_i |K_i|``.  ``WIDE_FAMILY`` names the operand precision this contract assumes above 64 epochs: a
  tensor-core replacement changes that one constant to "tf32" and is then held to check_K's "tf32" family on
  ``tf32_rna(z)`` instead.
* E <= 64: the tf32 plain SYRK, ``check_K``'s "tf32" family of test_gpu_norm_syrk.py on ``tf32_rna(z)``.
* the normaliser: ``wsc_ref`` of test_generic_pipeline_cpu.py (IEEE sequential sums over eps, var = sq/eps - mean^2,
  correctly rounded 1/sqrt, logf within 1 ulp on a rounded quotient), derivation there, ill-conditioned subjects left out
  by zref's rule (with one mask this includes the self column where r is clamped).
* summed classifier kernels: ``sum_i`` of the per-row bound, plus ``nb u sum_i |K_i|`` for the atomics; the decimal
  shrink's digit count of K[0, 0] equals the fp64 one unless K[0, 0] lies within the bound of a power of ten.
* ``k_shrink_kernels``: bit-exact, the rule of test_shrink_digits_and_factor_bit_exact.

Measured on one H100 80GB HBM3 (700 W power limit), largest fraction of each bound used: normaliser 0.19; k_syrk_simt
chain 0.19 inside the pipeline (V2 = 40) and 0.005 at n2 = 50 000 (0.005 with beta, 0.004 summed over rows); tf32 plain
SYRK 0.51; summed classifier kernels 0.015 (chain) and 0.24 (tf32); the reference's fixture kernels 0.011.  The file
runs in about 40 s there, the E = 256, n2 = 50 000 case in 0.9 s.

Coverage (path x edge -> test):

| path                                  | edge                                                         | test                                      |
|---------------------------------------|--------------------------------------------------------------|-------------------------------------------|
| kernel_matrices, k_syrk_simt          | E = 65, 100, 127, 128, 129, 140, 200, 256 (pair blocks of 4096) | test_simt_dyadic_exact                 |
|                                       | n2 = 1, 63, 64, 65, 127, 4099 (64-column chunks)             | test_simt_dyadic_exact                    |
|                                       | dense, ld % 32, stride_i > E ld, odd offset; NaN pad         | test_simt_dyadic_exact                    |
|                                       | nb = 1, 3 (one pass of the grid), 1185, 1300 (grid stride)   | test_simt_dyadic_exact                    |
|                                       | beta = 0 over NaN, 0.5 and -1 over dyadic K_old              | test_simt_dyadic_exact                    |
|                                       | sum_over_rows at nb = 1300, two calls into one out           | test_simt_dyadic_sum_over_rows            |
|                                       | Gaussian, n2 = 50 000, E = 140 and 256                       | test_simt_gaussian_long_rows              |
| voxel_kernels, generic, E > 64        | (140, 20), (256, 16), (65, 13), (100, 12) trailing 4, (200, 64) | test_voxel_kernels_stages             |
| voxel_kernels, generic, E <= 64       | (60, 12), (64, 20), (48, 3), (33, 5)                         | test_voxel_kernels_stages                 |
|   each of them                        | one and two masks, start != 0, ragged nb, V2 = 40 and 4129   | test_voxel_kernels_stages                 |
|   stage 1 (GEMM -> strided block)     | trailing epochs bit-identical to corr_block, finite z        | test_voxel_kernels_stages                 |
|   stage 2 (k_within_subject_norm)     | normalised epochs against wsc_ref                            | test_voxel_kernels_stages                 |
|   stage 3 (SIMT / tf32 SYRK)          | K against the workspace z                                    | test_voxel_kernels_stages                 |
|   several passes                      | 100-row and 512-row passes == one pass, nb = 1300            | test_voxel_kernels_passes_bit_identical   |
| classifier_kernel (portion mode)      | (140, 20), (100, 12), (60, 12), eps = 1, several passes      | test_classifier_kernel_generic            |
| kernel_matrices(sum_over_rows) small mask | E = 140, n2 = V V2                                       | test_classifier_small_mask_path           |
| k_shrink_kernels                      | E = 140, 256; nv % 4 != 0                                    | test_shrink_wide_bit_exact                |
"""
import numpy as np
import pytest
import torch
from sklearn import svm

from brainiak_b200 import _lib
from brainiak_b200.fcma import engine, synthetic
from brainiak_b200.fcma.voxelselector import VoxelSelector
from test_generic_pipeline_cpu import (compare_shrunk, digits, fixture_inputs, kernel_pair_bound, near_power_of_ten,
                                       ref_rho, wsc_ref)
from test_gpu_norm_syrk import U, Ref, check_K, tf32_rna
from test_gpu_pack_and_side_kernels import _k00_values

pytestmark = pytest.mark.gpu

NAN = float("nan")
# operand precision of the kernel-matrix stage above 64 epochs: "fp32" = k_syrk_simt's sequential FMA chain
WIDE_FAMILY = "fp32"
STATS = {}


@pytest.fixture(scope="module")
def dev():
    assert _lib.device_count() > 0, "no sm_90 device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    for k, v in sorted(STATS.items()):
        print("generic pipeline %s: %.3g of the bound" % (k, v))


def record(key, frac):
    STATS[key] = max(STATS.get(key, 0.0), float(frac))


# ------------------------------------------------------------------------------- helpers
def lay(x, layout, dev):
    """Copy x [nb, E, n2] into a NaN-filled buffer in one of four layouts; returns the strided view."""
    nb, E, n2 = x.shape
    pad = -(-n2 // 32) * 32
    ld, si, off = {"dense": (n2, E * n2, 0), "pad32": (pad, E * pad, 0), "gap": (pad, E * pad + 96, 0),
                   "odd": (n2 + 1, E * (n2 + 1) + 5, 3)}[layout]
    buf = torch.full((off + nb * si,), NAN, dtype=torch.float32, device=dev)
    v = buf.as_strided((nb, E, n2), (si, ld, 1), off)
    v.copy_(x)
    return v


def dyadic(gen, shape, dev, scale=8):
    """Integers in [-scale, scale] divided by scale (k/8: products multiples of 2^-6)."""
    return (torch.randint(-scale, scale + 1, shape, generator=gen, device=dev).float() / scale)


def gram64(z):
    return torch.einsum("iaj,ibj->iab", z.double(), z.double())


def chain_bound(z):
    """n2 u sum_j |z_aj z_bj| per row: the worst case of a sequential fp32 FMA chain over the n2 columns."""
    a = z.double().abs()
    return z.shape[2] * U * torch.einsum("iaj,ibj->iab", a, a)


def check_wide(K, z, what, extra=None, K_want=None):
    """K of exact fp32 operands z ([nb, E, n2]) against their fp64 product, with the bound of WIDE_FAMILY."""
    K = K.double()
    assert torch.isfinite(K).all(), what
    if WIDE_FAMILY != "fp32":
        t = tf32_rna(z.double())
        a = t.abs()
        ref = Ref(gram64(t) if K_want is None else K_want, torch.einsum("iaj,ibj->iab", a, a), 0.0, gram64(z))
        st = check_K(K, ref, WIDE_FAMILY, what, extra=extra, bias=False)
        record("wide " + WIDE_FAMILY, st["ratio"])
        return
    want = gram64(z) if K_want is None else K_want
    lim = chain_bound(z) + (0.0 if extra is None else extra)
    err = (K - want).abs()
    bad = err > lim
    assert not bad.any(), "%s: %d entries outside the chain bound, e.g. %s" % (what, int(bad.sum()),
                                                                              bad.nonzero()[:3].tolist())
    record("chain " + what.split()[0], (err / lim.clamp(min=1e-300)).max())


def check_tf32(K, z, what):
    t = tf32_rna(z.double())
    a = t.abs()
    st = check_K(K, Ref(gram64(t), torch.einsum("iaj,ibj->iab", a, a), 0.0, gram64(z)), "tf32", what, bias=False)
    record("tf32 " + what.split()[0], st["ratio"])


# ------------------------------------------------------------------------------- (a) kernel_matrices above 64 epochs
E_WIDE = (65, 100, 127, 128, 129, 140, 200, 256)
N2_SWEEP = (1, 63, 64, 65, 127, 4099)
LAYOUTS = ("dense", "pad32", "gap", "odd")
BETAS = (0.0, 0.5, -1.0)


def run_dyadic(dev, gen, E, n2, nb, layout, beta, what):
    x = dyadic(gen, (nb, E, n2), dev)
    blk = lay(x, layout, dev)
    if beta == 0.0:
        out = torch.full((nb, E, E), NAN, dtype=torch.float32, device=dev)
        old = torch.zeros((nb, E, E), dtype=torch.float64, device=dev)
    else:
        out = dyadic(gen, (nb, E, E), dev, scale=64) * 16
        old = out.double().clone()
    K = engine.kernel_matrices(blk, beta=beta, out=out)
    want = beta * old + gram64(x)
    assert K.data_ptr() == out.data_ptr()
    bad = K.double() != want
    assert not bad.any(), "%s E=%d n2=%d nb=%d %s beta=%g: %d of %d entries differ, e.g. %s" % (
        what, E, n2, nb, layout, beta, int(bad.sum()), bad.numel(), bad.nonzero()[:3].tolist())


@pytest.mark.parametrize("E", E_WIDE)
def test_simt_dyadic_exact(dev, E):
    """k_syrk_simt on dyadic data, bit for bit: every n2 across the 64-column chunk edges in the four layouts, beta 0
    (NaN-filled K), 0.5 and -1, one and three rows; then 1185 and 1300 rows (more than the grid of 1184 blocks)."""
    gen = torch.Generator(device=dev).manual_seed(1000 + E)
    k = 0
    for n2 in N2_SWEEP:
        for nb in (1, 3):
            run_dyadic(dev, gen, E, n2, nb, LAYOUTS[k % 4], BETAS[k % 3], "sweep")
            k += 1
    for j, nb in enumerate((1185, 1300)):
        for n2 in (1, 65):
            run_dyadic(dev, gen, E, n2, nb, LAYOUTS[(j + n2) % 4], BETAS[(j + n2) % 3], "grid")


@pytest.mark.parametrize("E", (65, 140, 256))
def test_simt_dyadic_sum_over_rows(dev, E):
    """sum_over_rows at nb = 1300 (k_scale, then fp32 atomics from the grid-stride loop), into a NaN-filled K with
    beta = 0 and over a dyadic K with beta 0.5; two calls accumulating into one K (beta 0, then 1).  nb n2 < 2^18: exact."""
    gen = torch.Generator(device=dev).manual_seed(2000 + E)
    nb, n2 = 1300, 65
    for beta in (0.0, 0.5):
        x = dyadic(gen, (nb, E, n2), dev)
        if beta == 0.0:
            out = torch.full((E, E), NAN, dtype=torch.float32, device=dev)
            want = gram64(x).sum(0)
        else:
            out = dyadic(gen, (E, E), dev, scale=64) * 16
            want = beta * out.double() + gram64(x).sum(0)
        K = engine.kernel_matrices(lay(x, "gap", dev), beta=beta, out=out, sum_over_rows=True)
        assert torch.equal(K.double(), want), "sum_over_rows E=%d beta=%g" % (E, beta)
    out = torch.full((E, E), NAN, dtype=torch.float32, device=dev)
    x1 = dyadic(gen, (nb, E, n2), dev)
    x2 = dyadic(gen, (7, E, 127), dev)
    engine.kernel_matrices(lay(x1, "odd", dev), beta=0.0, out=out, sum_over_rows=True)
    engine.kernel_matrices(lay(x2, "pad32", dev), beta=1.0, out=out, sum_over_rows=True)
    assert torch.equal(out.double(), gram64(x1).sum(0) + gram64(x2).sum(0)), "two calls E=%d" % E


@pytest.mark.parametrize("E", (140, 256))
def test_simt_gaussian_long_rows(dev, E):
    """Gaussian z, n2 = 50 000, a few rows: the precision contract of the kernel-matrix stage above 64 epochs, against
    the fp64 product of the exact fp32 inputs; beta over old values and sum_over_rows with their terms."""
    gen = torch.Generator(device=dev).manual_seed(3000 + E)
    nb, n2 = 3, 50000
    z = torch.randn((nb, E, n2), generator=gen, device=dev)
    K = engine.kernel_matrices(lay(z, "pad32", dev))
    check_wide(K, z, "gaussian E=%d" % E)
    old = torch.randn((nb, E, E), generator=gen, device=dev) * 1000
    want = 0.5 * old.double() + gram64(z)
    K = engine.kernel_matrices(lay(z, "odd", dev), beta=0.5, out=old.clone())
    check_wide(K, z, "gaussian_beta E=%d" % E, extra=2 * U * (0.5 * old.double().abs() + want.abs()), K_want=want)
    Ks = engine.kernel_matrices(lay(z, "dense", dev), sum_over_rows=True)
    Ki = gram64(z)
    lim = chain_bound(z).sum(0) + nb * U * Ki.abs().sum(0)
    err = (Ks.double() - Ki.sum(0)).abs()
    assert torch.all(err <= lim), "gaussian sum E=%d" % E
    record("chain gaussian_sum", (err / lim).max())


# ------------------------------------------------------------------------------- (b) voxel_kernels, stage by stage
STAGE_CASES = [(140, 20), (256, 16), (65, 13), (100, 12), (200, 64), (60, 12), (64, 20), (48, 3), (33, 5)]


def operands(E, V, V2, dev, seed, T=24):
    """(rows, cols) operands: one mask (V2 None) or two."""
    raw, _ = synthetic.make_epochs(V, T, E, seed=seed)
    ep, T_e = engine.stack_epochs(raw, dev)
    op = engine.pack_epochs(ep, T_e, "fp32")
    if V2 is None:
        return op, op
    raw2, _ = synthetic.make_epochs(V2, T, E, seed=seed + 1)
    ep2, _ = engine.stack_epochs(raw2, dev)
    return op, engine.pack_epochs(ep2, T_e, "fp32")


@pytest.mark.parametrize("E,eps", STAGE_CASES)
def test_voxel_kernels_stages(dev, E, eps):
    """One pass of voxel_kernels on the generic path, the 0xFF-filled workspace read back as the strided [nb][E][ld]
    z the SYRK consumed: (1) trailing epochs bit-identical to corr_block, z finite; (2) normalised epochs against
    wsc_ref of corr_block's r; (3) K against the fp64 product of that z."""
    assert not engine.fused_supported(E, eps)
    S = (E // eps) * eps
    for two in (False, True):
        for V2 in (40, 4129):
            V = 300 if two else V2
            start, nb = (3, 37) if V > 40 else (2, 37)
            op, op2 = operands(E, V, V2 if two else None, dev, seed=E * 31 + eps + V2 + two)
            ld = -(-V2 // 32) * 32
            assert ld != V2
            work = engine.Workspace(E, V2, nb, dev)
            work.buf.fill_(255)
            K = engine.voxel_kernels(op, op2, start, nb, eps, work=work)
            torch.cuda.synchronize()
            z = work.buf.view(torch.float32)[:nb * E * ld].view(nb, E, ld)[..., :V2]
            what = "E=%d eps=%d two=%d V2=%d" % (E, eps, two, V2)
            assert torch.isfinite(z).all(), what
            r = engine.corr_block(op, op2, start, nb)
            assert torch.equal(z[:, S:], r[:, S:]), what + ": trailing epochs differ from corr_block"
            z64, delta, ill = wsc_ref(r.double(), eps)
            err = (z.double() - z64).abs()
            bad = (err > delta) & ~ill
            assert not bad.any(), "%s: %d normalised values outside the bound, e.g. %s (err %s, bound %s)" % (
                what, int(bad.sum()), bad.nonzero()[:3].tolist(), err[bad][:3].tolist(), delta[bad][:3].tolist())
            assert float(ill.double().mean()) <= 0.15, what
            ok = ~ill & (delta > 0)
            if ok.any():
                record("normaliser", (err[ok] / delta[ok]).max())
            if E > 64:
                check_wide(K, z, "stages " + what)
            else:
                check_tf32(K, z, "stages " + what)


@pytest.mark.parametrize("E,eps", [(140, 20), (48, 3)])
def test_voxel_kernels_passes_bit_identical(dev, E, eps):
    """nb = 1300 in passes of 100 rows and of 512 rows (a 700-row workspace: whole 256-row blocks) equals one pass."""
    V2 = 40
    op, op2 = operands(E, 1400, V2, dev, seed=E + eps)
    one = engine.voxel_kernels(op, op2, 50, 1300, eps, work=engine.Workspace(E, V2, 1536, dev))
    for rows in (100, 700):
        K = engine.voxel_kernels(op, op2, 50, 1300, eps, work=engine.Workspace(E, V2, rows, dev))
        assert torch.equal(K, one), "E=%d eps=%d: %d-row workspace differs from one pass" % (E, eps, rows)


# ------------------------------------------------------------------------------- (c) summed classifier kernels
def per_row_z(op, op2, start, nb, eps):
    """The fp32 z the classifier path forms for each row: raw r, normalised by within_subject_norm_ when eps > 1."""
    r = engine.corr_block(op, op2, start, nb).contiguous()
    return engine.within_subject_norm_(r, eps) if eps > 1 else r


def check_summed(K, z, E, what):
    """K [E, E] against sum_i Z_i Z_i^T in fp64: the per-row bound summed, plus nb u sum_i |K_i| (atomics); the shrink's
    digit count of K[0, 0]."""
    nb = z.shape[0]
    Ki = gram64(z)
    want = Ki.sum(0)
    if E > 64:
        lim = chain_bound(z).sum(0)
    else:
        t = tf32_rna(z.double())
        a = t.abs()
        lim = 50.0 * U * torch.einsum("iaj,ibj->ab", a, a) + (gram64(t) - Ki).abs().sum(0)
    lim = lim + nb * U * Ki.abs().sum(0)
    err = (K.double() - want).abs()
    assert torch.isfinite(K).all() and torch.all(err <= lim), "%s: worst excess %.3g" % (what, float((err - lim).max()))
    record("summed " + ("chain" if E > 64 else "tf32"), (err / lim).max())
    k00, w00 = float(K[0, 0]), float(want[0, 0])
    if not near_power_of_ten(w00, float(lim[0, 0]) + abs(k00 - w00)):
        assert digits(k00) == digits(w00), "%s: digit count of K00 %g vs %g" % (what, k00, w00)


@pytest.mark.parametrize("E,eps", [(140, 20), (100, 12), (60, 12), (140, 1)])
def test_classifier_kernel_generic(dev, E, eps):
    """classifier_kernel(symmetric=False), portion mode: one pass, and a 40-row workspace (several passes, k_scale
    with beta = 1 before each); eps = 1 skips the normalisation."""
    V, V2, start, nb = 300, 700, 11, 250
    op, op2 = operands(E, V, V2, dev, seed=E * 3 + eps)
    z = per_row_z(op, op2, start, nb, eps)
    for rows in (nb, 40):
        K = engine.classifier_kernel(op, op2, start, nb, eps, work=engine.Workspace(E, V2, rows, dev), symmetric=False)
        check_summed(K, z, E, "classifier E=%d eps=%d rows=%d" % (E, eps, rows))


def test_classifier_small_mask_path(dev):
    """The Classifier's small-mask path: corr_block in layout 1 flattened to [1, E, V V2], normalised, one
    kernel_matrices(sum_over_rows=True) call (k_syrk_simt, one row, n2 = V V2)."""
    E, eps, V, V2 = 140, 20, 30, 200
    op, op2 = operands(E, V, V2, dev, seed=77)
    corr = engine.corr_block(op, op2, 0, V, layout=1).contiguous()
    flat = engine.within_subject_norm_(corr.view(1, E, V * V2), eps)
    K = engine.kernel_matrices(flat, sum_over_rows=True)
    check_summed(K, flat, E, "small mask")


# ------------------------------------------------------------------------------- (d) decimal shrink at wide E
@pytest.mark.parametrize("E", (140, 256))
def test_shrink_wide_bit_exact(dev, E):
    """k_shrink_kernels at E = 140 and 256 (19 600 / 65 536 entries per warp), nv not a multiple of 4: digit counts and
    the scaled kernels bit for bit against the reference's rule."""
    k00 = _k00_values()
    assert len(k00) % 4                                  # the last block of 4 warps is partly empty
    rng = np.random.RandomState(E)
    K = (rng.rand(len(k00), E, E) * 2 - 0.5).astype(np.float32)
    K[:, 0, 0] = k00
    K[:, E - 1, E - 1] = k00 * np.float32(0.75)
    want = K.copy()
    nd = np.ones(len(k00), np.int32)
    for i, v in enumerate(k00):
        if np.isfinite(v):
            nd[i] = len(str(int(v)))
            if nd[i] > 2:
                want[i] = K[i] * np.float32(10 ** (2 - int(nd[i])))
    t = torch.from_numpy(K.copy()).to(dev)
    got_nd = engine.shrink_kernels_(t, return_digits=True).cpu().numpy()
    assert np.array_equal(got_nd, nd)
    got = t.cpu().numpy()
    bad = np.flatnonzero((got.view(np.int32) != want.view(np.int32)).any(axis=(1, 2)))
    assert not bad.size, "E=%d: scaled kernels differ for K00 = %s" % (E, k00[bad[:5]].tolist())


# ------------------------------------------------------------------------------- the reference's precomputed fixtures
def _probe(raw):
    return np.stack([raw[e][:4, ::997][:, :16] for e in (0, len(raw) - 1)])


@pytest.mark.parametrize("precision", ["fp32", "tf32x3"])
@pytest.mark.parametrize("gpu_cv", [True, False])
@pytest.mark.parametrize("name", ["w1", "w2"])
def test_run_matches_reference_precomputed(dev, golden, name, gpu_cv, precision):
    """VoxelSelector.run(SVC(kernel='precomputed')) in the fp32-faithful modes returns the unmodified reference's voxel
    list and accuracies (tests/golden/make_golden_precomputed_wide.py): w1 E = 140, eps 20, 7 folds, one mask with 8
    planted voxels; w2 E = 100, eps 12 (4 trailing raw epochs), 5 folds, three classes, two masks."""
    g = golden("vs_pre_" + name)
    raw, raw2, eps = fixture_inputs(name)
    assert np.array_equal(_probe(raw), g["probe"])
    labels = [int(x) for x in g["labels"]]
    vs = VoxelSelector(labels, eps, int(g["num_folds"]), raw, raw2, device=dev, gpu_cv=gpu_cv, process_num=0,
                       precision=precision)
    got = vs.run(svm.SVC(kernel="precomputed", shrinking=False, C=1))
    want = [(int(v), float(a)) for v, a in zip(g["vids"], g["accs"])]
    assert [v for v, _ in got] == [v for v, _ in want]
    assert [a for _, a in got] == [a for _, a in want]


def gpu_rho(P, N, T):
    """|r_gpu - r_oracle|: the fp32-faithful GEMM (max(1e-6 |x| |y|, 2 T u sum |x y|) of the exact r, as
    test_gpu_corr_gemm.py holds it) plus the oracle's fp32 chain (T u sum |x y|)."""
    return np.maximum(1e-6 * N, 2 * T * U * P) + T * U * P


@pytest.mark.parametrize("name", ["w1", "w2"])
def test_sampled_kernels_match_reference(dev, golden, name):
    """The shrunk kernels of the sampled voxels (voxel_kernels on the generic path, then k_shrink_kernels) against the
    reference's, within both fp32 chains' bound (test_generic_pipeline_cpu.py: kernel_pair_bound)."""
    g = golden("vs_pre_" + name)
    raw, raw2, eps = fixture_inputs(name)
    for precision in ("fp32", "tf32x3"):
        ep, T_e = engine.stack_epochs(raw, dev)
        op = engine.pack_epochs(ep, T_e, precision)
        op2 = op
        if raw2 is not None:
            ep2, _ = engine.stack_epochs(raw2, dev)
            op2 = engine.pack_epochs(ep2, T_e, precision)
        for v, K_ref in zip(g["sample_vids"], g["sample_kernels"]):
            v = int(v)
            K = engine.voxel_kernels(op, op2, v, 1, eps)
            K_unshrunk = K[0].double().cpu().numpy()
            nd = engine.shrink_kernels_(K, return_digits=True)
            _, bound = kernel_pair_bound(raw, raw2, v, eps, gpu_rho, ref_rho)
            frac = compare_shrunk(K[0].cpu().numpy(), int(nd[0]), K_ref, K_unshrunk, bound[0],
                                  "%s %s voxel %d" % (name, precision, v))
            record("fixture kernels", frac)
