"""Element-wise tests of stage 2 of the hot path -- Fisher-z, within-subject z-score and ``K_i = Z_i Z_i^T`` -- against
an fp64 reference computed from the exact values the kernels read.

Kernels under test: ``k_norm_syrk<R, EPS, FISHER, VEC>`` (row pass), the column passes ``k_norm_syrk_cols16``,
``k_norm_syrk_cols<EPS, 4, HALF>``, ``k_norm_syrk_cols2``, ``k_norm_syrk_cols_tma`` and ``k_norm_syrk_cols64``, the
tf32 plain SYRK (``EPS = 0``) and ``k_syrk_simt`` (E > 64).

Reference (``zref``), from a block ``x`` [rows, E, n2] in fp32 (or the fp16 block widened):
1. Fisher ``log2((1 + x) / (1 - x))`` in fp64 with the clamps of fcma_extension.cc:68-72 (``1 +- x`` replaced by 1e-4
   where it is <= 0), only where the kernel applies it (raw-input ``norm_kernel_matrices``, FCMA_FLAG_FISHER_IN_PASS2);
   the kernels use log2, a constant factor that the z-score cancels;
2. z-score of every (subject, column) over its ``eps`` epochs in fp64, population variance, ``var == 0`` -> 0; epochs
   past the last whole subject pass through unchanged (fcma_extension.cc:52), so for ``eps > E`` nothing is normalised;
3. the self column (if any) set to 0 after the normalisation.
This is ``z64``.  The kernels' MMA operand is ``z16 = fp16(fp32(z64))`` (``cvt.rn.f16x2``; plain SYRK: tf32 rounded
ties away, ``(bits + 0x1000) & ~0x1fff``, of the exact input), ``K16 = sum_j z16 z16^T`` in fp64; ``K64`` from ``z64``.

Bound, element by element: ``|K - K16|_ab <= A_ab + F_ab`` (+ the terms of beta and sum_over_rows below), u = 2^-24:
* ``A_ab = c_A u sum_j |z16_aj z16_bj|``: accumulation.  The fp16 (tf32) products are exact in fp32; the warp MMA adds
  them with truncation (at most 2u relative per add) for FLUSH = 8 chunks (16 m16n8k16 or 32 m16n8k8 adds) before the
  round-to-nearest fp32 partials take over (one add per flush, then 8 warps); a column pass folds every
  COLS_SEG_STEPS = 64 16-row steps.  The worst case of such a chain is ~70 (row pass at n2 = 50 000) and ~130 (column
  pass), so ``C_A`` holds calibrated constants: the measured maximum of ``(|K - K16| - F) / (u sum |z16 z16|)`` on one
  H100 times ~2 (row pass 40, tf32 50).  The column passes need 96 (measured 73.8): a 64-step chain of truncating
  adds, mostly on the diagonal, where every add truncates the same way (bias -4.3e-6 against -1.0e-6 for the row pass).
* ``F_ab = sum_j (D_aj |z16_bj| + D_bj |z16_aj| + D_aj D_bj)``: fp16 rounding flips.  The kernel's fp32 z differs from
  z64 by at most ``delta``; where ``fp16(fp32(z64 - delta)) != fp16(fp32(z64 + delta))`` (z64 within delta of an fp16
  rounding midpoint) the kernel may have rounded to either side and ``D`` is the distance of the two; elsewhere D = 0.
* ``delta = (3 eps + 8) u (1 + m^2/var) max(1, |z|)`` (normaliser, fp32): the kernels sum x and x^2 in fp32 (error <=
  eps u sum |x|, eps u sum x^2), form ``var = m^2 - E[x^2]`` with one FMA (error <= (3 eps + 1) u E[x^2] =
  (3 eps + 1) u var (1 + m^2/var), as |m| E|x| <= E[x^2]), take ``rsqrt.approx`` (<= 2^-22.9 relative), round ``m inv``
  once and ``x inv + (-m inv)`` once.  Collecting: ``|dz| <= u (1 + m^2/var) max(1, |z|) (2.5 eps + 6.5)``, using
  |m|/sigma <= 1 + m^2/var.  Plus, where the kernel applies Fisher itself, ``(2 + |z| zmax) eF / sigma``: eF =
  ``2^-21 (2 + |lg2 num| + |lg2 den|) + u (2/ln2 + |x|)`` bounds ``lg2.approx`` (2^-22 absolute / relative), the fp32
  rounding of 1 +- r and of the difference, sigma is the fp64 spread of the subject's log2 values, zmax its largest
  |z|; an error eF moves the mean by eF and the variance by 2 sigma zmax eF.  ``var == 0``: delta = 0 (z must be 0).
* no first-order bound exists where ``(3 eps + 1) u (1 + m^2/var) >= 1/16`` (or the Fisher term reaches 1/16 of
  max(1, |z|)): two near-equal values at eps = 2, the self column of a one-mask block (r = 1 +- ulp).  The fp32
  normaliser of the reference is just as ill-conditioned there; the K entries of such a subject's epochs are left out
  (``Ref.free``), at most 15 % of the entries for eps >= 4.
* beta: ``+ 2u (|beta K_old| + |K16|)``; sum_over_rows (fp32 atomics in any order): ``+ nb u sum_i |K16_i|``.
* plain SYRK of caller data (EPS = 0): the inputs are exact, D = 0, only A (family "tf32").
* ``k_syrk_simt``: a sequential fp32 FMA chain over n2 terms per entry: ``n2 u sum_j |z_aj z_bj|`` (worst case).

Bias: ``mean((K - K16) / K16)`` over all diagonal entries must stay below ``BIAS_MAX``.  Rounding noise averages out in
this mean, truncation bias does not: a lost flush of the MMA accumulators (an unflushed chain biased the diagonal by
5e-5 at n2 = 50 000) or a lost fold of the column pass shows here first.

Coverage of ``launch_norm_syrk`` (E <= 16 and eps <= 16, fp32 vector block, no Fisher -> R = 2; E <= 32 -> R = 4;
else R = 8; VEC 0 = scalar loads (ld or stride_i not a multiple of 4, or a misaligned base), 1 = cp.async fp32,
2 = fp16 tiled block of the pipelines, only without Fisher):

| R | FISHER | VEC | EPS                        | covered by                                                            |
|---|--------|-----|----------------------------|-----------------------------------------------------------------------|
| 2 | 0      | 1   | 0, 1, 2, 4, 8, 16          | test_row_kernel_sweep (E <= 16, layout "vec"), test_plain_syrk_and_simt |
| 4 | 0      | 0   | 0 .. 32                    | test_row_kernel_sweep (layout "offset1"), test_plain_syrk_and_simt  |
| 4 | 0      | 1   | 0 .. 32                    | test_row_kernel_sweep (17 <= E <= 32, and eps = 32 at E <= 16)        |
| 4 | 1      | 0/1 | 1 .. 32                    | test_row_kernel_sweep (fisher), test_pipeline_row_pass (PASS2)        |
| 4 | 0      | 2   | 1 .. 32                    | test_pipeline_row_pass ("f16_E20", "f16_E32")                         |
| 8 | 0      | 0/1 | 0 .. 64                    | test_row_kernel_sweep (E >= 33), test_plain_syrk_and_simt             |
| 8 | 1      | 0/1 | 1 .. 64                    | test_row_kernel_sweep (E >= 33, fisher)                               |
| 8 | 0      | 2   | 1 .. 64                    | test_pipeline_row_pass ("f16_E40", "f16_E64")                         |

and of ``launch_norm_syrk_cols`` (through ``voxel_kernels_sym``; eps <= 32 for E <= 32, <= 64 for E > 32):

| kernel                         | EPS       | HALF | covered by (test_sym_column_pass case)                        |
|--------------------------------|-----------|------|---------------------------------------------------------------|
| k_norm_syrk_cols16             | 1 .. 16   | 0    | "cols16" (E = 12, 16), "n4096_cols16", "n1280_cols16"         |
| k_norm_syrk_cols<EPS, 4, 0>    | 1 .. 32   | 0    | "cols" (E = 24, 32), "pad32" (E = 12), "n4096_cols", "n1024_cols" |
| k_norm_syrk_cols<EPS, 4, 1>    | 1 .. 32   | 1    | "half" (E = 20, 32)                                           |
| k_norm_syrk_cols2<EPS, 4>      | 1 .. 32   | 0    | "v2" (E = 24, 32)                                             |
| k_norm_syrk_cols_tma<EPS, H,4> | 1 .. 32   | 0, 1 | "tma" (E = 24, 32), "tma_half" (E = 24, 32)                   |
| k_norm_syrk_cols64<EPS>        | 1 .. 64   | 0    | "wide" (E = 40, 64)                                           |
| transposed copy + row pass     | 1 .. 32   | 0    | "transposed" (E = 24)                                         |

Not covered: ``k_norm_syrk_cols<EPS, 2, false>`` and ``k_norm_syrk_cols2<EPS, 2>`` (2 columns per warp) are only
reachable in the diagnostic build (``FCMA_COLS_CPW`` / ``FCMA_COLS_V2_CPW``), which the product library never selects.
"""
import math

import numpy as np
import pytest
import torch

from brainiak_b200 import _lib
from brainiak_b200.fcma import engine, synthetic
from oracle import fcma_oracle as orc

gpu = pytest.mark.gpu

U = 2.0 ** -24
NAN = float("nan")
# accumulation constants (units of u * sum |z16 z16|) and diagonal bias limits, calibrated on one H100 80GB HBM3 (700 W limit):
# measured c_A 19.6 (row pass), 24.7 (tf32 plain SYRK), 73.8 (column passes); bias -1.0e-6 (row), -4.3e-6 (columns)
C_A = {"row": 40.0, "tf32": 50.0, "cols": 96.0}
BIAS_MAX = {"row": 2e-6, "cols": 6e-6}
E_LIST = (1, 2, 3, 5, 8, 12, 16, 17, 24, 31, 32, 33, 40, 48, 63, 64)
N2_LIST = (1, 3, 4, 5, 31, 32, 33, 255, 257, 2047, 2048, 2049, 4129)
STATS = {}


def accepted_eps(E):
    return [e for e in (1, 2, 4, 8, 16, 32, 64) if e <= (32 if E <= 32 else 64)]


# ------------------------------------------------------------------------------- reference helpers (CPU or device)
def f16(x):
    """fp16(fp32(x)) of a float64 tensor, back in float64."""
    return x.float().half().double()


def tf32_rna(x):
    """tf32 operand of the plain SYRK: fp32 bits + 0x1000 with the low 13 bits cleared (round to nearest, ties away)."""
    b = x.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32).double()


def flip_width(z, delta):
    """Distance of the fp16 roundings of z - delta and z + delta (0 where every value within delta rounds alike)."""
    return (f16(z + delta) - f16(z - delta)).abs()


def zref(x, eps, fisher=False, self_cols=None):
    """fp64 reference of the kernels' normalisation of a block ``x`` (float64 [rows, E, n2]).
    Returns (z64, z16, D, ill): the normalised block, the fp16 operand the kernel should multiply, the flip widths, and
    the values whose subject is too ill-conditioned for a first-order bound (bool [rows, E, n2])."""
    rows, E, n2 = x.shape
    z = x.clone()
    delta = torch.zeros_like(x)
    ill = torch.zeros(x.shape, dtype=torch.bool, device=x.device)
    S = (E // eps) * eps
    if S:
        v = x[:, :S]
        if fisher:
            num = torch.where(1 + v <= 0, torch.full_like(v, 1e-4), 1 + v)
            den = torch.where(1 - v <= 0, torch.full_like(v, 1e-4), 1 - v)
            lnum, lden = torch.log2(num), torch.log2(den)
            v = lnum - lden
            ef = 2.0 ** -21 * (2 + lnum.abs() + lden.abs()) + U * (2 / math.log(2) + v.abs())
        g = v.reshape(rows, S // eps, eps, n2)
        m = g.mean(2, keepdim=True)
        var = ((g - m) ** 2).mean(2, keepdim=True)
        pos = var > 0
        sd = torch.sqrt(torch.where(pos, var, torch.ones_like(var)))
        zz = torch.where(pos, (g - m) / sd, torch.zeros_like(g))
        cond = 1 + m * m / torch.where(pos, var, torch.ones_like(var))
        d = (3 * eps + 8) * U * cond * zz.abs().clamp(min=1)
        bad = (3 * eps + 1) * U * cond >= 1.0 / 16
        if fisher:
            efm = ef.reshape(g.shape).amax(2, keepdim=True) / sd
            zmax = zz.abs().amax(2, keepdim=True)
            d = d + (2 + zz.abs() * zmax) * efm
            bad = bad | ((2 + zmax * zmax) * efm >= 1.0 / 16)
        bad = pos & bad
        d = torch.where(pos & ~bad, d, torch.zeros_like(d))
        z[:, :S] = zz.reshape(rows, S, n2)
        delta[:, :S] = d.reshape(rows, S, n2)
        ill[:, :S] = bad.expand(g.shape).reshape(rows, S, n2)
    z16 = f16(z)
    D = flip_width(z, delta)
    if self_cols is not None:
        ii = torch.arange(rows, device=x.device)
        sc = torch.as_tensor(self_cols, device=x.device)
        ok = (sc >= 0) & (sc < n2)
        for t in (z, z16, D):
            t[ii[ok], :, sc[ok]] = 0.0
        ill[ii[ok], :, sc[ok]] = False
    return z, z16, D, ill


def kterms(z64, z16, D, dim=2):
    """(K16, S = sum |z16 z16^T|, F, K64) summed over columns (dim = 2: per row) or over rows (dim = 0: per column)."""
    spec = "iaj,ibj->iab" if dim == 2 else "iaj,ibj->jab"
    a = z16.abs()
    K16 = torch.einsum(spec, z16, z16)
    S = torch.einsum(spec, a, a)
    DA = torch.einsum(spec, D, a)
    F = DA + DA.transpose(1, 2) + torch.einsum(spec, D, D)
    K64 = torch.einsum(spec, z64, z64)
    return K16, S, F, K64


class Ref:
    """K16, S, F, K64 of a block ([voxels, E, E]) and ``free`` [voxels, E]: epochs of a voxel whose kernel entries depend
    on an ill-conditioned subject (eps <= 2: two near-equal values; 1 + m^2/var beyond 1/(16 (3 eps + 1) u)), where the
    fp32 normaliser, in the kernels as in the reference, has no first-order error bound."""

    def __init__(self, K16, S, F, K64, free=None, eps=None):
        self.K16, self.S, self.F, self.K64, self.eps = K16, S, F, K64, eps
        self.free = torch.zeros(K16.shape[:2], dtype=torch.bool, device=K16.device) if free is None else free

    @classmethod
    def of_block(cls, x, eps, fisher=False, self_cols=None, dim=2, chunk=256):
        """Reference kernels of block x (float tensor [rows, E, n2], any device); dim = 0 sums over the rows (column
        voxels' kernels), in row chunks."""
        acc = None
        for r0 in range(0, x.shape[0], chunk):
            sc = None if self_cols is None else self_cols[r0:r0 + chunk]
            z64, z16, D, ill = zref(x[r0:r0 + chunk].double(), eps, fisher, sc)
            t = list(kterms(z64, z16, D, dim)) + [ill.any(dim).transpose(0, 1) if dim == 0 else ill.any(dim)]
            if acc is None:
                acc = t
            elif dim == 2:
                acc = [torch.cat((p, q)) for p, q in zip(acc, t)]
            else:
                acc = [p + q for p, q in zip(acc[:4], t[:4])] + [acc[4] | t[4]]
        return cls(*acc, eps=eps)


def record(family, **kw):
    s = STATS.setdefault(family, {})
    for k, v in kw.items():
        s[k] = max(s.get(k, 0.0), v) if k != "bias" else (v if abs(v) > abs(s.get(k, 0.0)) else s.get(k, 0.0))


def check_K(K, ref, family, what, extra=None, K16=None, bias=True):
    """|K - K16| <= C_A u S + F (+ extra) element by element; records the calibration figures."""
    K = K.double()
    K16 = ref.K16 if K16 is None else K16
    assert torch.isfinite(K).all(), "%s: non-finite kernel entries" % what
    err = (K - K16).abs()
    bound = C_A[family] * U * ref.S + ref.F + (0.0 if extra is None else extra)
    free = ref.free[:, :, None] | ref.free[:, None, :]
    if ref.eps is not None and ref.eps >= 4:      # only the self column of a one-mask block (r = 1 +- ulp) is ill there
        assert float(free.double().mean()) <= 0.15, "%s: %.3f of the entries unbounded" % (what, float(free.double().mean()))
    bad = (err > bound) & ~free
    pos = (ref.S > 0) & ~free
    resid = ((err - ref.F - (0.0 if extra is None else extra)).clamp(min=0) / (U * torch.where(pos, ref.S, 1.0)))
    stats = {"c_A": float(resid[pos].max()) if pos.any() else 0.0,
             "ratio": float((err / torch.where(bound > 0, bound, 1.0))[~free].max()) if (~free).any() else 0.0,
             "rel64": float((K - ref.K64).abs()[~free].max() / ref.K64.abs().max().clamp(min=1e-300)) if (~free).any() else 0.0,
             "free": float(free.double().mean())}
    if bias:
        d = torch.diagonal(K, dim1=1, dim2=2)
        d16 = torch.diagonal(K16, dim1=1, dim2=2)
        keep = (d16 > 0) & ~ref.free
        if keep.any():
            stats["bias"] = float(((d - d16)[keep] / d16[keep]).mean())
    record(family, **stats)
    if bad.any():
        idx = bad.nonzero()[:4].tolist()
        pytest.fail("%s: %d of %d entries outside the bound, e.g. %s: got %s, K16 %s, bound %s" % (
            what, int(bad.sum()), bad.numel(), idx, [float(K[tuple(i)]) for i in idx],
            [float(K16[tuple(i)]) for i in idx], [float(bound[tuple(i)]) for i in idx]))
    return stats


def check_bias(stats, family, what):
    assert abs(stats["bias"]) <= BIAS_MAX[family], "%s: diagonal bias %.3g > %.1g" % (what, stats["bias"], BIAS_MAX[family])


# ------------------------------------------------------------------------------- CPU self-tests of the reference
def test_zref_matches_oracle_within_subject_norm():
    """zref equals the oracle's fp32 restatement of fcma_extension.cc within fp32 tolerance: Fisher + z-score,
    trailing epochs, var = 0 (a constant subject and a dead column) and eps > E."""
    rng = np.random.RandomState(5)
    for E, eps in ((7, 2), (12, 4), (9, 4), (3, 4), (16, 16), (6, 1)):
        r = np.tanh(rng.randn(3, E, 40) * 0.4).astype(np.float32)
        r[0, :, 3] = 0.0                                 # dead column
        if E >= 4 and eps == 4:
            r[1, 0:4, 5] = np.float32(0.25)              # constant subject
        want = orc.within_subject_norm(r.copy(), eps).astype(np.float64)
        z64, z16, D, ill = zref(torch.from_numpy(r).double(), eps, fisher=True)
        S = (E // eps) * eps
        np.testing.assert_array_equal(z64[:, S:].numpy(), r[:, S:].astype(np.float64))
        ok = ~ill.numpy()                                # the oracle's fp32 has no first-order bound there either
        assert ok.mean() > 0.9
        d = np.abs(z64.numpy() - want)[ok]
        assert np.all(d <= 2e-5 * (np.abs(want[ok]) + 1)), (E, eps, d.max())
        assert np.all(z64[0, :S, 3].numpy() == 0)
        if E >= 4 and eps == 4:
            assert np.all(z64[1, 0:4, 5].numpy() == 0) and np.all(D[1, 0:4, 5].numpy() == 0)


def test_f16_and_tf32_emulation_bit_patterns():
    """fp16(fp32(x)) rounds to nearest even; the tf32 operand rounds ties away from zero."""
    h = 2.0 ** -10                                         # fp16 spacing on [1, 2)
    x = torch.tensor([1 + h / 2, 1 + 1.5 * h, 1 + h / 2 + 2.0 ** -20, -(1 + 1.5 * h), 65504.0, 2.0 ** -25, 3 * 2.0 ** -25],
                     dtype=torch.float64)
    want = [1.0, 1 + 2 * h, 1 + h, -(1 + 2 * h), 65504.0, 0.0, 2.0 ** -24 * 2]
    assert f16(x).tolist() == want
    t = 2.0 ** -10                                         # tf32 spacing on [1, 2)
    y = torch.tensor([1 + t / 2, 1 + 1.5 * t, 1 + t / 2 - 2.0 ** -23, -(1 + t / 2), 3.0 + 2.0 ** -22], dtype=torch.float64)
    assert tf32_rna(y).tolist() == [1 + t, 1 + 2 * t, 1.0, -(1 + t), 3.0]


def test_flip_mask_at_fp16_midpoints():
    """A value within delta of an fp16 rounding midpoint is flagged with the width of one fp16 step; others are not."""
    h = 2.0 ** -10
    z = torch.tensor([1 + h / 2, 1 + h / 2 + 1e-7, 1 + h / 2 + 1e-4, 0.5 + h / 4, 1.0, 2 - h / 2, 2 - h / 4],
                     dtype=torch.float64)
    D = flip_width(z, torch.full_like(z, 1e-6))
    assert D.tolist() == [h, h, 0.0, h / 2, 0.0, h, 0.0]
    assert flip_width(z, torch.zeros_like(z)).abs().max() == 0


# ------------------------------------------------------------------------------- GPU fixtures and block builders
@pytest.fixture(scope="module")
def dev():
    assert _lib.device_count() > 0, "no sm_90 device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    for fam, s in sorted(STATS.items()):
        print("norm_syrk %s: %s" % (fam, ", ".join("%s %.3g" % kv for kv in sorted(s.items()))))


def make_block(gen, nb, E, n2, raw, dev):
    """[nb, E, n2] float32: raw r in (-1, 1) (raw=True) or Fisher-z-like values, trailing structure included."""
    x = torch.randn((nb, E, n2), generator=gen, dtype=torch.float64) * 0.45
    x = torch.tanh(x) if raw else x
    return x.float().to(dev)


def place(x, layout, dev, fill=NAN):
    """Copy x [nb, E, n2] into a NaN-filled buffer with the given layout; returns the strided view."""
    nb, E, n2 = x.shape
    if layout == "vec":            # ld a multiple of 4 with pad columns, gaps between rows
        ld = (n2 + 3) // 4 * 4 + 4
        si, off = E * ld + 8, 4
    elif layout == "offset1":      # base pointer one float past a 16-byte boundary: scalar loads
        ld, si, off = n2, E * n2, 1
    else:                          # "dense"
        ld, si, off = n2, E * n2, 0
    buf = torch.full((off + nb * si + 64,), fill, dtype=torch.float32, device=dev)
    v = buf.as_strided((nb, E, n2), (si, ld, 1), off)
    v.copy_(x)
    return v


def run_row_case(dev, gen, E, n2, eps, fisher, layout, self_col0=-1, nb=5, beta=0.0, sum_rows=False, misalign=False,
                 what=""):
    x = make_block(gen, nb, E, n2, raw=fisher, dev=dev)
    blk = place(x, layout, dev)
    EE = E * E
    old = None
    if sum_rows:
        out = torch.randn((E, E), generator=gen).float().to(dev) if beta else torch.full((E, E), NAN, device=dev)
    else:
        base = torch.full((1 + nb * EE,), NAN, dtype=torch.float32, device=dev)
        out = (base[1:] if misalign else base[:nb * EE]).view(nb, E, E)
        if beta:
            out.copy_(torch.randn((nb, E, E), generator=gen).float())
    if beta:
        old = out.double().clone()
    K = engine.norm_kernel_matrices(blk, eps, fisher_done=not fisher, self_col0=self_col0, beta=beta, out=out,
                                    sum_over_rows=sum_rows)
    torch.cuda.synchronize()
    sc = [self_col0 + i for i in range(nb)] if self_col0 >= 0 else None
    ref = Ref.of_block(x, eps, fisher, sc)
    name = "%s E=%d n2=%d eps=%d fisher=%d %s self=%d beta=%g sum=%d" % (what, E, n2, eps, fisher, layout, self_col0,
                                                                          beta, sum_rows)
    if sum_rows:
        K16 = ref.K16.sum(0, keepdim=True)
        extra = nb * U * ref.K16.abs().sum(0, keepdim=True)
        if beta:
            K16 = K16 + beta * old
            extra = extra + 2 * U * (beta * old.abs() + K16.abs())
        tot = Ref(K16, ref.S.sum(0, keepdim=True), ref.F.sum(0, keepdim=True), ref.K64.sum(0, keepdim=True),
                  ref.free.any(0, keepdim=True), ref.eps)
        return check_K(K.view(1, E, E), tot, "row", name, extra=extra, bias=False)
    extra = None
    K16 = None
    if beta:
        K16 = ref.K16 + beta * old
        extra = 2 * U * (beta * old.abs() + K16.abs())
    return check_K(K, ref, "row", name, extra=extra, K16=K16, bias=False)


# ------------------------------------------------------------------------------- (a) the row kernel on constructed blocks
@gpu
@pytest.mark.parametrize("E", E_LIST)
def test_row_kernel_sweep(dev, E):
    """norm_kernel_matrices on constructed blocks: every eps the dispatch accepts (trailing epochs, eps > E), Fisher in
    the kernel or done, a vector and a scalar layout, n2 rotating through the chunk / flush edges, self columns at 0,
    inside the ragged last chunk and past n2; then the full n2 sweep at one eps."""
    gen = torch.Generator().manual_seed(100 + E)
    k = 0
    for eps in accepted_eps(E):
        for fisher in (False, True):
            for layout in ("vec", "offset1"):
                n2 = N2_LIST[k % len(N2_LIST)]
                self_col0 = (-1, 0, max(n2 - 3, 0))[k % 3]
                k += 1
                run_row_case(dev, gen, E, n2, eps, fisher, layout, self_col0, what="sweep")
    eps = accepted_eps(E)[min(2, len(accepted_eps(E)) - 1)]
    for j, n2 in enumerate(N2_LIST):
        run_row_case(dev, gen, E, n2, eps, bool(j & 1), ("dense", "vec", "offset1")[j % 3], (-1, 0, max(n2 - 3, 0))[j % 3],
                     what="n2 sweep")


@gpu
def test_row_kernel_beta_layouts_and_sum(dev):
    """beta = 0 into a NaN-filled K, beta = 1 and 0.5 over old values, a K pointer off a 16-byte boundary (scalar
    writes), E*E % 4 != 0, sum_over_rows (fp32 atomics) with and without beta."""
    gen = torch.Generator().manual_seed(7)
    for E in (12, 24, 31, 40):
        for beta in (0.0, 1.0, 0.5):
            for misalign in (False, True):
                run_row_case(dev, gen, E, 300, 4, False, "vec", beta=beta, misalign=misalign, what="beta")
        for beta in (0.0, 1.0):
            run_row_case(dev, gen, E, 300, 4, True, "vec", nb=9, beta=beta, sum_rows=True, what="sum")


@gpu
def test_row_kernel_long_rows_bias(dev):
    """nb = 64, E = 32, n2 = 50 000: every warp runs ~196 chunks, 24 flushes of its MMA accumulators.  Element-wise
    bound and the mean signed error of the diagonal (truncation bias)."""
    gen = torch.Generator(device=dev).manual_seed(64)
    nb, E, n2, eps = 64, 32, 50000, 8
    x = (torch.randn((nb, E, n2), generator=gen, device=dev, dtype=torch.float64) * 0.45).float()
    K = engine.norm_kernel_matrices(x, eps, fisher_done=True)
    torch.cuda.synchronize()
    ref = Ref.of_block(x, eps, chunk=16)
    st = check_K(K, ref, "row", "long rows n2=50000")
    record("long_rows", bias=st["bias"], c_A=st["c_A"], rel64=st["rel64"])
    print("long rows: bias %.3g, c_A %.3g, rel64 %.3g" % (st["bias"], st["c_A"], st["rel64"]))
    check_bias(st, "row", "long rows n2=50000")


@gpu
def test_plain_syrk_and_simt(dev):
    """kernel_matrices (EPS = 0): tf32 operands rounded ties away, exact inputs, at E = 1 .. 64, vector and scalar
    layouts; k_syrk_simt at E = 65 and 96 (two pair blocks) against its worst-case chain bound."""
    gen = torch.Generator().manual_seed(11)
    for E in (1, 5, 16, 17, 32, 33, 64):
        for n2, layout in ((257, "vec"), (2049, "offset1"), (4129, "vec"), (33, "dense")):
            x = make_block(gen, 4, E, n2, raw=False, dev=dev)
            blk = place(x, layout, dev)
            K = engine.kernel_matrices(blk)
            torch.cuda.synchronize()
            z = tf32_rna(x.double())
            a = z.abs()
            ref = Ref(torch.einsum("iaj,ibj->iab", z, z), torch.einsum("iaj,ibj->iab", a, a), 0.0,
                      torch.einsum("iaj,ibj->iab", x.double(), x.double()))
            check_K(K, ref, "tf32", "plain E=%d n2=%d %s" % (E, n2, layout), bias=False)
    for E in (65, 96):
        for n2 in (1, 63, 300):
            x = make_block(gen, 3, E, n2, raw=False, dev=dev)
            K = engine.kernel_matrices(place(x, "offset1", dev)).double()
            torch.cuda.synchronize()
            z = x.double()
            want = torch.einsum("iaj,ibj->iab", z, z)
            lim = n2 * U * torch.einsum("iaj,ibj->iab", z.abs(), z.abs())
            assert torch.all((K - want).abs() <= lim), "simt E=%d n2=%d" % (E, n2)
            record("simt", frac_of_bound=float(((K - want).abs() / lim.clamp(min=1e-300)).max()))


# ------------------------------------------------------------------------------- (c) planted edges
@gpu
def test_planted_edges(dev):
    """A dead row gives K = 0 exactly; a dead column and a subject constant at a dyadic value give z = 0 exactly (K
    bit-identical to the block with those values replaced by another exact-zero pattern); |r| = 1 and 1 - ulp at the
    Fisher clamps; subjects with large mean / sigma (1 + m^2/var up to ~1e4)."""
    gen = torch.Generator().manual_seed(3)
    E, n2, eps, nb = 24, 700, 4, 6
    for layout in ("vec", "offset1"):
        x = make_block(gen, nb, E, n2, raw=False, dev=dev)
        x[0] = 0.0                                       # dead row
        x[1, :, 10] = 0.0                                # dead column
        x[2, 4:8, 40] = 0.375                            # constant subject, dyadic
        x[3, :8, 100:110] = 0.9 + 0.05 * x[3, :8, 100:110]
        x[3, 8:16, 200:210] = -0.5 + 0.02 * x[3, 8:16, 200:210]
        K = engine.norm_kernel_matrices(place(x, layout, dev), eps, fisher_done=True)
        y = x.clone()
        y[1, :, 10] = -0.75
        y[2, 4:8, 40] = 0.0
        K2 = engine.norm_kernel_matrices(place(y, layout, dev), eps, fisher_done=True)
        torch.cuda.synchronize()
        assert torch.all(K[0] == 0), "dead row"
        assert torch.equal(K[1:3], K2[1:3]), "dead column / constant subject are not exactly zero"
        check_K(K, Ref.of_block(x, eps), "row", "planted %s" % layout, bias=False)
        # Fisher in the kernel at the clamps
        r = make_block(gen, nb, E, n2, raw=True, dev=dev)
        one = 1 - 2.0 ** -24
        r[:, 0, 0:5] = torch.tensor([1.0, -1.0, one, -one, 1 - 2.0 ** -23])
        r[:, 5, 7] = 1.0
        r[:, 6, 7] = -one
        r[1, 8:12, 300] = torch.tensor([1.0, one, -1.0, -one])
        K = engine.norm_kernel_matrices(place(r, layout, dev), eps, fisher_done=False)
        torch.cuda.synchronize()
        check_K(K, Ref.of_block(r, eps, fisher=True), "row", "clamps %s" % layout, bias=False)


# ------------------------------------------------------------------------------- (b) stage 2 inside the pipelines
def _detile(flat, row_tiles, col_tiles, E):
    """[row_tiles][col_tiles][E][256][256] -> [row_tiles*256, E, col_tiles*256] (same dtype, on the device)."""
    a = flat[:row_tiles * col_tiles * E * 65536].view(row_tiles, col_tiles, E, 256, 256)
    return a.permute(0, 3, 2, 1, 4).reshape(row_tiles * 256, E, col_tiles * 256)


def _operand(V, T, E, dev, seed):
    raw, _ = synthetic.make_epochs(V, T, E, seed=seed)
    ep, T_e = engine.stack_epochs(raw, dev)
    return engine.pack_epochs(ep, T_e, "fp32")


PIPE_CASES = {
    # name: (E, eps list, flags)
    "f32_E12": (12, (1, 2, 4, 8, 16), 0),                                 # tiled fp32, R = 2
    "f32_E24": (24, (1, 2, 4, 8, 16, 32), 0),                             # tiled fp32, R = 4
    "f16_E20": (20, (1, 2, 4, 8, 16), _lib.FLAG_F16_INTERMEDIATE),        # fp16 block, R = 4
    "f16_E32": (32, (32,), _lib.FLAG_F16_INTERMEDIATE),
    "f16_E40": (40, (1, 2, 4, 8, 16, 32), _lib.FLAG_F16_INTERMEDIATE),    # fp16 block, R = 8
    "f16_E64": (64, (64,), _lib.FLAG_F16_INTERMEDIATE),
    "strided_E24": (24, (4, 8), _lib.FLAG_STRIDED_BLOCK),
    "pass2_E12": (12, (1, 4, 16), _lib.FLAG_FISHER_IN_PASS2),             # Fisher in the row kernel, R = 4
    "pass2_E40": (40, (2, 8, 64), _lib.FLAG_FISHER_IN_PASS2),             # R = 8
    "mask_self_E24": (24, (8,), _lib.FLAG_MASK_SELF),
}


@gpu
@pytest.mark.parametrize("case", sorted(PIPE_CASES))
def test_pipeline_row_pass(dev, case):
    """voxel_kernels, one pass: read the block the GEMM left in the workspace and check the kernels against the
    reference of that block (GEMM error excluded): tiled fp32 (R = 2, 4), tiled fp16 (R = 4, 8), strided, Fisher in the
    row kernel, the self column masked."""
    E, eps_list, flags = PIPE_CASES[case]
    V, T, start, nb = 700, 40, 77, 600
    op = _operand(V, T, E, dev, seed=50 + E)
    work = engine.Workspace(E, V, 768, dev)
    half = bool(flags & _lib.FLAG_F16_INTERMEDIATE)
    for eps in eps_list:
        work.buf.fill_(255)
        K = engine.voxel_kernels(op, op, start, nb, eps, flags=flags, work=work)
        torch.cuda.synchronize()
        if flags & _lib.FLAG_STRIDED_BLOCK:
            ld = -(-V // 32) * 32
            blk = work.buf.view(torch.float32)[:nb * E * ld].view(nb, E, ld)[..., :V]
        else:
            blk = _detile(work.buf.view(torch.float16 if half else torch.float32), -(-nb // 256), -(-V // 256), E)[:nb, :, :V]
        assert torch.isfinite(blk).all()
        sc = list(range(start, start + nb)) if flags & _lib.FLAG_MASK_SELF else None
        ref = Ref.of_block(blk, eps, fisher=bool(flags & _lib.FLAG_FISHER_IN_PASS2), self_cols=sc)
        check_K(K, ref, "row", "voxel_kernels %s eps=%d" % (case, eps))


SYM_CASES = {
    # name: (E list with eps lists, flags, pass rows n, V)
    "cols16": (((12, (1, 2, 4, 8)), (16, (16,))), 0, 256, 556),
    "pad32": (((12, (1, 2, 4, 8, 16)),), _lib.FLAG_COLS_PAD32, 256, 556),
    "cols": (((24, (1, 2, 4, 8, 16)), (32, (32,))), 0, 256, 556),
    "v2": (((24, (1, 2, 4, 8, 16)), (32, (32,))), _lib.FLAG_COLS_V2, 256, 556),
    "tma": (((24, (1, 2, 4, 8, 16)), (32, (32,))), _lib.FLAG_COLS_TMA, 256, 556),
    "tma_half": (((24, (1, 2, 4, 8, 16)), (32, (32,))), _lib.FLAG_COLS_TMA | _lib.FLAG_F16_INTERMEDIATE, 256, 556),
    "half": (((20, (1, 2, 4, 8, 16)), (32, (32,))), _lib.FLAG_F16_INTERMEDIATE, 256, 556),
    "wide": (((40, (1, 2, 4, 8, 16, 32)), (64, (64,))), _lib.FLAG_COLS_WIDE, 256, 556),
    "transposed": (((24, (1, 4, 8)),), _lib.FLAG_SYM_TRANSPOSED, 256, 556),
    "n1024_cols": (((24, (8,)),), 0, 1024, 1024 + 333),
    "n1280_cols16": (((16, (4,)),), 0, 1280, 1280 + 333),
    "n1280_v2": (((24, (4,)),), _lib.FLAG_COLS_V2, 1280, 1280 + 333),
    "n1280_wide": (((40, (8,)),), _lib.FLAG_COLS_WIDE, 1280, 1280 + 333),
    "n4096_cols16": (((16, (4,)),), 0, 4096, 4096 + 4314),           # 4 folds, more strips (135) than SMs
    "n4096_cols": (((24, (8,)),), 0, 4096, 4096 + 4314),
}


@gpu
@pytest.mark.parametrize("case", sorted(SYM_CASES))
def test_sym_column_pass(dev, case):
    """voxel_kernels_sym, start = 0, one pass of n < V rows: K[i] (i < n) from the row pass over block A, K[j] (j >= n)
    from the column pass over the same block (or the row pass over the transposed copy), both against the reference of
    the block read back from the workspace; ragged last strip (V - n = 300, 333, 4314 columns)."""
    Es, flags, n, V = SYM_CASES[case]
    T = 24
    half = bool(flags & _lib.FLAG_F16_INTERMEDIATE)
    transposed = bool(flags & _lib.FLAG_SYM_TRANSPOSED)
    for E, eps_list in Es:
        op = _operand(V, T, E, dev, seed=70 + E + n)
        for eps in eps_list:
            assert _lib.load().fcma_sym_uses_column_pass(_lib.PREC[op.precision], E, eps, flags) == (not transposed)
            work = engine.SymWorkspace.for_operand(op, n, eps, flags)
            work.buf.fill_(255)
            K = engine.voxel_kernels_sym(op, 0, n, eps, flags=flags, work=work)
            torch.cuda.synchronize()
            flat = work.buf.view(torch.float16 if half else torch.float32)
            nt, t256 = -(-n // 256), -(-V // 256)
            A = _detile(flat, nt, t256, E)[:n, :, :V]
            what = "sym %s E=%d eps=%d n=%d" % (case, E, eps, n)
            rows = Ref.of_block(A, eps)
            check_K(K[:n], rows, "row", what + " rows")
            if transposed:
                B = _detile(flat[nt * t256 * E * 65536:], t256 - nt, nt, E)[:V - n, :, :n]
                cols = Ref.of_block(B, eps)
                st = check_K(K[n:], cols, "row", what + " transposed copy")
            else:
                cols = Ref.of_block(A[:, :, n:], eps, dim=0)
                st = check_K(K[n:], cols, "cols", what + " columns")
                if n >= 1024:
                    check_bias(st, "cols", what)
