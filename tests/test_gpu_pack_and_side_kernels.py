"""Element-wise tests of the kernels that feed the correlation GEMM or sit beside it on public API paths: the operand
packer, the two z-score normalisers, the fp32 side GEMMs, the standalone within-subject normaliser and the decimal
shrink.  Each is compared with a plain reference of the same operation, computed in this file in numpy / fp64 or by the
C oracle (``oracle/fcma_oracle.c``), at the shapes and values where these kernels go wrong.

References and bounds
---------------------
* ``k_pack_operand`` planes, **bit for bit** (raw bit patterns, not values), emulated in numpy from the packer's input x
  (``normalize = 0``) or from ``epoch_normalize_`` of it (``normalize = 1``, exact by the next item):
  bf16 ``hi = RN_bf16(x)``, ``lo = RN_bf16(x - hi)``; tf32 ``hi = RNA_tf32(x)`` (``cvt.rna``: ``(bits + 0x1000) &
  ~0x1fff``, ties away, low 13 bits zero), ``lo = RNA_tf32(x - hi)``; fp16x3 ``hi = RN_fp16(64 x)``, ``lo = RN_fp16(64 x
  - hi)``; single-plane modes store hi only.  Rows ``t in [T_e, Kp)`` are +0 in every plane; the source holds NaN there,
  so a packer that reads them fails.  Layout ``[planes][E][V][Kp]``, the planes' bytes rounded up to 256, then the
  ``[E][V]`` fp32 diagonal; ``Kp`` and the byte count come from ``fcma_operand_kp`` / ``fcma_operand_bytes``.
* the packer's diagonal, ``k_gemm_nt`` and ``k_corr_simt``, **bit for bit**: each is a sequential fp32 FMA chain over
  t (k), restated by ``orc.corr_block(..., f64=False)``.  The kernels' zero-padded steps ``fmaf(0, b, acc)`` may turn
  -0 into +0, which ``np.array_equal`` treats as equal.
* ``pack_epochs(normalize=True)`` against ``pack_epochs(epoch_normalize_(x))``: **bit for bit** (same arithmetic).
* ``k_epoch_normalize`` / ``k_row_normalize`` against the fp64 z-score of the float32 input (population sigma over the
  n = T_e (D) values, then ``/ sqrt(n)``).  The kernels: fp64 sum, mean rounded to fp32 (|dm| <= u |m|, u = 2^-24);
  d = fp32(x - mean) (relative u) summed squared in fp64, sigma rounded to fp32 (sigma relative 2u; the shifted mean
  adds dm^2 / 2 sigma^2 <= (u |m| / sigma)^2 / 2); then ``scale = 1 / (sigma sqrt(n))`` with three roundings and
  ``(x - mean) * scale`` with two (k_row_normalize: ``(x - mean) / sigma / sqrt(n)``, one rounding fewer).  So the
  result is the exact z of the rounded mean to relative 7u, and the rounded mean moves z by ``u |m| / (sigma sqrt(n))``:
  ``|dz| <= 2 u ((7 + |m| / sigma) |z| + |m| / (sigma sqrt(n))) + 2^-50 sqrt(n) (1 + |m| / sigma)``.  The factor 2
  covers second-order products of the (1 + delta) factors (the shifted-mean term is below ``u |m| / sigma |z| / 32``
  where it is first-order, see next); the last term is the fp64 sums (n 2^-53 of sum |x|).  Where ``u |m| / sigma >=
  1/16`` no first-order bound exists (scipy's fp32 z-score is no better); such values are exempt, and the tests assert
  that their generic data has none.  sigma == 0 (constant) gives exactly 0; a NaN gives 0 (packer / epoch normaliser,
  ``nan_to_num`` of a NaN mean), and 0 or NaN by ``nan_to_zero`` in the row normaliser.
* ``compute_correlation`` against fp64 ``corrcoef`` of the float32 inputs: ``tol_r`` of test_gpu_corr_gemm.py
  (``max(1e-6, 2 e32)``, e32 = error of the fp32 chain at the shape) plus the propagated normaliser bound
  ``sum_t (B_it |z_jt| + |z_it| B_jt + B_it B_jt)``, B the per-element bound above.
* ``k_within_subject_norm`` against ``orc.within_subject_norm`` (fp32 restatement of fcma_extension.cc:52-84) with
  ``norm_tolerance`` of test_gpu_parity.py (CUDA vs glibc ``logf``, amplified by the ``E[x^2] - m^2`` cancellation),
  most values bit-identical, trailing epochs ``E % eps`` untouched bit for bit.
* ``k_shrink_kernels`` against Python: ``nd = len(str(int(K00)))`` and ``K * float32(10 ** (2 - nd))`` for nd > 2,
  **bit for bit**; NaN and +-inf (where the reference's ``int()`` raises) give nd = 1 and leave K untouched.

Coverage
--------
| kernel / instantiation                   | covered by                                                                  |
|------------------------------------------|-----------------------------------------------------------------------------|
| ``k_pack_operand<0, 1>`` (bf16)           | test_pack_operand_bit_exact[bf16], test_pack_range_keeps_other_voxels[bf16]  |
| ``k_pack_operand<0, 2>`` (bf16x3)         | test_pack_operand_bit_exact[bf16x3], test_pack_range_keeps_other_voxels[bf16x3] |
| ``k_pack_operand<1, 1>`` (tf32)           | test_pack_operand_bit_exact[tf32], test_pack_range_keeps_other_voxels[tf32]  |
| ``k_pack_operand<1, 2>`` (tf32x3)         | test_pack_operand_bit_exact[tf32x3], test_pack_range_keeps_other_voxels[tf32x3], test_grouped_packing_matches_one_shot_pack[tf32x3] |
| ``k_pack_operand<2, 2>`` (fp16x3)         | test_pack_operand_bit_exact[fp16x3], test_pack_range_keeps_other_voxels[fp16x3], test_grouped_packing_matches_one_shot_pack[fp16x3] |
| each of the five, ``normalize`` = 1       | test_pack_operand_bit_exact and test_pack_range_keeps_other_voxels (normalize = 1 half of every case) |
| ``k_epoch_normalize``                     | test_pack_operand_bit_exact (exact agreement), test_epoch_normalize_against_fp64 |
| ``fcma_epoch_normalize`` T_e validation   | test_epoch_normalize_rejects_long_epochs                                     |
| ``k_row_normalize``                       | test_row_normalize_against_fp64                                              |
| ``util.compute_correlation``              | test_compute_correlation_against_fp64                                        |
| ``k_gemm_nt`` (+ the cython_blas shim)    | test_gemm_nt_bit_exact, test_side_gemm_argument_checks                       |
| ``k_corr_simt`` (+ the cython_blas shims) | test_corr_simt_bit_exact                                                     |
| ``k_within_subject_norm``                 | test_within_subject_norm_at_scale                                            |
| ``k_shrink_kernels``                      | test_shrink_digits_and_factor_bit_exact; CPU: test_pow10_table_...          |

CPU self-tests (no ``gpu`` mark): the rounding emulations on hand-built ties and the power-of-ten table of
``k_shrink_kernels`` against Python integers.
"""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

from brainiak_b200 import _lib

U = 2.0 ** -24
NAN = float("nan")
PRECS = ("bf16", "bf16x3", "tf32", "tf32x3", "fp16x3")
SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "brainiak_b200", "csrc", "fcma_b200.cu")


@pytest.fixture(scope="module")
def dev():
    assert _lib.device_count() > 0, "no sm_90 device"
    return torch.device("cuda:0")


# ------------------------------------------------------------------------------- rounding emulations (numpy)
def bf16_rn(x):
    """float32 -> bf16 bit patterns (int16), round to nearest even."""
    b = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16).view(np.int16)


def bf16_value(bits):
    return (np.asarray(bits).view(np.uint16).astype(np.uint32) << 16).view(np.float32)


def tf32_rna(x):
    """float32 -> tf32 bit patterns (int32, low 13 bits zero), round to nearest, ties away (cvt.rna.tf32.f32)."""
    b = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return (((b + 0x1000) & ~np.uint64(0x1FFF)) & 0xFFFFFFFF).astype(np.uint32).view(np.int32)


def fp16_rn(x):
    """float32 -> fp16 bit patterns (int16), round to nearest even (subnormals included)."""
    return np.asarray(x, np.float32).astype(np.float16).view(np.int16)


def split_planes(x, prec):
    """The packer's planes of float32 values x, as bit patterns: [hi] or [hi, lo]."""
    x = np.asarray(x, np.float32)
    if prec.startswith("bf16"):
        hi = bf16_rn(x)
        lo = bf16_rn(x - bf16_value(hi))
    elif prec.startswith("tf32"):
        hi = tf32_rna(x)
        lo = tf32_rna(x - hi.view(np.float32))
    else:
        xs = x * np.float32(64.0)                       # FCMA_FP16_SCALE: exact
        hi = fp16_rn(xs)
        lo = fp16_rn(xs - hi.view(np.float16).astype(np.float32))
    return [hi] if prec in ("bf16", "tf32") else [hi, lo]


def pow10_table():
    """kPow10Ceil of k_shrink_kernels, read from the source."""
    src = open(SRC).read()
    body = re.search(r"kPow10Ceil\[38\]\s*=\s*\{([^}]*)\}", src).group(1)
    return [float.fromhex(s.strip().rstrip("f")) for s in body.split(",") if s.strip()]


def digits_by_table(f, table):
    """k_shrink_kernels' digit count of a finite float32 f."""
    a = abs(float(f))
    return 1 + sum(a >= t for t in table) + (1 if f <= -1.0 else 0)


def zscore64(x, axis):
    """fp64 z-score of float32 data along `axis` (population sigma), divided by sqrt(n); also the mean, sigma, n."""
    x = np.asarray(x, np.float64)
    n = x.shape[axis]
    m = x.mean(axis, keepdims=True)
    sd = np.sqrt(((x - m) ** 2).mean(axis, keepdims=True))
    with np.errstate(invalid="ignore", divide="ignore"):
        z = (x - m) / sd / math.sqrt(n)
    return z, m, sd, n


def z_bound(z, m, sd, n):
    """Per-element bound of the fp32 normalisers (module docstring) and the mask of values without one."""
    with np.errstate(invalid="ignore", divide="ignore"):
        ratio = np.abs(m) / sd
    b = 2 * U * ((7 + ratio) * np.abs(z) + ratio / math.sqrt(n)) + 2.0 ** -50 * math.sqrt(n) * (1 + ratio)
    return b, np.broadcast_to(U * ratio >= 1.0 / 16, z.shape)


# ------------------------------------------------------------------------------- CPU self-tests of the helpers
def test_rounding_emulations_on_hand_built_ties():
    f = np.float32
    # bf16: 7 fraction bits; 1 + 2^-8 is the midpoint of 1 and 1 + 2^-7 -> even (1.0); 1 + 3 * 2^-8 -> 1 + 2^-6
    assert bf16_rn(f(1 + 2 ** -8)).view(np.uint16) == 0x3F80
    assert bf16_rn(f(1 + 3 * 2 ** -8)).view(np.uint16) == 0x3F82
    assert bf16_rn(f(-(1 + 2 ** -8))).view(np.uint16) == 0xBF80
    assert bf16_rn(f(1 + 2 ** -8 + 2 ** -23)).view(np.uint16) == 0x3F81
    assert bf16_rn(f(-0.0)).view(np.uint16) == 0x8000
    # tf32: 10 fraction bits, ties away from zero
    assert tf32_rna(f(1 + 2 ** -11)).view(np.uint32) == 0x3F802000
    assert tf32_rna(f(-(1 + 2 ** -11))).view(np.uint32) == 0xBF802000
    assert tf32_rna(f(1 + 2 ** -11 - 2 ** -23)).view(np.uint32) == 0x3F800000
    assert tf32_rna(f(1 + 3 * 2 ** -11)).view(np.uint32) == 0x3F804000
    # fp16: even ties, normal and subnormal (2^-25 is the midpoint of 0 and the smallest subnormal 2^-24)
    assert fp16_rn(f(1 + 2 ** -11)).view(np.uint16) == 0x3C00
    assert fp16_rn(f(1 + 3 * 2 ** -11)).view(np.uint16) == 0x3C02
    assert fp16_rn(f(-(1 + 3 * 2 ** -11))).view(np.uint16) == 0xBC02
    assert fp16_rn(f(2 ** -25)).view(np.uint16) == 0x0000
    assert fp16_rn(f(3 * 2 ** -25)).view(np.uint16) == 0x0002
    assert fp16_rn(f(65504.0)).view(np.uint16) == 0x7BFF
    # splits: hi + lo reproduces x where the format pair holds it; lo-plane ties follow each format's rule
    x = f(1 + 2 ** -12 + 2 ** -23)                        # tf32: hi = 1, lo = 2^-12 (1 + 2^-11), a tie -> away
    hi, lo = split_planes(x, "tf32x3")
    assert hi.view(np.uint32) == 0x3F800000 and lo.view(np.float32) == f(2 ** -12 * (1 + 2 ** -10))
    x = f(1 + 2 ** -9 + 2 ** -17)                         # bf16: hi = 1, lo = 2^-9 (1 + 2^-8), a tie -> even
    hi, lo = split_planes(x, "bf16x3")
    assert bf16_value(hi) == 1 and bf16_value(lo) == f(2 ** -9)
    rng = np.random.RandomState(0)
    v = (rng.randn(1000) * 0.3).astype(np.float32)
    hi, lo = split_planes(v, "fp16x3")
    back = hi.view(np.float16).astype(np.float64) + lo.view(np.float16).astype(np.float64)
    assert np.all(np.abs(back / 64 - v) <= 2.0 ** -21 * np.abs(v) + 2.0 ** -31)
    for p in PRECS:
        assert len(split_planes(v, p)) == (1 if p in ("bf16", "tf32") else 2)


def test_pow10_table_matches_python_integers():
    table = pow10_table()
    assert len(table) == 38
    for k, t in enumerate(table, start=1):
        f = np.float32(t)
        assert float(f) == t, "entry %d is not a float32" % k
        below = np.nextafter(f, np.float32(0))
        assert int(t) >= 10 ** k > int(below), "entry %d is not the smallest float32 >= 10^%d" % (k, k)
    # the digit rule of the kernel against len(str(int(f))) over every power of ten and its neighbours
    vals = [0.0, -0.0, 0.5, -0.5, 0.999, -1.0, 1.0, 9.99, -9.99, 3.4028235e38, -3.4028235e38, 9e18, 1e19]
    for k in range(0, 39):
        p = np.float32(10.0 ** k)
        vals += [p, np.nextafter(p, np.float32(0)), np.nextafter(p, np.float32(np.inf))]
    vals += [-v for v in vals]
    for v in vals:
        v = np.float32(v)
        if np.isfinite(v):
            assert digits_by_table(v, table) == len(str(int(v))), v


def test_z_bound_helper():
    """The fp64 reference and its bound on a hand-checked case; a constant column has sigma 0 and is not bounded."""
    x = np.array([[1.0, 2.0], [3.0, 2.0]], np.float32)
    z, m, sd, n = zscore64(x, 0)
    assert np.allclose(z[:, 0], [-1 / math.sqrt(2), 1 / math.sqrt(2)]) and np.isnan(z[:, 1]).all()
    b, free = z_bound(z[:, :1], m[:, :1], sd[:, :1], n)
    assert np.all(b > 0) and np.all(b < 1e-5) and not free.any()


# ------------------------------------------------------------------------------- operand readback
def read_operand(op):
    """(planes [P, E, V, Kp] int16 / int32 bit patterns, diagonal [E, V] float32, Kp) of a PackedOperand."""
    lib = _lib.load()
    code = _lib.PREC[op.precision]
    Kp = lib.fcma_operand_kp(code, op.T)
    nbytes = lib.fcma_operand_bytes(code, op.E, op.T, op.V)
    P = lib.fcma_operand_planes(code)
    esz = 4 if op.precision.startswith("tf32") else 2
    raw = op.buf[:nbytes].cpu().numpy()
    planes = raw[:P * op.E * op.V * Kp * esz].view(np.int32 if esz == 4 else np.int16).reshape(P, op.E, op.V, Kp)
    diag = raw[nbytes - op.E * op.V * 4:].view(np.float32).reshape(op.E, op.V)
    return planes, diag, Kp


def expected_operand(x, T_e, prec, Kp):
    """Planes and diagonal the packer must write for the float32 epochs x [E, T, V] (rows >= T_e[e] ignored)."""
    from oracle import fcma_oracle as orc
    E, _, V = x.shape
    P = 1 if prec in ("bf16", "tf32") else 2
    planes = np.zeros((P, E, V, Kp), np.int32 if prec.startswith("tf32") else np.int16)
    for e in range(E):
        for p, pl in enumerate(split_planes(x[e, :T_e[e]].T, prec)):
            planes[p, e, :, :T_e[e]] = pl
    diag = np.empty((E, V), np.float32)
    for c0 in range(0, V, 64):
        c1 = min(V, c0 + 64)
        chunk = [np.ascontiguousarray(x[e, :T_e[e], c0:c1]) for e in range(E)]
        r = orc.corr_block(chunk, None, 0, c1 - c0, f64=False)
        diag[:, c0:c1] = r[np.arange(c1 - c0), :, np.arange(c1 - c0)].T
    return planes, diag


def planted_values():
    """Rounding ties of each format (hi and lo plane, both signs), +-0, fp16x3 values whose lo plane is subnormal, and
    |x| just under 65504 / 64."""
    f = np.float32
    ties = [1 + 2 ** -8, 1 + 3 * 2 ** -8, 1 + 2 ** -9 + 2 ** -17,            # bf16 hi / lo
            1 + 2 ** -11, 1 + 3 * 2 ** -11, 1 + 2 ** -12 + 2 ** -23,         # tf32 hi / lo
            (1 + 2 ** -11) / 64, (1 + 3 * 2 ** -11) / 64, 0.375 + 2 ** -13]  # fp16 (x 64) hi ties
    vals = ties + [-t for t in ties] + [0.0, -0.0]
    rng = np.random.RandomState(7)
    for k in range(9, 17):
        vals += list(rng.randn(3) * 2.0 ** -k)
    top = np.nextafter(f(65504.0 / 64), f(0))
    vals += [top, -top, f(1023.0)]
    return np.array(vals, np.float32)


def pack_case_data(T, V, T_e, seed, normalize):
    """[E, T, V] float32 with NaN in the rows t >= T_e[e]; raw data carries the planted values in epoch 0, data to be
    normalised has a mean offset, a constant voxel, a voxel with a NaN and a voxel at scale 1e-30."""
    rng = np.random.RandomState(seed)
    E = len(T_e)
    x = (rng.randn(E, T, V) * 0.3).astype(np.float32)
    if normalize:
        x = (x * 3 + 5).astype(np.float32)
        if V > 3:
            x[:, :, 1] = 0.7
            x[:, 0, 2] = NAN
            x[:, :, 3] = (rng.randn(E, T) * 1e-30).astype(np.float32)
    else:
        flat = x[0].reshape(-1)
        pv = planted_values()
        k = min(flat.size, pv.size)
        flat[:k] = pv[:k]
    for e in range(E):
        x[e, T_e[e]:] = NAN
    return x


def _pack_cases():
    cases = []
    for T in (1, 7, 8, 9, 15, 16, 17, 63, 64, 65, 127, 128, 129, 200, 500):
        lens = [T, 1, max(1, (T + 1) // 2)] if T > 1 else [1, 1]
        cases.append((T, 33, lens))
    for V in (1, 31, 32, 33):
        cases.append((65, V, [65, 64, 63]))
    cases.append((129, 1000, [129, 65, 64, 63, 1]))
    cases.append((500, 1000, [500, 1]))
    return cases


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECS)
def test_pack_operand_bit_exact(dev, prec):
    """k_pack_operand planes, padding rows and diagonal bit for bit, normalize = 0 and 1, T across the 8 / 16 Kp rounding
    and the 64-row slab loop, ragged epochs (1 and lengths on both sides of 64), V across the 32-voxel blocks; the fused
    normaliser equals pack(epoch_normalize_(x)) bit for bit, and epoch_normalize_ leaves the rows t >= T_e alone."""
    from brainiak_b200.fcma import engine
    for T, V, lens in _pack_cases():
        for normalize in (False, True):
            what = "%s T=%d V=%d T_e=%s normalize=%d" % (prec, T, V, lens, normalize)
            x = pack_case_data(T, V, lens, T * 131 + V, normalize)
            ep = torch.from_numpy(x).to(dev)
            op = engine.pack_epochs(ep, lens, prec, normalize=normalize)
            planes, diag, Kp = read_operand(op)
            if normalize:
                xn = engine.epoch_normalize_(ep.clone(), lens)
                op2 = engine.pack_epochs(xn, lens, prec)
                planes2, diag2, _ = read_operand(op2)
                assert np.array_equal(planes, planes2), what + ": fused normaliser != k_epoch_normalize (planes)"
                assert np.array_equal(diag.view(np.int32), diag2.view(np.int32)), what + ": fused normaliser diagonal"
                src = xn.cpu().numpy()
                for e, t in enumerate(lens):
                    assert np.isnan(src[e, t:]).all(), what + ": epoch_normalize_ wrote rows past T_e"
                if V > 3:
                    assert not src[:, :, 1:3][np.arange(T)[None, :] < np.array(lens)[:, None]].any(), \
                        what + ": constant / NaN voxel not exactly 0"
            else:
                src = x
            want_p, want_d = expected_operand(src, lens, prec, Kp)
            if not np.array_equal(planes, want_p):
                bad = np.argwhere(planes != want_p)[:5]
                pytest.fail("%s: %d plane elements differ, e.g. [p, e, v, t] %s: got %s, want %s (x %s)" % (
                    what, int((planes != want_p).sum()), bad.tolist(), planes[tuple(bad.T)].tolist(),
                    want_p[tuple(bad.T)].tolist(), src[bad[:, 1], np.minimum(bad[:, 3], T - 1), bad[:, 2]].tolist()))
            if not np.array_equal(diag, want_d):
                bad = np.argwhere(diag != want_d)[:5]
                pytest.fail("%s: diagonal differs at [e, v] %s: got %s, want %s" % (
                    what, bad.tolist(), diag[tuple(bad.T)].tolist(), want_d[tuple(bad.T)].tolist()))
            if prec.startswith("tf32"):
                assert not (planes & 0x1FFF).any(), what + ": tf32 plane with low mantissa bits set"


def _patterned(op_like, pattern=0xA5):
    from brainiak_b200.fcma import engine
    buf = torch.full_like(op_like.buf, pattern)
    return engine.PackedOperand(buf, op_like.E, op_like.T, op_like.V, op_like.precision, op_like.T_e)


def _expect_voxels(full, pattern_op, v0):
    """Bytes of `pattern_op` with the voxels [v0, V) of `full` (planes and diagonal) written in."""
    lib = _lib.load()
    code = _lib.PREC[full.precision]
    E, V = full.E, full.V
    Kp = lib.fcma_operand_kp(code, full.T)
    nbytes = lib.fcma_operand_bytes(code, E, full.T, V)
    P = lib.fcma_operand_planes(code)
    esz = 4 if full.precision.startswith("tf32") else 2
    src = full.buf[:nbytes].cpu().numpy()
    out = pattern_op.buf[:nbytes].cpu().numpy().copy()
    pb = P * E * V * Kp * esz
    o4 = out[:pb].reshape(P, E, V, Kp * esz)
    o4[:, :, v0:] = src[:pb].reshape(P, E, V, Kp * esz)[:, :, v0:]
    od = out[nbytes - E * V * 4:].reshape(E, V, 4)
    od[:, v0:] = src[nbytes - E * V * 4:].reshape(E, V, 4)[:, v0:]
    return out, nbytes


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECS)
def test_pack_range_keeps_other_voxels(dev, prec):
    """fcma_pack_operand_range into a byte-pattern buffer: exactly the voxels [v_begin, V) are written, in every plane and
    in the diagonal, bit-identical to a one-shot pack; every other byte keeps the pattern."""
    from brainiak_b200.fcma import engine
    V, T, lens = 300, 40, [40, 17, 33]
    for normalize in (False, True):
        x = pack_case_data(T, V, lens, 99, normalize)
        ep = torch.from_numpy(x).to(dev)
        full = engine.pack_epochs(ep, lens, prec, normalize=normalize)
        for vb in (1, 31, 32, 33, 255, 256, V - 1):
            op = _patterned(full)
            engine.pack_epochs(ep, lens, prec, normalize=normalize, v_begin=vb, out=op)
            want, nbytes = _expect_voxels(full, _patterned(full), vb)
            got = op.buf.cpu().numpy()
            assert np.array_equal(got[:nbytes], want), "%s normalize=%d v_begin=%d: %d bytes differ" % (
                prec, normalize, vb, int((got[:nbytes] != want).sum()))
            assert (got[nbytes:] == 0xA5).all()


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ("fp16x3", "tf32x3"))
def test_grouped_packing_matches_one_shot_pack(dev, prec):
    """voxel_kernels_sym_grouped packs epoch group by group (epoch sub-range launches) into the operand: afterwards the
    buffer equals a one-shot pack_epochs bit for bit over the voxels [start, V) it owns; everything else keeps the
    pattern."""
    from brainiak_b200.fcma import engine, synthetic
    V, T, E, eps = 1100, 40, 8, 4
    raw, _ = synthetic.make_epochs(V, T, E, seed=555)
    ep, T_e = engine.stack_epochs(raw, dev)
    full = engine.pack_epochs(ep, T_e, prec)
    groups = [(0, 2), (2, 2), (4, 2), (6, 2)]
    for start in (0, 512):
        op = _patterned(full)
        engine.voxel_kernels_sym_grouped(ep, op, start, V - start, eps, groups, [None] * 4, flags=_lib.FLAG_MASK_SELF)
        torch.cuda.synchronize()
        want, nbytes = _expect_voxels(full, _patterned(full), start)
        got = op.buf.cpu().numpy()[:nbytes]
        assert np.array_equal(got, want), "%s start=%d: %d bytes differ" % (prec, start, int((got != want).sum()))


# ------------------------------------------------------------------------------- k_epoch_normalize
def _check_z(got, x, axis, what, nan_to_zero=True):
    """got (float32) against the fp64 z-score of x along axis; sigma == 0 or NaN lanes must be exactly 0 (NaN when
    not nan_to_zero).  Returns the largest error / bound."""
    z, m, sd, n = zscore64(x, axis)
    b, free = z_bound(z, m, sd, n)
    lane_ok = np.broadcast_to((sd > 0) & np.isfinite(sd), z.shape)
    assert not free[lane_ok].any(), "%s: generic data without a first-order bound" % what
    got = np.asarray(got, np.float64)
    dead = ~lane_ok
    if nan_to_zero:
        assert np.all(got[dead] == 0), "%s: constant / NaN lanes not exactly 0" % what
    else:
        assert np.isnan(got[dead]).all(), "%s: constant / NaN lanes not NaN" % what
    err = np.abs(got - z)
    bad = lane_ok & ~(err <= b)
    if bad.any():
        idx = np.argwhere(bad)[:5]
        pytest.fail("%s: %d of %d beyond the bound, e.g. %s: got %s, want %s, bound %s" % (
            what, int(bad.sum()), int(lane_ok.sum()), idx.tolist(), got[tuple(idx.T)].tolist(),
            z[tuple(idx.T)].tolist(), b[tuple(idx.T)].tolist()))
    return float(np.max(err[lane_ok] / b[lane_ok], initial=0.0))


@pytest.mark.gpu
def test_epoch_normalize_against_fp64(dev):
    """epoch_normalize_ element by element against the fp64 z-score of the float32 input over T_e (preprocessing.py:
    80-84): ragged epochs with a NaN sentinel in the rows t >= T_e (left untouched), a pitched layout through the ABI
    (ld > V, pad columns NaN and untouched), dead, constant and NaN voxels, a mean far from 0, a voxel at 1e-30."""
    from brainiak_b200.fcma import engine
    rng = np.random.RandomState(11)
    E, T, V, ld = 5, 203, 700, 737
    lens = [203, 1, 64, 65, 130]
    x = (rng.randn(E, T, V) * 2 + 20).astype(np.float32)
    x[:, :, 5] = 0.0
    x[:, :, 6] = 3.25
    x[:, 7, 7] = NAN
    x[:, :, 8] = (rng.randn(E, T) * 1e-30).astype(np.float32)
    x[:, :, 9] = (rng.randn(E, T) * 1e3 - 4e3).astype(np.float32)
    for e in range(E):
        x[e, lens[e]:] = NAN
    worst = 0.0
    for pitched in (False, True):
        if pitched:
            buf = torch.full((E, T, ld), NAN, device=dev)
            buf[:, :, :V] = torch.from_numpy(x).to(dev)
            te = (ctypes.c_int * E)(*lens)
            lib = _lib.load()
            _lib.check(lib.fcma_epoch_normalize(ctypes.c_void_p(buf.data_ptr()), E, T, V, ld, te,
                                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
            out = buf.cpu().numpy()
            assert np.isnan(out[:, :, V:]).all(), "write into the pad columns"
            out = out[:, :, :V]
        else:
            out = engine.epoch_normalize_(torch.from_numpy(x).to(dev), lens).cpu().numpy()
        for e, t in enumerate(lens):
            assert np.isnan(out[e, t:]).all(), "pitched=%d: epoch %d rows >= T_e written" % (pitched, e)
            worst = max(worst, _check_z(out[e, :t], x[e, :t], 0, "pitched=%d epoch %d" % (pitched, e)))
    print("k_epoch_normalize: max |dz| / bound = %.3f" % worst)


@pytest.mark.gpu
def test_epoch_normalize_rejects_long_epochs(dev):
    """T_e[e] outside (0, T] is refused before any kernel runs (a longer epoch would read the next epoch's rows, or
    past the allocation for the last one); the data is left as it was."""
    from brainiak_b200.fcma import engine
    lib = _lib.load()
    ep = torch.randn(3, 16, 40, device=dev)
    before = ep.clone()
    for lens in ([16, 16, 17], [17, 16, 16], [16, 0, 16], [16, -1, 8]):
        n0 = lib.fcma_launch_count()
        with pytest.raises(ValueError, match="outside"):
            engine.epoch_normalize_(ep, lens)
        assert lib.fcma_launch_count() == n0
    torch.cuda.synchronize()
    assert torch.equal(ep, before)


# ------------------------------------------------------------------------------- k_row_normalize, compute_correlation
@pytest.mark.gpu
def test_row_normalize_against_fp64(dev):
    """row_normalize_ (util.py:32-60: zscore(axis=1, ddof=0), nan -> 0, / sqrt(D)) element by element: D across the
    256-thread reduction, R across the 148 * 8 = 1 184-row grid cap (grid-stride loop), a row pitch ld > D with the pad
    untouched, constant rows and rows with a NaN (0 with nan_to_zero, NaN without)."""
    from brainiak_b200.fcma import engine
    rng = np.random.RandomState(12)
    worst = 0.0
    cases = [(D, R) for D in (1, 2, 255, 256, 257) for R in (1, 1184, 1185, 3000)] + [(4097, 1), (4097, 1185)]
    for D, R in cases:
        x = (rng.randn(R, D) * 1.5 - 3).astype(np.float32)
        if R > 3:
            x[1] = 3.7
            x[2, D // 2] = NAN
            x[3] *= np.float32(1e-20)
        for nan_to_zero in (True, False):
            ld = D + 5
            buf = torch.full((R, ld), NAN, device=dev)
            buf[:, :D] = torch.from_numpy(x).to(dev)
            engine.row_normalize_(buf[:, :D], nan_to_zero=nan_to_zero)
            out = buf.cpu().numpy()
            assert np.isnan(out[:, D:]).all(), "D=%d R=%d: write into the pad" % (D, R)
            worst = max(worst, _check_z(out[:, :D], x, 1, "D=%d R=%d nan_to_zero=%d" % (D, R, nan_to_zero),
                                        nan_to_zero))
    print("k_row_normalize: max |dz| / bound = %.3f" % worst)


@pytest.mark.gpu
def test_compute_correlation_against_fp64(dev):
    """util.compute_correlation against the fp64 corrcoef of the float32 inputs, element by element: r1, r2 across the
    256-row tiles, D across the 16 / 64 k-block edges up to 2 000; the self case (diagonal within tol_r of 1, the rest
    bit-identical to the two-argument call on a copy); return_nans=True (exactly the NaN rows and columns are NaN)."""
    from brainiak_b200.fcma import util
    from oracle import fcma_oracle as orc
    rng = np.random.RandomState(13)
    shapes = [(1, 255, 2), (255, 256, 15), (256, 257, 16), (257, 1, 17), (600, 255, 63), (1, 600, 64),
              (257, 256, 65), (600, 600, 2000), (255, 257, 1000)]
    for r1, r2, D in shapes:
        m1 = (rng.randn(r1, D) * 2 + 1).astype(np.float32)
        m2 = (rng.randn(r2, D) * 0.5 - 2).astype(np.float32)
        if r1 > 2:
            m1[1] = 0.25                                     # constant row -> 0 correlations
        got = util.compute_correlation(m1, m2).astype(np.float64)
        z1, _, _, _ = zscore64(m1, 1)
        z2, _, _, _ = zscore64(m2, 1)
        z1, z2 = np.nan_to_num(z1), np.nan_to_num(z2)
        b1 = z_bound(*zscore64(m1, 1))[0]
        b2 = z_bound(*zscore64(m2, 1))[0]
        b1, b2 = (np.where(np.isfinite(b), b, 0.0) for b in (b1, b2))    # constant rows: exactly 0
        r64 = z1 @ z2.T
        e1 = [np.ascontiguousarray(z1.T, np.float32)]
        e2 = [np.ascontiguousarray(z2.T, np.float32)]
        e32 = float(np.max(np.abs(orc.corr_block(e1, e2, 0, r1, f64=False)[:, 0, :] -
                                  orc.corr_block(e1, e2, 0, r1, f64=True)[:, 0, :])))
        tol_r = max(1e-6, 2 * e32)
        prop = b1 @ np.abs(z2).T + np.abs(z1) @ b2.T + b1 @ b2.T
        err = np.abs(got - r64)
        bad = err > tol_r + prop
        assert not bad.any(), "r1=%d r2=%d D=%d: %d bad, max err %.3g (tol_r %.3g)" % (
            r1, r2, D, int(bad.sum()), err.max(), tol_r)
    # the self case
    m = (rng.randn(300, 129) * 3).astype(np.float32)
    s = util.compute_correlation(m, m)
    two = util.compute_correlation(m, m.copy())
    off = ~np.eye(300, dtype=bool)
    assert np.array_equal(s[off], two[off])
    z, _, _, _ = zscore64(m, 1)
    e1 = [np.ascontiguousarray(z.T, np.float32)]
    tol_r = max(1e-6, 2 * float(np.max(np.abs(orc.corr_block(e1, None, 0, 300, f64=False)[:, 0, :] -
                                              orc.corr_block(e1, None, 0, 300, f64=True)[:, 0, :]))))
    assert np.all(np.abs(np.diag(s).astype(np.float64) - 1) <= tol_r)
    # return_nans: the rows / columns of NaN or constant rows are NaN, nothing else
    m1 = (rng.randn(70, 45)).astype(np.float32)
    m2 = (rng.randn(80, 45)).astype(np.float32)
    m1[3, 7] = NAN
    m1[10] = 2.0
    m2[5] = -1.0
    m2[60, 0] = NAN
    got = util.compute_correlation(m1, m2, return_nans=True)
    want = np.zeros(got.shape, bool)
    want[[3, 10], :] = True
    want[:, [5, 60]] = True
    assert np.array_equal(np.isnan(got), want)


# ------------------------------------------------------------------------------- k_gemm_nt, k_corr_simt
@pytest.mark.gpu
def test_gemm_nt_bit_exact(dev):
    """gemm_nt (C = A B^T, fp32 FFMA) bit for bit against the sequential FMA chain over k: M, N across the 64-row /
    column tiles, K across the 16-wide k-blocks, operands that are row slices of wider tensors (lda, ldb > K); and the
    compute_single_matrix_multiplication shim, which passes such slices."""
    from brainiak_b200.fcma import cython_blas, engine
    from oracle import fcma_oracle as orc
    rng = np.random.RandomState(14)
    for M in (1, 63, 64, 65, 129):
        for N in (1, 63, 64, 65, 129):
            for K in (1, 15, 16, 17, 1000):
                wide = (M + N + K) % 2 == 1
                A = rng.randn(M, K + (7 if wide else 0)).astype(np.float32)
                B = rng.randn(N, K + (3 if wide else 0)).astype(np.float32)
                a = torch.from_numpy(A).to(dev)[:, :K]
                b = torch.from_numpy(B).to(dev)[:, :K]
                got = engine.gemm_nt(a, b).cpu().numpy()
                want = orc.corr_block([np.ascontiguousarray(A[:, :K].T)], [np.ascontiguousarray(B[:, :K].T)], 0, M,
                                      f64=False)[:, 0, :]
                assert np.array_equal(got, want), "M=%d N=%d K=%d wide=%d: %d differ" % (
                    M, N, K, wide, int((got != want).sum()))
    # cython_blas.pyx:480-560 call pattern: C[n, m] = B[n, :k] @ A[m, :k]^T with k < the operands' width
    A = rng.randn(65, 40).astype(np.float32)
    B = rng.randn(70, 40).astype(np.float32)
    C = np.full((70, 65), NAN, np.float32)
    cython_blas.compute_single_matrix_multiplication('T', 'N', 65, 70, 33, 1.0, A, 40, B, 40, 0.0, C, 65)
    want = orc.corr_block([np.ascontiguousarray(B[:, :33].T)], [np.ascontiguousarray(A[:, :33].T)], 0, 70,
                          f64=False)[:, 0, :]
    assert np.array_equal(C, want)


def _simt_cases():
    """(V, V2 or None, lens, start, nb)."""
    return [(130, None, [16] * 3, 0, 130), (130, None, [15, 16, 17], 3, 64), (200, 63, [17] * 2, 0, 65),
            (200, 64, [1, 31, 32, 33], 100, 63), (200, 65, [16, 9], 5, 129), (129, 129, [40, 7, 33], 64, 65),
            (300, 191, [100, 100], 170, 130), (64, 1, [16], 0, 64)]


@pytest.mark.gpu
def test_corr_simt_bit_exact(dev):
    """corr_block_f32 (k_corr_simt) bit for bit against the sequential fp32 FMA chain: nb and V2 across the 64-wide
    tiles, T across the 16-step k-blocks, start offsets, one mask and two masks of different widths (ldr != ldc), ragged
    epochs (the zero rows add fmaf(0, b, acc)), both layouts; and the cython_blas shims once each."""
    from brainiak_b200.fcma import cython_blas, engine
    from oracle import fcma_oracle as orc
    rng = np.random.RandomState(15)
    for V, V2, lens, start, nb in _simt_cases():
        d1 = [rng.randn(t, V).astype(np.float32) for t in lens]
        d2 = [rng.randn(t, V2).astype(np.float32) for t in lens] if V2 else None
        ep1, _ = engine.stack_epochs(d1, dev)
        ep2 = engine.stack_epochs(d2, dev)[0] if d2 else ep1
        want = orc.corr_block(d1, d2, start, nb, f64=False)
        for layout in (0, 1):
            got = engine.corr_block_f32(ep1, ep2, start, nb, layout=layout).cpu().numpy()
            if layout == 1:
                got = np.transpose(got, (1, 0, 2))
            assert np.array_equal(got, want), "V=%d V2=%s T_e=%s start=%d nb=%d layout %d: %d differ" % (
                V, V2, lens, start, nb, layout, int((got != want).sum()))
    # cython_blas.pyx:20-116 and :388-478: one epoch of [T, V] (rows operand) against [T, V2]
    T, V, V2, s, n = 37, 150, 90, 20, 70
    Bm = rng.randn(T, V).astype(np.float32)
    Am = rng.randn(T, V2).astype(np.float32)
    want = orc.corr_block([Bm], [Am], s, n, f64=False)[:, 0, :]
    C = np.full((n, 3, V2), NAN, np.float32)
    cython_blas.compute_self_corr_for_voxel_sel('N', 'T', V2, n, T, 1.0, Am, V2, s, Bm, V, 0.0, C, 3 * V2, 1)
    assert np.array_equal(C[:, 1, :], want) and np.isnan(C[:, [0, 2]]).all()
    C = np.full((4, n, V2), NAN, np.float32)
    cython_blas.compute_corr_vectors('N', 'T', V2, n, T, 1.0, Am, V2, Bm, V, 0.0, C, V2, s, 2)
    assert np.array_equal(C[2], want) and np.isnan(C[[0, 1, 3]]).all()


@pytest.mark.gpu
def test_side_gemm_argument_checks(dev):
    """gemm_nt and row_normalize_ refuse what their kernels cannot read (they take stride(0) as the row pitch): a
    transposed view, float64, a host tensor -- ValueError, not a silently wrong result."""
    from brainiak_b200.fcma import engine
    a = torch.randn(8, 5, device=dev)
    b = torch.randn(6, 5, device=dev)
    assert engine.gemm_nt(a, b).shape == (8, 6)
    for x, y in ((torch.randn(5, 8, device=dev).t(), b), (a, torch.randn(5, 6, device=dev).t()),
                 (a.double(), b), (a, b.double()), (a.cpu(), b), (a, b.cpu()), (a, torch.randn(6, 4, device=dev))):
        with pytest.raises(ValueError):
            engine.gemm_nt(x, y)
    for x in (torch.randn(5, 8, device=dev).t(), torch.randn(8, 5, device=dev, dtype=torch.float64),
              torch.randn(8, 5), torch.randn(2, 8, 5, device=dev)):
        with pytest.raises(ValueError):
            engine.row_normalize_(x)


# ------------------------------------------------------------------------------- k_within_subject_norm
def norm_tolerance(raw_r, eps):
    """Per-element bound for the exact normaliser (as in test_gpu_parity.py): the reference's var = E[x^2] - mean^2
    in fp32 amplifies 1-ulp differences (CUDA logf vs glibc logf) by (1 + mean^2/var)."""
    n0, E, n2 = raw_r.shape
    S = E // eps
    r = raw_r[:, :S * eps].astype(np.float64).reshape(n0, S, eps, n2)
    num, den = 1 + r, 1 - r
    num[num <= 0] = 1e-4
    den[den <= 0] = 1e-4
    fz = 0.5 * np.log(num / den)
    m = fz.mean(2, keepdims=True)
    var = np.maximum(fz.var(2, keepdims=True), 1e-30)
    z = (fz - m) / np.sqrt(var)
    amp = 1 + m * m / var
    tol = 4e-6 * amp * np.maximum(1, np.abs(z))
    full = np.full(raw_r.shape, 0.0)
    full[:, :S * eps] = tol.reshape(n0, S * eps, n2)
    return full


@pytest.mark.gpu
def test_within_subject_norm_at_scale(dev):
    """within_subject_norm_ against the fp32 C restatement: eps 1 .. 8 (3 and 5 not powers of two) with E % eps != 0
    (trailing epochs bit-identical), r at +-1 and beyond (the clamps), and the Classifier's shape n0 = 1, E = 12, eps = 4,
    n2 = 1 000 003 (3 million elements: the grid-stride loop past 148 * 64 blocks of 256)."""
    from brainiak_b200.fcma import engine
    from oracle import fcma_oracle as orc
    rng = np.random.RandomState(16)
    cases = [(3, 5, 1, 700)] + [(3, 3 * eps + 1 + (eps > 2), eps, 700) for eps in (2, 3, 4, 5, 8)] + \
        [(1, 12, 4, 1000003)]
    for n0, E, eps, n2 in cases:
        r = rng.uniform(-0.95, 0.95, (n0, E, n2)).astype(np.float32)
        edge = np.array([1.0, -1.0, 1.0000001, -1.0000001, 1.5, -2.0, 0.9999999, -0.9999999], np.float32)
        r[:, :, :len(edge)] = edge[None, None, :]                 # constant across epochs -> 0
        r[0, ::2, 8:8 + len(edge)] = edge[None, :]                # every other epoch clamped
        want = orc.within_subject_norm(r.copy(), eps)
        t = torch.from_numpy(r.copy()).to(dev)
        engine.within_subject_norm_(t, eps)
        got = t.cpu().numpy()
        S = E // eps
        what = "n0=%d E=%d eps=%d n2=%d" % (n0, E, eps, n2)
        assert np.array_equal(got[:, S * eps:].view(np.int32), r[:, S * eps:].view(np.int32)), what + ": trailing"
        tol = norm_tolerance(r, eps)
        err = np.abs(got.astype(np.float64) - want)
        bad = ~(err <= tol)
        assert not bad.any(), "%s: %d bad, e.g. %s" % (what, int(bad.sum()), np.argwhere(bad)[:5].tolist())
        same = float(np.mean(got[:, :S * eps] == want[:, :S * eps]))
        assert same > 0.7, "%s: only %.2f bit-identical" % (what, same)


# ------------------------------------------------------------------------------- k_shrink_kernels
def _k00_values():
    f = np.float32
    vals = [0.0, -0.0, 0.3, -0.3, 0.999, -0.999, -1.0, 9e18, 1e19, -9e18, -1e19, 3.4028235e38, -3.4028235e38,
            99.9, 100.0, 4321.0, 123456.7]
    for k in range(0, 39):
        p = f(10.0 ** k)
        vals += [p, np.nextafter(p, f(0)), np.nextafter(p, f(np.inf))]
    vals += [-v for v in vals[-3 * 39:]]
    return np.array(vals + [NAN, np.inf, -np.inf], np.float32)


@pytest.mark.gpu
def test_shrink_digits_and_factor_bit_exact(dev):
    """k_shrink_kernels against the reference's rule in Python: nd = len(str(int(K00))) for every digit count 1 .. 39
    (and 40 with the sign), 10^k and its two float neighbours, negative values, +-0, 9e18 and 1e19; K scaled by
    float32(10 ** (2 - nd)) bit for bit; NaN and +-inf give nd = 1 and leave K untouched."""
    from brainiak_b200.fcma import engine
    k00 = _k00_values()
    E = 7                                                    # 49 entries: the lanes loop
    rng = np.random.RandomState(17)
    K = (rng.rand(len(k00), E, E) * 2 - 0.5).astype(np.float32)
    K[:, 0, 0] = k00
    K[:, 3, 4] = k00 * np.float32(0.75)
    want = K.copy()
    nd = np.ones(len(k00), np.int32)
    for i, v in enumerate(k00):
        if np.isfinite(v):
            nd[i] = len(str(int(v)))
            if nd[i] > 2:
                want[i] = K[i] * np.float32(10 ** (2 - int(nd[i])))
    assert set(range(1, 41)) <= set(nd.tolist())
    t = torch.from_numpy(K.copy()).to(dev)
    digits = engine.shrink_kernels_(t, return_digits=True).cpu().numpy()
    bad = np.flatnonzero(digits != nd)
    assert not bad.size, "digits differ for K00 = %s: got %s, want %s" % (
        k00[bad[:5]].tolist(), digits[bad[:5]].tolist(), nd[bad[:5]].tolist())
    got = t.cpu().numpy()
    bad = np.flatnonzero((got.view(np.int32) != want.view(np.int32)).any(axis=(1, 2)))
    assert not bad.size, "scaled kernels differ for K00 = %s (nd %s)" % (k00[bad[:5]].tolist(), nd[bad[:5]].tolist())
