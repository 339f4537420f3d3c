"""GPU parity tests: the CUDA path, called through the C ABI (ctypes -> libfcma_b200.so), against
 * the CPU oracle (oracle/, test infrastructure) on seeded inputs,
 * golden fixtures produced by the UNMODIFIED reference (tests/golden/make_golden.py),
 * size-independent invariants at the BASELINE.json shape (V=50 000, T=200, E=32).

Stated tolerances (fp32 work, DESIGN.md "Parity"):
  raw correlation r          |dr| <= 1e-6 (fp16x3 / tf32x3: the default "fp32" mode)   4e-5 (bf16x3)  1e-3 (tf32)  8e-3 (bf16)
  Fisher-z / z-score (exact kernel)  |dz| <= 4e-6 * (1 + mean^2/var) * max(1,|z|)   [E[x^2]-mean^2 cancellation]
  kernel matrices            max|dK| <= (5e-4 * sqrt(256 / V2) + 2e-6) * max|K|   (tf32 SYRK; 3.8e-5 at V2 = 50 000)
"""
import math

import numpy as np
import pytest
import torch
from numpy.random import RandomState
from scipy.spatial.distance import hamming
from scipy.stats.mstats import zscore
from sklearn import svm
from sklearn.linear_model import LogisticRegression

from brainiak_b200 import _lib
from brainiak_b200.fcma import engine, synthetic
from brainiak_b200.fcma.classifier import Classifier
from brainiak_b200.fcma.voxelselector import VoxelSelector, shrink_kernels_
from oracle import fcma_oracle as orc

pytestmark = pytest.mark.gpu

R_TOL = {"fp16x3": 1e-6, "tf32x3": 1e-6, "bf16x3": 4e-5, "tf32": 1e-3, "bf16": 8e-3}


@pytest.fixture(scope="module")
def dev():
    assert _lib.device_count() > 0, "no sm_90 device"
    return torch.device("cuda:0")


def k_tol(V2):
    return 5e-4 * math.sqrt(256.0 / max(V2, 1)) + 2e-6


def zero_self(z, start):
    z = z.copy()
    for i in range(z.shape[0]):
        z[i, :, start + i] = 0
    return z


def norm_tolerance(raw_r, eps):
    """Per-element bound for the exact normaliser: the reference's var = E[x^2] - mean^2 in fp32
    amplifies 1-ulp differences (CUDA logf vs glibc logf) by (1 + mean^2/var)."""
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


# ------------------------------------------------------------------------------- a4
@pytest.mark.parametrize("prec", ["fp16x3", "tf32x3", "bf16x3", "tf32", "bf16"])
def test_corr_block_vs_oracle(dev, prec):
    V, V2, T, E = 300, 333, 50, 8
    d1, d2, _ = synthetic.make_two_masks(V, V2, T, E)
    ep1, T_e = engine.stack_epochs(d1, dev)
    ep2, _ = engine.stack_epochs(d2, dev)
    r1, r2 = engine.pack_epochs(ep1, T_e, prec), engine.pack_epochs(ep2, T_e, prec)
    for (a, b, ra, rb, start, nb) in ((d1, d2, r1, r2, 33, 70), (d1, None, r1, r1, 0, 300),
                                      (d2, d1, r2, r1, 300, 33)):
        ref = orc.corr_block(a, b, start, nb, f64=True)
        for layout in (0, 1):
            got = engine.corr_block(ra, rb, start, nb, layout=layout).cpu().numpy()
            if layout == 1:
                got = np.transpose(got, (1, 0, 2))
            assert got.shape == ref.shape
            assert np.max(np.abs(got - ref)) <= R_TOL[prec]


def test_corr_block_f32_simt_and_ragged_epochs(dev):
    # epochs of different length (voxelselector.py:317 uses mat.shape[0] per epoch)
    rng = RandomState(5)
    lens = [7, 12, 9, 12]
    raw = [synthetic.normalize_epoch(rng.randn(t, 77).astype(np.float32)) for t in lens]
    ep, T_e = engine.stack_epochs(raw, dev)
    assert T_e == lens and ep.shape == (4, 12, 77)
    ref = orc.corr_block(raw, None, 5, 40, f64=True)
    got = engine.corr_block_f32(ep, ep, 5, 40).cpu().numpy()
    assert np.max(np.abs(got - ref)) <= 1e-6
    op = engine.pack_epochs(ep, T_e, "tf32x3")
    got = engine.corr_block(op, op, 5, 40).cpu().numpy()
    assert np.max(np.abs(got - ref)) <= 1e-6
    # normalise prologue with ragged epochs == preprocessing.py:80-84 per epoch
    rawu = [rng.randn(t, 77).astype(np.float32) * 2 + 1 for t in lens]
    epu, T_e = engine.stack_epochs(rawu, dev)
    opn = engine.pack_epochs(epu, T_e, "tf32x3", normalize=True)
    refn = orc.corr_block([orc.epoch_normalize(m) for m in rawu], None, 0, 77, f64=True)
    assert np.max(np.abs(engine.corr_block(opn, opn, 0, 77).cpu().numpy() - refn)) <= 2e-6


def test_corr_vs_reference_golden(dev, golden):
    g = golden("vs_mid")
    raw = list(g["raw"])
    ep, T_e = engine.stack_epochs(raw, dev)
    op = engine.pack_epochs(ep, T_e, "tf32x3")
    s, nb = (int(x) for x in g["task"])
    got = engine.corr_block(op, op, s, nb).cpu().numpy()
    assert np.max(np.abs(got - g["corr_raw"])) <= 1e-6         # vs the reference's OpenBLAS sgemm
    # the self-correlation entries are the reference's, bit for bit (exact FMA-chain diagonal)
    ii = np.arange(nb)
    assert np.array_equal(got[ii, :, s + ii], g["corr_raw"][ii, :, s + ii])
    # the FFMA path accumulates like the reference's sgemm (sequential fp32 FMA over t): bit-exact
    got32 = engine.corr_block_f32(ep, ep, s, nb).cpu().numpy()
    assert np.array_equal(got32, g["corr_raw"])
    d1, d2 = list(g["d1"]), list(g["d2"])
    e1, T1 = engine.stack_epochs(d1, dev)
    e2, _ = engine.stack_epochs(d2, dev)
    o1, o2 = engine.pack_epochs(e1, T1, "tf32x3"), engine.pack_epochs(e2, T1, "tf32x3")
    s2, nb2 = (int(x) for x in g["task2"])
    got2 = engine.corr_block(o1, o2, s2, nb2).cpu().numpy()
    assert np.max(np.abs(got2 - g["corr_raw2"])) <= 1e-6
    assert np.array_equal(engine.corr_block_f32(e1, e2, s2, nb2).cpu().numpy(), g["corr_raw2"])


# ------------------------------------------------------------------------------- a6
def test_within_subject_norm_vs_reference_golden(dev, golden):
    g = golden("vs_mid")
    eps = int(g["eps"])
    for raw_key, norm_key, e in (("corr_raw", "corr_norm", eps), ("corr_raw2", "corr_norm2", 4)):
        r = g[raw_key]
        t = torch.from_numpy(r.copy()).to(dev)
        engine.within_subject_norm_(t, e)
        got = t.cpu().numpy()
        tol = norm_tolerance(r, e)
        bad = np.abs(got.astype(np.float64) - g[norm_key]) > tol
        # the self-correlation column (r == 1 +- ulp) is clamp noise in the reference itself
        if raw_key == "corr_raw":
            s = int(g["task"][0])
            for i in range(r.shape[0]):
                bad[i, :, s + i] = False
        assert not bad.any(), (np.argwhere(bad)[:5], np.abs(got - g[norm_key])[bad][:5])
        S = r.shape[1] // e
        # trailing epochs untouched (fcma_extension.cc:52)
        assert np.array_equal(got[:, S * e:], r[:, S * e:])
        assert np.mean(got == g[norm_key]) > 0.7      # mostly bit-identical to the reference's C++
    # known-answer block of the reference's own test (test_voxel_selection.py:58-65)
    gs = golden("vs_small")
    t = torch.from_numpy(gs["fake_corr"].copy()).to(dev)
    engine.within_subject_norm_(t, 4)
    assert np.allclose(t.cpu().numpy(), gs["scipy_norm"])
    # host-buffer entry point with the reference module's signature
    from brainiak_b200.fcma import fcma_extension
    buf = gs["fake_corr"].copy()
    fcma_extension.normalization(buf, 4)
    assert np.allclose(buf, gs["cpp_norm"], atol=1e-6)
    with pytest.raises(RuntimeError):
        engine.within_subject_norm_(torch.zeros((4, 4), device=dev), 2)


def test_norm_degenerate_inputs(dev):
    # var == 0 -> 0 (fcma_extension.cc:78); r >= 1 / r <= -1 clamps (fcma_extension.cc:68-72)
    r = np.zeros((2, 4, 6), np.float32)
    r[0, :, 0] = 0.3                       # constant across epochs -> var 0 -> zeros
    r[0, :, 1] = [1.0, 1.0000001, -1.0, 0.2]
    r[1, :2, 2] = [0.5, -0.5]
    ref = orc.within_subject_norm(r.copy(), 2)
    t = torch.from_numpy(r.copy()).to(dev)
    engine.within_subject_norm_(t, 2)
    got = t.cpu().numpy()
    assert np.all(np.isfinite(got))
    assert np.allclose(got, ref, atol=2e-6)
    assert np.all(got[0, :, 0] == 0)


# ------------------------------------------------------------------------------- a7 / fused a6+a7
@pytest.mark.parametrize("case", ["self_eps4", "two_eps8", "trailing", "generic_eps3", "wide_E48"])
def test_kernels_and_pipeline_vs_oracle(dev, case):
    cfg = {"self_eps4": dict(V=300, V2=None, T=50, E=8, eps=4, start=33, nb=70),
           "two_eps8": dict(V=260, V2=333, T=40, E=16, eps=8, start=5, nb=131),
           "trailing": dict(V=157, V2=None, T=24, E=10, eps=4, start=40, nb=37),
           "generic_eps3": dict(V=128, V2=200, T=24, E=12, eps=3, start=0, nb=128),
           "wide_E48": dict(V=96, V2=200, T=30, E=48, eps=16, start=0, nb=96)}[case]
    V, V2, T, E, eps, start, nb = (cfg[k] for k in ("V", "V2", "T", "E", "eps", "start", "nb"))
    raw, _ = synthetic.make_epochs(V, T, E, seed=4321)
    raw2 = synthetic.make_epochs(V2, T, E, seed=99)[0] if V2 else None
    n2 = V2 or V
    r, z, _ = orc.voxel_block(raw, raw2, start, nb, eps, shrink=False)
    zz = zero_self(z, start) if raw2 is None else z
    Kref = orc.kernel_matrices(zz, f64=True)
    scale = np.max(np.abs(Kref))
    # a7 alone on normalised data
    got = engine.kernel_matrices(torch.from_numpy(zz).to(dev)).cpu().numpy()
    assert np.max(np.abs(got - Kref)) <= k_tol(n2) * scale
    assert np.array_equal(got, np.transpose(got, (0, 2, 1)))            # mirrored triangle
    # fused a6+a7 from raw r
    if engine.fused_supported(E, eps):
        got = engine.norm_kernel_matrices(torch.from_numpy(r).to(dev), eps,
                                          self_col0=start if raw2 is None else -1).cpu().numpy()
        assert np.max(np.abs(got - Kref)) <= k_tol(n2) * scale
    # full pipeline a4->a6->a7 (default precision), both Fisher placements
    ep, T_e = engine.stack_epochs(raw, dev)
    rows = engine.pack_epochs(ep, T_e, "tf32x3")
    cols = engine.pack_epochs(engine.stack_epochs(raw2, dev)[0], T_e, "tf32x3") if raw2 else rows
    fused = engine.fused_supported(E, eps)
    fl = 0
    for fl in (0, _lib.FLAG_FISHER_IN_PASS2):
        if raw2 is None and fused:
            fl |= _lib.FLAG_MASK_SELF
        got = engine.voxel_kernels(rows, cols, start, nb, eps, flags=fl).cpu().numpy()
        if raw2 is None and not fused:
            continue      # generic-eps path keeps the (noisy) self column: covered by two-mask cases
        assert np.max(np.abs(got - Kref)) <= k_tol(n2) * scale
    # small scratch buffer -> several passes give the same result
    if fused or raw2 is not None:
        small = engine.Workspace(E, n2, 32, dev)
        got2 = engine.voxel_kernels(rows, cols, start, nb, eps, flags=fl, work=small).cpu().numpy()
        assert np.max(np.abs(got2 - Kref)) <= k_tol(n2) * scale
    # host-buffer C-ABI entry point (numpy in, numpy out)
    if raw2 is not None:
        Kh = engine.host_voxel_kernels(raw, raw2, start, nb, eps, "tf32x3")
        assert np.max(np.abs(Kh - Kref)) <= k_tol(n2) * scale


@pytest.mark.gpu
@pytest.mark.parametrize("two", [False, True])
def test_tiled_intermediate_equals_strided(dev, two):
    """Fused pipeline with >= 256 rows of workspace stores the correlation block tiled
    [nb/256][V2/256][E][256][256]; FCMA_FLAG_STRIDED_BLOCK forces the reference's [nb][E][V2] layout.  Ragged last
    row tile (600 = 2*256 + 88), ragged last column tile, self columns crossing tile borders."""
    V, V2, T, E, eps, start, nb = 700, (530 if two else None), 40, 8, 4, 77, 600
    raw, _ = synthetic.make_epochs(V, T, E, seed=777)
    raw2 = synthetic.make_epochs(V2, T, E, seed=778)[0] if two else None
    n2 = V2 or V
    _, z, _ = orc.voxel_block(raw, raw2, start, nb, eps, shrink=False)
    Kref = orc.kernel_matrices(z if two else zero_self(z, start), f64=True)
    ep, T_e = engine.stack_epochs(raw, dev)
    rows = engine.pack_epochs(ep, T_e, "fp32")
    cols = engine.pack_epochs(engine.stack_epochs(raw2, dev)[0], T_e, rows.precision) if two else rows
    fl = 0 if two else _lib.FLAG_MASK_SELF
    work = engine.Workspace(E, n2, 768, dev)
    out = {}
    for no_tiled in ("0", "1"):
        work.buf.view(torch.float32).fill_(float("nan"))   # stale padding must never reach the kernels
        out[no_tiled] = engine.voxel_kernels(rows, cols, start, nb, eps, work=work,
                                             flags=fl | (_lib.FLAG_STRIDED_BLOCK if no_tiled == "1" else 0)).cpu().numpy()
    assert np.array_equal(out["0"], out["1"])
    assert np.max(np.abs(out["0"] - Kref)) <= k_tol(n2) * np.max(np.abs(Kref))
    # fp16 intermediate (opt-in flag): same result up to the averaged rounding of the stored Fisher-z values
    got16 = engine.voxel_kernels(rows, cols, start, nb, eps, flags=fl | _lib.FLAG_F16_INTERMEDIATE, work=work).cpu().numpy()
    d16 = np.max(np.abs(got16 - out["0"]))
    assert 0 < d16 <= 4e-3 / math.sqrt(n2) * np.max(np.abs(Kref))
    # several passes through a 256-row workspace (tiled, one row tile per pass)
    small = engine.Workspace(E, n2, 256, dev)
    got = engine.voxel_kernels(rows, cols, start, nb, eps, flags=fl, work=small).cpu().numpy()
    assert np.array_equal(got, out["0"])


@pytest.mark.parametrize("case", ["ragged_multi_pass", "whole_tiles_sharded", "wide_E64", "long_column_walk"])
def test_symmetric_pipeline_vs_oracle_and_plain(dev, case):
    """fcma_voxel_kernels_sym (self-correlation: only blocks on/above the diagonal are contracted, every block is
    used for its row voxels and -- transposed -- for its column voxels) against the CPU oracle and the plain
    pipeline: ragged last pass (V not a multiple of 256), several passes through a small workspace, shards that
    accumulate into one K (the multi-GPU scheme: sum of the shards' K arrays), self-column masking, E > 32."""
    cfg = {"ragged_multi_pass": dict(V=1100, T=40, E=8, eps=4, rows=256, shards=1),
           "whole_tiles_sharded": dict(V=1536, T=50, E=16, eps=8, rows=512, shards=3),
           "wide_E64": dict(V=900, T=30, E=64, eps=16, rows=512, shards=2),
           # 2048-row pass = 128 row steps of the column pass: two accumulator folds, the brick ring wraps 42 times
           "long_column_walk": dict(V=2600, T=24, E=8, eps=4, rows=2048, shards=1)}[case]
    V, T, E, eps, rows, shards = (cfg[k] for k in ("V", "T", "E", "eps", "rows", "shards"))
    raw, _ = synthetic.make_epochs(V, T, E, seed=2468)
    ep, T_e = engine.stack_epochs(raw, dev)
    op = engine.pack_epochs(ep, T_e, "fp32")
    # (a buffer sized for block + transposed copy gives the column-pass variant twice the rows per pass)
    work = engine.SymWorkspace(E, V, rows, dev, transposed_copy=(case != "long_column_walk"))
    fls = (_lib.FLAG_MASK_SELF, 0)
    if case == "long_column_walk":      # also the TMA-fed column pass: ring wrap-around and folds over a long walk
        fls = (_lib.FLAG_MASK_SELF, _lib.FLAG_MASK_SELF | _lib.FLAG_COLS_TMA, _lib.FLAG_MASK_SELF | _lib.FLAG_COLS_V2, 0)
    for fl in fls:
        plain = engine.voxel_kernels(op, op, 0, V, eps, flags=fl & _lib.FLAG_MASK_SELF)
        work.buf.view(torch.float32).fill_(float("nan"))       # stale scratch must never reach the kernels
        K = torch.zeros((V, E, E), device=dev)
        for s, n in engine.sym_row_partition(V, shards):
            if n > 0:
                engine.voxel_kernels_sym(op, s, n, eps, flags=fl, work=work, out=K)
        scale = float(plain.abs().max())
        assert torch.isfinite(K).all()
        assert float((K - K.transpose(1, 2)).abs().max()) == 0.0
        # same values, summed in a different order: fp32 rounding of the partial sums only
        assert float((K - plain).abs().max()) <= 1e-5 * scale      # measured 4e-7 .. 4e-6 (E = 64)
        if fl & _lib.FLAG_MASK_SELF:   # the oracle comparison uses the masked self column (the raw one is rounding noise)
            sel = np.r_[0:40, V // 2:V // 2 + 40, V - 40:V]
            for blk in (slice(0, 40), slice(V // 2, V // 2 + 40), slice(V - 40, V)):
                _, z, _ = orc.voxel_block(raw, None, blk.start, 40, eps, shrink=False)
                Kref = orc.kernel_matrices(zero_self(z, blk.start), f64=True)
                got = K[blk].cpu().numpy()
                assert np.max(np.abs(got - Kref)) <= k_tol(V) * np.max(np.abs(Kref))
            del sel
    # argument checks: ragged row count that does not end at V, workspace below 256 rows
    with pytest.raises(ValueError):
        engine.voxel_kernels_sym(op, 0, 300, eps, work=work, out=K)
    tiny = engine.Workspace(E, V, 64, dev)
    with pytest.raises(MemoryError):
        engine.voxel_kernels_sym(op, 0, V, eps, work=tiny, out=K)


@pytest.mark.parametrize("E,eps", [(5, 1), (7, 2), (10, 2), (12, 4), (16, 16), (32, 32), (24, 8), (9, 4)])
def test_symmetric_column_pass_all_eps(dev, E, eps):
    """Every instantiation of the column-direction pass (eps = 1 .. 32), epoch counts that are not multiples of 4
    (scalar K folds), trailing epochs outside a complete subject (left un-normalised, fcma_extension.cc:52) and a
    block that needs several folds of the accumulators: symmetric == plain pipeline, and against the oracle."""
    V, T = 1300, 24
    raw, _ = synthetic.make_epochs(V, T, E, seed=1000 + 37 * E + eps)
    ep, T_e = engine.stack_epochs(raw, dev)
    op = engine.pack_epochs(ep, T_e, "fp32")
    assert _lib.load().fcma_sym_uses_column_pass(_lib.PREC[op.precision], E, eps, 0) == 1
    fl = _lib.FLAG_MASK_SELF
    plain = engine.voxel_kernels(op, op, 0, V, eps, flags=fl)
    K = torch.zeros((V, E, E), device=dev)
    work = engine.Workspace(E, V, 256, dev)            # the column-pass variant keeps only the block itself
    work.buf.view(torch.float32).fill_(float("nan"))
    engine.voxel_kernels_sym(op, 0, V, eps, flags=fl, work=work, out=K)      # 6 passes of <= 256 rows
    # scale floor V: with eps = 1 every z-score is 0 and so is K
    scale = max(float(plain.abs().max()), float(V))
    assert torch.isfinite(K).all()
    assert float((K - K.transpose(1, 2)).abs().max()) == 0.0
    # eps = 2: the z-score of two values is sign(x1 - x2) -- a step function, so the rare pair of near-equal Fisher
    # values flips with the last bit of r (the plain pipeline adds the three split products of r(j, i) in another order
    # than those of r(i, j)); a flipped pair moves one K entry by 2 of ~V
    loose = eps <= 2
    assert float((K - plain).abs().max()) <= (2e-3 if loose else 1e-5) * scale
    # the three column-pass kernels (default fragment-layout kernel; version 2 = thread-per-row normalisation +
    # ldmatrix; the TMA-fed variant when E % 4 == 0) and the transposed-copy variant agree to the order of the fp32 sums
    # (E <= 16 takes the 16-epoch kernel by default: FLAG_COLS_PAD32 selects the padded 32-epoch one)
    for extra in (_lib.FLAG_COLS_PAD32, _lib.FLAG_COLS_V2, _lib.FLAG_COLS_TMA, _lib.FLAG_SYM_TRANSPOSED):
        K2 = torch.zeros((V, E, E), device=dev)
        w2 = engine.SymWorkspace(E, V, 256, dev)
        w2.buf.view(torch.float32).fill_(float("nan"))
        engine.voxel_kernels_sym(op, 0, V, eps, flags=fl | extra, work=w2, out=K2)
        assert float((K2 - K).abs().max()) <= (2e-3 if loose else 1e-5) * scale
    for s0 in (0, 700, V - 30):
        _, z, _ = orc.voxel_block(raw, None, s0, 30, eps, shrink=False)
        Kref = orc.kernel_matrices(zero_self(z, s0), f64=True)
        tol = (1e-2 if loose else k_tol(V)) * max(np.max(np.abs(Kref)), float(V))   # measured 4.5e-3 for eps = 2
        assert np.max(np.abs(K[s0:s0 + 30].cpu().numpy() - Kref)) <= tol


@pytest.mark.parametrize("E,eps,rows", [(64, 1, 256), (64, 2, 256), (64, 4, 256), (64, 8, 256), (64, 16, 256), (64, 32, 256),
                                        (64, 64, 256), (48, 16, 256), (40, 8, 256), (33, 1, 256), (36, 4, 256), (64, 8, 2048)])
def test_symmetric_column_pass_wide(dev, E, eps, rows):
    """32 < E <= 64: the 64-epoch column kernel (k_norm_syrk_cols64: one column voxel per warp, 8-column strips, bricks
    scattered column-major by 4-byte cp.async) for every eps instantiation, epoch counts that are not multiples of 8 or 4,
    trailing epochs outside a complete subject, a ragged last strip (V % 8 = 4), and a 2048-row pass that folds the
    accumulators twice: equal to the plain pipeline, to the transposed-copy variant and to the oracle."""
    V, T = (1300, 24) if rows == 256 else (2604, 20)
    raw, _ = synthetic.make_epochs(V, T, E, seed=2000 + 41 * E + eps)
    ep, T_e = engine.stack_epochs(raw, dev)
    op = engine.pack_epochs(ep, T_e, "fp32")
    wide = _lib.FLAG_COLS_WIDE
    assert _lib.load().fcma_sym_uses_column_pass(_lib.PREC[op.precision], E, eps, 0) == 0      # opt-in (4 % slower at scale)
    assert _lib.load().fcma_sym_uses_column_pass(_lib.PREC[op.precision], E, eps, wide) == 1
    assert _lib.load().fcma_sym_uses_column_pass(_lib.PREC[op.precision], E, eps, wide | _lib.FLAG_F16_INTERMEDIATE) == 0
    fl = _lib.FLAG_MASK_SELF
    plain = engine.voxel_kernels(op, op, 0, V, eps, flags=fl)
    K = torch.zeros((V, E, E), device=dev)
    work = engine.Workspace(E, V, rows, dev)
    work.buf.view(torch.float32).fill_(float("nan"))
    engine.voxel_kernels_sym(op, 0, V, eps, flags=fl | wide, work=work, out=K)
    scale = max(float(plain.abs().max()), float(V))
    loose = eps <= 2
    assert torch.isfinite(K).all()
    assert float((K - K.transpose(1, 2)).abs().max()) == 0.0
    assert float((K - plain).abs().max()) <= (2e-3 if loose else 1e-5) * scale
    K2 = torch.zeros((V, E, E), device=dev)
    w2 = engine.SymWorkspace(E, V, rows, dev)
    w2.buf.view(torch.float32).fill_(float("nan"))
    engine.voxel_kernels_sym(op, 0, V, eps, flags=fl, work=w2, out=K2)          # the default: transposed copy + row pass
    assert float((K2 - K).abs().max()) <= (2e-3 if loose else 1e-5) * scale
    for s0 in (0, 700, V - 30):
        _, z, _ = orc.voxel_block(raw, None, s0, 30, eps, shrink=False)
        Kref = orc.kernel_matrices(zero_self(z, s0), f64=True)
        if loose:
            # eps <= 2: z = sign(x1 - x2) -- and where fp32 E[x^2] - m^2 of two near-equal Fisher values cancels, 0 or a huge
            # value, in the reference as on the GPU but not the same one (tools/r2_wide_eps_probe.py: a single such pair moves a
            # diagonal entry by 40 .. 500 of V = 1300): compare all but the few entries such pairs touch
            d = np.abs(K[s0:s0 + 30].cpu().numpy() - Kref)
            assert np.mean(d > 1e-2 * float(V)) < 0.02
            continue
        tol = k_tol(V) * max(np.max(np.abs(Kref)), float(V))
        assert np.max(np.abs(K[s0:s0 + 30].cpu().numpy() - Kref)) <= tol


@pytest.mark.parametrize("prec,flag", [("fp32", True), ("bf16", False)])
def test_symmetric_fp16_block_column_pass(dev, prec, flag):
    """fp16 Fisher-z block (opt-in flag, or implied by the single-product operand modes): the symmetric pipeline's column
    pass reads 64-byte lines of the fp16 block; same stored values as the plain fp16-block pipeline, so the kernels
    agree to the order of the fp32 partial sums, and both stay within the fp16-block tolerance of the fp32 block."""
    V, T, E, eps = 1400, 40, 16, 8
    raw, _ = synthetic.make_epochs(V, T, E, seed=8642)
    ep, T_e = engine.stack_epochs(raw, dev)
    op = engine.pack_epochs(ep, T_e, prec)
    fl = _lib.FLAG_MASK_SELF | (_lib.FLAG_F16_INTERMEDIATE if flag else 0)
    assert _lib.load().fcma_sym_uses_column_pass(_lib.PREC[op.precision], E, eps, fl) == 1
    plain = engine.voxel_kernels(op, op, 0, V, eps, flags=fl)
    scale = float(plain.abs().max())
    out = {}
    # column pass over the block (cp.async bricks / TMA bricks) / transposed copy + row pass
    for cols, extra in (("1", 0), ("tma", _lib.FLAG_COLS_TMA), ("0", _lib.FLAG_SYM_TRANSPOSED)):
        K = torch.zeros((V, E, E), device=dev)
        work = engine.SymWorkspace(E, V, 512, dev)
        work.buf.view(torch.float32).fill_(float("nan"))
        for s0, n0 in engine.sym_row_partition(V, 2):
            engine.voxel_kernels_sym(op, s0, n0, eps, flags=fl | extra, work=work, out=K)
        assert torch.isfinite(K).all()
        assert float((K - K.transpose(1, 2)).abs().max()) == 0.0
        assert float((K - plain).abs().max()) <= 1e-5 * scale
        out[cols] = K
    if flag:     # against the fp32 block: the averaged rounding of the stored values (DESIGN.md 3.3)
        K32 = engine.voxel_kernels(op, op, 0, V, eps, flags=_lib.FLAG_MASK_SELF)
        assert 0 < float((out["1"] - K32).abs().max()) <= 4e-3 / math.sqrt(V) * float(K32.abs().max())


def test_pipeline_vs_reference_golden_kernels(dev, golden):
    g = golden("vs_mid")
    d1, d2 = list(g["d1"]), list(g["d2"])
    e1, T1 = engine.stack_epochs(d1, dev)
    e2, _ = engine.stack_epochs(d2, dev)
    for prec, tol in (("fp32", 1.0), ("tf32x3", 1.0), ("bf16x3", 1.0), ("bf16", 60.0)):
        o1, o2 = engine.pack_epochs(e1, T1, prec), engine.pack_epochs(e2, T1, prec)
        s2, nb2 = (int(x) for x in g["task2"])
        K = engine.voxel_kernels(o1, o2, s2, nb2, 4).cpu().numpy()
        shrink_kernels_(K)
        ref = g["kernels2"]                    # reference kernels AFTER its decimal shrink
        assert np.max(np.abs(K - ref)) <= tol * k_tol(136) * np.max(np.abs(ref))


def test_classifier_kernel_is_sum_of_voxel_kernels(dev):
    d1, d2, _ = synthetic.make_two_masks(90, 70, 16, 12)
    e1, T1 = engine.stack_epochs(d1, dev)
    e2, _ = engine.stack_epochs(d2, dev)
    o1, o2 = engine.pack_epochs(e1, T1, "tf32x3"), engine.pack_epochs(e2, T1, "tf32x3")
    Ksum = engine.classifier_kernel(o1, o2, 0, 90, 4).cpu().numpy()
    Kv = engine.voxel_kernels(o1, o2, 0, 90, 4).cpu().numpy().astype(np.float64).sum(0)
    assert np.max(np.abs(Ksum - Kv)) <= 2e-5 * np.max(np.abs(Kv))
    Kref, _ = orc.classifier_kernel(d1, d2, 4, 32, shrink=False)
    assert np.max(np.abs(Ksum - Kref)) <= 4 * k_tol(70 * 90) * np.max(np.abs(Kref))
    # two calls over disjoint row ranges accumulate (beta = 1, classifier.py:334-339)
    K2 = torch.zeros((12, 12), device=dev)
    engine.classifier_kernel(o1, o2, 0, 40, 4, out=K2)
    engine.classifier_kernel(o1, o2, 40, 50, 4, out=K2)
    assert np.max(np.abs(K2.cpu().numpy() - Ksum)) <= 2e-5 * np.max(np.abs(Ksum))
    # eps <= 1: no normalisation at all (classifier.py:204)
    K0 = engine.classifier_kernel(o1, o2, 0, 90, 0).cpu().numpy()
    c = orc.corr_block(d1, d2, 0, 90, layout=1).reshape(12, -1).astype(np.float64)
    assert np.max(np.abs(K0 - c @ c.T)) <= 5e-4 * np.max(np.abs(c @ c.T))


# ------------------------------------------------------------------------------- reference tests, ported
def _create_epoch(prng, row=12, col=5):
    mat = prng.rand(row, col).astype(np.float32)
    mat = zscore(mat, axis=0, ddof=0)
    mat = np.nan_to_num(mat)
    return mat / math.sqrt(mat.shape[0])


def test_voxel_selection(dev, golden):
    """Port of reference tests/fcma/test_voxel_selection.py:39-89 (same inputs, same assertions)."""
    prng = RandomState(1234567890)
    fake_raw_data = [_create_epoch(prng) for i in range(8)]
    labels = [0, 1, 0, 1, 0, 1, 0, 1]
    vs = VoxelSelector(labels, 4, 2, fake_raw_data, voxel_unit=1, process_num=0)
    fake_corr = prng.rand(1, 4, 5).astype(np.float32)
    fake_corr = vs._correlation_normalization(fake_corr)
    expected_fake_corr = [[[1.06988919, 0.51641309, -0.46790636, -1.31926763, 0.2270218],
                           [-1.22142744, -1.39881694, -1.2979387, 1.05702305, -0.6525566],
                           [0.89795232, 1.27406132, 0.36460185, 0.87538344, 1.5227468],
                           [-0.74641371, -0.39165771, 1.40124381, -0.61313909, -1.0972116]]]
    assert np.allclose(fake_corr, expected_fake_corr), \
        'within-subject normalization does not provide correct results'
    clf = svm.SVC(kernel='precomputed', shrinking=False, C=1, gamma='auto')
    results = vs.run(clf)
    output = [None] * len(results)
    for tup in results:
        output[tup[0]] = int(8 * tup[1])
    assert np.allclose(output, [7, 4, 6, 4, 4], atol=1), \
        'voxel selection via SVM does not provide correct results'
    clf = LogisticRegression()
    results = vs.run(clf)
    output = [None] * len(results)
    for tup in results:
        output[tup[0]] = int(8 * tup[1])
    assert np.allclose(output, [6, 3, 6, 4, 4], atol=1)
    # stage methods keep the reference's contracts
    corr = vs._correlation_computation((1, 3))
    g = golden("vs_small")
    assert corr.shape == (3, 8, 5) and np.max(np.abs(corr - g["corr_raw"][1:4])) <= 2e-6


def test_voxel_selection_with_two_masks(dev, golden):
    """Port of reference tests/fcma/test_voxel_selection.py:92-130."""
    prng = RandomState(1234567890)
    fake_raw_data1 = [_create_epoch(prng) for i in range(8)]
    fake_raw_data2 = [_create_epoch(prng) for i in range(8)]
    labels = [0, 1, 0, 1, 0, 1, 0, 1]
    vs = VoxelSelector(labels, 4, 2, fake_raw_data1, raw_data2=fake_raw_data2, voxel_unit=1,
                       process_num=0)
    clf = svm.SVC(kernel='precomputed', shrinking=False, C=1, gamma='auto')
    results = vs.run(clf)
    output = [None] * len(results)
    for tup in results:
        output[tup[0]] = int(8 * tup[1])
    assert np.allclose(output, [3, 3, 7, 5, 7], atol=1)
    # no self column with two masks: exactly the accuracies the reference produced here
    g = golden("vs_small")
    acc = np.zeros(5)
    for v, a in results:
        acc[v] = a
    assert np.array_equal(acc, g["acc2_svm"])
    clf = LogisticRegression()
    results = vs.run(clf)
    output = [None] * len(results)
    for tup in results:
        output[tup[0]] = int(8 * tup[1])
    assert np.allclose(output, [4, 3, 7, 4, 6], atol=1)


def test_voxel_selection_ranking_vs_reference(dev, golden):
    """Full run on a planted-signal case: selected voxels and accuracies vs the reference's run."""
    g = golden("vs_full")
    raw = list(g["rawf"])
    labels = [int(x) for x in g["labelsf"]]
    clf = svm.SVC(kernel='precomputed', shrinking=False, C=1)
    # per-precision bounds (measured, tools/tolerance_probe.py: the fp32-faithful modes reproduce the reference's accuracies
    # of all 128 voxels exactly -- its self column included, thanks to the exact diagonal; tf32 0.992, bf16 0.977)
    bounds = {"fp32": (1.0, 0.0, 12), "tf32x3": (1.0, 0.0, 12), "bf16x3": (0.99, 1.0 / 16, 12),
              "tf32": (0.97, 1.0 / 16, 12), "bf16": (0.95, 2.0 / 16, 11)}
    for prec, (min_same, max_diff, min_top) in bounds.items():
        vs = VoxelSelector(labels, int(g["epsf"]), 4, raw, voxel_unit=32, process_num=2, precision=prec)
        res = vs.run(clf)
        acc = np.zeros(raw[0].shape[1])
        for v, a in res:
            acc[v] = a
        ref = g["accf"]
        assert [a for _, a in res] == sorted((a for _, a in res), reverse=True)
        # planted voxels 0..11 are the top of both rankings
        top_ref = set(int(v) for v in np.argsort(-ref, kind="stable")[:12])
        top_got = set(v for v, _ in res[:12])
        assert len(top_ref & top_got) >= min_top, prec
        assert np.mean(acc == ref) >= min_same, (prec, np.mean(acc == ref))
        assert np.max(np.abs(acc - ref)) <= max_diff + 1e-9, (prec, np.max(np.abs(acc - ref)))


def _create_clf_epoch(prng, idx, num_voxels):
    mat = prng.rand(12, num_voxels).astype(np.float32)
    if idx % 2 == 0:
        mat = np.sort(mat, axis=0)
    mat = zscore(mat, axis=0, ddof=0)
    mat = np.nan_to_num(mat)
    return mat / math.sqrt(mat.shape[0])


@pytest.mark.parametrize("two", [False, True])
def test_classification(dev, golden, two):
    """Port of reference tests/fcma/test_classification.py:43-217 (Hamming <= 1 assertions)."""
    prng = RandomState(1234567890)
    d5 = [_create_clf_epoch(prng, i, 5) for i in range(20)]
    d6 = [_create_clf_epoch(prng, i, 6) for i in range(20)] if two else None
    a, b = d5, (d6 if two else d5)
    labels = [0, 1] * 10
    if two:
        expected_confidence = np.array([-1.23311606, 1.02440964, -0.93898336, 1.07028798,
                                        -1.04420007, 0.97647772, -1.0498268, 1.04970111])
        expected_output = [0, 1, 0, 1, 0, 1, 0, 1]
    else:
        expected_confidence = np.array([-1.18234421, 0.97403604, -1.04005679, 0.92403019,
                                        -0.95567738, 1.11746593, -0.83275891, 0.9486868])
        expected_output = [0, 0, 0, 1, 0, 1, 0, 1]
    svm_clf = svm.SVC(kernel='precomputed', shrinking=False, C=1, gamma='auto')
    clf = Classifier(svm_clf, epochs_per_subj=4)
    clf.fit(list(zip(a[:12], b[:12])), labels[:12])
    test = list(zip(a[12:], b[12:]))
    conf = clf.decision_function(test)
    assert hamming(np.sign(expected_confidence), np.sign(conf)) * 8 <= 1
    y_pred = clf.predict(test)
    assert hamming(y_pred, expected_output) * 8 <= 1
    conf2 = clf.decision_function(test)          # cached test_data_ path
    assert np.array_equal(conf, conf2)
    y = [0, 1, 0, 1, 0, 1, 0, 1]
    score = clf.score(test, y)
    assert np.isclose(hamming(y_pred, y), 1 - score)
    # against what the unmodified reference produced on the same inputs (two masks: no self column)
    g = golden("clf")
    tag = "two" if two else "one"
    assert clf.num_digits_ == int(g[tag + "_num_digits"])
    if two:
        assert np.allclose(clf.training_data_, g["two_train_features"], atol=2e-5)
        assert np.allclose(conf, g["two_decision"], atol=2e-3)
        assert np.array_equal(y_pred, g["two_predict"])
    # partial similarity matrix computation
    clf = Classifier(svm_clf, num_processed_voxels=2, epochs_per_subj=4)
    clf.fit(list(zip(a, b)), labels, num_training_samples=12)
    y_pred = clf.predict()
    assert hamming(y_pred, expected_output) * 8 <= 1
    conf = clf.decision_function()
    assert hamming(np.sign(expected_confidence), np.sign(conf)) * 8 <= 1
    assert clf.training_data_ is None and clf.test_data_.shape == (8, 12)
    if two:
        assert np.allclose(clf.test_data_, g["two_portion_test_sim"], rtol=2e-3, atol=2e-3)
    # logistic regression
    clf = Classifier(LogisticRegression(), epochs_per_subj=4)
    clf.fit(list(zip(a[:12], b[:12])), labels[:12], num_training_samples=12 if two else None)
    y_pred = clf.predict(test)
    assert hamming(y_pred, expected_output) * 8 <= 1
    if two:
        assert np.allclose(clf.decision_function(test), g["two_lr_decision"], atol=2e-3)


def test_classifier_big_kernel_vs_reference(dev, golden):
    g = golden("clf")
    x1, x2 = list(g["big_x1"]), list(g["big_x2"])
    c = Classifier(svm.SVC(kernel='precomputed'), num_processed_voxels=32, epochs_per_subj=int(g["big_eps"]))
    c.num_voxels_, c.num_features_, c.num_samples_ = 90, 90 * 70, 12
    K, feats = c._compute_kernel_matrix_in_portion(x1, x2)
    assert feats is None and c.num_digits_ == int(g["big_num_digits"])
    assert np.max(np.abs(K - g["big_kernel"])) <= 2e-5 * np.max(np.abs(g["big_kernel"]))


def test_compute_correlation(dev, golden):
    """Port of reference tests/fcma/test_util.py:23-54 + fixtures from the reference itself."""
    from brainiak_b200.fcma.util import compute_correlation
    prng = RandomState(1234567890)
    mat1 = prng.rand(5, 10).astype(np.float32)
    mat2 = prng.rand(6, 10).astype(np.float32)
    corr = compute_correlation(mat1, mat1)
    assert np.allclose(corr, np.corrcoef(mat1), atol=1e-5)
    corr = compute_correlation(mat1, mat2)
    mat = np.concatenate((mat1, mat2), axis=0)
    assert np.allclose(corr, np.corrcoef(mat)[0:5, 5:], atol=1e-5)
    assert corr.dtype == np.float32 and corr.flags.c_contiguous
    mat1 = prng.rand(5, 10).astype(np.float32)
    mat2 = prng.rand(6, 10).astype(np.float32)
    mat1[0, 0] = np.nan
    corr = compute_correlation(mat1, mat2, return_nans=False)
    assert np.all(corr == 0, axis=1)[0]
    assert np.sum(corr == 0) == 6
    corr = compute_correlation(mat1, mat2, return_nans=True)
    assert np.all(np.isnan(corr), axis=1)[0]
    assert np.sum(np.isnan(corr)) == 6
    with pytest.raises(ValueError, match="Dimension discrepancy"):
        compute_correlation(mat1, mat2[:, :9])
    g = golden("util")
    assert np.allclose(compute_correlation(g["big1"], g["big2"]), g["cb"], atol=1e-5)


def test_separate_epochs_vs_reference_golden_file(dev, golden):
    """a14 against the reference's own golden file tests/fcma/data/expected_raw_data.npy."""
    from brainiak_b200.fcma.preprocessing import separate_epochs
    g = golden("preproc")
    raw, labels = separate_epochs(list(g["activity"]), list(g["epochs"]))
    assert np.array_equal(labels, [0, 1, 0, 1])            # test_preprocessing.py:29,41
    assert len(raw) == len(g["expected_raw_data"])
    for a, b in zip(raw, g["expected_raw_data"]):
        assert np.allclose(a, b)
    raw2, labels2 = separate_epochs(list(g["act2"]), list(g["ep2"]))
    assert np.array_equal(labels2, g["labels2"])
    for k, a in enumerate(raw2):
        ref = g["raw2_%d" % k]
        live = np.ones(a.shape[1], bool)
        if 4 <= k < 8:
            live[7] = False                    # constant voxel: exact 0 here, rounding residue in scipy
            assert np.all(a[:, 7] == 0)
        assert a.shape == ref.shape and np.allclose(a[:, live], ref[:, live], atol=2e-6)


def test_cython_blas_shims(dev, golden):
    from brainiak_b200.fcma import cython_blas as blas
    g = golden("vs_small")
    raw = [np.ascontiguousarray(m) for m in g["raw1"]]
    raw2 = [np.ascontiguousarray(m) for m in g["raw2"]]
    corr = np.zeros((3, 8, 5), np.float32)
    for e in range(8):       # the reference's call, voxelselector.py:316-322
        blas.compute_self_corr_for_voxel_sel('N', 'T', 5, 3, 12, 1.0, raw2[e], 5, 1, raw[e], 5, 0.0,
                                             corr, 5 * 8, e)
    assert np.max(np.abs(corr - g["corr_raw2"][1:4])) <= 2e-6
    K = np.zeros((8, 8), np.float32)
    z = g["corr_norm2"]
    blas.compute_kernel_matrix('L', 'T', 8, 5, 1.0, z, 2, 5, 0.0, K, 8)
    ref = z[2].astype(np.float64) @ z[2].astype(np.float64).T
    assert np.max(np.abs(K - ref)) <= 2e-3 * np.max(np.abs(ref)) and np.array_equal(K, K.T)
    cv = np.zeros((8, 2, 5), np.float32)
    blas.compute_corr_vectors('N', 'T', 5, 2, 12, 1.0, raw2[3], 5, raw[3], 5, 0.0, cv, 5, 0, 3)
    assert np.max(np.abs(cv[3] - g["corr_raw2"][0:2, 3, :])) <= 2e-6


# ------------------------------------------------------------------------------- full-size invariants
@pytest.mark.timeout(900)
def test_full_size_invariants(dev):
    """BASELINE.json shape (V=50 000, T=200, E=32, eps=8) on a block of 512 voxel rows.

    Size-independent properties of the pipeline (z-scored within subject over eps epochs):
      * r is symmetric: corr[i, e, j] == corr[j, e, i];  r_self == 1
      * trace(K_i) == E * (V - 1)      (every (subject, column) group has sum z^2 == eps)
      * every subject block of K_i sums to 0 along rows  (sum_b z_b == 0)
      * permuting the TRs of every epoch changes nothing (same math, different summation order)
      * the classifier kernel is the sum of the voxel kernels
    """
    V, T, E, eps, nb, start = 50000, 200, 32, 8, 512, 24960
    g = torch.Generator(device=dev).manual_seed(1234)
    ep = torch.randn((E, T, V), device=dev, generator=g)
    common = torch.randn((E, T, 1), device=dev, generator=g)
    ep[1::2, :, :500] += 0.6 * common[1::2]
    engine.epoch_normalize_(ep)
    op = engine.pack_epochs(ep, None, "fp32")
    assert op.precision == "fp16x3"           # normalised data -> the fast fp32-faithful split
    # symmetry of r on a diagonal block
    blk = engine.corr_block(op, op, start, nb)[:, :, start:start + nb]
    assert float((blk - blk.transpose(0, 2)).abs().max()) <= 1e-6
    ar = torch.arange(nb, device=dev)
    diag = blk[ar, :, ar]
    assert float((diag - 1).abs().max()) <= 2e-6
    del blk
    work = engine.Workspace(E, V, nb, dev)
    fl = _lib.FLAG_MASK_SELF
    K = engine.voxel_kernels(op, op, start, nb, eps, flags=fl, work=work).double()
    tr = torch.diagonal(K, dim1=1, dim2=2).sum(1)
    assert float((tr / (E * (V - 1.0)) - 1).abs().max()) <= 1e-4
    Kb = K.view(nb, E // eps, eps, E).sum(2)
    assert float(Kb.abs().max()) <= 1e-4 * V                 # ~0 compared with diag ~ V
    assert float((K - K.transpose(1, 2)).abs().max()) == 0.0
    # TR permutation invariance
    perm = torch.randperm(T, device=dev, generator=g)
    op2 = engine.pack_epochs(ep[:, perm, :].contiguous(), None, "fp32")
    K2 = engine.voxel_kernels(op2, op2, start, nb, eps, flags=fl, work=work).double()
    assert float((K2 - K).abs().max()) <= 2e-5 * float(K.abs().max())
    # Fisher in the GEMM epilogue == Fisher in pass 2
    K3 = engine.voxel_kernels(op, op, start, nb, eps, flags=fl | _lib.FLAG_FISHER_IN_PASS2, work=work).double()
    assert float((K3 - K).abs().max()) <= 2e-5 * float(K.abs().max())
    # opt-in fp16 intermediate (default in the bf16 / tf32 operand modes): rounding errors of the stored Fisher-z
    # values average out over the V columns -> max|dK| <= 4e-3 / sqrt(V) * max|K|  (1.8e-5 here)
    K16 = engine.voxel_kernels(op, op, start, nb, eps, flags=fl | _lib.FLAG_F16_INTERMEDIATE, work=work).double()
    assert 0 < float((K16 - K).abs().max()) <= 4e-3 / math.sqrt(V) * float(K.abs().max())
    # classifier kernel == sum of voxel kernels (no self masking on either side)
    Kn = engine.voxel_kernels(op, op, start, nb, eps, work=work).double().sum(0)
    Kc = engine.classifier_kernel(op, op, start, nb, eps, work=work).double()
    assert float((Kc - Kn).abs().max()) <= 1e-5 * float(Kn.abs().max())
    # reduced-precision modes stay within their stated tolerance of the fp32-faithful result
    for prec, tol in (("tf32x3", 2e-5), ("bf16x3", 2e-5), ("bf16", 2e-3)):
        opp = engine.pack_epochs(ep, None, prec)
        Kp = engine.voxel_kernels(opp, opp, start, nb, eps, flags=fl, work=work).double()
        assert float((Kp - K).abs().max()) <= tol * float(K.abs().max())


# ------------------------------------------------------------------------------- a8 on the GPU
def _sklearn_cv(K, labels, folds, **kw):
    from sklearn import model_selection
    out = np.zeros(K.shape[0])
    for v in range(K.shape[0]):
        skf = model_selection.StratifiedKFold(n_splits=folds, shuffle=False)
        clf = svm.SVC(kernel='precomputed', **kw)
        out[v] = model_selection.cross_val_score(clf, K[v], y=labels, cv=skf, n_jobs=1).mean()
    return out


def test_gpu_shrink_matches_reference_rule(dev):
    rng = RandomState(0)
    K = (rng.rand(9, 6, 6).astype(np.float32) + 0.5)
    K[:, 0, 0] = [0.3, 5, 50, 99.9, 100, 4321, 1e6, 99.99999, 123456.7]
    ref = shrink_kernels_(K.copy())
    t = torch.from_numpy(K.copy()).to(dev)
    digits = engine.shrink_kernels_(t, return_digits=True).cpu().numpy()
    assert list(digits) == [len(str(int(x))) for x in K[:, 0, 0]]
    assert np.array_equal(t.cpu().numpy(), ref)


def test_gpu_svm_cv_matches_sklearn(dev, golden):
    """Batched GPU SMO (libsvm restatement) vs sklearn.cross_val_score on the same kernels."""
    g = golden("vs_full")
    # (a) the kernels the unmodified reference built in its full run -> the accuracies it reported
    Kf = np.ascontiguousarray(g["kernelsf"])
    labels = [int(x) for x in g["labelsf"]]
    acc = engine.svm_cv_precomputed(torch.from_numpy(Kf).to(dev), labels, 4, C=1.0, tol=1e-3)
    assert np.array_equal(acc, g["accf"])
    # (b) random correlation-like kernels, several (C, tol, folds); shrinking=False is reproduced
    #     exactly, shrinking=True (sklearn's default) may differ only on near-zero margins
    rng = RandomState(42)
    E, nv = 32, 300
    Z = rng.randn(nv, E, 200).astype(np.float32)
    Z[:, 1::2, :20] += 0.35            # some signal
    K = np.einsum('vej,vfj->vef', Z, Z).astype(np.float32)
    shrink_kernels_(K)
    lab = [e % 2 for e in range(E)]
    Kd = torch.from_numpy(K).to(dev)
    for folds, C, tol in ((4, 1.0, 1e-3), (8, 0.05, 1e-3), (2, 10.0, 1e-4)):
        ref = _sklearn_cv(K, lab, folds, C=C, tol=tol, shrinking=False)
        got, iters = engine.svm_cv_precomputed(Kd, lab, folds, C=C, tol=tol, return_iters=True)
        assert np.array_equal(got, ref), (folds, C, tol, np.flatnonzero(got != ref)[:5])
        assert iters.max() < 100000 and iters.min() >= 1
    # scikit-learn's default shrinking=True against the solver WITHOUT the heuristic: same optimum within tol
    ref = _sklearn_cv(K, lab, 4, C=1.0, shrinking=True)
    got = engine.svm_cv_precomputed(Kd, lab, 4, C=1.0)
    assert np.mean(got == ref) >= 0.99
    # ... and against the restatement of the heuristic: exact
    got = engine.svm_cv_precomputed(Kd, lab, 4, C=1.0, shrinking=True)
    assert np.array_equal(got, ref)
    # unbalanced labels / odd fold sizes / label values other than 0,1
    lab2 = [3 if e < 14 else 7 for e in range(E)]
    ref = _sklearn_cv(K[:60], lab2, 3, C=1.0, shrinking=False)
    got = engine.svm_cv_precomputed(Kd[:60], lab2, 3, C=1.0)
    assert np.array_equal(got, ref)


def test_gpu_svm_shrinking_follows_libsvm_iteration_by_iteration(dev):
    """libsvm's shrinking heuristic (do_shrinking / be_shrunk / reconstruct_gradient / the counter and unshrink logic of
    Solver::Solve) restated in k_svm_cv<KT, true>: on problems that need several hundred iterations -- where variables
    are shrunk, swapped and the gradient is reconstructed -- the iteration count of EVERY problem equals scikit-learn's
    SVC.n_iter_ and the accuracies are identical; the counts differ from the unshrunk solver's, i.e. the heuristic ran."""
    from sklearn import model_selection
    rng = RandomState(11)
    heuristic_ran = False
    for E, folds, C, T, nv in ((64, 4, 1.0, 60, 60), (48, 3, 1.0, 20, 60), (64, 2, 100.0, 30, 40)):
        Z = rng.randn(nv, E, T).astype(np.float32)
        lab = np.asarray([e % 2 for e in range(E)])
        Z[:, lab == 1, :5] += 0.2
        K = np.einsum('vej,vfj->vef', Z, Z).astype(np.float32)
        shrink_kernels_(K)
        Kd = torch.from_numpy(K).to(dev)
        got, it_s = engine.svm_cv_precomputed(Kd, list(lab), folds, C=C, return_iters=True, shrinking=True)
        _, it_n = engine.svm_cv_precomputed(Kd, list(lab), folds, C=C, return_iters=True, shrinking=False)
        ref_it = np.zeros_like(it_s)
        ref_acc = np.zeros(nv)
        skf = model_selection.StratifiedKFold(n_splits=folds, shuffle=False)
        for v in range(nv):
            accs = []
            for f, (tr, te) in enumerate(skf.split(np.zeros((E, 1)), lab)):
                clf = svm.SVC(kernel="precomputed", C=C, shrinking=True)
                clf.fit(K[v][np.ix_(tr, tr)].astype(np.float64), lab[tr])
                ref_it[v, f] = int(np.asarray(clf.n_iter_).ravel()[0])
                accs.append(np.mean(clf.predict(K[v][np.ix_(te, tr)].astype(np.float64)) == lab[te]))
            ref_acc[v] = np.mean(accs)
        assert np.array_equal(it_s, ref_it), (E, folds, C, int(np.sum(it_s != ref_it)))
        assert np.array_equal(got, ref_acc)
        heuristic_ran |= bool(np.any(it_s != it_n))
    assert heuristic_ran


def test_gpu_svm_cv_multiclass_matches_sklearn(dev):
    """More than two conditions: one-vs-one problems on the GPU solver + libsvm's vote (first maximum wins) give the
    accuracies of sklearn.cross_val_score, exactly, including label values other than 0..k-1, unbalanced classes and
    folds whose held-out part is not the same size."""
    rng = RandomState(77)
    E, nv = 36, 250
    for k, folds, lab in ((3, 3, [e % 3 for e in range(36)]),
                          (4, 3, [(7, 2, 11, 5)[e % 4] for e in range(36)]),
                          (3, 4, [0] * 9 + [1] * 14 + [2] * 13)):
        Z = rng.randn(nv, E, 120).astype(np.float32)
        code = np.searchsorted(np.unique(lab), lab)
        for c in range(k):
            Z[:, code == c, 10 * c:10 * c + 10] += 0.3      # some signal: accuracies spread between chance and 1
        K = np.einsum('vej,vfj->vef', Z, Z).astype(np.float32)
        shrink_kernels_(K)
        for C, tol in ((1.0, 1e-3), (0.02, 1e-3)):
            for shrinking in (False, True):
                ref = _sklearn_cv(K, lab, folds, C=C, tol=tol, shrinking=shrinking)
                got = engine.svm_cv_precomputed(torch.from_numpy(K).to(dev), lab, folds, C=C, tol=tol, shrinking=shrinking)
                assert np.array_equal(got, ref), (k, folds, C, shrinking, np.flatnonzero(got != ref)[:5])
            assert ref.std() > 0.02                          # not a degenerate comparison
    # and through VoxelSelector: three conditions stay on the device, same result list as the host scikit-learn loop
    clf = svm.SVC(kernel='precomputed', shrinking=False, C=1)
    lab3 = [e % 3 for e in range(24)]
    assert engine.svm_cv_supported(clf, lab3, 2, 24)
    raw = [rng.randn(40, 150).astype(np.float32) for _ in range(24)]
    for e in range(24):
        raw[e][:, :20] += 0.4 * rng.randn(40, 1).astype(np.float32) * (lab3[e] + 1)
    a = VoxelSelector(lab3, 12, 2, raw, voxel_unit=64, process_num=0, gpu_cv=True).run(clf)
    b = VoxelSelector(lab3, 12, 2, raw, voxel_unit=64, process_num=0, gpu_cv=False).run(clf)
    assert a == b


def test_voxel_selector_gpu_cv_equals_host_cv(dev, golden):
    g = golden("vs_full")
    raw = list(g["rawf"])
    labels = [int(x) for x in g["labelsf"]]
    clf = svm.SVC(kernel='precomputed', shrinking=False, C=1)
    assert engine.svm_cv_supported(clf, labels, 4, 16)
    assert not engine.svm_cv_supported(LogisticRegression(), labels, 4, 16)
    assert not engine.svm_cv_supported(svm.SVC(kernel='precomputed', class_weight='balanced'), labels, 4, 16)
    a = VoxelSelector(labels, int(g["epsf"]), 4, raw, voxel_unit=32, process_num=0, gpu_cv=True).run(clf)
    b = VoxelSelector(labels, int(g["epsf"]), 4, raw, voxel_unit=32, process_num=0, gpu_cv=False).run(clf)
    assert a == b
    # scikit-learn's default classifier (shrinking=True) stays on the device too, same result list
    clf_d = svm.SVC(kernel='precomputed')
    assert engine.svm_cv_supported(clf_d, labels, 4, 16)
    a = VoxelSelector(labels, int(g["epsf"]), 4, raw, voxel_unit=32, process_num=0, gpu_cv=True).run(clf_d)
    b = VoxelSelector(labels, int(g["epsf"]), 4, raw, voxel_unit=32, process_num=0, gpu_cv=False).run(clf_d)
    assert a == b


def test_symmetric_pipeline_vs_reference_golden(dev, golden):
    """vs_sym fixture: the UNMODIFIED reference's shrunk kernels and cross-validation accuracies of all 560 voxels of
    a one-mask run.  The symmetric pipeline takes three passes here (256 + 256 + 48 rows: diagonal mirroring, row pass,
    column pass, ragged tail); VoxelSelector.run picks it by default (V >= 512)."""
    g = golden("vs_sym")
    raw, eps, folds = list(g["raw"]), int(g["eps"]), int(g["folds"])
    labels = [int(x) for x in g["labels"]]
    V, E = raw[0].shape[1], len(raw)
    ep, T_e = engine.stack_epochs(raw, dev)
    ref = g["kernels"]
    for prec in ("fp32", "tf32x3"):
        op = engine.pack_epochs(ep, T_e, prec)
        K = torch.zeros((V, E, E), device=dev)
        engine.voxel_kernels_sym(op, 0, V, eps, work=engine.Workspace(E, V, 256, dev), out=K)
        K = K.cpu().numpy()
        shrink_kernels_(K)
        assert np.max(np.abs(K - ref)) <= k_tol(V) * np.max(np.abs(ref))
    clf = svm.SVC(kernel="precomputed", shrinking=False, C=1)
    vs = VoxelSelector(labels, eps, folds, raw, process_num=0, block_rows=256)
    assert vs._symmetric_ok()
    res = vs.run(clf)
    acc = np.zeros(V)
    for v, a in res:
        acc[v] = a
    assert np.mean(acc == g["acc"]) >= 0.99             # measured 0.9964: 2 of 560 chance-level voxels move by one test sample of 8
    assert np.max(np.abs(acc - g["acc"])) <= 1.0 / 8 + 1e-9


def test_classifier_kernel_single_mask_uses_symmetry(dev):
    """One mask, all voxels in one call: engine.classifier_kernel sums the symmetric pipeline's voxel kernels; same
    [E, E] matrix as the plain accumulation (classifier.py:334-339) and as the oracle."""
    V, T, E, eps = 900, 30, 16, 4
    raw, _ = synthetic.make_epochs(V, T, E, seed=515)
    ep, T_e = engine.stack_epochs(raw, dev)
    op = engine.pack_epochs(ep, T_e, "fp32")
    Ks = engine.classifier_kernel(op, op, 0, V, eps).cpu().numpy()
    Kp = engine.classifier_kernel(op, op, 0, V, eps, symmetric=False).cpu().numpy()
    assert np.max(np.abs(Ks - Kp)) <= 2e-5 * np.max(np.abs(Kp))
    # accumulates into `out` like the plain path (beta = 1)
    out = torch.ones((E, E), device=dev)
    engine.classifier_kernel(op, op, 0, V, eps, out=out)
    assert np.max(np.abs(out.cpu().numpy() - 1 - Ks)) <= 1e-6 * np.max(np.abs(Ks))
    # row portions (start > 0) keep the plain path
    K2 = torch.zeros((E, E), device=dev)
    engine.classifier_kernel(op, op, 0, 400, eps, out=K2)
    engine.classifier_kernel(op, op, 400, 500, eps, out=K2)
    assert np.max(np.abs(K2.cpu().numpy() - Kp)) <= 2e-5 * np.max(np.abs(Kp))
    # fcma_classifier_kernel_sym in several 256-row passes (diagonal squares once, the blocks right of them twice), with the
    # self column masked, with E > 32 (no transposed copy needed here) and with the fp16 block: always the fp64 sum of the
    # symmetric pipeline's per-voxel kernels
    for (E2, eps2, fl) in ((16, 4, _lib.FLAG_MASK_SELF), (48, 8, 0), (24, 8, _lib.FLAG_F16_INTERMEDIATE)):
        raw2, _ = synthetic.make_epochs(V, T, E2, seed=900 + E2)
        ep2, T2 = engine.stack_epochs(raw2, dev)
        op2 = engine.pack_epochs(ep2, T2, "fp32")
        small = engine.SymWorkspace(E2, V, 256, dev, transposed_copy=False)
        small.buf.view(torch.float32).fill_(float("nan"))
        Kc = engine.classifier_kernel(op2, op2, 0, V, eps2, flags=fl, work=small)
        Kv = engine.voxel_kernels_sym(op2, 0, V, eps2, flags=fl).to(torch.float64).sum(0)
        assert torch.isfinite(Kc).all()
        assert float((Kc.to(torch.float64) - Kv).abs().max()) <= 2e-6 * float(Kv.abs().max()), (E2, eps2, fl)


def test_voxel_selector_symmetric_equals_plain(dev):
    """Public API: one mask -> the symmetric pipeline by default; same (voxel, accuracy) list as the plain
    pipeline (the kernels differ only in the order of fp32 partial sums), host and GPU cross-validation."""
    V, T, E, eps = 700, 40, 16, 4
    raw, labels = synthetic.make_epochs(V, T, E, informative=12, signal=1.2, seed=31)
    clf = svm.SVC(kernel="precomputed", shrinking=False, C=1)
    a = VoxelSelector(labels, eps, 4, raw, process_num=0, block_rows=256)
    assert a._symmetric_ok()
    ra = a.run(clf)
    assert isinstance(a._work, engine.SymWorkspace)
    b = VoxelSelector(labels, eps, 4, raw, process_num=0, symmetric=False)
    assert not b._symmetric_ok()
    rb = b.run(clf)
    da, db = dict(ra), dict(rb)
    assert sorted(da) == list(range(V)) == sorted(db)
    assert sum(1 for v in da if da[v] != db[v]) <= 1
    assert [x for _, x in ra] == sorted((x for _, x in ra), reverse=True)
    # two masks never take the symmetric path
    c = VoxelSelector(labels, eps, 4, raw, raw_data2=raw, process_num=0)
    assert not c._symmetric_ok()


def test_voxel_selector_multi_gpu_nccl(dev):
    """N>1 product path (NCCL broadcast of the epochs, static row shards, all-gather of the scores):
    runs tools/run_vs_multi.py under torchrun when the box has >= 2 GPUs."""
    import os
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs (covered on CPU by tests/test_distributed_cpu.py with gloo)")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                          "--master-addr", "127.0.0.1", "--master-port", "29533",
                          os.path.join(root, "tools", "run_vs_multi.py")],
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    assert "multi-GPU == single-GPU result: OK" in out.stdout


# ------------------------------------------------------------------------------- round 2: BASELINE config shapes,
# noise floor, host entry point of the symmetric pipeline, range packing
def _probe_matches(raw, probe):
    """the seeded synthetic inputs are those the stored reference outputs were computed from"""
    return np.array_equal(np.stack([raw[e][:4, ::997][:, :16] for e in (0, len(raw) - 1)]), probe)


def _gpu_rows_acc(K_rows, labels, folds):
    Kg = K_rows.clone()
    engine.shrink_kernels_(Kg)
    return Kg.cpu().numpy(), engine.svm_cv_precomputed(Kg, labels, folds, C=1.0, tol=1e-3)


@pytest.mark.timeout(600)
def test_config1_shape_vs_reference(dev, golden):
    """BASELINE configs[1] at FULL size (V=30 000, T=200, E=16, eps=8, fp32-faithful, one GPU): the symmetric pipeline
    (E=16 instantiations of the row and column passes, 8 passes of 4096 rows, ragged tail 30 000 = 117*256 + 48) against
    the unmodified reference on three 32-row samples: first pass, a middle pass, the ragged tail (its kernels and
    accuracies stored in tests/golden/config1.npz)."""
    g = golden("config1")
    V, T, E, eps, folds = 30000, 200, 16, 8, 2
    raw, labels = synthetic.make_epochs(V, T, E)
    assert _probe_matches(raw, g["c1_probe"])
    ep, T_e = engine.stack_epochs(raw, dev)
    op = engine.pack_epochs(ep, T_e, "fp32")
    K = torch.zeros((V, E, E), device=dev)
    work = engine.SymWorkspace(E, V, 4096, dev, transposed_copy=False)
    engine.voxel_kernels_sym(op, 0, V, eps, work=work, out=K)
    same, total = 0, 0
    for s0 in (64, 15008, V - 32):
        Kref, acc_ref = g["c1_K_%d" % s0], g["c1_acc_%d" % s0]
        Kg, acc = _gpu_rows_acc(K[s0:s0 + 32], labels, folds)
        assert np.max(np.abs(Kg - Kref)) <= 3e-5 * np.max(np.abs(Kref))      # measured 1.3e-5 (reference's own ssyrk noise ~1e-5)
        same += int(np.sum(acc == acc_ref))
        total += 32
        assert np.max(np.abs(acc - acc_ref)) <= 2.0 / E + 1e-9
    assert same >= total - 4          # measured: all identical


@pytest.mark.timeout(600)
def test_config4_classifier_kernel_at_scale(dev, golden):
    """BASELINE configs[4] shape class (Classifier precomputed kernel, one mask, V = 20 000, E = 32): the one [E, E]
    kernel of engine.classifier_kernel equals the fp64 sum of the per-voxel kernels, and sampled per-voxel kernels equal
    the unmodified reference's (its own full classifier run at this size is ~10 min of CPU: classifier.py:279-348 is the
    same per-row arithmetic summed over rows, pinned at small size by test_classifier_big_kernel_vs_reference; the
    sampled reference kernels are stored in tests/golden/config4.npz)."""
    g = golden("config4")
    V, T, E, eps = 20000, 200, 32, 8
    raw, labels = synthetic.make_epochs(V, T, E)
    assert _probe_matches(raw, g["c4_probe"])
    ep, T_e = engine.stack_epochs(raw, dev)
    op = engine.pack_epochs(ep, T_e, "fp32")
    Kc = engine.classifier_kernel(op, op, 0, V, eps)
    Kv = engine.voxel_kernels_sym(op, 0, V, eps)
    Ksum = Kv.to(torch.float64).sum(0)
    assert float((Kc.to(torch.float64) - Ksum).abs().max()) <= 2e-6 * float(Ksum.abs().max())
    assert float((Kc - Kc.t()).abs().max()) == 0.0 or float((Kc - Kc.t()).abs().max()) <= 1e-6 * float(Kc.abs().max())
    for s0 in (256, 10016, V - 32):
        Kref = g["c4_K_%d" % s0]
        Kg, _ = _gpu_rows_acc(Kv[s0:s0 + 32], labels, 4)
        assert np.max(np.abs(Kg - Kref)) <= 3e-5 * np.max(np.abs(Kref))
    # the classifier's decimal shrink rule (classifier.py:343-347) on the summed kernel
    nd = len(str(int(float(Kc[0, 0]))))
    assert nd > 2       # ~1e8: the shrink matters at this size


@pytest.mark.timeout(900)
def test_result_level_noise_floor(dev, golden):
    """SURVEY Appendix B.2 result-level contract, measured in this run: with the self column present ("drop-in" mode)
    even the reference re-run on TR-permuted inputs (identical mathematics) changes the accuracy of a large share of the
    chance-level voxels; a precision mode must not disagree with the reference more than that noise floor (plus a small
    margin), and must agree almost everywhere once the self column is masked on both sides.  The reference's accuracies
    (on the inputs, on TR-permuted inputs, and with the self column masked, each through its own scikit-learn
    cross-validation) are stored in tests/golden/noise_floor.npz."""
    g = golden("noise_floor")
    V, T, E, eps, folds = 768, 200, 32, 8, 4
    raw, labels = synthetic.make_epochs(V, T, E)
    assert _probe_matches(raw, g["probe"])
    acc_ref, acc_perm = g["acc"], g["acc_perm"]
    floor = float(np.mean(acc_ref != acc_perm))            # e.g. 0.1 - 0.2 (SURVEY: 352 / 2000)
    acc_ref_m = g["acc_masked"]
    planted = set(range(V // 100))
    clf = svm.SVC(kernel='precomputed', shrinking=False, C=1)
    bounds = {"fp32": (1.25, 0.02, 0.99), "tf32x3": (1.25, 0.02, 0.99), "bf16x3": (1.25, 0.02, 0.985),
              "tf32": (1.5, 0.03, 0.90), "bf16": (1.5, 0.04, 0.80)}
    for prec, (mult, add, masked_min) in bounds.items():
        res = VoxelSelector(labels, eps, folds, raw, process_num=0, precision=prec).run(clf)
        acc = np.zeros(V)
        for v, a in res:
            acc[v] = a
        differ = float(np.mean(acc != acc_ref))
        assert differ <= mult * floor + add, (prec, differ, floor)
        assert np.max(np.abs(acc - acc_ref)) <= 3.0 / E + 1e-9
        # the informative (planted) voxels score like the reference says, whatever the chance-level ones do
        pl = sorted(planted)
        assert np.max(np.abs(acc[pl] - acc_ref[pl])) <= 1.0 / E + 1e-9
        res_m = VoxelSelector(labels, eps, folds, raw, process_num=0, precision=prec, mask_self=True).run(clf)
        acc_m = np.zeros(V)
        for v, a in res_m:
            acc_m[v] = a
        assert float(np.mean(acc_m == acc_ref_m)) >= masked_min, (prec, float(np.mean(acc_m == acc_ref_m)))


def test_host_entry_point_symmetric_and_range_packing(dev):
    """fcma_host_voxel_kernels_sym (host buffers in, host buffers out, everything inside the call) restores the caller's
    device (its values: test_gpu_sym_entry_points.py); fcma_pack_operand_range packs exactly the voxels it is asked for,
    bit-identically to a full pack."""
    V, T, E, eps = 1100, 40, 8, 4
    raw, _ = synthetic.make_epochs(V, T, E, seed=4242)
    ep, T_e = engine.stack_epochs(raw, dev)
    op = engine.pack_epochs(ep, T_e, "fp16x3")
    host = torch.from_numpy(np.stack(raw)).pin_memory()
    out = torch.empty((V, E, E), dtype=torch.float32).pin_memory()
    engine.host_voxel_kernels_sym(host, eps, precision="fp16x3", out=out, rows_per_pass=256)
    assert torch.cuda.current_device() == dev.index          # the entry point restores the caller's device
    # range packing: voxels >= 512 only, into a buffer pre-filled with a pattern
    full = op.buf.clone()
    part = engine.PackedOperand(torch.full_like(op.buf, 0x5A), E, T, V, op.precision, op.T_e)
    engine.pack_epochs(ep, T_e, "fp16x3", v_begin=512, out=part)
    kp = _lib.load().fcma_operand_kp(_lib.PREC["fp16x3"], T)
    planes = full[: 2 * E * V * kp * 2].view(2, E, V, kp * 2)
    got = part.buf[: 2 * E * V * kp * 2].view(2, E, V, kp * 2)
    assert torch.equal(got[:, :, 512:], planes[:, :, 512:])
    assert bool((got[:, :, :512] == 0x5A).all())
    Kp = engine.voxel_kernels_sym(part, 512, V - 512, eps).cpu().numpy()
    Kf = engine.voxel_kernels_sym(op, 512, V - 512, eps).cpu().numpy()
    assert np.array_equal(Kp, Kf)


def test_epoch_exchange_single_rank(dev):
    """EpochExchange without a process group: the share is everything, gather is one H2D copy."""
    from brainiak_b200.fcma.exchange import EpochExchange, epoch_partition
    assert epoch_partition(32, 8) == [(4 * r, 4) for r in range(8)]
    assert epoch_partition(10, 4) == [(0, 3), (3, 3), (6, 2), (8, 2)]
    x = EpochExchange(4, 8, 64, dev, nbuf=2)
    host = torch.randn((4, 8, 64)).pin_memory()
    out = x.gather(1, host)
    torch.cuda.synchronize()
    assert x.mode == "single" and torch.equal(out.cpu(), host)


@pytest.mark.parametrize("two", [False, True])
def test_classifier_streamed_prediction(dev, two):
    """SURVEY §8f rank 4: after a portion-mode fit (training_data_ is None) predict / decision_function on NEW data
    stream the test-vs-train similarity portion by portion from the raw training epochs; same decision values as the
    small-mask path that materialises training_data_ (classifier.py:222-277, 506-566)."""
    prng = RandomState(1234567890)
    nv1, nv2 = (9, 6) if two else (9, 9)
    a = [_create_clf_epoch(prng, i, nv1) for i in range(20)]
    b = [_create_clf_epoch(prng, i, nv2) for i in range(20)] if two else a
    labels = [0, 1] * 10
    X = list(zip(a, b))
    full = Classifier(svm.SVC(kernel='precomputed', shrinking=False, C=1), epochs_per_subj=4)
    full.fit(X[:12], labels[:12])
    assert full.training_data_ is not None
    conf_full = full.decision_function(X[12:])
    # portion mode: 2 voxel rows per portion, the kernel over all 20 samples, the first 12 for training
    part = Classifier(svm.SVC(kernel='precomputed', shrinking=False, C=1), num_processed_voxels=2, epochs_per_subj=4)
    part.fit(X, labels, num_training_samples=12)
    assert part.training_data_ is None and part._train_raw_ is not None and len(part._train_raw_[0]) == 12
    sim_full = full.test_data_.copy()               # [8, 12] similarity from the materialised features
    conf = part.decision_function(X[12:])            # NEW data after a portion-mode fit -> streamed similarity
    assert part.test_data_.shape == (8, 12)
    assert np.allclose(part.test_data_, sim_full, rtol=2e-4, atol=2e-4 * np.max(np.abs(sim_full)))
    assert np.allclose(conf, conf_full, atol=2e-3)
    assert np.array_equal(part.predict(X[12:]), full.predict(X[12:]))
    # score() in portion mode scores the cached test part (classifier.py:652-690): here the same 8 samples
    assert np.isclose(part.score(X[12:], labels[12:]), full.score(X[12:], labels[12:]))


def test_prepare_fcma_data_matches_reference_arithmetic(dev):
    """prepare_fcma_data (reference preprocessing.py:156-232) on synthetic 4-D images: masking (image.py:107-140),
    voxel randomisation with the reference's seeding, epoch separation + z-score on the GPU -- against the same steps in
    numpy / scipy."""
    from brainiak_b200.fcma.preprocessing import RandomType, prepare_fcma_data
    prng = RandomState(42)
    nsub, shape, ntr = 3, (5, 4, 3), 40
    images = [prng.randn(*shape, ntr).astype(np.float32) * 3 + 10 for _ in range(nsub)]
    mask1 = prng.rand(*shape) > 0.4
    mask2 = prng.rand(*shape) > 0.6
    cond = np.zeros((2, 4, ntr), np.int8)       # 2 conditions, 4 epochs of 8 TRs each
    for e in range(4):
        cond[e % 2, e, 2 + 9 * e: 10 + 9 * e] = 1
    conditions = [cond] * nsub

    def expected(mask, random):
        act = [im.astype(np.float32)[mask] for im in images]
        if random == RandomType.REPRODUCIBLE:
            for i in range(len(act)):
                np.random.seed(i)
                np.random.shuffle(act[i])
        raw, labels = [], []
        for sid in range(nsub):
            for c in range(2):
                for e in range(4):
                    sel = cond[c, e] == 1
                    if sel.sum() > 0:
                        mat = np.ascontiguousarray(act[sid][:, sel].T)
                        mat = np.nan_to_num(zscore(mat, axis=0, ddof=0)) / math.sqrt(sel.sum())
                        raw.append(mat.astype(np.float32))
                        labels.append(c)
        return raw, labels
    for random in (RandomType.NORANDOM, RandomType.REPRODUCIBLE):
        r1, r2, labels = prepare_fcma_data(images, conditions, mask1, mask2, random=random)
        e1, el = expected(mask1, random)
        e2, _ = expected(mask2, random)
        assert list(labels) == el and len(r1) == len(e1) == 12 and len(r2) == 12
        for got, ref in zip(r1 + r2, e1 + e2):
            assert got.shape == ref.shape and got.dtype == np.float32 and np.allclose(got, ref, atol=2e-6)
    r1, r2, labels = prepare_fcma_data(images, conditions, mask1)
    assert r2 is None and len(r1) == 12
    (ep, T_e), none2, labels = prepare_fcma_data(images, conditions, mask1, return_device=True)
    assert none2 is None and ep.is_cuda and tuple(ep.shape) == (12, 8, int(mask1.sum())) and T_e == [8] * 12
    with pytest.raises(ValueError, match="different shapes"):
        prepare_fcma_data(images, conditions, mask1[:-1])


def test_host_entry_point_tiny_mask(dev):
    """fcma_host_voxel_kernels_sym on a mask smaller than one 256-voxel tile (single ragged tile, one pass, no column pass)."""
    V, T, E, eps = 70, 20, 4, 2
    raw, _ = synthetic.make_epochs(V, T, E, seed=99)
    Kh = engine.host_voxel_kernels_sym(raw, eps, precision="tf32x3", flags=_lib.FLAG_MASK_SELF)
    ep, T_e = engine.stack_epochs(raw, dev)
    op = engine.pack_epochs(ep, T_e, "tf32x3")
    Kp = engine.voxel_kernels(op, op, 0, V, eps, flags=_lib.FLAG_MASK_SELF).cpu().numpy()
    assert np.isfinite(Kh).all() and np.max(np.abs(Kh - Kp)) <= 1e-5 * max(np.max(np.abs(Kp)), 1.0)
