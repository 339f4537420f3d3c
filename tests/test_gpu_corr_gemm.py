"""Element-wise tests of the correlation GEMM (k_corr_wgmma, its epilogue and k_self_corr_fixup) against an fp64
contraction of the same float32 epochs, at the shapes where a tiled, pipelined kernel goes wrong.

Reference: ``orc.corr_block(..., f64=True)`` (fp64 sums of the float32 products) for small shapes, a float64
``torch.einsum`` on the device for the large one.  Fisher reference: ``fz(r) = 0.5 * log(num / den)`` in fp64 with the
clamps of fcma_extension.cc:68-72 (``num = 1 + r``, ``den = 1 - r``, each replaced by 1e-4 when it is <= 0).

Tolerances:
* fp32-faithful modes (fp16x3, tf32x3): ``tol_r = max(1e-6, 2 * e32)``, e32 = max error of the fp32 sequential-FMA
  chain (``orc.corr_block(f64=False)``, which the reference's sgemm matches bit for bit) against fp64 at the same
  shape: "no worse than the reference's own fp32";
* other modes: ``R_TOL`` of the parity tests;
* Fisher-z where |r| <= 1 - 1e-5: ``|z - fz(r64)| <= 2 tol_r / (1 - r64^2) + 1e-6 (1 + |fz|)`` (dz/dr = 1 / (1 - r^2));
  beyond, the reference's own value depends on the last bit of r: z finite, with the sign of r, 4.9 <= |z| <= 8.7;
* self-correlation entries: the exact chain value (bit for bit), or fz of it to 1e-5.

Layouts read back by the white-box test of the fused pipelines (the only check on the per-element mapping of the
tiled stores; kernel matrices are blind to a permutation of the columns inside a row):
* tiled block, fp32 or fp16: ``[ceil(n/256)][ceil(V2/256)][E][256 i][256 j]``, element (i, e, j) at
  ``[i // 256][j // 256][e][i % 256][j % 256]``; rows >= n and columns >= V2 are padding;
* strided block (FCMA_FLAG_STRIDED_BLOCK): ``[n][E][round_up(V2, 32)]``;
* symmetric pipeline: block A = rows [a, a+n) x columns [a, V) tiled as above (inside the diagonal n x n part the
  tiles tj < ti hold the transposed tiles (ti, tj)); with FCMA_FLAG_SYM_TRANSPOSED block B follows A at byte offset
  ``nt * t256 * E * 65536 * esz`` (nt = ceil(n/256), t256 = ceil((V-a)/256)) and holds
  ``[t256 - nt][nt][E][256 j][256 i]``: the transposed off-diagonal tiles, rows = column voxels.
"""
import numpy as np
import pytest
import torch

from brainiak_b200 import _lib
from brainiak_b200.fcma import engine, synthetic
from oracle import fcma_oracle as orc

pytestmark = pytest.mark.gpu

R_TOL = {"fp16x3": 1e-6, "tf32x3": 1e-6, "bf16x3": 4e-5, "tf32": 1e-3, "bf16": 8e-3}
FAITHFUL = ("fp16x3", "tf32x3")
PRECS = ("fp16x3", "tf32x3", "bf16x3", "tf32", "bf16")
NAN = float("nan")


@pytest.fixture(scope="module")
def dev():
    assert _lib.device_count() > 0, "no sm_90 device"
    return torch.device("cuda:0")


def fz(r):
    r = np.asarray(r, np.float64)
    num, den = 1.0 + r, 1.0 - r
    num = np.where(num <= 0, 1e-4, num)
    den = np.where(den <= 0, 1e-4, den)
    return 0.5 * np.log(num / den)


def unit_columns(rng, T, V, center=False):
    """[T, V] float32 with unit-norm columns (centred first if asked: z-scored data)."""
    g = rng.randn(T, V)
    if center:
        g -= g.mean(0, keepdims=True)
    return np.ascontiguousarray(g / np.linalg.norm(g, axis=0, keepdims=True), dtype=np.float32)


def tol_for(prec, r64, r32):
    if prec in FAITHFUL:
        return max(1e-6, 2.0 * float(np.max(np.abs(r32 - r64))))
    return R_TOL[prec]


def check_values(got, r64, fisher_e, tol_r, self_j=None, chain_self=None, half=False, what=""):
    """Element-wise check of a block [n, E, m]: raw r (fisher_e[e] False) or Fisher-z (True) per epoch; the
    self-correlation entries (column self_j[i] of row i) against the chain values.  Returns the max errors."""
    got = np.asarray(got, np.float64)
    n, E, m = got.shape
    assert got.shape == r64.shape, what
    assert np.isfinite(got).all(), "%s: non-finite values at %s" % (what, np.argwhere(~np.isfinite(got))[:5])
    selfm = np.zeros(got.shape, bool)
    ii = np.arange(n)
    if self_j is not None:
        selfm[ii, :, self_j] = True
    stats = {"raw": 0.0, "fisher": 0.0, "clamp": 0}
    for e in range(E):
        g, r, off = got[:, e], r64[:, e], ~selfm[:, e]
        extra = 2.0 ** -11 * np.abs(g) if half else 0.0
        ref = fz(r) if fisher_e[e] else r
        if fisher_e[e]:
            inner = off & (np.abs(r) <= 1 - 1e-5)
            rr = np.where(inner, r, 0.0)
            bound = 2 * tol_r / (1 - rr * rr) + 1e-6 * (1 + np.abs(ref)) + extra
            err = np.abs(g - ref)
            bad = inner & (err > bound)
            clamp = off & ~inner
            bad |= clamp & ~((np.sign(g) == np.sign(r)) & (np.abs(g) >= 4.9) & (np.abs(g) <= 8.7))
            stats["fisher"] = max(stats["fisher"], float(np.max(err[inner], initial=0.0)))
            stats["clamp"] += int(clamp.sum())
        else:
            err = np.abs(g - r)
            bad = off & (err > tol_r + extra)
            stats["raw"] = max(stats["raw"], float(np.max(err[off], initial=0.0)))
        if bad.any():
            idx = np.argwhere(bad)[:5]
            pytest.fail("%s: epoch %d (%s), %d bad of %d, e.g. (i, j) %s: got %s, want %s (r64 %s)" % (
                what, e, "fisher" if fisher_e[e] else "raw", int(bad.sum()), bad.size, idx.tolist(),
                g[tuple(idx.T)].tolist(), ref[tuple(idx.T)].tolist(), r[tuple(idx.T)].tolist()))
        if self_j is not None:
            c = chain_self[:, e].astype(np.float64)
            want = fz(c) if fisher_e[e] else c
            d = np.abs(g[ii, self_j] - want)
            lim = 1e-5 + (2.0 ** -11 * np.abs(want) if half else 0.0)
            assert np.all(d <= lim), "%s: self column, epoch %d: max %g" % (what, e, d.max())
    return stats


# ------------------------------------------------------------------------------- a: raw r over a shape sweep
def _case_list(prec):
    """(name, V, V2 or None (one mask), T or list of T_e, E, start, nb)."""
    ts = [1, 2, 15, 16, 17, 63, 64, 65, 127, 128, 129, 200, 500]
    if prec in ("tf32x3", "tf32"):
        ts += [7, 8, 9, 31, 32, 33]
    cases = []
    for T in ts:
        cases.append(("T%d_self" % T, 300, None, T, 3, 17, 260))
        cases.append(("T%d_two" % T, 300, 333, T, 3, 5, 290))
    cases.append(("ragged_self", 300, None, [200, 129, 64, 17], 4, 0, 300))
    cases.append(("ragged500_self", 300, None, [500, 333, 65, 499], 4, 40, 257))
    for V2 in (1, 127, 128, 129, 255, 256, 257, 385):
        cases.append(("V2_%d_two" % V2, 300, V2, 65, 3, 0, 300))
        cases.append(("V_%d_self" % V2, V2, None, 65, 3, 0, V2))
    for start, nb in ((0, 1), (255, 2), (100, 256), (3, 257), (599, 1)):
        cases.append(("rows%d+%d_self" % (start, nb), 600, None, 129, 3, start, nb))
        cases.append(("rows%d+%d_two" % (start, nb), 600, 333, 129, 3, start, nb))
    return cases


_DATA = {}


def _case_data(V, V2, T, E):
    """Seeded epochs (unit-norm columns) and their fp64 / fp32-chain references, shared by every precision."""
    key = (V, V2, tuple(T) if isinstance(T, list) else T, E)
    if key not in _DATA:
        lens = T if isinstance(T, list) else [T] * E
        rng = np.random.RandomState((V * 1009 + (V2 or 0) * 31 + sum(lens) * 7 + E) % (2 ** 31))
        d1 = [unit_columns(rng, t, V) for t in lens]
        d2 = [unit_columns(rng, t, V2) for t in lens] if V2 else None
        _DATA[key] = (d1, d2, {})
    return _DATA[key]


def _refs(d1, d2, start, nb, cache):
    if (start, nb) not in cache:
        cache[(start, nb)] = (orc.corr_block(d1, d2, start, nb, f64=True), orc.corr_block(d1, d2, start, nb, f64=False))
    return cache[(start, nb)]


def _guarded_call(ra, rb, start, nb, layout, ld, E, V2, dev, fisher_epochs=0):
    """corr_block into a view of a NaN-filled buffer with guard regions; checks that nothing outside [nb][E][V2]
    (guards, pad columns of the pitch ld) was written and returns the [nb, E, V2] result in that order."""
    G = 4096
    n = nb * E * ld
    buf = torch.full((G + n + G,), NAN, dtype=torch.float32, device=dev)
    shape = (nb, E, ld) if layout == 0 else (E, nb, ld)
    out = buf[G:G + n].view(shape)
    got = engine.corr_block(ra, rb, start, nb, layout=layout, fisher_epochs=fisher_epochs, out=out, ld=ld)
    torch.cuda.synchronize()
    assert got.shape == shape[:2] + (V2,)
    assert torch.isnan(buf[:G]).all() and torch.isnan(buf[G + n:]).all(), "write outside the output"
    if ld > V2:
        assert torch.isnan(out[..., V2:]).all(), "write into the pad columns of the output pitch"
    g = got.cpu().numpy()
    return np.transpose(g, (1, 0, 2)) if layout == 1 else g


@pytest.mark.parametrize("prec", PRECS)
def test_raw_r_shape_sweep(dev, prec):
    """Raw r, element by element, with T across the k-block edges (16-bit modes: 64 TRs per k-block, a partial last
    block when Kp % 64 != 0; tf32 modes: 32), V2 and (start, nb) across the 128 / 256 tile edges, one and two masks,
    both layouts, an output pitch ld = V2 + 37 and guard regions; self-correlation entries bit-identical to the
    sequential fp32 chain (the packer accumulates them across 64-row slabs), ragged epochs included."""
    worst = {}
    for name, V, V2, T, E, start, nb in _case_list(prec):
        d1, d2, cache = _case_data(V, V2, T, E)
        r64, r32 = _refs(d1, d2, start, nb, cache)
        tol = tol_for(prec, r64, r32)
        ep1, T_e = engine.stack_epochs(d1, dev)
        ra = engine.pack_epochs(ep1, T_e, prec)
        rb = engine.pack_epochs(engine.stack_epochs(d2, dev)[0], T_e, prec) if d2 else ra
        n2 = r64.shape[2]
        self_j = None if d2 else start + np.arange(nb)
        for layout, ld in ((0, n2 + 37), (1, n2)):
            got = _guarded_call(ra, rb, start, nb, layout, ld, E, n2, dev)
            st = check_values(got, r64, [False] * E, tol, self_j, None if d2 else r32[np.arange(nb), :, self_j],
                              what="%s %s layout %d" % (prec, name, layout))
            if self_j is not None:
                ii = np.arange(nb)
                assert np.array_equal(got[ii, :, self_j], r32[ii, :, self_j]), "%s: diagonal != fp32 chain" % name
            worst[name] = (max(worst.get(name, (0, 0))[0], st["raw"]), tol)
    big = {k: v for k, v in worst.items() if k.startswith(("T500", "T200", "ragged500"))}
    print("%s max|dr| (tol): %s" % (prec, {k: "%.2e (%.1e)" % v for k, v in big.items()}))
    print("%s max|dr| over all %d cases: %.2e" % (prec, len(worst), max(v[0] for v in worst.values())))


@pytest.mark.parametrize("prec", PRECS)
def test_raw_r_many_tiles_per_cta(dev, prec):
    """E = 64, V = V2 = 600, T = 500: 576 tiles of 256 x 256 on the persistent grid (66 CTA pairs on an H100 SXM), so
    every CTA runs several tiles and the stage ring wraps inside and across tiles; fp64 reference on the device."""
    V, T, E = 600, 500, 64
    rng = np.random.RandomState(600)
    d = [unit_columns(rng, T, V) for _ in range(E)]
    ep, T_e = engine.stack_epochs(d, dev)
    x = ep.double()
    r64 = torch.einsum("eti,etj->iej", x, x).cpu().numpy()
    # the fp32 chain at this shape (k_corr_simt is bit-identical to it) for the faithful tolerance
    r32 = engine.corr_block_f32(ep, ep, 0, V).cpu().numpy()
    tol = tol_for(prec, r64, r32)
    op = engine.pack_epochs(ep, T_e, prec)
    ii = np.arange(V)
    for layout in (0, 1):
        got = _guarded_call(op, op, 0, V, layout, V, E, V, dev)
        st = check_values(got, r64, [False] * E, tol, ii, r32[ii, :, ii], what="%s many tiles layout %d" % (prec, layout))
    print("%s E=64 T=500 max|dr| %.2e (tol %.1e)" % (prec, st["raw"], tol))


# ------------------------------------------------------------------------------- b: the Fisher epilogue
RHOS = (0.34, 0.349, 0.351, 0.36, 0.9, 0.99, 0.999, 0.9999)


def _planted_epochs(V, T, E, seed):
    """Centred unit-norm columns with voxel pairs planted at r = +-RHOS, one exact duplicate and one exact negation
    (every epoch, different vectors, same voxels).  Returns the epochs and the planted (a, b, rho) triples."""
    rng = np.random.RandomState(seed)
    idx = rng.permutation(V)[:2 * (2 * len(RHOS) + 2)].reshape(-1, 2)
    pairs = [(int(a), int(b), s * rho) for (a, b), (s, rho) in zip(idx, [(s, r) for s in (1, -1) for r in RHOS])]
    dup, neg = idx[-2], idx[-1]
    data = []
    for _ in range(E):
        m = unit_columns(rng, T, V, center=True).astype(np.float64)
        for a, b, rho in pairs:
            u = m[:, a]
            w = m[:, b] - (m[:, b] @ u) * u
            w /= np.linalg.norm(w)
            m[:, b] = rho * u + np.sqrt(1 - rho * rho) * w
        m = m.astype(np.float32)
        m[:, dup[1]] = m[:, dup[0]]
        m[:, neg[1]] = -m[:, neg[0]]
        data.append(np.ascontiguousarray(m))
    return data, pairs


@pytest.mark.parametrize("prec", ("fp16x3", "tf32x3", "bf16x3"))
@pytest.mark.parametrize("F", (3, 6))
def test_fisher_epilogue_elementwise(dev, prec, F):
    """corr_block(..., fisher_epochs=F): the series form below |r| = 0.35 and the two-logarithm form above (a warp
    block with one large value switches every element to the logarithms), the clamps next to |r| = 1, Fisher-z on
    the fixed-up diagonal, raw r for the epochs >= F."""
    V, T, E = 512, 40, 6
    data, pairs = _planted_epochs(V, T, E, seed=35 + F)
    r64 = orc.corr_block(data, None, 0, V, f64=True)
    r32 = orc.corr_block(data, None, 0, V, f64=False)
    for a, b, rho in pairs:                     # the planted values sit where they are meant to
        assert np.all(np.abs(r64[a, :, b] - rho) < 2e-6 + 1e-3 * (1 - abs(rho))), (rho, r64[a, :, b])
    tol = tol_for(prec, r64, r32)
    ep, T_e = engine.stack_epochs(data, dev)
    op = engine.pack_epochs(ep, T_e, prec)
    ii = np.arange(V)
    fisher = [e < F for e in range(E)]
    for layout in (0, 1):
        got = _guarded_call(op, op, 0, V, layout, V, E, V, dev, fisher_epochs=F)
        st = check_values(got, r64, fisher, tol, ii, r32[ii, :, ii], what="%s F=%d layout %d" % (prec, F, layout))
        assert st["clamp"] == 4 * min(F, E)     # duplicate and negation, both triangles, every Fisher epoch
        for e in range(F, E):
            assert np.array_equal(got[ii, e, ii], r32[ii, e, ii])
    near = {}
    for a, b, rho in pairs:
        for e in range(min(F, E)):
            err = abs(float(got[a, e, b]) - float(fz(r64[a, e, b])))
            near[abs(rho)] = max(near.get(abs(rho), 0.0), err)
    print("%s F=%d tol_r %.1e, max|dz| at planted |r|: %s, raw %.2e" % (
        prec, F, tol, {k: "%.1e" % v for k, v in sorted(near.items())}, st["raw"]))


# ------------------------------------------------------------------------------- c: the fused pipelines' block
def _detile(flat, row_tiles, col_tiles, E):
    """[row_tiles][col_tiles][E][256][256] -> [row_tiles*256, E, col_tiles*256] (float64 numpy)."""
    a = flat[:row_tiles * col_tiles * E * 65536].view(row_tiles, col_tiles, E, 256, 256)
    return a.permute(0, 3, 2, 1, 4).reshape(row_tiles * 256, E, col_tiles * 256).double().cpu().numpy()


def _pipeline_data(V, V2, T, E, dev):
    raw, _ = synthetic.make_epochs(V, T, E, seed=4040)
    raw2 = synthetic.make_epochs(V2, T, E, seed=4041)[0] if V2 else None
    ep, T_e = engine.stack_epochs(raw, dev)
    rows = engine.pack_epochs(ep, T_e, "fp32")
    cols = engine.pack_epochs(engine.stack_epochs(raw2, dev)[0], T_e, rows.precision) if V2 else rows
    return raw, raw2, rows, cols


@pytest.mark.parametrize("two", (False, True))
def test_pipeline_block_readback(dev, two):
    """fcma_voxel_kernels leaves the GEMM's block in the workspace (normalised values are never written back): read it
    back after a single pass, de-tile it and compare every element -- Fisher-z for the epochs < S * eps, raw r for the
    trailing epochs, the chain value (or its Fisher-z) in the self column; raw r everywhere with FISHER_IN_PASS2; the
    fp16 block to an extra 2^-11 |z|."""
    V, T, E, eps, start, nb = 700, 40, 6, 4, 77, 600
    V2 = 530 if two else None
    raw, raw2, rows, cols = _pipeline_data(V, V2, T, E, dev)
    n2 = V2 or V
    r64 = orc.corr_block(raw, raw2, start, nb, f64=True)
    r32 = orc.corr_block(raw, raw2, start, nb, f64=False)
    tol = tol_for(rows.precision, r64, r32)
    S = (E // eps) * eps
    ii = np.arange(nb)
    self_j = None if two else start + ii
    chain = None if two else r32[ii, :, self_j]
    work = engine.Workspace(E, n2, 768, dev)            # one pass: all 600 rows
    for flags in (0, _lib.FLAG_STRIDED_BLOCK, _lib.FLAG_FISHER_IN_PASS2, _lib.FLAG_F16_INTERMEDIATE):
        work.buf.fill_(255)                             # NaN in fp32 and in fp16: unwritten elements show
        engine.voxel_kernels(rows, cols, start, nb, eps, flags=flags, work=work)
        torch.cuda.synchronize()
        half = bool(flags & _lib.FLAG_F16_INTERMEDIATE)
        if flags & _lib.FLAG_STRIDED_BLOCK:
            ld = -(-n2 // 32) * 32
            blk = work.buf.view(torch.float32)[:nb * E * ld].view(nb, E, ld)[..., :n2].double().cpu().numpy()
        else:
            blk = _detile(work.buf.view(torch.float16 if half else torch.float32), -(-nb // 256), -(-n2 // 256), E)
            blk = blk[:nb, :, :n2]
        fisher = [e < S and not (flags & _lib.FLAG_FISHER_IN_PASS2) for e in range(E)]
        st = check_values(blk, r64, fisher, tol, self_j, chain, half=half, what="voxel_kernels flags %d" % flags)
        print("two=%s flags %d: max|dr| %.2e, max|dz| %.2e (tol_r %.1e)" % (two, flags, st["raw"], st["fisher"], tol))


def test_symmetric_pipeline_block_readback(dev):
    """fcma_voxel_kernels_sym: (1) V = 700 in one pass with the column-direction variant -- block A is the whole
    3 x 3 tile square, the tiles below the diagonal filled by the mirrored stores; (2) rows [0, 256) with
    FCMA_FLAG_SYM_TRANSPOSED -- block B, right after A, holds the transposed tiles of the columns [256, 700)."""
    V, T, E, eps = 700, 40, 6, 4
    raw, _, op, _ = _pipeline_data(V, None, T, E, dev)
    r64 = orc.corr_block(raw, None, 0, V, f64=True)
    r32 = orc.corr_block(raw, None, 0, V, f64=False)
    tol = tol_for(op.precision, r64, r32)
    S = (E // eps) * eps
    fisher = [e < S for e in range(E)]
    ii = np.arange(V)
    assert _lib.load().fcma_sym_uses_column_pass(_lib.PREC[op.precision], E, eps, 0) == 1
    work = engine.SymWorkspace(E, V, 768, dev, transposed_copy=False)
    work.buf.fill_(255)
    engine.voxel_kernels_sym(op, 0, V, eps, work=work)
    torch.cuda.synchronize()
    A = _detile(work.buf.view(torch.float32), 3, 3, E)[:V, :, :V]
    st = check_values(A, r64, fisher, tol, ii, r32[ii, :, ii], what="sym one pass, block A")
    print("sym one pass: max|dr| %.2e, max|dz| %.2e (tol_r %.1e)" % (st["raw"], st["fisher"], tol))

    nb = 256
    work = engine.SymWorkspace(E, V, nb, dev, transposed_copy=True)
    work.buf.fill_(255)
    engine.voxel_kernels_sym(op, 0, nb, eps, flags=_lib.FLAG_SYM_TRANSPOSED, work=work)
    torch.cuda.synchronize()
    flat = work.buf.view(torch.float32)
    nt, t256 = 1, 3
    A = _detile(flat, nt, t256, E)[:nb, :, :V]
    ia = np.arange(nb)
    check_values(A, r64[:nb], fisher, tol, ia, r32[ia, :, ia], what="sym transposed, block A")
    B = _detile(flat[nt * t256 * E * 65536:], t256 - nt, nt, E)[:V - nb]          # rows j = 256 .. 699, columns i
    check_values(B, np.ascontiguousarray(np.transpose(r64[:nb, :, nb:], (2, 1, 0))), fisher, tol,
                 what="sym transposed, block B")


# ------------------------------------------------------------------------------- d: data scale
def test_fp32_default_is_faithful_at_any_data_scale(dev):
    """pack_epochs(..., 'fp32') then corr_block: |dr_ij| <= 1e-6 * |x_i| |x_j| per epoch for unit-norm columns scaled
    by s (the fp16 split goes subnormal below |x| ~ 2^-9 and must not be chosen there), and for normalised data with
    8 voxels at a small scale.  The diagonal is the exact chain value (checked above) and is left out.  Explicit
    fp16x3 on data whose x * 2^6 overflows fp16 is refused."""
    V, T, E = 256, 200, 4
    rng = np.random.RandomState(16)
    unit = [unit_columns(rng, T, V) for _ in range(E)]
    cases = [("s=%g" % s, [np.ascontiguousarray(m * np.float32(s)) for m in unit])
             for s in (8.0, 1.0, 2.0 ** -4, 2.0 ** -8, 2.0 ** -12, 2.0 ** -16, 2.0 ** -20)]
    mixed, _ = synthetic.make_epochs(V, T, E, seed=17)
    mixed = [m.copy() for m in mixed]
    for m in mixed:
        m[:, 100:108] *= np.float32(2.0 ** -14)
    cases.append(("mixed", mixed))
    off = ~np.eye(V, dtype=bool)
    failed = []
    for name, data in cases:
        ep, T_e = engine.stack_epochs(data, dev)
        op = engine.pack_epochs(ep, T_e, "fp32")
        got = engine.corr_block(op, op, 0, V).cpu().numpy().astype(np.float64)
        r64 = orc.corr_block(data, None, 0, V, f64=True)
        worst = 0.0
        for e in range(E):
            nrm = np.linalg.norm(data[e].astype(np.float64), axis=0)
            rel = np.abs(got[:, e] - r64[:, e]) / np.outer(nrm, nrm)
            worst = max(worst, float(rel[off].max()))
        print("%s (%s): max |dr| / (|x_i| |x_j|) = %.2e" % (name, op.precision, worst))
        if not worst <= 1e-6:
            failed.append("%s: %s gives %.2e" % (name, op.precision, worst))
    assert not failed, "normwise error above 1e-6: " + "; ".join(failed)
    big = torch.full((2, 16, 64), 1024.0, device=dev)
    with pytest.raises(ValueError):
        engine.pack_epochs(big, None, "fp16x3")
    assert engine.pack_epochs(big, None, "fp32").precision == "tf32x3"
    ok = torch.full((2, 16, 64), 1000.0, device=dev)          # 64 * 1000 < 65504: still representable
    op = engine.pack_epochs(ok, None, "fp16x3")
    assert torch.isfinite(engine.corr_block(op, op, 0, 64)).all()
