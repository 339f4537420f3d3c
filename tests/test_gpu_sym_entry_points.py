"""The two entry points the benchmark's symmetric step runs through, against the device pipeline on the same tiles:

* ``fcma_host_voxel_kernels_sym`` (host epochs in, host kernels out): the epochs go up in four groups on a copy stream (one
  when E < 4), each group is packed and multiplied as it lands, and each pass's rows of K are read back on that stream;
* ``fcma_voxel_kernels_sym_grouped`` (epochs still arriving on the device, EpochExchange.gather_groups): one packing and one
  GEMM launch per epoch group, the diagonal fix-up with the last group, and with room for two blocks the GEMMs of passes
  0 and 1 both follow the upload.

Both run the same kernels on the same tiles as ``fcma_voxel_kernels_sym`` with the same pass partition (R rows per pass,
asserted through ``fcma_sym_rows_per_pass``), so the device pipeline -- pinned element by element to fp64 by
test_gpu_corr_gemm.py, test_gpu_norm_syrk.py and test_gpu_parity.py -- is the reference:

* E <= 32: bit for bit.  The R <= 4 row kernel reduces across warps in a fixed order and the column kernels use no atomics.
* E > 32: the R = 8 row kernel (k_norm_syrk) adds its 8 warps' accumulators into shared memory with atomics in no fixed
  order.  Everything else is the same on both sides: the leaves of each entry's sum (a warp's MMA accumulator at a flush,
  a column kernel's segment fold) are identical values, only the order in which the atomics add them differs.  Row i of a
  pass's block has n2 columns, ceil(n2 / 32) chunks of 32, dealt to the 8 warps round robin; a warp flushes every FLUSH = 8
  of its trips and once at the end, so one row-pass result is the sum of A(n2) = 8 (floor(trips / 8) + 1) atomic terms,
  trips = ceil(ceil(n2 / 32) / 8).  K[j] then takes one addition per contribution across passes: its own row pass (block
  A, n2 = V - a), one row pass of each earlier pass's transposed copy (n2 = that pass's rows), or the ceil(n / 1024)
  segment folds of each earlier pass's 64-epoch column kernel (COLS_WIDE).  A leaf of K[j] so passes through at most
  m = max A + (number of contributions) additions, and each side's sum differs from the exact sum of the common leaves
  by at most gamma_m sum|leaves|, gamma_m = m u / (1 - m u), u = 2^-24.  By Cauchy-Schwarz
  sum|leaves| <= sum_j |z_aj z_bj| <= sqrt(K_aa K_bb), taken from the reference's diagonal, so
  |K - K_ref| <= 2 gamma_m sqrt(K_aa K_bb)  (the 1 / (1 - m u) also covers the rounding of K_aa, K_bb themselves).

Every case with an fp32 block (fp16x3, tf32x3) is also anchored to the fp64 oracle on three 32-row samples (the first
pass, a pass boundary, the ragged tail) within test_gpu_parity.py's k_tol (1e-2 at eps = 2, where the z-score of two
values is a step function), with the self column masked: where a case keeps its self column, r = 1 +- ulp there and its
z-score is rounding noise in any fp32 pipeline, so the anchor is taken on the same pipeline run with FLAG_MASK_SELF.

Measured on one H100 80GB HBM3 (700 W power limit): largest fraction of the E > 32 bound used 0.23 (0.19 .. 0.23 over the
host wide48 / wide64_cols and grouped E = 48, 64 cases); the whole file runs in about 30 s.
"""
import numpy as np
import pytest
import torch

from brainiak_b200 import _lib
from brainiak_b200.fcma import engine, synthetic
from brainiak_b200.fcma.exchange import EpochExchange, epoch_groups
from oracle import fcma_oracle as orc
from test_gpu_parity import k_tol, zero_self

pytestmark = pytest.mark.gpu

NAN = float("nan")
U = 2.0 ** -24
FLUSH = 8             # k_norm_syrk: trips between flushes of a warp's MMA accumulators
WARPS = 8             # k_norm_syrk: warps per row, chunks dealt round robin
CHUNK = 32            # k_norm_syrk: columns per chunk
COLS64_SEGMENT = 16 * 64   # k_norm_syrk_cols64: rows between folds into K (COLS_SEG_STEPS 16-row steps)
DELAY = 1 << 20       # cycles of the delay kernel in front of each group's upload (~0.5 ms at 1.98 GHz)
STATS = {}


@pytest.fixture(scope="module")
def dev():
    assert _lib.device_count() > 0, "no sm_90 device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    for k, v in sorted(STATS.items()):
        print("symmetric entry points %s: %.3g of the bound" % (k, v))


def cdiv(a, b):
    return -(-a // b)


def make_raw(V, T, E, seed, ragged):
    raw, _ = synthetic.make_epochs(V, T, E, seed=seed)
    if ragged:
        raw = [np.ascontiguousarray(m[:T - 3 * (e % 4)]) for e, m in enumerate(raw)]
    return raw


def packed(raw, dev, prec, normalize):
    ep, T_e = engine.stack_epochs(raw, dev)
    return ep, engine.pack_epochs(ep, T_e, prec, normalize=bool(normalize))


def uses_cols(op, eps, flags):
    return bool(_lib.load().fcma_sym_uses_column_pass(_lib.PREC[op.precision], op.E, eps, flags))


def rows_per_pass(op, eps, flags, start, nbytes):
    return _lib.load().fcma_sym_rows_per_pass(_lib.PREC[op.precision], op.E, eps, flags, op.V, start, nbytes)


def device_sym(op, shards, eps, flags, R):
    """The reference: fcma_voxel_kernels_sym over the shards, R rows per pass, NaN-filled scratch, one K."""
    K = torch.zeros((op.V, op.E, op.E), dtype=torch.float32, device=op.device)
    for s, n in shards:
        work = engine.SymWorkspace.for_operand(op, R, eps, flags, s)
        work.buf.view(torch.float32).fill_(NAN)
        assert rows_per_pass(op, eps, flags, s, work.buf.numel()) == R
        engine.voxel_kernels_sym(op, s, n, eps, flags=flags, work=work, out=K)
    torch.cuda.synchronize()
    assert torch.isfinite(K).all()
    return K


def atomic_terms(n2):
    trips = cdiv(cdiv(n2, CHUNK), WARPS)
    return WARPS * (trips // FLUSH + 1)


def additions(V, shards, R, cols):
    """m of the module docstring for every row of K: the most atomic terms of one row-pass result that reaches the row plus
    the number of contributions the row receives across the passes of all shards."""
    A = np.zeros(V, np.int64)
    C = np.zeros(V, np.int64)
    for s, n in shards:
        for a in range(s, s + n, R):
            n_p = min(R, s + n - a)
            A[a:a + n_p] = np.maximum(A[a:a + n_p], atomic_terms(V - a))
            C[a:a + n_p] += 1
            if cols:
                C[a + n_p:] += cdiv(n_p, COLS64_SEGMENT)
            else:
                A[a + n_p:] = np.maximum(A[a + n_p:], atomic_terms(n_p))
                C[a + n_p:] += 1
    return A + C


def where(row, shards, R):
    for s, n in shards:
        if s <= row < s + n:
            return "row pass %d of the shard at %d" % ((row - s) // R, s)
    return "no shard's row passes (column contributions only)"


def compare(got, ref, shards, R, cols, what):
    """E <= 32: bit for bit; E > 32: within 2 gamma_m sqrt(K_aa K_bb).  Returns the fraction of the bound used (0 if equal)."""
    E = ref.shape[1]
    if E <= 32:
        if torch.equal(got, ref):
            return 0.0
        bad = torch.nonzero(~(got == ref))[0].tolist()
        row, a, b = bad
        raise AssertionError("%s: first difference at K[%d, %d, %d] (%s): %r != %r, %d entries differ"
                             % (what, row, a, b, where(row, shards, R), float(got[row, a, b]), float(ref[row, a, b]),
                                int((~(got == ref)).sum())))
    assert torch.isfinite(got).all(), what
    m = torch.from_numpy(additions(ref.shape[0], shards, R, cols)).to(ref.device)
    mu = m.to(torch.float64) * U
    gamma = (mu / (1 - mu))[:, None, None]
    d = torch.diagonal(ref, dim1=1, dim2=2).to(torch.float64).clamp_min(0)
    lim = 2 * gamma * torch.sqrt(d[:, :, None] * d[:, None, :])
    diff = (got.to(torch.float64) - ref.to(torch.float64)).abs()
    assert bool((diff[lim == 0] == 0).all()), what
    frac = float((diff / lim.clamp_min(1e-300)).max())
    if frac > 1:
        idx = int(torch.argmax(diff / lim.clamp_min(1e-300)))
        row, a, b = idx // (E * E), (idx // E) % E, idx % E
        raise AssertionError("%s: K[%d, %d, %d] (%s) differs by %.3g of its bound" % (what, row, a, b,
                                                                                       where(row, shards, R), frac))
    return frac


def check(got, ref, op, eps, flags, shards, R, what):
    frac = compare(got, ref, shards, R, uses_cols(op, eps, flags), what)
    if op.E > 32:
        STATS[what] = max(STATS.get(what, 0.0), frac)


def anchor(K, raw, normalize, eps, rows, col0):
    """fp64 oracle on 32-row samples starting at `rows`; `K` was computed with the self column masked over the columns
    [col0, V) (a shard that starts at row col0 contracts its rows with those columns only)."""
    ref_raw = [orc.epoch_normalize(m) for m in raw] if normalize else raw
    V = raw[0].shape[1]
    for s0 in rows:
        _, z, _ = orc.voxel_block(ref_raw, None, s0, 32, eps, shrink=False)
        Kref = orc.kernel_matrices(np.ascontiguousarray(zero_self(z, s0)[:, :, col0:]), f64=True)
        got = K[s0:s0 + 32].cpu().numpy()
        # eps = 2: the z-score of two values is a step function (test_gpu_parity.py: measured 4.5e-3 of max(|K|, V))
        scale = max(np.max(np.abs(Kref)), float(V))
        err = np.max(np.abs(got - Kref)) / scale
        assert err <= (1e-2 if eps <= 2 else k_tol(V)), (s0, err)


def anchor_rows(V, start, R):
    """first pass, the boundary between the first two passes, the ragged tail"""
    return [start, min(start + R, V - 32) - 16, V - 32]


def anchor_case(K, op, raw, normalize, eps, flags, shards, R):
    if op.precision not in ("fp16x3", "tf32x3"):
        return                                # fp16 block / bf16x3: pinned elsewhere; bit identity is the check here
    if not flags & _lib.FLAG_MASK_SELF:
        K = device_sym(op, shards, eps, flags | _lib.FLAG_MASK_SELF, R)
    anchor(K, raw, normalize, eps, anchor_rows(op.V, shards[0][0], R), shards[0][0])


# ------------------------------------------------------------------------------------- fcma_host_voxel_kernels_sym
MS, TMA, WIDE = _lib.FLAG_MASK_SELF, _lib.FLAG_COLS_TMA, _lib.FLAG_COLS_WIDE
HOST_CASES = {
    # id: V, T, E, eps, precision, flags, R (0: the entry point's own choice), ragged, normalize
    "bench32": (2600, 60, 32, 8, "fp16x3", 0, 512, False, 0),
    "bench32_masked_tma": (2600, 60, 32, 8, "fp16x3", MS | TMA, 512, False, 0),
    "ragged_norm": (1300, 50, 12, 4, "tf32x3", 0, 256, True, 1),
    "odd_groups": (900, 40, 6, 2, "bf16x3", MS, 256, False, 0),          # upload groups of 1, 1, 2, 2 epochs
    "one_group": (600, 40, 3, 2, "fp16x3", 0, 256, False, 0),            # E < 4: one group; epoch 2 outside a subject
    "e16": (1100, 40, 16, 16, "fp16x3", 0, 256, False, 0),               # 16-epoch column kernel
    "f16_block": (1400, 40, 24, 8, "bf16", 0, 512, False, 0),            # fp16 Fisher-z block, column pass
    "wide48": (1100, 30, 48, 16, "fp16x3", 0, 256, False, 0),            # transposed copy B + row pass
    "wide64_cols": (900, 30, 64, 8, "tf32x3", WIDE, 256, False, 0),      # 64-epoch column kernel
    "single_pass": (700, 40, 32, 8, "fp16x3", 0, 0, False, 0),           # one pass of one block
}


@pytest.mark.parametrize("case", list(HOST_CASES))
def test_host_entry_point(dev, case):
    """fcma_host_voxel_kernels_sym == fcma_voxel_kernels_sym with the same pass partition, into a pinned tensor (from a
    pinned epoch tensor when the epochs are equal) and into a pageable numpy array; every element of `out` is written
    and the caller's device is restored."""
    V, T, E, eps, prec, flags, R, ragged, normalize = HOST_CASES[case]
    raw = make_raw(V, T, E, 7000 + E + V, ragged)
    ep, op = packed(raw, dev, prec, normalize)
    assert op.precision == prec
    # the entry point's own choice: every row in one block when it fits
    R_ref = R or cdiv(V, 256) * 256
    K = device_sym(op, [(0, V)], eps, flags, R_ref)
    torch.cuda.set_device(dev)
    pinned = torch.full((V, E, E), NAN, dtype=torch.float32).pin_memory()
    src = raw if ragged else torch.from_numpy(np.stack(raw)).pin_memory()
    engine.host_voxel_kernels_sym(src, eps, precision=prec, normalize=bool(normalize), flags=flags, device=dev.index,
                                  rows_per_pass=R, out=pinned)
    assert torch.cuda.current_device() == dev.index
    pageable = np.full((V, E, E), NAN, np.float32)
    engine.host_voxel_kernels_sym(raw, eps, precision=prec, normalize=bool(normalize), flags=flags, device=dev.index,
                                  rows_per_pass=R, out=pageable)
    assert torch.cuda.current_device() == dev.index
    Kc = K.cpu()
    for name, out in (("pinned", pinned), ("pageable", torch.from_numpy(pageable))):
        assert not torch.isnan(out).any(), "%s: %d entries of out are NaN" % (name, int(torch.isnan(out).sum()))
        check(out, Kc, op, eps, flags, [(0, V)], R_ref, "host %s (%s out)" % (case, name))
    anchor_case(K, op, raw, normalize, eps, flags, [(0, V)], R_ref)


# ------------------------------------------------------------------------------------- fcma_voxel_kernels_sym_grouped
def uneven(E):
    return [(0, 1), (1, E - 3), (E - 2, 2)]


GROUPED_CASES = {
    # id: V, T, E, eps, precision, flags, groups, shards ("partition": the two of sym_row_partition), two blocks, normalize
    "e32_whole": (1300, 40, 32, 8, "fp16x3", 0, "whole", 0, True, 0),
    "e32_uneven_start512_masked": (1300, 40, 32, 8, "fp16x3", MS, "uneven", 512, False, 1),
    "e16_subject_cuts_shards": (1100, 40, 16, 4, "tf32x3", 0, [(0, 3), (3, 6), (9, 7)], "partition", True, 0),
    "e48_subject_cuts_start512": (1100, 30, 48, 16, "fp16x3", 0, [(0, 20), (20, 20), (40, 8)], 512, True, 1),
    "e64_single_epochs_cols_wide": (900, 30, 64, 8, "tf32x3", WIDE, "single", 0, True, 0),
    "e64_whole_shards": (900, 30, 64, 16, "fp16x3", 0, "whole", "partition", False, 1),
    "f16_block_uneven_shards": (1400, 40, 24, 8, "bf16", 0, "uneven", "partition", False, 0),
}


def arrive(buf, host, groups, dev):
    """NaN-fill the epoch buffer, then upload each group on a stream of its own behind a delay kernel (later groups later)
    and record its event: a launch that does not wait for its group reads NaN."""
    buf.fill_(NAN)
    cur = torch.cuda.current_stream(dev)
    events = []
    for g, (e0, c) in enumerate(groups):
        s = torch.cuda.Stream(device=dev)
        s.wait_stream(cur)
        with torch.cuda.stream(s):
            torch.cuda._sleep(DELAY * (g + 1))
            buf[e0:e0 + c].copy_(host[e0:e0 + c], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(s)
        events.append(ev)
    return events


def grouped_case(dev, what, V, T, E, eps, prec, flags, layout, shards, two, normalize):
    """fcma_voxel_kernels_sym_grouped == fcma_voxel_kernels_sym over the same shards and pass partition, with the epochs
    arriving group by group into a NaN-filled buffer and packed into a NaN-filled operand."""
    raw = make_raw(V, T, E, 555 if layout == "exchange" else 9000 + E + V, False)
    ep, op = packed(raw, dev, prec, normalize)
    host = torch.from_numpy(np.stack(raw)).pin_memory()
    shards = engine.sym_row_partition(V, 2) if shards == "partition" else [(shards, V - shards)]
    if isinstance(layout, list):
        groups = layout
    elif layout != "exchange":        # gather_groups returns its own four groups
        groups = {"whole": [(0, E)], "uneven": uneven(E), "single": [(e, 1) for e in range(E)]}[layout]
    R = 256
    K_ref = device_sym(op, shards, eps, flags, R)
    K = torch.zeros_like(K_ref)
    assert not two or max(n for _, n in shards) > R        # two blocks: passes 0 and 1 both follow the upload
    for s, n in shards:
        op2 = engine.PackedOperand(torch.full_like(op.buf, 0xFF), E, T, V, op.precision, op.T_e)
        work = engine.SymWorkspace.for_operand(op, (2 if two else 1) * R, eps, flags, s)
        work.buf.view(torch.float32).fill_(NAN)
        assert rows_per_pass(op, eps, flags, s, work.buf.numel() // (2 if two else 1)) == R
        if layout == "exchange":
            x = EpochExchange(E, T, V, dev, nbuf=1)
            assert x.interleaved_share() == list(range(E)) and epoch_groups(E, 4) == [(0, 2), (2, 2), (4, 2), (6, 2)]
            x.buffers[0].fill_(NAN)
            cs = torch.cuda.Stream(device=dev)
            cs.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(cs):
                torch.cuda._sleep(DELAY)
            buf, groups, events = x.gather_groups(0, host, stream=cs, ngroups=4)
        else:
            buf = torch.empty_like(ep)
            events = arrive(buf, host, groups, dev)
        engine.voxel_kernels_sym_grouped(buf, op2, s, n, eps, groups, events, flags=flags, work=work, out=K,
                                         normalize=bool(normalize))
    torch.cuda.synchronize()
    check(K, K_ref, op, eps, flags, shards, R, "grouped %s" % what)
    anchor_case(K, op, raw, normalize, eps, flags, shards, R)


@pytest.mark.parametrize("case", list(GROUPED_CASES))
def test_grouped_entry_point(dev, case):
    grouped_case(dev, case, *GROUPED_CASES[case])


def test_grouped_symmetric_pipeline_follows_arriving_epochs(dev):
    """The production caller, EpochExchange.gather_groups (four groups of two epochs, behind a delay on the copy stream),
    feeding the grouped entry point with two blocks of workspace: a shard that starts at row 0 and one that starts at 512."""
    for start in (0, 512):
        grouped_case(dev, "exchange start %d" % start, 1100, 40, 8, 4, "fp16x3", MS, "exchange", start, True, 0)


def test_grouped_entry_point_arguments(dev):
    """No events (the epochs are all there) in one group equals the device pipeline; groups that do not tile [0, E), more
    than 64 groups and a packed-operand buffer below the operand's size are refused."""
    V, T, E, eps = 1100, 40, 8, 4
    raw = make_raw(V, T, E, 556, False)
    ep, op = packed(raw, dev, "fp16x3", 0)
    op2 = engine.PackedOperand(torch.full_like(op.buf, 0xFF), E, T, V, op.precision, op.T_e)
    K = engine.voxel_kernels_sym_grouped(ep, op2, 0, V, eps, [(0, E)], [None], flags=MS,
                                         work=engine.SymWorkspace.for_operand(op, 256, eps, MS))
    assert torch.equal(K, device_sym(op, [(0, V)], eps, MS, 256))
    with pytest.raises(ValueError, match="cover"):
        engine.voxel_kernels_sym_grouped(ep, op2, 0, V, eps, [(0, 3), (4, 4)], [None, None])
    with pytest.raises(ValueError, match="cover"):
        engine.voxel_kernels_sym_grouped(ep, op2, 0, V, eps, [(0, 3), (3, 4)], [None, None])
    with pytest.raises(ValueError, match="bad arguments"):
        engine.voxel_kernels_sym_grouped(ep, op2, 0, V, eps, [(0, 1)] * 65, [None] * 65)
    small = engine.PackedOperand(op2.buf[:-16], E, T, V, op.precision, op.T_e)
    with pytest.raises(MemoryError):
        engine.voxel_kernels_sym_grouped(ep, small, 0, V, eps, [(0, E)], [None])
