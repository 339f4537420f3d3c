"""Element-wise tests of the pipelines past 32-bit element offsets: correlation blocks, packed operands and kernel arrays
of more than 2^31 elements, checked where their last part lies past element offset 2^31 (and past byte offset 2^32
where the type allows).

The fused pipelines size their scratch from free device memory (up to 4096 block rows, tens of GB): one tiled block at
the benchmark's shape (V = 50 000, E = 32, 4096 rows) holds 6.6e9 elements.  An offset computed in 32 bits, or wrapped in
a TMA descriptor, shows only at such sizes.  Every case below builds one buffer whose last part lies past 2^31 elements,
picks the rows, epochs or items that live there, checks them element by element against a plain fp64 reference and,
where it is cheap, checks that they are bit-identical to the same items computed by a small call whose buffers stay
below 2^31.  Each assertion message names the element offsets its items reach.

References and bounds (the helpers are imported from the files that define them):
* correlation block read back from the workspace: ``check_values`` of test_gpu_corr_gemm.py against the fp64
  contraction of the float32 epochs on the device, ``tol_r = max(1e-6, 2 e32)`` with e32 the error of the sequential
  fp32 chain (``corr_block_f32``, bit-identical to it), Fisher-z to ``2 tol_r / (1 - r^2) + 1e-6 (1 + |z|)``, the fp16
  block to an extra ``2^-11 |z|``, the self column against the chain value;
* kernel matrices: ``check_K`` of test_gpu_norm_syrk.py against ``Ref.of_block`` of the block read back from the
  workspace (rows: dim 2; column voxels of the symmetric column pass: dim 0), ``|K - K16| <= C_A u S + F``;
  ``classifier_kernel``: the same bound summed over every row, plus ``2 u |K16|`` for its one fp32 rounding, against the
  per-row ``Ref`` kernels of standalone ``corr_block`` rows (no workspace, no pipeline);
* fp64 feature kernels: ``_check_against_exact`` of test_gpu_feature_svc_wide.py (error-free sums of the fp64 products
  of ``within_subject_norm_(corr_block(...))`` of the same rows, ``gamma_n sum |z_a z_b| + u |G|``), moments with
  ``_check_moments`` of test_gpu_svc_scale.py (hi within an ulp of ``math.fsum``, hi + lo within 2^-100 sum |x|);
* packed operand: planes bit for bit against ``split_planes`` and the diagonal against the sequential fp32 chain of the
  C oracle (``expected_operand`` of test_gpu_pack_and_side_kernels.py), ``normalize = 1`` against
  ``epoch_normalize_`` of the same columns; ``corr_block`` of the last rows with ``check_values``;
* searchlight kernels: ``math.fsum`` of the fp64 products of each centre's features, ``gamma_n sum |x_a x_b| + u |G|``
  (the linear bound of test_gpu_mvpa_wide.py); kernel arrays under ``subset_kernels`` bit for bit against torch
  indexing and the decimal shrink (``K * float32(10^(2 - nd))``, nd the digits of the compacted K00); the solvers'
  accuracies and iteration counts equal to those of a call on a small copy of the same items.

Every check would fail on a wrap: the data are random, so the values 2^31 elements before a sampled item belong to other
rows, epochs or items and differ from its reference by far more than the bounds (order 0.1 against 1e-6 for r).
``test_fused_pipeline_block_past_2_31`` asserts this once on the device: the tiled block 2^31 elements before the last
row block fails the reference of that row block almost everywhere.

Coverage:

| kernel                                      | buffer past 2^31 elements                         | covered by                                    |
|---------------------------------------------|---------------------------------------------------|-----------------------------------------------|
| k_corr_wgmma TMA stores (fp32 / fp16 tiled) | 4096-row block, last row block at 2.49e9          | test_fused_pipeline_block_past_2_31           |
| k_corr_wgmma strided stores                 | [4096][32][20000] block, last row block at 2.46e9 | test_fused_pipeline_block_past_2_31[strided]  |
| k_self_corr_fixup                           | the same blocks (self column of the last rows)     | test_fused_pipeline_block_past_2_31           |
| k_norm_syrk row pass (VEC 1, 2, FISHER)     | the same blocks                                   | test_fused_pipeline_block_past_2_31           |
| k_corr_wgmma symmetric (mirrored tiles)     | block A, 4096 x 20096 x 32                        | test_symmetric_pipeline_past_2_31             |
| k_norm_syrk_cols<8, 4, 0> column pass       | block A, last column tiles in row blocks >= 12    | test_symmetric_pipeline_past_2_31[cols]       |
| transposed copy (block B) + row pass        | block B, starts at 2.21e9                         | test_symmetric_pipeline_past_2_31[transposed] |
| k_norm_syrk_cols64 (FCMA_FLAG_COLS_WIDE)    | block A at E = 64, 2.95e9 elements                | test_symmetric_pipeline_past_2_31[wide]       |
| fcma_classifier_kernel_sym (fp64 sums)      | first pass's block A, 2.65e9 elements             | test_symmetric_pipeline_past_2_31[cols]       |
| k_block_within_subject_norm, k_block_moments | E = 140 block, last row block at 2.18e9          | test_feature_route_past_2_31                  |
| k_feature_gram_tiled<1> (+ rbf epilogue)    | the same block                                    | test_feature_route_past_2_31                  |
| k_pack_operand (fp16x3, tf32x3, normalize)  | operand, lo plane of the last epochs at 2.28e9    | test_packed_operand_past_2_31                 |
| k_corr_wgmma operand TMA loads              | the same operands                                 | test_packed_operand_past_2_31                 |
| k_searchlight_kernels_tiled<0>              | fp64 [46208][216][216], 2.16e9 elements           | test_searchlight_kernels_and_solver_past_2_31 |
| k_svm_cv (fp64, wide)                       | the same array                                    | test_searchlight_kernels_and_solver_past_2_31 |
| k_subset_kernels<float, 0 / 1>              | in [34500][256][256], out [34500][250][250]       | test_fp32_kernel_arrays_past_2_31             |
| k_svm_cv (fp32, wide)                       | in [34500][256][256]                              | test_fp32_kernel_arrays_past_2_31             |

Each test allocates at most about 20 GB, skips (naming the bytes it needs) when the device has less free memory, frees
its buffers before it returns and prints its wall time and peak ``torch.cuda.max_memory_allocated``.
"""
import gc
import math
import time

import numpy as np
import pytest
import torch

from brainiak_b200 import _lib
from brainiak_b200.fcma import engine, synthetic
from test_gpu_corr_gemm import check_values, fz, tol_for
from test_gpu_feature_svc import U as U64, _operands
from test_gpu_feature_svc_wide import _check_against_exact
from test_gpu_mvpa import _features
from test_gpu_norm_syrk import U, Ref, _detile, check_K
from test_gpu_pack_and_side_kernels import expected_operand
from test_gpu_svc_scale import _check_moments

pytestmark = pytest.mark.gpu
LIM = 2 ** 31
GB = 1 << 30


@pytest.fixture(scope="module")
def dev():
    assert _lib.device_count() > 0, "no sm_90 device"
    return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def _measure(request):
    """Wall time and peak device memory of the test; the buffers are released afterwards."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print("\n%s: wall %.1f s, peak max_memory_allocated %.2f GB" % (
        request.node.name, time.perf_counter() - t0, torch.cuda.max_memory_allocated() / GB))
    _release()


def _release():
    gc.collect()
    torch.cuda.empty_cache()


def _need(nbytes):
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip("needs %d bytes (%.1f GB) of free device memory, %d free" % (nbytes, nbytes / GB, free))


def _at(off):
    """An element offset as the assertion messages state it."""
    return "element %d (%.3g, %.2f x 2^31)" % (off, off, off / LIM)


def _epochs(V, T, E, dev, seed):
    raw, _ = synthetic.make_epochs(V, T, E, seed=seed)
    ep, T_e = engine.stack_epochs(raw, dev)
    return ep, engine.pack_epochs(ep, T_e, "fp32")


def _r64_rows(ep, rows):
    """fp64 r[i, e, j] of the float32 epochs for the voxel rows ``rows`` (all columns), on the device, as numpy."""
    x = ep.double()
    return torch.einsum("eti,etj->iej", x[:, :, rows], x).cpu().numpy()


# ------------------------------------------------------------------------------- 1: plain fused pipeline
PLAIN_FLAGS = {"default": 0, "f16": _lib.FLAG_F16_INTERMEDIATE, "pass2": _lib.FLAG_FISHER_IN_PASS2,
               "strided": _lib.FLAG_STRIDED_BLOCK}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("case", sorted(PLAIN_FLAGS))
def test_fused_pipeline_block_past_2_31(dev, case):
    """voxel_kernels, one pass of 4096 rows (E = 32, eps = 8, T = 24, V = V2 = 20 000, one mask): the last 256-row block
    lies past 2^31 elements of the workspace.  Its block read back against the fp64 correlations (the GEMM's stores and
    the self-column fix-up), its kernels against Ref of that block (the row pass's loads), and bit-identical to
    voxel_kernels started at that row block with a 256-row workspace."""
    flags = PLAIN_FLAGS[case]
    E, eps, T, V, n = 32, 8, 24, 20000, 4096
    r0 = n - 256
    per_row = _lib.load().fcma_work_bytes_per_row(E, V)
    _need(n * per_row + 6 * GB)
    ep, op = _epochs(V, T, E, dev, seed=3101)
    assert op.precision == "fp16x3"
    work = engine.Workspace(E, V, n, dev)
    work.buf.fill_(255)
    K = engine.voxel_kernels(op, op, 0, n, eps, flags=flags, work=work)
    torch.cuda.synchronize()
    half = bool(flags & _lib.FLAG_F16_INTERMEDIATE)
    pass2 = bool(flags & _lib.FLAG_FISHER_IN_PASS2)
    flat = work.buf.view(torch.float16 if half else torch.float32)
    if flags & _lib.FLAG_STRIDED_BLOCK:
        ld = -(-V // 32) * 32
        off0, span = r0 * E * ld, 256 * E * ld
        blk = flat[off0:off0 + span].view(256, E, ld)[..., :V]
        wrapped = flat[off0 - LIM:off0 - LIM + span].view(256, E, ld)[..., :V]
    else:
        t256 = -(-V // 256)
        off0, span = (r0 // 256) * t256 * E * 65536, t256 * E * 65536
        blk = _detile(flat[off0:], 1, t256, E)[:, :, :V]
        wrapped = _detile(flat[off0 - LIM:], 1, t256, E)[:, :, :V]
    assert off0 > LIM and off0 * flat.element_size() > 2 ** 32
    where = "%s: rows %d-%d, from %s to %s" % (case, r0, n - 1, _at(off0), _at(off0 + span))

    # (a) the block, element by element, on the first and last 32 rows of the row block
    sample = np.r_[0:32, 224:256]
    rows = r0 + sample
    r64 = _r64_rows(ep, torch.as_tensor(rows, device=dev))
    r32 = engine.corr_block_f32(ep, ep, r0, 256).cpu().numpy()[sample]
    tol = tol_for(op.precision, r64, r32)
    fisher = [not pass2] * E                                     # E // eps * eps = E epochs normalised
    got = blk[torch.as_tensor(sample, device=dev)].double().cpu().numpy()
    st = check_values(got, r64, fisher, tol, rows, r32[np.arange(len(rows)), :, rows], half=half,
                      what="block " + where)
    # a wrapped offset would read the block 2^31 elements earlier: other rows' values, far outside the bound
    wr = wrapped[torch.as_tensor(sample, device=dev)].double().cpu().numpy()
    want = fz(r64) if not pass2 else r64
    near = np.abs(wr - want) <= 1e3 * tol + (2.0 ** -11 * np.abs(want) if half else 0.0)
    assert near.mean() < 0.01, "%s: the block 2^31 elements earlier matches the reference at %.3f of its entries" % (
        where, near.mean())

    # (b) the kernels of the whole row block against Ref of the block read back
    ref = Ref.of_block(blk, eps, fisher=pass2, chunk=64)
    check_K(K[r0:n], ref, "row", "kernels " + where)
    # (c) bit-identical to a call whose workspace stays below 2^31 elements
    small = engine.Workspace(E, V, 256, dev)
    K2 = engine.voxel_kernels(op, op, r0, 256, eps, flags=flags, work=small)
    torch.cuda.synchronize()
    assert torch.equal(K[r0:n], K2), "kernels %s differ from a 256-row call in %d entries" % (
        where, int((K[r0:n] != K2).sum()))
    print("%s: max|dr| %.2e, max|dz| %.2e (tol_r %.1e)" % (where, st["raw"], st["fisher"], tol))
    del work, flat, blk, wrapped, K, K2, small, ref


# ------------------------------------------------------------------------------- 2: symmetric pipeline
SYM_CASES = {
    # name: (E, eps, V, flags)
    "cols": (32, 8, 4096 + 16000, 0),                            # column pass, block A 2.65e9 elements
    "transposed": (32, 8, 4096 + 12800, _lib.FLAG_SYM_TRANSPOSED),  # block B from 2.21e9
    "wide": (64, 8, 4096 + 7104, _lib.FLAG_COLS_WIDE),          # k_norm_syrk_cols64, block A 2.95e9 elements
}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("case", sorted(SYM_CASES))
def test_symmetric_pipeline_past_2_31(dev, case):
    """voxel_kernels_sym, one pass of n = 4096 rows over V columns: K[i] of the last row block (row pass over block A's
    last row block), K[j] of the last column tiles (column pass over those tiles in every row block, the far ones past
    2^31), or with FCMA_FLAG_SYM_TRANSPOSED the last column voxels from block B, which starts past 2^31 -- each against
    Ref of the block read back.  "cols" then runs classifier_kernel (fcma_classifier_kernel_sym, fp64 sums) on the same
    operand and workspace, against the fp64 sum of the per-row Ref kernels of standalone corr_block rows."""
    E, eps, V, flags = SYM_CASES[case]
    n = 4096
    nt, t256 = n // 256, -(-V // 256)
    transposed = bool(flags & _lib.FLAG_SYM_TRANSPOSED)
    per_row = (2 if transposed else 1) * _lib.load().fcma_work_bytes_per_row(E, V)
    _need(n * per_row + 3 * GB)
    ep, op = _epochs(V, 24, E, dev, seed=3200 + E + V)
    assert _lib.load().fcma_sym_uses_column_pass(_lib.PREC[op.precision], E, eps, flags) == (not transposed)
    work = engine.SymWorkspace.for_operand(op, n, eps, flags)
    work.buf.fill_(255)
    K = engine.voxel_kernels_sym(op, 0, n, eps, flags=flags, work=work)
    torch.cuda.synchronize()
    flat = work.buf.view(torch.float32)
    tile = E * 65536                                             # elements of one (row block, column tile)
    a_end = nt * t256 * tile
    assert a_end > LIM

    # rows of the last row block
    off = (nt - 1) * t256 * tile
    A_rows = _detile(flat[off:], 1, t256, E)[:, :, :V]
    what = "sym %s E=%d V=%d: rows %d-%d, block A elements from %s to %s" % (case, E, V, n - 256, n - 1, _at(off),
                                                                           _at(off + t256 * tile))
    check_K(K[n - 256:n], Ref.of_block(A_rows, eps, chunk=64), "row", what)
    del A_rows

    if transposed:
        # block B [t256 - nt][nt][E][256 j][256 i]: its last column tile-row = the last 256 column voxels
        jt = t256 - nt - 1
        off = a_end + jt * nt * tile
        B_last = _detile(flat[off:], 1, nt, E)[:, :, :n]
        j0 = n + jt * 256
        what = "sym %s: column voxels %d-%d, block B elements from %s to %s" % (case, j0, V - 1, _at(off),
                                                                              _at(off + nt * tile))
        assert off > LIM
        check_K(K[j0:V], Ref.of_block(B_last[:V - j0], eps, chunk=64), "row", what)
        del B_last
    else:
        # the last two column tiles of block A in every row block: [nt][2][E][256][256] -> [n, E, 512]
        tj0 = t256 - 2
        A = flat[:a_end].view(nt, t256, E, 256, 256)[:, tj0:]
        A_cols = A.permute(0, 3, 2, 1, 4).reshape(n, E, 512)[:, :, :V - tj0 * 256]
        far = [rb for rb in range(nt) if (rb * t256 + tj0) * tile > LIM]
        what = "sym %s E=%d: column voxels %d-%d, read in row blocks %s at or past %s" % (
            case, E, tj0 * 256, V - 1, far, _at((far[0] * t256 + tj0) * tile))
        assert far
        check_K(K[tj0 * 256:V], Ref.of_block(A_cols, eps, dim=0, chunk=256), "cols", what)
        del A, A_cols

    if case == "cols":
        # the summed one-mask kernel from the same workspace: its first pass's block is this block A
        Kc = engine.classifier_kernel(op, op, 0, V, eps, work=work)
        torch.cuda.synchronize()
        del work, flat
        _release()
        K16 = S = F = K64 = free = None
        for s in range(0, V, 256):
            r = engine.corr_block(op, op, s, min(256, V - s), fisher_epochs=E)
            ref = Ref.of_block(r, eps, chunk=128)
            parts = (ref.K16.sum(0), ref.S.sum(0), ref.F.sum(0), ref.K64.sum(0), ref.free.any(0))
            if K16 is None:
                K16, S, F, K64, free = parts
            else:
                K16, S, F, K64, free = K16 + parts[0], S + parts[1], F + parts[2], K64 + parts[3], free | parts[4]
            del r, ref
        tot = Ref(K16[None], S[None], F[None], K64[None], free[None], eps)
        check_K(Kc.view(1, E, E), tot, "row", "classifier_kernel V=%d (first pass block A up to %s)" % (V, _at(a_end)),
                extra=2 * U * K16.abs()[None], bias=False)
        del Kc


# ------------------------------------------------------------------------------- 3: fp64 feature route
@pytest.mark.timeout(900)
def test_feature_route_past_2_31(dev):
    """feature_gram_wide and feature_kernels_f64_wide (rbf), E = 140, eps = 20, 2048 rows against V2 = 8600 columns (two
    masks): the tiled block holds 2.50e9 elements, its last row block starts at 2.18e9.  For the first and last row of
    that block: G, K_fit and K_pred against exact sums of within_subject_norm_(corr_block(...)) of the row, the
    moments against math.fsum; the whole row block bit-identical to a 256-row call, and the linear G of that call equal to
    feature_gram_wide's G."""
    E, eps, T, V, V2, n = 140, 20, 24, 2048, 8600, 2048
    per_row = _lib.load().fcma_work_bytes_per_row(E, V2)
    _need(n * per_row + 4 * n * E * E * 8 + 2 * GB)
    op, op2 = _operands(V, V2, T, E, dev, seed=3300)
    t256 = -(-V2 // 256)
    r0 = n - 256
    off0 = (r0 // 256) * t256 * E * 65536
    assert off0 > LIM
    where = "rows %d-%d, block elements from %s to %s" % (r0, n - 1, _at(off0), _at(off0 + t256 * E * 65536))
    work = engine.Workspace(E, V2, n, dev)
    G, D, mom = engine.feature_gram_wide(op, op2, 0, n, eps, work=work)
    gamma = 0.37 / V2
    Kf, Kp = engine.feature_kernels_f64_wide(op, op2, 0, n, eps, "rbf", gamma, work=work)
    torch.cuda.synchronize()
    del work
    _release()
    for i in (r0, n - 1):
        _check_against_exact(op, op2, i, 1, eps, G[i:i + 1].cpu().numpy(), Kf[i:i + 1].cpu().numpy(),
                             Kp[i:i + 1].cpu().numpy(), gamma, "row %d of %s" % (i, where))
        z = engine.within_subject_norm_(engine.corr_block(op, op2, i, 1).contiguous(), eps).cpu().numpy()
        _check_moments(z.astype(np.float64), mom[i:i + 1].cpu().numpy(), "moments, row %d of %s" % (i, where))
    small = engine.Workspace(E, V2, 256, dev)
    G2, D2, mom2 = engine.feature_gram_wide(op, op2, r0, 256, eps, work=small)
    Kf2, Kp2 = engine.feature_kernels_f64_wide(op, op2, r0, 256, eps, "rbf", gamma, work=small)
    Gl, _ = engine.feature_kernels_f64_wide(op, op2, r0, 256, eps, "linear", work=small)
    torch.cuda.synchronize()
    for name, big, sm in (("G", G, G2), ("D", D, D2), ("moments", mom, mom2), ("K_fit", Kf, Kf2), ("K_pred", Kp, Kp2),
                          ("linear G", G, Gl)):
        assert torch.equal(big[r0:n], sm), "%s of %s differs from a 256-row call" % (name, where)
    del G, D, mom, Kf, Kp, G2, D2, mom2, Kf2, Kp2, Gl, small


# ------------------------------------------------------------------------------- 4: packed operand
@pytest.mark.timeout(900)
@pytest.mark.parametrize("prec", ("fp16x3", "tf32x3"))
def test_packed_operand_past_2_31(dev, prec):
    """pack_epochs of E = 64 epochs, T = 256, V = 70 000 (raw epochs 4.6 GB): the lo plane of the last epochs lies past
    2^31 elements (and 2^32 bytes).  The last two epochs' planes and diagonal on the last 2048 voxels bit for bit, raw
    (normalize = 0) and normalised on the fly (normalize = 1); then corr_block of the last 4 rows against the fp64
    contraction, every epoch, the GEMM reading operand elements past 2^31 for the epochs named in the message."""
    E, T, V, nv = 64, 256, 70000, 2048
    lib = _lib.load()
    code = _lib.PREC[prec]
    nbytes = lib.fcma_operand_bytes(code, E, T, V)
    _need(E * T * V * 4 + nbytes + 2 * GB)
    g = torch.Generator(device=dev).manual_seed(3400)
    ep = torch.randn((E, T, V), device=dev, generator=g).mul_(0.4).add_(2.0)
    Kp = lib.fcma_operand_kp(code, T)
    P = lib.fcma_operand_planes(code)
    esz = 4 if prec.startswith("tf32") else 2
    plane = E * V * Kp                                           # elements of one plane
    e0, v0 = E - 2, V - nv
    last = (P - 1) * plane + (e0 * V + v0) * Kp                  # first sampled element of the last plane
    diag0 = (nbytes - E * V * 4) // 4 + e0 * V + v0              # first sampled diagonal element (fp32)
    assert last > LIM and last * esz > 2 ** 32
    where = "%s: epochs %d-%d, voxels %d-%d, last plane from %s, diagonal from %s" % (prec, e0, E - 1, v0, V - 1,
                                                                                      _at(last), _at(diag0))

    def sampled(op):
        pl = op.buf[:P * plane * esz].view(torch.int32 if esz == 4 else torch.int16).view(P, E, V, Kp)
        d = op.buf[nbytes - E * V * 4:nbytes].view(torch.float32).view(E, V)
        return pl[:, e0:, v0:].cpu().numpy(), d[e0:, v0:].cpu().numpy()

    op = engine.pack_epochs(ep, None, prec)
    for normalize in (False, True):
        if normalize:
            engine.pack_epochs(ep, None, prec, normalize=True, out=op)
            x = engine.epoch_normalize_(ep[e0:, :, v0:].contiguous()).cpu().numpy()
        else:
            x = ep[e0:, :, v0:].contiguous().cpu().numpy()
        torch.cuda.synchronize()
        planes, diag = sampled(op)
        want_p, want_d = expected_operand(x, [T, T], prec, Kp)
        what = "%s normalize=%d" % (where, normalize)
        if not np.array_equal(planes, want_p):
            bad = np.argwhere(planes != want_p)[:5]
            pytest.fail("%s: %d plane elements differ, e.g. [p, e - %d, v - %d, t] %s: got %s, want %s" % (
                what, int((planes != want_p).sum()), e0, v0, bad.tolist(), planes[tuple(bad.T)].tolist(),
                want_p[tuple(bad.T)].tolist()))
        assert np.array_equal(diag, want_d), "%s: diagonal differs at %d entries" % (what, int((diag != want_d).sum()))

    # the operand now holds the normalised epochs: corr_block of the last rows reads every epoch of every column
    engine.epoch_normalize_(ep)                                  # bit-identical to the packer's normaliser
    nb, s = 4, V - 4
    got = engine.corr_block(op, op, s, nb).double().cpu().numpy()
    r32 = engine.corr_block_f32(ep, ep, s, nb).cpu().numpy()
    r64 = np.empty((nb, E, V))
    for e in range(E):
        xe = ep[e].double()
        r64[:, e] = (xe[:, s:].t() @ xe).cpu().numpy()
        del xe
    tol = tol_for(prec, r64, r32)
    far = [e for e in range(E) if (P - 1) * plane + e * V * Kp > LIM]
    ii = np.arange(nb)
    check_values(got, r64, [False] * E, tol, s + ii, r32[ii, :, s + ii],
                 what="corr_block %s rows %d-%d (epochs %d-%d read the last plane past 2^31, from %s)" % (
                     prec, s, V - 1, far[0], E - 1, _at((P - 1) * plane + far[0] * V * Kp)))
    del ep, op


# ------------------------------------------------------------------------------- 5: kernel arrays
@pytest.mark.timeout(900)
def test_searchlight_kernels_and_solver_past_2_31(dev):
    """searchlight_kernels_wide (linear), E = 216, a 40 x 40 x 34 mask (46 208 centres, sl_rad 1, cube): the fp64 array
    holds 2.16e9 elements, centres >= 46 029 lie wholly past 2^31 and centre 46 028 straddles it.  Those centres
    element by element against math.fsum of their features; svm_cv_f64 (wide solver) on the whole array gives every
    centre from 46 028 on the accuracy and iteration counts of a call on a copy of those centres."""
    E, r, dims = 216, 1, (40, 40, 34)
    M = (dims[0] - 2) * (dims[1] - 2) * (dims[2] - 2)
    EE = E * E
    assert M * EE > LIM
    _need(M * EE * 8 + 2 * GB)
    rng = np.random.RandomState(3500)
    vol = rng.randn(*dims, E).astype(np.float32)
    y = np.arange(E) % 2
    vol[28:, :, :] += (0.3 * y).astype(np.float32)             # signal in the last centres' cubes
    mask = np.ones(dims, dtype=bool)
    shape = np.ones((3, 3, 3), dtype=bool)
    centres, nfeat = engine.searchlight_centres(mask, r, shape, 0)
    assert len(centres) == M and (nfeat == 27).all()
    vt = torch.from_numpy(vol).to(dev)
    mt = torch.from_numpy(mask).to(dev)
    st = torch.from_numpy(shape).to(dev)
    G, G2 = engine.searchlight_kernels_wide(vt, mt, r, st, centres, "linear")
    assert G2 is G
    m0 = LIM // EE                                               # the first centre that reaches past 2^31
    for m in (m0, m0 + 1, M - 2, M - 1):
        Gm = G[m].cpu().numpy()
        X = _features(vol, mask, shape, r, int(centres[m]))
        gn = X.shape[1] * U64 / (1 - X.shape[1] * U64)
        assert np.array_equal(Gm, Gm.T), "centre %d at %s: not symmetric" % (m, _at(m * EE))
        P = np.einsum("af,bf->abf", X, X)                        # exact in fp64
        gx = np.array([[math.fsum(P[a, b]) for b in range(E)] for a in range(E)])
        bound = gn * np.abs(P).sum(axis=2) + U64 * np.abs(gx)
        assert np.all(np.abs(Gm - gx) <= bound), "centre %d (elements %s to %s): max excess %g" % (
            m, _at(m * EE), _at((m + 1) * EE), np.max(np.abs(Gm - gx) - bound))
    folds = engine.make_svm_folds_wide(y, 4)
    acc, it = engine.svm_cv_f64(G, G, y, 4, folds=folds, return_iters=True)
    tail = G[m0:].clone()
    acc2, it2 = engine.svm_cv_f64(tail, tail, y, 4, folds=folds, return_iters=True)
    assert np.array_equal(acc[m0:], acc2) and np.array_equal(it[m0:], it2), \
        "svm_cv_f64 on centres %d-%d (from %s) differs from a call on their copy at %s" % (
            m0, M - 1, _at(m0 * EE), np.flatnonzero((acc[m0:] != acc2) | (it[m0:] != it2).any(1))[:5] + m0)
    assert 0.5 < acc[m0:].max()
    del G, G2, tail, vt


@pytest.mark.timeout(900)
def test_fp32_kernel_arrays_past_2_31(dev):
    """A float32 [34 500][256][256] kernel array (2.26e9 elements; voxels >= 32 768 past 2^31): subset_kernels to 250
    epochs (output 2.16e9 elements; voxels >= 34 360 past 2^31) with and without the decimal shrink, the last 64 voxels
    bit for bit against torch indexing and the shrink rule; svm_cv_precomputed (wide solver) gives them the accuracies and
    iteration counts of a call on a copy of those voxels."""
    nv, E, d = 34500, 256, 16
    keep = np.array([e for e in range(E) if e not in (0, 17, 100, 128, 200, 255)])
    Ek = len(keep)
    assert nv * E * E > LIM and nv * Ek * Ek > LIM
    _need((nv * E * E + nv * Ek * Ek + nv * E * d) * 4 + 2 * GB)
    g = torch.Generator(device=dev).manual_seed(3600)
    y = np.arange(E) % 2
    # linear kernels of 16 features, the classes well apart: K_11 ~ 600 has three digits, so the shrink scales most of the
    # compacted kernels by 0.1, and libsvm needs a few hundred iterations per problem (with entries of 1e5 and classes
    # that overlap, a fp32 kernel takes it tens of millions)
    X = torch.randn((nv, E, d), device=dev, generator=g) * 4.0
    X[:, torch.as_tensor(y == 1, device=dev), 0] += 20.0
    K = torch.bmm(X, X.transpose(1, 2))
    del X
    sel = torch.arange(nv - 64, nv, device=dev)
    kt = torch.as_tensor(keep, device=dev)
    want = K[sel][:, kt][:, :, kt].cpu()
    where = "voxels %d-%d: input from %s, output from %s" % (nv - 64, nv - 1, _at((nv - 64) * E * E),
                                                            _at((nv - 64) * Ek * Ek))
    out = engine.subset_kernels(K, keep)
    assert torch.equal(out[sel].cpu(), want), "subset_kernels %s" % where
    out, digits = engine.subset_kernels(K, keep, shrink=True, out=out, return_digits=True)
    got, dg = out[sel].cpu(), digits[sel].cpu().numpy()
    nd = np.array([len(str(int(float(k)))) for k in want[:, 0, 0]])
    assert np.array_equal(dg, nd) and (nd > 2).mean() > 0.5, "shrink digits %s" % where
    fac = torch.tensor([np.float32(10.0 ** (2 - int(k))) for k in nd])
    assert torch.equal(got, want * fac[:, None, None]), "shrunk subset_kernels %s" % where
    del out, digits
    _release()
    acc, it = engine.svm_cv_precomputed(K, y, 4, return_iters=True)
    m0 = LIM // (E * E)
    tail = K[m0:].clone()
    acc2, it2 = engine.svm_cv_precomputed(tail, y, 4, return_iters=True)
    assert np.array_equal(acc[m0:], acc2) and np.array_equal(it[m0:], it2), \
        "svm_cv_precomputed on voxels %d-%d (from %s) differs from a call on their copy" % (m0, nv - 1, _at(m0 * E * E))
    assert acc[m0:].min() > 0.5
    del K, tail
