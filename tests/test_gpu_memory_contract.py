"""Memory and stream contract of the fp64 kernel builders, the batched solvers and the gamma='scale' kernels.

Every device argument of an entry point is a view inside a ``[guard | payload | guard]`` byte arena (guards of 1 MiB,
payload offsets a multiple of 256 bytes, payloads of exactly the documented size), and every call runs twice:

* pattern A: every guard, workspace and overwritten output filled with ``0xFF`` bytes (NaN in every float type, -1 in
  integers, "set" in masks and bit words);
* pattern B: ``0x7F`` for float and double buffers (a huge finite value), ``0x01`` guards for byte masks and shapes (an
  out-of-range read finds a voxel "in the mask"), ``0x00`` for integer and bit buffers.

The inputs hold the same valid values in both runs.  Asserted: every guard byte unchanged; every device input and host
array byte-identical before and after the call; runs A and B bit-identical (nothing stale or outside is read); the
outputs bit-identical to the engine wrapper's (which the element-wise and libsvm tests pin) -- for the older fp32
pipelines, whose partial sums meet in atomics in no fixed order, both within 1e-5 of max|K| instead; the extents the
header states: decision words past the held-out samples 0, optional solver outputs independent of each other, accumulated
outputs accumulated only where documented, a linear builder's separate K_pred untouched.  Every solver call is capped at
100 000 iterations and every count must stay below the cap.

The stream tests run one entry point of each family on a fresh ``torch.cuda.Stream`` behind a ~50 ms sleep, after which
the real inputs replace a decoy input on that stream: an internal upload, memset or launch on another stream would read
the decoy and give a well-formed wrong answer.
"""
import ctypes
import time

import numpy as np
import pytest
import torch

from brainiak_b200 import _lib
from brainiak_b200 import searchlight as slm
from brainiak_b200.fcma import engine, synthetic
from test_gpu_feature_svc import _operands

pytestmark = pytest.mark.gpu

GUARD = 1 << 20
ALIGN = 256
PAT_B = {"f": 0x7F, "b": 0x01, "i": 0x00}
MAX_ITER = 100000
SLEEP_CYCLES = 100_000_000          # ~50 ms at the H100's clocks
T = 40
_T0 = [None]


@pytest.fixture(scope="module")
def dev():
    assert _lib.device_count() > 0, "no sm_90 device"
    _T0[0] = time.time()
    yield torch.device("cuda:0")
    print("\ntest_gpu_memory_contract: %.1f s" % (time.time() - _T0[0]))


def _sp(stream=None):
    return ctypes.c_void_p((stream or torch.cuda.current_stream()).cuda_stream)


def _pattern(cls, run):
    return 0xFF if run == "A" else PAT_B[cls]


class Buf:
    """A payload of ``dtype`` and ``shape`` inside a ``[guard | payload | guard]`` uint8 arena (device or host).

    cls: 'f' float / double (and packed operands and workspaces), 'b' byte masks, 'i' integers and bit words.
    role: 'in' (``init``, read only), 'out' (overwritten: filled with the pattern), 'work' (scratch: the pattern),
    'acc' (``init``, accumulated into / updated in place), 'keep' (the pattern, must not be written)."""

    def __init__(self, name, shape, dtype, cls, role, init=None, device="cuda"):
        self.name, self.cls, self.role = name, cls, role
        self.shape = tuple(int(s) for s in shape)
        self.nbytes = int(np.prod(self.shape)) * torch.empty((), dtype=dtype).element_size()
        assert self.nbytes > 0
        self.raw = torch.empty(2 * GUARD + self.nbytes + ALIGN, dtype=torch.uint8, device=device)
        self.off = GUARD + (-(self.raw.data_ptr() + GUARD)) % ALIGN
        self.bytes = self.raw[self.off:self.off + self.nbytes]
        self.t = self.bytes.view(dtype).view(self.shape)
        assert self.t.data_ptr() % ALIGN == 0
        self.item = self.nbytes // self.shape[0]
        self.init = None
        if init is not None:
            init = torch.as_tensor(init).to(device=device, dtype=dtype).reshape(self.shape).contiguous()
            self.init = init
        assert (self.init is not None) == (role in ("in", "acc")), name

    @property
    def ptr(self):
        return ctypes.c_void_p(self.t.data_ptr())

    def fill(self, run, init=None):
        self.raw.fill_(_pattern(self.cls, run))
        src = self.init if init is None else init
        if self.role in ("in", "acc"):
            self.t.copy_(src)


def _first(mask):
    idx = torch.nonzero(mask.reshape(-1))
    return int(idx[0]) if len(idx) else None


def _bytes_of(t):
    return t.contiguous().reshape(-1).view(torch.uint8)


def _check_buf(who, b, run):
    p = _pattern(b.cls, run)
    head, tail = b.raw[:b.off], b.raw[b.off + b.nbytes:]
    k = _first(head != p)
    assert k is None, "%s: %s: guard byte %d before the payload written (pattern %s, now 0x%02x)" % (
        who, b.name, b.off - k, run, int(head[k]))
    k = _first(tail != p)
    assert k is None, "%s: %s: byte %d past the end written (item %d of %d, pattern %s, now 0x%02x)" % (
        who, b.name, k, (b.nbytes + k) // b.item, b.shape[0], run, int(tail[k]))
    if b.role == "in":
        k = _first(_bytes_of(b.init) != b.bytes)
        assert k is None, "%s: input %s changed at byte %d (item %d, pattern %s)" % (who, b.name, k, k // b.item, run)
    if b.role == "keep":
        k = _first(b.bytes != p)
        assert k is None, "%s: %s must not be written; byte %d (item %d) is (pattern %s)" % (
            who, b.name, k, k // b.item, run)


def assert_bits(who, what, got, want):
    """got and want bit-identical (NaN-safe); the message names the first differing byte and its item."""
    assert tuple(got.shape) == tuple(want.shape), (who, what, tuple(got.shape), tuple(want.shape))
    g, w = _bytes_of(got), _bytes_of(want.to(got.device))
    k = _first(g != w)
    per = max(1, g.numel() // max(1, got.shape[0] if got.dim() else 1))
    assert k is None, "%s: %s differs at byte %d (item %d): 0x%02x != 0x%02x" % (who, what, k, k // per, int(g[k]),
                                                                                   int(w[k]))


def assert_near(who, what, got, want, rel=1e-5):
    """For the fp32 pipelines, whose partial sums meet in atomics (order not fixed): finite and within ``rel`` of
    max|want|; the message names the first item out of bounds."""
    g, w = got.double().cpu(), want.double().cpu()
    assert g.shape == w.shape, (who, what, tuple(g.shape), tuple(w.shape))
    bad = ~torch.isfinite(g) | ((g - w).abs() > rel * w.abs().max())
    k = _first(bad)
    per = max(1, g.numel() // max(1, g.shape[0]))
    assert k is None, "%s: %s differs at element %d (item %d): %r vs %r" % (who, what, k, k // per,
                                                                            float(g.reshape(-1)[k]), float(w.reshape(-1)[k]))


def _host_bytes(h):
    return h.tobytes() if isinstance(h, np.ndarray) else bytes(h)


def guarded(who, bufs, invoke, host=(), near=()):
    """Runs ``invoke(stream)`` under patterns A and B and checks guards, inputs, host arrays and A == B (within
    ``assert_near`` for the outputs named in ``near``).  Returns the outputs of run A: {name: tensor} of every 'out'
    and 'acc' buffer ('keep' buffers hold their pattern, which _check_buf checks)."""
    outs = {}
    for run in "AB":
        for b in bufs:
            b.fill(run)
        snap = [_host_bytes(h) for h in host]
        torch.cuda.synchronize()
        rc = invoke(_sp())
        torch.cuda.synchronize()
        assert rc == 0, (who, rc, _lib.last_error())
        for b in bufs:
            _check_buf(who, b, run)
        for i, (h, s) in enumerate(zip(host, snap)):
            assert _host_bytes(h) == s, "%s: host array %d changed (pattern %s)" % (who, i, run)
        outs[run] = {b.name: b.t.clone() for b in bufs if b.role in ("out", "acc")}
    for name in outs["A"]:
        (assert_near if name in near else assert_bits)(who + " (A vs B)", name, outs["A"][name], outs["B"][name])
    return outs["A"]


def on_stream(who, bufs, decoys, invoke, want, near=()):
    """Inputs prefilled with ``decoys`` ({name: tensor}), then on a new stream: a ~50 ms sleep, the real inputs copied in,
    the call, the outputs copied out; one synchronisation, then bit-identical to ``want`` ({name: tensor})."""
    for b in bufs:
        b.fill("A", decoys.get(b.name))
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        for b in bufs:
            if b.role in ("in", "acc"):
                b.t.copy_(b.init)
        rc = invoke(_sp(s))
        got = {name: next(b for b in bufs if b.name == name).t.clone() for name in want}
    s.synchronize()
    assert rc == 0, (who, rc, _lib.last_error())
    for name, w in want.items():
        (assert_near if name in near else assert_bits)(who + " (stream)", name, got[name], w)


def _entry(name):
    """The entry point ``name`` of the searchlight builders and the solvers."""
    lib = _lib.load()
    return {"fcma_searchlight_kernels": lib.fcma_searchlight_kernels,
            "fcma_searchlight_kernels_wide": lib.fcma_searchlight_kernels_wide,
            "fcma_svm_cv_solve": lib.fcma_svm_cv_solve, "fcma_svm_cv_solve_f64": lib.fcma_svm_cv_solve_f64,
            "fcma_svm_cv_solve_wide": lib.fcma_svm_cv_solve_wide,
            "fcma_svm_cv_solve_f64_wide": lib.fcma_svm_cv_solve_f64_wide,
            "fcma_svm_cv_precomputed": lib.fcma_svm_cv_precomputed}[name]


def _op_buf(name, op):
    return Buf(name, (op.buf.numel(),), torch.uint8, "f", "in", op.buf)


# ---------------------------------------------------------------------------------------------- feature builders
def _feature_case(E, V2, nb, rows, start, eps, seed, V=300):
    op, op2 = _operands(V, V2, T, E, torch.device("cuda"), seed=seed)
    n2 = op2.V
    per_row = _lib.load().fcma_work_bytes_per_row(E, n2)
    return op, op2, n2, per_row


def _feature_bufs(op, op2, E, nb, per_row, rows, outs):
    ops = [_op_buf("rows_op", op)]
    if op2 is not op:
        ops.append(_op_buf("cols_op", op2))
    work = Buf("work", (per_row * rows,), torch.uint8, "f", "work")
    return ops, work, [Buf(n, s, torch.float64, "f", r) for n, s, r in outs]


# E, V2 (None: one mask), nb, workspace rows, start, eps
NARROW = [(1, 33, 3, 3, 0, 1), (33, None, 3, 3, 7, 3), (64, 257, 257, 256, 5, 16), (33, 33, 257, 256, 40, 4),
          (16, 257, 3, 3, 290, 4)]
WIDE = [(1, 33, 3, 3, 0, 1), (65, 257, 257, 256, 5, 20), (127, None, 3, 3, 9, 16), (129, 33, 3, 3, 0, 16),
        (140, 257, 3, 3, 17, 20), (255, None, 257, 256, 3, 16), (256, 33, 257, 256, 0, 3)]


def _feature_call(entry, op, op2, ops, E, start, nb, eps, kind, gamma, work, Kf, Kp):
    cols = ops[-1]
    return lambda st: entry(ops[0].ptr, cols.ptr, _lib.PREC[op.precision], E, op.T, op.V, op2.V, start, nb, eps, kind,
                            gamma, work.ptr, work.nbytes, Kf.ptr, Kp.ptr if Kp is not None else None, st)


@pytest.mark.parametrize("wide,E,V2,nb,rows,start,eps", [(False,) + c for c in NARROW] + [(True,) + c for c in WIDE])
def test_feature_kernels_guarded(dev, wide, E, V2, nb, rows, start, eps):
    lib = _lib.load()
    entry = lib.fcma_voxel_feature_kernels_wide if wide else lib.fcma_voxel_feature_kernels
    who = "%s E=%d V2=%s nb=%d rows=%d start=%d eps=%d" % (
        "fcma_voxel_feature_kernels_wide" if wide else "fcma_voxel_feature_kernels", E, V2, nb, rows, start, eps)
    op, op2, n2, per_row = _feature_case(E, V2, nb, rows, start, eps, seed=E * 31 + (V2 or 0) + rows)
    wrapper = engine.feature_kernels_f64_wide if wide else engine.feature_kernels_f64
    ew = engine.Workspace(E, n2, rows, dev)
    gamma = 0.41 / n2
    for kind in ("linear", "rbf"):
        # linear with a separate, non-null K_pred: pinned as untouched
        ops, work, (Kf, Kp) = _feature_bufs(op, op2, E, nb, per_row, rows,
                                            [("K_fit", (nb, E, E), "out"),
                                             ("K_pred", (nb, E, E), "keep" if kind == "linear" else "out")])
        k = 0 if kind == "linear" else 1
        out = guarded("%s %s" % (who, kind), ops + [work, Kf, Kp],
                      _feature_call(entry, op, op2, ops, E, start, nb, eps, k, gamma if k else 0.0, work, Kf, Kp))
        want = wrapper(op, op2, start, nb, eps, kind, gamma if k else None, work=ew)
        assert_bits(who, kind + " K_fit", out["K_fit"], want[0])
        if k:
            assert_bits(who, kind + " K_pred", out["K_pred"], want[1])
        else:
            # and with K_pred null (what the wrapper passes) the same K_fit
            out0 = guarded(who + " linear, null K_pred", ops + [work, Kf],
                           _feature_call(entry, op, op2, ops, E, start, nb, eps, 0, 0.0, work, Kf, None))
            assert_bits(who, "linear K_fit (null K_pred)", out0["K_fit"], want[0])


@pytest.mark.parametrize("E,V2,nb,rows,start,eps", WIDE)
def test_feature_gram_wide_guarded(dev, E, V2, nb, rows, start, eps):
    lib = _lib.load()
    who = "fcma_voxel_feature_gram_wide E=%d V2=%s nb=%d rows=%d start=%d eps=%d" % (E, V2, nb, rows, start, eps)
    op, op2, n2, per_row = _feature_case(E, V2, nb, rows, start, eps, seed=E * 37 + (V2 or 0) + rows)
    ops, work, (G, D, mo) = _feature_bufs(op, op2, E, nb, per_row, rows, [("G", (nb, E, E), "out"),
                                                                        ("D", (nb, E, E), "out"),
                                                                        ("moments", (nb, E, 4), "out")])
    out = guarded(who, ops + [work, G, D, mo], lambda st: lib.fcma_voxel_feature_gram_wide(
        ops[0].ptr, ops[-1].ptr, _lib.PREC[op.precision], E, op.T, op.V, n2, start, nb, eps, work.ptr, work.nbytes,
        G.ptr, D.ptr, mo.ptr, st))
    want = engine.feature_gram_wide(op, op2, start, nb, eps, work=engine.Workspace(E, n2, rows, dev))
    for name, w in zip(("G", "D", "moments"), want):
        assert_bits(who, name, out[name], w)


def test_feature_kernels_wide_stream(dev):
    E, V2, nb, rows, start, eps = 140, 257, 257, 256, 5, 20
    lib = _lib.load()
    op, op2, n2, per_row = _feature_case(E, V2, nb, rows, start, eps, seed=901)
    dop, dop2, _, _ = _feature_case(E, V2, nb, rows, start, eps, seed=902)
    ops, work, (Kf, Kp) = _feature_bufs(op, op2, E, nb, per_row, rows, [("K_fit", (nb, E, E), "out"),
                                                                        ("K_pred", (nb, E, E), "out")])
    gamma = 0.3 / n2
    want = engine.feature_kernels_f64_wide(op, op2, start, nb, eps, "rbf", gamma, work=engine.Workspace(E, n2, rows, dev))
    on_stream("fcma_voxel_feature_kernels_wide", ops + [work, Kf, Kp], {"rows_op": dop.buf, "cols_op": dop2.buf},
              _feature_call(lib.fcma_voxel_feature_kernels_wide, op, op2, ops, E, start, nb, eps, 1, gamma, work, Kf, Kp),
              {"K_fit": want[0], "K_pred": want[1]})


# ---------------------------------------------------------------------------------------------- searchlight builders
def _sl_case(E, r, shape_i, seed):
    """A volume with mask holes; centres: the inner corner (exactly r from three faces), the opposite corner (its cube
    holds the volume's last voxel, which is in the mask) and random interior mask voxels."""
    rng = np.random.RandomState(seed)
    dims = (2 * r + 4, 2 * r + 5, 2 * r + 3)
    vol = (rng.randn(*dims, E) * rng.choice([0.01, 1.0, 30.0], size=dims + (1,))).astype(np.float32)
    mask = rng.rand(*dims) > 0.3
    mask[r, r, r] = True
    mask[-1, -1, -1] = True
    far = (dims[0] - 1 - r, dims[1] - 1 - r, dims[2] - 1 - r)
    mask[far] = True
    inner = np.zeros(dims, dtype=bool)
    inner[r:dims[0] - r, r:dims[1] - r, r:dims[2] - r] = True
    cand = np.flatnonzero((mask & inner).ravel())
    extra = rng.choice(cand, size=min(3, len(cand)), replace=False)
    centres = np.unique(np.concatenate([[np.ravel_multi_index((r, r, r), dims), np.ravel_multi_index(far, dims)],
                                        extra])).astype(np.int64)
    shape = [slm.Cube, slm.Diamond, slm.Ball][shape_i](r).mask_.astype(np.uint8)
    gamma = rng.uniform(0.01, 0.5, size=len(centres))
    return vol, mask.astype(np.uint8), shape, centres, gamma


def _sl_bufs(vol, mask, shape, outs):
    return [Buf("vol", vol.shape, torch.float32, "f", "in", vol), Buf("mask", mask.shape, torch.uint8, "b", "in", mask),
            Buf("shape", shape.shape, torch.uint8, "b", "in", shape)] + \
        [Buf(n, s, torch.float64, "f", role) for n, s, role in outs]


SL_NARROW = [(1, 0, 0), (63, 1, 1), (64, 2, 2), (64, 1, 0), (33, 2, 1)]
SL_WIDE = [(1, 2, 1), (63, 0, 2), (64, 1, 0), (65, 2, 2), (216, 1, 0), (255, 2, 0), (255, 1, 1)]


@pytest.mark.parametrize("entry_name,E,r,shape_i",
                         [("fcma_searchlight_kernels",) + c for c in SL_NARROW] +
                         [("fcma_searchlight_kernels_wide",) + c for c in SL_WIDE])
def test_searchlight_kernels_guarded(dev, entry_name, E, r, shape_i):
    entry = _entry(entry_name)
    wrapper = engine.searchlight_kernels_wide if entry_name.endswith("wide") else engine.searchlight_kernels
    vol, mask, shape, centres, gamma = _sl_case(E, r, shape_i, seed=E * 11 + r * 3 + shape_i)
    M = len(centres)
    nx, ny, nz = mask.shape
    vt, mt, st_ = (torch.from_numpy(a).to(dev) for a in (vol, mask, shape))
    for kind in ("linear", "rbf"):
        who = "%s E=%d sl_rad=%d shape=%d %s" % (entry_name, E, r, shape_i, kind)
        k = 0 if kind == "linear" else 1
        bufs = _sl_bufs(vol, mask, shape, [("K_fit", (M, E, E), "out"), ("K_pred", (M, E, E), "keep" if k == 0 else "out")])
        v, m, s, Kf, Kp = bufs
        g = gamma.copy()
        out = guarded(who, bufs, lambda st: entry(v.ptr, nx, ny, nz, E, m.ptr, r, s.ptr,
                                                  centres.ctypes.data_as(ctypes.c_void_p), M, k,
                                                  g.ctypes.data_as(ctypes.c_void_p) if k else None, Kf.ptr, Kp.ptr, st),
                      host=(centres, g))
        want = wrapper(vt, mt, r, st_, centres, kind, gamma if k else None)
        assert_bits(who, "K_fit", out["K_fit"], want[0])
        if k:
            assert_bits(who, "K_pred", out["K_pred"], want[1])


@pytest.mark.parametrize("E,r,shape_i", SL_WIDE)
def test_searchlight_gram_wide_guarded(dev, E, r, shape_i):
    lib = _lib.load()
    vol, mask, shape, centres, _ = _sl_case(E, r, shape_i, seed=E * 13 + r * 5 + shape_i)
    M = len(centres)
    nx, ny, nz = mask.shape
    who = "fcma_searchlight_gram_wide E=%d sl_rad=%d shape=%d" % (E, r, shape_i)
    bufs = _sl_bufs(vol, mask, shape, [("G", (M, E, E), "out"), ("D", (M, E, E), "out"), ("moments", (M, E, 4), "out")])
    v, m, s, G, D, mo = bufs
    out = guarded(who, bufs, lambda st: lib.fcma_searchlight_gram_wide(
        v.ptr, nx, ny, nz, E, m.ptr, r, s.ptr, centres.ctypes.data_as(ctypes.c_void_p), M, G.ptr, D.ptr, mo.ptr, st),
        host=(centres,))
    want = engine.searchlight_gram_wide(*(torch.from_numpy(a).to(dev) for a in (vol, mask)), r,
                                        torch.from_numpy(shape).to(dev), centres)
    for name, w in zip(("G", "D", "moments"), want):
        assert_bits(who, name, out[name], w)


def test_searchlight_kernels_wide_stream(dev):
    E, r = 140, 1
    entry = _lib.load().fcma_searchlight_kernels_wide
    vol, mask, shape, centres, gamma = _sl_case(E, r, 2, seed=903)
    dvol = np.random.RandomState(904).randn(*vol.shape).astype(np.float32)
    M = len(centres)
    nx, ny, nz = mask.shape
    bufs = _sl_bufs(vol, mask, shape, [("K_fit", (M, E, E), "out"), ("K_pred", (M, E, E), "out")])
    v, m, s, Kf, Kp = bufs
    want = engine.searchlight_kernels_wide(*(torch.from_numpy(a).to(dev) for a in (vol, mask)), r,
                                           torch.from_numpy(shape).to(dev), centres, "rbf", gamma)
    on_stream("fcma_searchlight_kernels_wide", bufs, {"vol": torch.from_numpy(dvol).to(dev)},
              lambda st: entry(v.ptr, nx, ny, nz, E, m.ptr, r, s.ptr, centres.ctypes.data_as(ctypes.c_void_p), M, 1,
                               gamma.ctypes.data_as(ctypes.c_void_p), Kf.ptr, Kp.ptr, st),
              {"K_fit": want[0], "K_pred": want[1]})


# ---------------------------------------------------------------------------------------------- gamma='scale' kernels
def _moments(n, E, seed):
    """Valid double-double moments [n][E][4] of random feature rows (s.lo = q.lo = 0) and the feature counts."""
    rng = np.random.RandomState(seed)
    nfeat = rng.randint(1, 40, size=n).astype(np.int64)
    mo = np.zeros((n, E, 4))
    for i in range(n):
        X = rng.randn(E, nfeat[i]) * rng.choice([0.1, 1.0, 5.0]) + rng.randn()
        mo[i, :, 0] = X.sum(axis=1)
        mo[i, :, 2] = (X * X).sum(axis=1)
    return mo, nfeat


def _train_masks(nfolds, E, seed):
    rng = np.random.RandomState(seed)
    train = (rng.rand(nfolds, E) > 0.3).astype(np.uint8)
    train[:, 0] = 1
    return train


@pytest.mark.parametrize("per_item", [False, True], ids=["nfeat", "nfeat_dev"])
@pytest.mark.parametrize("nfolds", [2, 64])
def test_fold_gammas_guarded(dev, nfolds, per_item):
    n, E = 37, 140                        # n * nfolds not a multiple of the 256-thread block
    lib = _lib.load()
    mo, nfeat = _moments(n, E, seed=nfolds * 3 + per_item)
    train = _train_masks(nfolds, E, seed=nfolds)
    who = "fcma_fold_gammas nfolds=%d %s" % (nfolds, "nfeat_dev" if per_item else "nfeat")
    bufs = [Buf("moments", (n, E, 4), torch.float64, "f", "in", mo),
            Buf("gamma", (n, nfolds), torch.float64, "f", "out"), Buf("flag", (n, nfolds), torch.uint8, "i", "out")]
    if per_item:
        bufs.append(Buf("nfeat", (n,), torch.int64, "i", "in", nfeat))
    m, g, f = bufs[:3]
    nf = bufs[3].ptr if per_item else None
    out = guarded(who, bufs, lambda st: lib.fcma_fold_gammas(m.ptr, n, E, nfolds, train.ctypes.data_as(ctypes.c_void_p),
                                                             nf, 0 if per_item else 17, g.ptr, f.ptr, st), host=(train,))
    want_g, want_f = engine.fold_gammas(torch.from_numpy(mo).to(dev), train, nfeat if per_item else 17)
    assert_bits(who, "gamma", out["gamma"], want_g)
    assert_bits(who, "flag", out["flag"], want_f.to(torch.uint8))


def test_fold_gammas_stream(dev):
    n, E, nfolds = 37, 140, 64
    lib = _lib.load()
    mo, nfeat = _moments(n, E, seed=905)
    dmo, _ = _moments(n, E, seed=906)
    train = _train_masks(nfolds, E, seed=907)
    bufs = [Buf("moments", (n, E, 4), torch.float64, "f", "in", mo), Buf("nfeat", (n,), torch.int64, "i", "in", nfeat),
            Buf("gamma", (n, nfolds), torch.float64, "f", "out"), Buf("flag", (n, nfolds), torch.uint8, "i", "out")]
    m, nf, g, f = bufs
    want_g, want_f = engine.fold_gammas(torch.from_numpy(mo).to(dev), train, nfeat)
    decoys = {"moments": torch.from_numpy(dmo).to(dev), "nfeat": torch.from_numpy(nfeat[::-1].copy()).to(dev)}
    on_stream("fcma_fold_gammas", bufs, decoys,
              lambda st: lib.fcma_fold_gammas(m.ptr, n, E, nfolds, train.ctypes.data_as(ctypes.c_void_p), nf.ptr, 0, g.ptr,
                                              f.ptr, st),
              {"gamma": want_g, "flag": want_f.to(torch.uint8)})


def _gd(n, E, nfolds, seed):
    rng = np.random.RandomState(seed)
    X = rng.randn(n, E, 9)
    G = np.einsum("nef,ngf->neg", X, X)
    D = ((X[:, :, None, :] - X[:, None, :, :]) ** 2).sum(axis=3)
    gamma = rng.uniform(0.01, 0.3, size=(n, nfolds))
    return G, D, gamma


def _rbf_bufs(G, D, gamma):
    n, E, _ = G.shape
    return [Buf("G", G.shape, torch.float64, "f", "in", G), Buf("D", D.shape, torch.float64, "f", "in", D),
            Buf("gamma", gamma.shape, torch.float64, "f", "in", gamma),
            Buf("K_fit", (n, E, E), torch.float64, "f", "out"), Buf("K_pred", (n, E, E), torch.float64, "f", "out")]


@pytest.mark.parametrize("E", [1, 65, 256])
@pytest.mark.parametrize("last", [False, True], ids=["fold0", "last_fold"])
def test_rbf_fold_kernels_guarded(dev, E, last):
    n, nfolds = 5, 7
    fold = nfolds - 1 if last else 0
    lib = _lib.load()
    G, D, gamma = _gd(n, E, nfolds, seed=E + last)
    bufs = _rbf_bufs(G, D, gamma)
    g, d, ga, Kf, Kp = bufs
    who = "fcma_rbf_fold_kernels E=%d fold=%d" % (E, fold)
    out = guarded(who, bufs, lambda st: lib.fcma_rbf_fold_kernels(g.ptr, d.ptr, n, E, ga.ptr, nfolds, fold, Kf.ptr,
                                                                  Kp.ptr, st))
    want = engine.rbf_fold_kernels(*(torch.from_numpy(a).to(dev) for a in (G, D, gamma)), fold)
    assert_bits(who, "K_fit", out["K_fit"], want[0])
    assert_bits(who, "K_pred", out["K_pred"], want[1])


def test_rbf_fold_kernels_stream(dev):
    n, E, nfolds, fold = 5, 256, 7, 6
    lib = _lib.load()
    G, D, gamma = _gd(n, E, nfolds, seed=908)
    dG, dD, dgamma = _gd(n, E, nfolds, seed=909)
    bufs = _rbf_bufs(G, D, gamma)
    g, d, ga, Kf, Kp = bufs
    want = engine.rbf_fold_kernels(*(torch.from_numpy(a).to(dev) for a in (G, D, gamma)), fold)
    on_stream("fcma_rbf_fold_kernels", bufs, {k: torch.from_numpy(a).to(dev) for k, a in
                                              (("G", dG), ("D", dD), ("gamma", dgamma))},
              lambda st: lib.fcma_rbf_fold_kernels(g.ptr, d.ptr, n, E, ga.ptr, nfolds, fold, Kf.ptr, Kp.ptr, st),
              {"K_fit": want[0], "K_pred": want[1]})


# ---------------------------------------------------------------------------------------------- batched solvers
def _problems(E, ncls, specs, wide, seed):
    """One fold per (n_train, n_test) of ``specs``, one problem per class pair (libsvm's one-vs-one order), as
    engine._build_svm_folds lays them out: training samples of the pair's first class first."""
    rng = np.random.RandomState(seed)
    y = rng.permutation(np.arange(E) % ncls)
    pairs = [(a, b) for a in range(ncls) for b in range(a + 1, ncls)]
    struct = engine._SvmFoldWide if wide else engine._SvmFold
    folds = (struct * (len(specs) * len(pairs)))()
    n_test, test_labels = [], []
    for f, (ntr, nte) in enumerate(specs):
        perm = rng.permutation(E)
        tr = perm[:ntr]
        te = perm[ntr:ntr + nte] if ntr + nte <= E else rng.choice(E, nte, replace=nte > E)
        for q, (a, b) in enumerate(pairs):
            pos, neg = [int(i) for i in tr if y[i] == a], [int(i) for i in tr if y[i] == b]
            assert pos and neg, "a training part misses a class"
            fd = folds[f * len(pairs) + q]
            fd.n_train, fd.n_pos, fd.n_test = len(pos) + len(neg), len(pos), nte
            for j, i in enumerate(pos + neg):
                fd.train_idx[j] = i
            for j, i in enumerate(te):
                fd.test_idx[j] = int(i)
                fd.test_pos[j] = 1 if y[i] == a else 0
        n_test.append(nte)
        test_labels.append(y[te].astype(np.int64))
    return engine.SvmFolds(folds, np.asarray(n_test, dtype=np.float64), np.arange(ncls), pairs, test_labels)


def _kernels(nv, E, seed):
    rng = np.random.RandomState(seed)
    X = rng.randn(nv, E, 12) + rng.randn(nv, 1, 12)
    K = np.einsum("nef,ngf->neg", X, X) / 12.0
    return K, np.exp(-0.05 * ((X[:, :, None, :] - X[:, None, :, :]) ** 2).sum(axis=3))


# E, classes, [(n_train, n_test)], shrinking; narrow problems: n_train, n_test <= 64
SOLVER_NARROW = [(2, 2, [(2, 1)], False), (64, 2, [(64, 63), (48, 64), (60, 1)], True),
                 (64, 3, [(64, 64), (50, 33)], False), (33, 2, [(30, 3), (20, 13)], True)]
SOLVER_WIDE = [(65, 2, [(64, 1), (65, 63), (50, 64), (40, 65)], True),
               (129, 2, [(128, 1), (128, 64), (100, 65), (128, 128)], False),
               (129, 3, [(129, 63), (120, 129)], True),
               (256, 2, [(129, 63), (200, 65), (256, 129), (128, 1)], False),
               (256, 3, [(129, 64), (250, 1)], True)]
SOLVERS = ["fcma_svm_cv_solve", "fcma_svm_cv_solve_f64", "fcma_svm_cv_solve_wide", "fcma_svm_cv_solve_f64_wide"]


def _solver_cases():
    out = []
    for name in SOLVERS:
        wide = name.endswith("wide")
        for i, c in enumerate(SOLVER_NARROW + (SOLVER_WIDE if wide else [])):
            out.append(pytest.param(name, c, id="%s-E%d-c%d-%d" % (name, c[0], c[1], i)))
    return out


def _solver_bufs(f64, nv, E, nprob, wide, K, Kp, outputs=("correct", "bits", "iters")):
    dt = torch.float64 if f64 else torch.float32
    bufs = [Buf("K_fit", (nv, E, E), dt, "f", "in", K)]
    if f64:
        bufs.append(Buf("K_pred", (nv, E, E), dt, "f", "in", Kp))
    shapes = {"correct": ((nv, nprob), torch.int32), "bits": ((nv, nprob, 4) if wide else (nv, nprob), torch.int64),
              "iters": ((nv, nprob), torch.int32)}
    for o in outputs:
        bufs.append(Buf(o, shapes[o][0], shapes[o][1], "i", "out"))
    return bufs


def _solver_call(entry, f64, bufs, nv, E, folds, shrinking, outputs):
    by = {b.name: b for b in bufs}
    kern = (by["K_fit"].ptr, by["K_pred"].ptr) if f64 else (by["K_fit"].ptr,)
    o = {n: (by[n].ptr if n in outputs else None) for n in ("correct", "bits", "iters")}
    return lambda st: entry(*kern, nv, E, folds.nproblems, ctypes.cast(folds.structs, ctypes.c_void_p), 1.0, 1e-3,
                            MAX_ITER, 1 if shrinking else 0, o["correct"], o["bits"], o["iters"], st)


@pytest.mark.parametrize("name,case", _solver_cases())
def test_solvers_guarded(dev, name, case):
    E, ncls, specs, shrinking = case
    nv = 5                                          # a partly filled block of 4 warps
    lib = _lib.load()
    entry = _entry(name)
    wide, f64 = name.endswith("wide"), "f64" in name
    folds = _problems(E, ncls, specs, wide, seed=E * 7 + ncls)
    nprob = folds.nproblems
    K, Kp = _kernels(nv, E, seed=E + ncls)
    if not f64:
        K = K.astype(np.float32)
    who = "%s E=%d classes=%d problems=%s shrinking=%d" % (name, E, ncls, specs, shrinking)
    full = ("correct", "bits", "iters")
    bufs = _solver_bufs(f64, nv, E, nprob, wide, K, Kp)
    out = guarded(who, bufs, _solver_call(entry, f64, bufs, nv, E, folds, shrinking, full), host=(folds.structs,))
    iters = out["iters"].cpu().numpy()
    assert iters.max() < MAX_ITER, (who, iters.max())
    # the words past the held-out samples are 0
    bits = out["bits"].cpu().numpy().view(np.uint64).reshape(nv, nprob, -1)
    words = [(int(folds.structs[p].n_test) + 63) // 64 for p in range(nprob)]
    for p, w in enumerate(words):
        assert not bits[:, p, w:].any(), (who, "bits past the held-out samples", p, w)
    # the engine wrapper on the same inputs (its own tensors)
    Kt = torch.from_numpy(K).to(dev)
    Kp_t = torch.from_numpy(Kp).to(dev) if f64 else None
    kern = (engine._ptr(Kt), engine._ptr(Kp_t)) if f64 else (engine._ptr(Kt),)
    correct, w_iters = engine._svm_correct(entry, kern, Kt, 1.0, 1e-3, MAX_ITER, shrinking, folds, True)
    assert_bits(who, "iters", out["iters"], w_iters)
    if ncls == 2:
        assert_bits(who, "correct", out["correct"], correct)
    else:
        assert_bits(who, "vote over bits", engine._ovo_vote(out["bits"], folds), correct)
    # each optional output null once: the others unchanged
    for drop in full:
        keep = tuple(o for o in full if o != drop)
        b2 = _solver_bufs(f64, nv, E, nprob, wide, K, Kp, keep)
        o2 = guarded(who + " %s=null" % drop, b2, _solver_call(entry, f64, b2, nv, E, folds, shrinking, keep),
                     host=(folds.structs,))
        for k in keep:
            assert_bits(who + " %s=null" % drop, k, o2[k], out[k])
    # fcma_svm_cv_precomputed: the two-class solver without shrinking
    if name == "fcma_svm_cv_solve" and ncls == 2:
        b3 = _solver_bufs(False, nv, E, nprob, False, K, None, ("correct", "iters"))
        kb, cb, ib = b3
        o3 = guarded("fcma_svm_cv_precomputed E=%d" % E, b3, lambda st: lib.fcma_svm_cv_precomputed(
            kb.ptr, nv, E, nprob, ctypes.cast(folds.structs, ctypes.c_void_p), 1.0, 1e-3, MAX_ITER, cb.ptr, ib.ptr, st),
            host=(folds.structs,))
        assert o3["iters"].max() < MAX_ITER
        c0, i0 = engine._svm_correct(entry, (engine._ptr(Kt),), Kt, 1.0, 1e-3, MAX_ITER, False, folds, True)
        assert_bits("fcma_svm_cv_precomputed", "correct", o3["correct"], c0)
        assert_bits("fcma_svm_cv_precomputed", "iters", o3["iters"], i0)


@pytest.mark.parametrize("name", SOLVERS + ["fcma_svm_cv_precomputed"])
def test_solvers_stream(dev, name):
    lib = _lib.load()
    wide, f64 = name.endswith("wide"), "f64" in name
    E, ncls, specs, shrinking = (129, 3, [(129, 63), (120, 129)], True) if wide else \
        (64, 2, [(64, 63), (48, 64)], name != "fcma_svm_cv_precomputed")
    nv = 5
    folds = _problems(E, ncls, specs, wide, seed=910)
    K, Kp = _kernels(nv, E, seed=911)
    dK, dKp = _kernels(nv, E, seed=912)
    if not f64:
        K, dK = K.astype(np.float32), dK.astype(np.float32)
    outs = ("correct", "iters") if name == "fcma_svm_cv_precomputed" else ("correct", "bits", "iters")
    bufs = _solver_bufs(f64, nv, E, folds.nproblems, wide, K, Kp, outs)
    entry = _entry(name)
    if name == "fcma_svm_cv_precomputed":
        kb, cb, ib = bufs

        def call(st):
            return entry(kb.ptr, nv, E, folds.nproblems, ctypes.cast(folds.structs, ctypes.c_void_p), 1.0, 1e-3,
                         MAX_ITER, cb.ptr, ib.ptr, st)
    else:
        call = _solver_call(entry, f64, bufs, nv, E, folds, shrinking, outs)
    guarded(name, bufs, call, host=(folds.structs,))
    want = {b.name: b.t.clone() for b in bufs if b.role == "out"}
    assert int(want["iters"].max()) < MAX_ITER, name
    decoys = {"K_fit": torch.from_numpy(dK).to(dev)}
    if f64:
        decoys["K_pred"] = torch.from_numpy(dKp).to(dev)
    on_stream(name, bufs, decoys, call, want)


# ---------------------------------------------------------------------------------------------- older entry points
def test_voxel_kernels_guarded(dev):
    E, eps, start, nb, rows = 16, 4, 3, 257, 256
    lib = _lib.load()
    op, op2, n2, per_row = _feature_case(E, 257, nb, rows, start, eps, seed=913)
    ops, work, _ = _feature_bufs(op, op2, E, nb, per_row, rows, [])
    K = Buf("K", (nb, E, E), torch.float32, "f", "out")
    who = "fcma_voxel_kernels E=%d nb=%d" % (E, nb)
    out = guarded(who, ops + [work, K], lambda st: lib.fcma_voxel_kernels(
        ops[0].ptr, ops[-1].ptr, _lib.PREC[op.precision], E, op.T, op.V, n2, start, nb, eps, 0, work.ptr, work.nbytes,
        K.ptr, st), near=("K",))
    assert_near(who, "K", out["K"], engine.voxel_kernels(op, op2, start, nb, eps, work=engine.Workspace(E, n2, rows, dev)))


def _sym_op(V, E, seed):
    raw, _ = synthetic.make_epochs(V, T, E, seed=seed)
    ep, T_e = engine.stack_epochs(raw, torch.device("cuda"))
    return engine.pack_epochs(ep, T_e, "fp32")


def _sym_call(op, opb, start, nb, eps, work, K):
    lib = _lib.load()
    return lambda st: lib.fcma_voxel_kernels_sym(opb.ptr, _lib.PREC[op.precision], op.E, op.T, op.V, start, nb, eps, 0,
                                                 work.ptr, work.nbytes, K.ptr, st)


def _sym_work(op, eps, start):
    lib = _lib.load()
    w = engine.SymWorkspace.for_operand(op, 256, eps, 0, start)
    nbytes = w.buf.numel()
    assert lib.fcma_sym_rows_per_pass(_lib.PREC[op.precision], op.E, eps, 0, op.V, start, nbytes) == 256
    return w, Buf("work", (nbytes,), torch.uint8, "f", "work")


@pytest.mark.parametrize("E,eps", [(16, 4), (48, 16)])
def test_voxel_kernels_sym_shards_guarded(dev, E, eps):
    """K is the full [V][E][E] array, accumulated into: a shard starting at 256 leaves rows < 256 bit-unchanged, and the
    two shards' sum equals the one-shot call."""
    V = 400                           # two 256-row passes: [0, 256) and the ragged [256, 400)
    op = _sym_op(V, E, seed=E)
    opb = _op_buf("op", op)
    sentinel = torch.full((V, E, E), -3.25, dtype=torch.float32)
    shards = []
    for start, nb in ((0, 256), (256, V - 256)):
        init = sentinel.clone()
        init[start:] = 0
        ew, work = _sym_work(op, eps, start)
        K = Buf("K", (V, E, E), torch.float32, "f", "acc", init)
        who = "fcma_voxel_kernels_sym E=%d start=%d nb=%d" % (E, start, nb)
        out = guarded(who, [opb, work, K], _sym_call(op, opb, start, nb, eps, work, K), near=("K",))["K"]
        assert_bits(who, "rows < start", out[:start], sentinel[:start])
        assert_near(who, "K", out, engine.voxel_kernels_sym(op, start, nb, eps, work=ew, out=init.to(dev)))
        shards.append(torch.where(torch.arange(V, device=dev)[:, None, None] >= start, out, torch.zeros_like(out)))
    one = engine.voxel_kernels_sym(op, 0, V, eps, work=_sym_work(op, eps, 0)[0])
    assert_near("fcma_voxel_kernels_sym E=%d" % E, "sum of shards vs one shot", shards[0] + shards[1], one)


def test_voxel_kernels_sym_stream(dev):
    V, E, eps, start = 600, 16, 4, 256
    op = _sym_op(V, E, seed=914)
    dop = _sym_op(V, E, seed=915)
    opb = _op_buf("op", op)
    ew, work = _sym_work(op, eps, start)
    init = torch.zeros((V, E, E), dtype=torch.float32)
    K = Buf("K", (V, E, E), torch.float32, "f", "acc", init)
    want = engine.voxel_kernels_sym(op, start, V - start, eps, work=ew, out=init.to(dev))
    on_stream("fcma_voxel_kernels_sym", [opb, work, K], {"op": dop.buf}, _sym_call(op, opb, start, V - start, eps, work, K),
              {"K": want}, near=("K",))


def test_classifier_kernels_guarded(dev):
    """K [E][E] += the sum over the rows (beta = 1 semantics): a finite prefill is accumulated into, not overwritten."""
    lib = _lib.load()
    E, eps, start, nb, rows = 16, 4, 3, 257, 256
    op, op2, n2, per_row = _feature_case(E, 257, nb, rows, start, eps, seed=916)
    prefill = torch.from_numpy(np.random.RandomState(1).randn(E, E).astype(np.float32))
    ops, work, _ = _feature_bufs(op, op2, E, nb, per_row, rows, [])
    K = Buf("K", (E, E), torch.float32, "f", "acc", prefill)
    who = "fcma_classifier_kernel E=%d nb=%d" % (E, nb)
    out = guarded(who, ops + [work, K], lambda st: lib.fcma_classifier_kernel(
        ops[0].ptr, ops[-1].ptr, _lib.PREC[op.precision], E, op.T, op.V, n2, start, nb, eps, 0, work.ptr, work.nbytes,
        K.ptr, st), near=("K",))
    want = engine.classifier_kernel(op, op2, start, nb, eps, work=engine.Workspace(E, n2, rows, dev),
                                    out=prefill.to(dev), symmetric=False)
    assert_near(who, "K", out["K"], want)
    # the symmetric form: one mask, all rows
    V = 600
    sop = _sym_op(V, E, seed=917)
    sopb = _op_buf("op", sop)
    per = lib.fcma_work_bytes_per_row(E, V)
    swork = Buf("work", (per * 256,), torch.uint8, "f", "work")
    K2 = Buf("K", (E, E), torch.float32, "f", "acc", prefill)
    who = "fcma_classifier_kernel_sym E=%d V=%d" % (E, V)
    out = guarded(who, [sopb, swork, K2], lambda st: lib.fcma_classifier_kernel_sym(
        sopb.ptr, _lib.PREC[sop.precision], E, sop.T, V, eps, 0, swork.ptr, swork.nbytes, K2.ptr, st), near=("K",))
    want = engine.classifier_kernel(sop, sop, 0, V, eps, work=engine.SymWorkspace(E, V, 256, dev, transposed_copy=False),
                                    out=prefill.to(dev))
    assert_near(who, "K", out["K"], want)


def test_shrink_kernels_guarded(dev):
    lib = _lib.load()
    nv, E = 5, 16
    rng = np.random.RandomState(2)
    K0 = (rng.randn(nv, E, E) * 10.0 ** rng.randint(0, 8, size=(nv, 1, 1))).astype(np.float32)
    K = Buf("K", (nv, E, E), torch.float32, "f", "acc", K0)
    dg = Buf("digits", (nv,), torch.int32, "i", "out")
    out = guarded("fcma_shrink_kernels", [K, dg], lambda st: lib.fcma_shrink_kernels(K.ptr, nv, E, dg.ptr, st))
    Kw = torch.from_numpy(K0).to(dev)
    digits = engine.shrink_kernels_(Kw, return_digits=True)
    assert_bits("fcma_shrink_kernels", "K", out["K"], Kw)
    assert_bits("fcma_shrink_kernels", "digits", out["digits"], digits)


# ---------------------------------------------------------------------------------------------- host entry points
def test_host_entry_points_guarded(dev):
    lib = _lib.load()
    E, eps, V, V2, start, nb = 16, 4, 300, 257, 3, 40
    raw, _ = synthetic.make_epochs(V, T, E, seed=918)
    raw2, _ = synthetic.make_epochs(V2, T, E, seed=919)
    raw = [np.ascontiguousarray(m[:T - 3 * (e % 3)]) for e, m in enumerate(raw)]
    raw2 = [np.ascontiguousarray(m[:T - 3 * (e % 3)]) for e, m in enumerate(raw2)]
    pp = ctypes.POINTER(ctypes.c_float)
    arr = (pp * E)(*[m.ctypes.data_as(pp) for m in raw])
    arr2 = (pp * E)(*[m.ctypes.data_as(pp) for m in raw2])
    te = (ctypes.c_int * E)(*[m.shape[0] for m in raw])
    host = tuple(raw) + tuple(raw2) + (te,)
    K = Buf("K", (nb, E, E), torch.float32, "f", "out", device="cpu")
    who = "fcma_host_voxel_kernels"
    out = guarded(who, [K], lambda st: lib.fcma_host_voxel_kernels(arr, arr2, te, E, V, V2, start, nb, eps,
                                                                  _lib.PREC["tf32x3"], 1, 0, dev.index,
                                                                  ctypes.c_void_p(K.t.data_ptr())), host=host, near=("K",))
    want = engine.host_voxel_kernels(raw, raw2, start, nb, eps, precision="tf32x3", normalize=True, device=dev.index)
    assert_near(who, "K", out["K"], torch.from_numpy(want))

    Vs = 600
    raws, _ = synthetic.make_epochs(Vs, T, E, seed=920)
    raws = [np.ascontiguousarray(m) for m in raws]
    arrs = (pp * E)(*[m.ctypes.data_as(pp) for m in raws])
    tes = (ctypes.c_int * E)(*[m.shape[0] for m in raws])
    Ks = Buf("K", (Vs, E, E), torch.float32, "f", "out", device="cpu")
    who = "fcma_host_voxel_kernels_sym"
    out = guarded(who, [Ks], lambda st: lib.fcma_host_voxel_kernels_sym(arrs, tes, E, Vs, eps, _lib.PREC["fp16x3"], 0, 0,
                                                                        dev.index, 256, ctypes.c_void_p(Ks.t.data_ptr())),
                  host=tuple(raws) + (tes,), near=("K",))
    want = engine.host_voxel_kernels_sym(raws, eps, precision="fp16x3", device=dev.index, rows_per_pass=256)
    assert_near(who, "K", out["K"], torch.from_numpy(want))

    n0, n2 = 7, 33
    corr = np.random.RandomState(3).uniform(-0.9, 0.9, size=(n0, E, n2)).astype(np.float32)
    C = Buf("corr", corr.shape, torch.float32, "f", "acc", corr, device="cpu")
    who = "fcma_host_within_subject_norm"
    out = guarded(who, [C], lambda st: lib.fcma_host_within_subject_norm(ctypes.c_void_p(C.t.data_ptr()), n0, E, n2, 3,
                                                                        dev.index))
    want = engine.within_subject_norm_(torch.from_numpy(corr).to(dev), 3)
    assert_bits(who, "corr", out["corr"], want)
