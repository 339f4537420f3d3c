#!/usr/bin/env python
"""Symmetric self-correlation pipeline (fcma_voxel_kernels_sym) against the plain pipeline
(fcma_voxel_kernels): parity on small / ragged / multi-pass / sharded cases, then step times at the bench
shape.  Run on an H100:  timeout 900 python tools/sym_check.py [--no-big]"""
import ctypes
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from brainiak_b200 import _lib  # noqa: E402
from brainiak_b200.fcma import engine  # noqa: E402

lib = _lib.load()
dev = torch.device("cuda:0")
FAILS = []


def make(V, T, E, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    ep = torch.randn((E, T, V), device=dev, generator=g)
    ep[1::2, :, : max(1, V // 100)] += 0.6 * torch.randn((E // 2, T, 1), device=dev, generator=g)
    engine.epoch_normalize_(ep)
    return ep


def parity(V, T, E, eps, rows_sym, shards=1, flags=0, prec="fp16x3", tol=1e-5):
    ep = make(V, T, E, seed=V)
    op = engine.pack_epochs(ep, None, prec)
    Kp = engine.voxel_kernels(op, op, 0, V, eps, flags=flags)
    Ks = torch.zeros((V, E, E), device=dev)
    work = engine.SymWorkspace(E, V, rows_sym, dev)
    for s, n in engine.sym_row_partition(V, shards):
        if n > 0:
            engine.voxel_kernels_sym(op, s, n, eps, flags=flags, work=work, out=Ks)
    torch.cuda.synchronize()
    d = (Ks - Kp).abs().max().item() / Kp.abs().max().item()
    asym = (Ks - Ks.transpose(1, 2)).abs().max().item()
    ok = d <= tol and asym == 0.0
    print("parity V=%d T=%d E=%d eps=%d rows/pass=%d shards=%d flags=%d %s: max|dK|/max|K| = %.3g  asym %.3g  %s"
          % (V, T, E, eps, rows_sym, shards, flags, prec, d, asym, "ok" if ok else "FAIL"), flush=True)
    if not ok:
        FAILS.append((V, T, E, eps, rows_sym, shards, flags))
        bad = ((Ks - Kp).abs().amax(dim=(1, 2)) > tol * Kp.abs().max()).nonzero().flatten()
        print("   bad voxels: %d, first %s last %s" % (bad.numel(), bad[:8].tolist(), bad[-8:].tolist()), flush=True)


def timed_step(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def kernel_times(fn, reps=2):
    lib.fcma_timing_enable(1)
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    g, s = ctypes.c_double(0), ctypes.c_double(0)
    n = lib.fcma_timing_read(ctypes.byref(g), ctypes.byref(s))
    lib.fcma_timing_enable(0)
    return g.value / reps, s.value / reps, n // reps


def big():
    V, T, E, eps = 50000, 200, 32, 8
    ep = make(V, T, E, seed=1)
    op = engine.pack_epochs(ep, None, "fp16x3")
    del ep
    K = torch.empty((V, E, E), device=dev)
    work = engine.Workspace(E, V, 4096, dev)
    plain = lambda: engine.voxel_kernels(op, op, 0, V, eps, work=work, out=K)   # noqa: E731
    ms = timed_step(plain, 3)
    g, s, n = kernel_times(plain)
    print("plain: step %.1f ms (%.3g corr/s); gemm %.1f ms, syrk %.1f ms per step over %d passes"
          % (ms, V * V * E / ms * 1e3, g, s, n), flush=True)
    Kp = K.clone()
    del work
    torch.cuda.empty_cache()
    Ks = torch.empty((V, E, E), device=dev)
    F16, TR = _lib.FLAG_F16_INTERMEDIATE, _lib.FLAG_SYM_TRANSPOSED
    for name, rows, fl in (("sym fp32 block, column-direction pass over the block (default)", 2048, 0),
                           ("sym fp32 block, transposed copy B + row pass over it", 4096, TR),
                           ("sym fp16 block, column pass", 2048, F16),
                           ("sym fp16 block, transposed copy B", 4096, F16 | TR)):
        work = engine.SymWorkspace(E, V, rows, dev)

        def sym():
            Ks.zero_()
            engine.voxel_kernels_sym(op, 0, V, eps, flags=fl, work=work, out=Ks)
        ms = timed_step(sym, 3)
        g, s, n = kernel_times(sym)
        d = (Ks - Kp).abs().max().item() / Kp.abs().max().item()
        print("%s: step %.1f ms (%.3g corr/s); gemm %.1f ms, syrk %.1f ms per step over %d passes; "
              "max|dK|/max|K| vs plain %.3g" % (name, ms, V * V * E / ms * 1e3, g, s, n, d), flush=True)
        del work
        torch.cuda.empty_cache()


if __name__ == "__main__":
    t0 = time.time()
    parity(2000, 64, 16, 4, 256)                     # ragged tail pass, several passes
    parity(2000, 64, 16, 4, 512, flags=_lib.FLAG_MASK_SELF)
    parity(3072, 200, 32, 8, 1024)                   # whole tiles, 3 passes
    parity(3000, 200, 32, 8, 1024, shards=2)         # two shards accumulate into one K
    parity(5000, 100, 8, 8, 2048, shards=3)
    parity(700, 50, 32, 16, 256)
    parity(2500, 120, 64, 8, 512)                    # E > 32 path
    parity(1500, 200, 32, 8, 512, prec="tf32x3")
    parity(3000, 200, 32, 8, 1024, shards=2, flags=_lib.FLAG_F16_INTERMEDIATE)     # fp16 blocks, both copies
    parity(2000, 64, 16, 4, 256, flags=_lib.FLAG_F16_INTERMEDIATE | _lib.FLAG_MASK_SELF)
    parity(1800, 200, 32, 8, 768, prec="bf16")
    # fp16 block with the column pass: same values as the plain fp16-block pipeline
    assert lib.fcma_sym_uses_column_pass(_lib.PREC["fp16x3"], 32, 8, _lib.FLAG_F16_INTERMEDIATE) == 1
    parity(3000, 200, 32, 8, 1024, shards=2, flags=_lib.FLAG_F16_INTERMEDIATE)
    parity(2000, 64, 16, 4, 256, flags=_lib.FLAG_F16_INTERMEDIATE | _lib.FLAG_MASK_SELF)
    parity(1800, 200, 32, 8, 768, prec="bf16")
    parity(1300, 24, 7, 2, 256, flags=_lib.FLAG_F16_INTERMEDIATE, tol=2e-3)
    parity(2600, 50, 24, 8, 512, flags=_lib.FLAG_F16_INTERMEDIATE)
    print("parity section: %.1f s, failures: %s" % (time.time() - t0, FAILS), flush=True)
    if "--no-big" not in sys.argv:
        big()
    sys.exit(1 if FAILS else 0)
