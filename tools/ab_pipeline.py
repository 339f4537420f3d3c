#!/usr/bin/env python
"""Per-kernel times of the fused pipeline (timing hook of the C library), tiled intermediate (default)
against the strided [i][e][j] block (FCMA_FLAG_STRIDED_BLOCK), plus max |K_tiled - K_strided|.
python tools/ab_pipeline.py [nb]"""
import ctypes, os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from brainiak_b200 import _lib
from brainiak_b200.fcma import engine
lib = _lib.load()
V, T, E, eps = 50000, 200, 32, 8
nb = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
dev = torch.device("cuda:0")
g = torch.Generator(device=dev).manual_seed(0)
ep = torch.randn((E, T, V), device=dev, generator=g)
engine.epoch_normalize_(ep)
work = engine.Workspace(E, V, nb, dev)
K = torch.empty((nb, E, E), device=dev)
start = 40000 if nb <= 8192 else 0     # self-correlation columns land in the last column tiles
for prec in sys.argv[2:] or ("fp16x3", "bf16", "tf32x3"):
    op = engine.pack_epochs(ep, None, prec)
    Ks = {}
    for rep in range(2):
        for flags in (0, _lib.FLAG_STRIDED_BLOCK):
            for _ in range(2):
                engine.voxel_kernels(op, op, start, nb, eps, flags=flags, work=work, out=K)
            torch.cuda.synchronize()
            Ks[flags] = K.clone()
            lib.fcma_timing_enable(1)
            for _ in range(5):
                engine.voxel_kernels(op, op, start, nb, eps, flags=flags, work=work, out=K)
            torch.cuda.synchronize()
            a, b = ctypes.c_double(0), ctypes.c_double(0)
            n = lib.fcma_timing_read(ctypes.byref(a), ctypes.byref(b))
            lib.fcma_timing_enable(0)
            print("%-7s nb=%d %-8s gemm %.3f ms  syrk %.3f ms  total %.3f ms" %
                  (prec, nb, "strided" if flags else "tiled", a.value / n, b.value / n, (a.value + b.value) / n), flush=True)
    d = (Ks[0] - Ks[_lib.FLAG_STRIDED_BLOCK]).abs().max().item()
    print("%-7s max|K_tiled - K_strided| = %.3g (max|K| %.3g)" % (prec, d, Ks[_lib.FLAG_STRIDED_BLOCK].abs().max().item()),
          flush=True)
    del op
