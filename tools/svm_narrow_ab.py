#!/usr/bin/env python
"""Time fcma_svm_cv_solve / fcma_svm_cv_solve_f64 of two builds of libfcma_b200.so in one process, alternating.

Both libraries are loaded side by side (ctypes, RTLD_LOCAL) and called on the same device arrays: float kernels
[50 000, 32, 32] and fp64 linear kernels of E = 32 and 64, 4 folds, shrinking off and on.  The kernels are Gram matrices
of random features with a class signal on one feature (features of 3 to 40 dimensions).  Each call is timed with CUDA
events; the script prints the median and minimum of every case for both libraries and checks that their outputs
(decision bits, correct counts, iterations) are identical.  The card's name and power limit are printed too.

    python tools/svm_narrow_ab.py OLD.so NEW.so [--calls 30]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from brainiak_b200 import _lib  # noqa: E402
from brainiak_b200.fcma import engine  # noqa: E402


def load(path):
    lib = ctypes.CDLL(os.path.abspath(path))
    for name in ("fcma_svm_cv_solve", "fcma_svm_cv_solve_f64", "fcma_last_error"):
        res, args = _lib.SIGNATURES[name]
        getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    return lib


def kernels(nv, E, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    y = torch.arange(E, device="cuda") % 2
    K = torch.empty((nv, E, E), dtype=dtype, device="cuda")
    for s in range(0, nv, 5000):
        d = int(3 + (s // 5000) * 37 // max(1, nv // 5000))
        X = torch.randn((min(5000, nv - s), E, d), generator=g, device="cuda", dtype=torch.float32)
        X[:, :, 0] += 0.7 * (2 * y - 1).float()
        X = X.to(dtype)
        K[s:s + X.shape[0]] = X @ X.transpose(1, 2)
    return K.contiguous(), y.cpu().numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--voxels", type=int, default=50000)
    a = ap.parse_args()
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    print("card (name, power limit, max SM clock):", out.stdout.strip(), flush=True)
    libs = {"old": load(a.old), "new": load(a.new)}
    cases = [("float", 32, torch.float32), ("f64", 32, torch.float64), ("f64", 64, torch.float64)]
    for kind, E, dtype in cases:
        K, labels = kernels(a.voxels, E, dtype, seed=E)
        folds = engine.make_svm_folds(labels, 4)
        nprob = folds.nproblems
        arr = ctypes.cast(folds.structs, ctypes.c_void_p)
        for shrinking in (0, 1):
            outs, ms = {}, {k: [] for k in libs}
            for call in range(a.calls + 2):                      # two warm-up rounds
                for name in (("old", "new") if call % 2 == 0 else ("new", "old")):
                    lib = libs[name]
                    correct = torch.empty((a.voxels, nprob), dtype=torch.int32, device="cuda")
                    bits = torch.empty((a.voxels, nprob), dtype=torch.int64, device="cuda")
                    iters = torch.empty((a.voxels, nprob), dtype=torch.int32, device="cuda")
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    if kind == "float":
                        rc = lib.fcma_svm_cv_solve(K.data_ptr(), a.voxels, E, nprob, arr, 1.0, 1e-3, -1, shrinking,
                                                   correct.data_ptr(), bits.data_ptr(), iters.data_ptr(), None)
                    else:
                        rc = lib.fcma_svm_cv_solve_f64(K.data_ptr(), K.data_ptr(), a.voxels, E, nprob, arr, 1.0, 1e-3,
                                                       -1, shrinking, correct.data_ptr(), bits.data_ptr(),
                                                       iters.data_ptr(), None)
                    e1.record()
                    e1.synchronize()
                    assert rc == 0, lib.fcma_last_error()
                    if call >= 2:
                        ms[name].append(e0.elapsed_time(e1))
                    outs[name] = (correct.cpu(), bits.cpu(), iters.cpu())
            same = all(torch.equal(x, y) for x, y in zip(outs["old"], outs["new"]))
            r = {"kernels": "%s [%d, %d, %d], 4 folds" % (kind, a.voxels, E, E), "shrinking": shrinking,
                 "identical": same, "mean_iters": round(float(outs["new"][2].double().mean()), 1)}
            for name in libs:
                r[name + "_median_ms"] = round(float(np.median(ms[name])), 3)
                r[name + "_min_ms"] = round(float(np.min(ms[name])), 3)
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
