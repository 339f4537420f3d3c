#!/usr/bin/env python
"""VoxelSelector.run with SVC(kernel='linear' | 'rbf') on the normalised correlation vectors above 64 epochs, on the GPU
(engine.feature_kernels_f64_wide + the wide fp64 solver), against the host path (scikit-learn per voxel, as the
reference does).

For each configuration (V = V2 voxels, T time points, E epochs, eps epochs per subject, folds) it reports:
* the stage times from CUDA events over the whole run: correlation GEMM, the kernel-matrix stage (normaliser, tiled Gram
  pass and rbf epilogue), cross validation; and the split of the kernel-matrix stage into its kernels, from a
  torch.profiler trace of one block;
* the kernel-matrix stage's bytes (the block normalised in place, read and written, then read by the tiles; fp64
  matrices written) and fp64 operations (G on the tensor cores, D on the FP64 pipe) over its time, against the H100
  SXM data sheet;
* the host path's time per voxel on a sample of voxels, extrapolated to V (labelled as such);
* the accuracies of sampled voxels, GPU against host.
The card's name and power limit are printed in the same run.

    python tools/feature_svc_wide_bench.py [--voxels 50000] [--T 15] [--configs 140:20:7,256:16:16] [--compare 256]
"""
import argparse
import ctypes
import json
import multiprocessing
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402
from sklearn import svm  # noqa: E402

from brainiak_b200 import _lib  # noqa: E402
from brainiak_b200.fcma import engine, synthetic  # noqa: E402
from brainiak_b200.fcma.voxelselector import VoxelSelector  # noqa: E402
from feature_svc_bench import FP64, FP64_TC, HBM, card, host_acc  # noqa: E402


def stage_split(vs, kind, gamma, eps, rows):
    """Kernel times (s) of one feature_kernels_f64_wide call on `rows` rows, by kernel name, from torch.profiler."""
    rows_op, cols_op = vs._operands()
    engine.feature_kernels_f64_wide(rows_op, cols_op, 0, rows, eps, kind, gamma, work=vs._work)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        engine.feature_kernels_f64_wide(rows_op, cols_op, 0, rows, eps, kind, gamma, work=vs._work)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for key in ("k_corr", "k_block_within_subject_norm", "k_feature_gram_tiled", "k_feature_rbf_epilogue"):
            if key in ev.key:
                t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                out[key] = out.get(key, 0.0) + t / 1e6
    return out


def run_config(V, T, E, eps, folds, kind, ncompare, ntime, pool):
    raw, labels = synthetic.make_epochs(V, T, E)
    clf = svm.SVC(kernel="linear", shrinking=False) if kind == "linear" else \
        svm.SVC(kernel="rbf", gamma="auto", shrinking=False)
    vs = VoxelSelector(labels, eps, folds, raw, device="cuda:0")
    assert vs._feature_kind(clf, max_epochs=engine.SVM_WIDE_MAX_EPOCHS) == kind
    gamma = None if kind == "linear" else 1.0 / V
    lib = _lib.load()
    cv_ms = []
    orig = engine.svm_cv_f64

    def timed_cv(*a, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = orig(*a, **kw)                 # ends with a device-to-host copy: synchronised
        e1.record()
        e1.synchronize()
        cv_ms.append(e0.elapsed_time(e1))
        return out

    # warm-up of the same kernels and solver on 512 voxels (module loads); the timed run includes the upload
    VoxelSelector(labels, eps, folds, [m[:, :512] for m in raw], device="cuda:0").run(clf)
    engine.svm_cv_f64 = timed_cv
    cv_ms.clear()
    lib.fcma_timing_enable(1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = vs.run(clf)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    print("E=%d %s: run() %.1f s" % (E, kind, wall), flush=True)
    gemm, stage = ctypes.c_double(), ctypes.c_double()
    passes = lib.fcma_timing_read(ctypes.byref(gemm), ctypes.byref(stage))
    lib.fcma_timing_enable(0)
    engine.svm_cv_f64 = orig
    split_rows = min(V, 2048)
    split = stage_split(vs, kind, gamma, eps, split_rows)
    acc = dict(res)
    nt = -(-E // 64)
    # the tiles' reads: a diagonal tile reads its 64 epochs once, an off-diagonal tile its row and column epochs
    tile_reads = sum(min(64, E - 64 * i) * (1 if i == j else 0) + (min(64, E - 64 * i) + min(64, E - 64 * j)) *
                     (0 if i == j else 1) for i in range(nt) for j in range(i, nt))
    block = 4.0 * V * V                       # bytes of one epoch of the block
    # normalise read and write, the tiles' reads (the GEMM's write is its own stage), the fp64 matrices written
    nbytes = block * (2 * E + tile_reads) + 8.0 * V * E * E * (2 if kind == "rbf" else 1)
    if kind == "rbf":
        nbytes += 8.0 * V * E * E * 4         # the epilogue reads and writes both matrices
    mma_blocks = sum(36 if i == j else 64 for i in range(nt) for j in range(i, nt))
    g_flops = 2.0 * V * V * mma_blocks * 64   # 8 x 8 blocks, every 64-epoch tile computed whole
    d_flops = 3.0 * V * V * sum((64 * 64 if i != j else 136 * 16) for i in range(nt) for j in range(i, nt)) \
        if kind == "rbf" else 0.0             # difference + fma per entry and column
    st = stage.value / 1e3
    rng = np.random.default_rng(1)
    sample = np.sort(rng.choice(V, size=max(ncompare, ntime), replace=False))
    rows_op, cols_op = vs._operands()
    feats = []
    for v in sample:
        c = engine.corr_block(rows_op, cols_op, int(v), 1, layout=0).contiguous()
        feats.append(engine.within_subject_norm_(c, eps)[0].cpu().numpy())
    print("E=%d %s: kernel split %s" % (E, kind, split), flush=True)
    t0 = time.perf_counter()
    for k in range(ntime):
        host_acc((clf, feats[k], labels, folds))
    host_per_voxel = (time.perf_counter() - t0) / ntime
    cmp = sample[:ncompare]
    host = pool.map(host_acc, [(clf, feats[k], labels, folds) for k in range(ncompare)])
    same = sum(acc[int(v)] == h for v, h in zip(cmp, host))
    return {
        "V": V, "T": T, "E": E, "eps": eps, "folds": folds, "kind": kind, "passes": passes,
        "run_s": round(wall, 3), "gemm_s": round(gemm.value / 1e3, 3), "kernel_stage_s": round(st, 3),
        "cv_s": round(sum(cv_ms) / 1e3, 3),
        "profiled_rows": split_rows, "profiled_kernel_s": {k: round(v, 4) for k, v in split.items()},
        "kernel_stage_GB": round(nbytes / 1e9, 1), "kernel_stage_GBps": round(nbytes / st / 1e9, 1),
        "kernel_stage_hbm_share": round(nbytes / HBM / st, 3),
        "kernel_stage_fp64_Tflop": round((g_flops + d_flops) / 1e12, 1),
        "kernel_stage_fp64_share": round((g_flops / FP64_TC + d_flops / FP64) / st, 3),
        "host_s_per_voxel": round(host_per_voxel, 3), "host_voxels_timed": ntime,
        "host_total_s_extrapolated": round(host_per_voxel * V, 1),
        "accuracies_compared": int(ncompare), "accuracies_identical": int(same),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voxels", type=int, default=50000)
    ap.add_argument("--T", type=int, default=15)
    ap.add_argument("--configs", default="140:20:7,256:16:16", help="E:eps:folds,...")
    ap.add_argument("--kinds", default="linear,rbf")
    ap.add_argument("--compare", type=int, default=256)
    ap.add_argument("--time-voxels", type=int, default=4)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    a = ap.parse_args()
    _lib.require_device()
    print("card (name, power limit, max SM clock):", card(), flush=True)
    out = []
    with multiprocessing.get_context("spawn").Pool(max(1, min(32, os.cpu_count() or 1))) as pool:
        for cfg in a.configs.split(","):
            E, eps, folds = (int(x) for x in cfg.split(":"))
            for kind in a.kinds.split(","):
                r = run_config(a.voxels, a.T, E, eps, folds, kind, a.compare, a.time_voxels, pool)
                print(json.dumps(r), flush=True)
                out.append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": card(), "results": out}, f, indent=1)


if __name__ == "__main__":
    main()
