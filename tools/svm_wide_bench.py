#!/usr/bin/env python
"""VoxelSelector.run with SVC(kernel='precomputed') above 64 epochs: the wide GPU solver (fcma_svm_cv_solve_wide)
against the host path (one scikit-learn cross_val_score per voxel, as the reference does).

Configurations (V voxels, T time points, E epochs, eps epochs per subject, folds): the reference's FCMA script shape,
E = 140, eps = 20, 7 folds (docs/examples/fcma/FCMA_script/fcma_voxel_selection_cv.py: VoxelSelector(labels, 20, 7, ...)
with SVC(kernel='precomputed', shrinking=False, C=1)), and E = 256, eps = 16, 16 folds.  For each it reports:
* cv_s: CUDA events around each block's svm_cv_precomputed call, the accuracies read back included;
* kernels_s: CUDA events around each block's voxel_kernels call (the generic pipeline: strided correlation block,
  k_within_subject_norm, k_syrk_simt), and the library's own GEMM / second-stage split of it;
* run_s: the whole run(), after a warm-up run;
* the host path's time per voxel over a block of voxels, in one process and with process_num = 4, extrapolated to V
  (labelled as such);
* the accuracies of that block, GPU against host.
The card's name and power limit are printed in the same run.

    python tools/svm_wide_bench.py [--voxels 50000] [--T 15] [--configs 140:20:7,256:16:16] [--host-voxels 256]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
from sklearn import svm  # noqa: E402

from brainiak_b200 import _lib  # noqa: E402
from brainiak_b200.fcma import engine, synthetic  # noqa: E402
from brainiak_b200.fcma.voxelselector import VoxelSelector, shrink_kernels_  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def timed(fn, sink):
    """fn wrapped in CUDA events; the elapsed ms of every call go to sink."""
    def call(*a, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn(*a, **kw)
        e1.record()
        e1.synchronize()
        sink.append(e0.elapsed_time(e1))
        return out
    return call


def run_config(V, T, E, eps, folds, shrinking, nhost):
    raw, labels = synthetic.make_epochs(V, T, E)
    clf = svm.SVC(kernel="precomputed", shrinking=shrinking, C=1)
    vs = VoxelSelector(labels, eps, folds, raw, device="cuda:0")
    assert engine.svm_cv_supported(clf, labels, folds, E, max_epochs=engine.SVM_WIDE_MAX_EPOCHS)
    lib = _lib.load()
    vs.run(clf)                               # warm-up: operands, scratch, module loads
    cv_ms, k_ms = [], []
    orig_cv, orig_k = engine.svm_cv_precomputed, engine.voxel_kernels
    engine.svm_cv_precomputed, engine.voxel_kernels = timed(orig_cv, cv_ms), timed(orig_k, k_ms)
    lib.fcma_timing_enable(1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    try:
        res = vs.run(clf)
        torch.cuda.synchronize()
    finally:
        engine.svm_cv_precomputed, engine.voxel_kernels = orig_cv, orig_k
    wall = time.perf_counter() - t0
    gemm, stage = ctypes.c_double(), ctypes.c_double()
    lib.fcma_timing_read(ctypes.byref(gemm), ctypes.byref(stage))
    lib.fcma_timing_enable(0)
    acc = dict(res)
    # host path on one block of voxels: the same GPU kernels, shrunk on the host, scikit-learn per voxel
    s = V // 3
    rows_op, cols_op = vs._operands()
    K = engine.voxel_kernels(rows_op, cols_op, s, nhost, eps)
    data = shrink_kernels_(K.cpu().numpy())
    host = {}
    for procs in (1, 4):
        vs.process_num, vs.use_multiprocessing = procs, procs > 1
        t0 = time.perf_counter()
        out = vs._do_cross_validation(clf, data, (s, nhost))
        host[procs] = (time.perf_counter() - t0) / nhost
    same = sum(acc[v] == a for v, a in out)
    cv_s = sum(cv_ms) / 1e3
    return {
        "V": V, "T": T, "E": E, "eps": eps, "folds": folds, "shrinking": shrinking,
        "run_s": round(wall, 3), "cv_s": round(cv_s, 3), "cv_us_per_voxel": round(cv_s / V * 1e6, 2),
        "kernels_s": round(sum(k_ms) / 1e3, 3), "kernels_gemm_s": round(gemm.value / 1e3, 3),
        "kernels_stage2_s": round(stage.value / 1e3, 3),
        "host_ms_per_voxel_1proc": round(host[1] * 1e3, 2), "host_ms_per_voxel_4proc": round(host[4] * 1e3, 2),
        "host_voxels_timed": nhost,
        "host_cv_s_extrapolated_1proc": round(host[1] * V, 1), "host_cv_s_extrapolated_4proc": round(host[4] * V, 1),
        "cv_speedup_vs_4proc": round(host[4] * V / cv_s, 1),
        "accuracies_compared": nhost, "accuracies_identical": int(same),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voxels", type=int, default=50000)
    ap.add_argument("--T", type=int, default=15)
    ap.add_argument("--configs", default="140:20:7,256:16:16", help="E:eps:folds,...")
    ap.add_argument("--shrinking", default="0", help="0, 1 or 0,1")
    ap.add_argument("--host-voxels", type=int, default=256)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    a = ap.parse_args()
    _lib.require_device()
    print("card (name, power limit, max SM clock):", card(), flush=True)
    out = []
    for cfg in a.configs.split(","):
        E, eps, folds = (int(x) for x in cfg.split(":"))
        for sh in a.shrinking.split(","):
            r = run_config(a.voxels, a.T, E, eps, folds, sh == "1", a.host_voxels)
            print(json.dumps(r), flush=True)
            out.append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": card(), "results": out}, f, indent=1)


if __name__ == "__main__":
    main()
