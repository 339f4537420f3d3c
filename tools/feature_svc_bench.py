#!/usr/bin/env python
"""VoxelSelector.run with SVC(kernel='linear' | 'rbf') on the normalised correlation vectors, on the GPU, against the host
path (scikit-learn per voxel, as the reference does).

For each configuration (V = V2 voxels, T time points, E epochs, eps epochs per subject) it reports:
* the stage times from CUDA events: correlation GEMM, fp64 kernel pass (k_norm_gram_f64), cross validation (svm_cv_f64),
  and the whole run;
* the kernel pass's bytes (the fp32 block it reads, the fp64 matrices it writes) and fp64 operations (G: E(E+1)/2 products
  and additions per column, D for rbf: E(E-1)/2 differences and fmas) over its time, against the H100 SXM data sheet;
* the host path's time per voxel on a sample of voxels, extrapolated to V (labelled as such);
* the accuracies of sampled voxels, GPU against host.
The card's name and power limit are printed in the same run.

    python tools/feature_svc_bench.py [--voxels 50000] [--T 200] [--configs 32:8,64:8] [--compare 256]
"""
import argparse
import ctypes
import json
import multiprocessing
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
from sklearn import model_selection, svm  # noqa: E402

from brainiak_b200 import _lib  # noqa: E402
from brainiak_b200.fcma import engine, synthetic  # noqa: E402
from brainiak_b200.fcma.voxelselector import VoxelSelector  # noqa: E402

HBM = 3.35e12          # bytes/s, H100 SXM data sheet
FP64_TC = 67e12        # flop/s, fp64 tensor cores
FP64 = 34e12           # flop/s, FP64 pipe


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def host_acc(args):
    clf, X, y, folds = args
    skf = model_selection.StratifiedKFold(n_splits=folds, shuffle=False)
    return model_selection.cross_val_score(clf, X, y=y, cv=skf, n_jobs=1).mean()


def run_config(V, T, E, eps, kind, ncompare, ntime, pool):
    raw, labels = synthetic.make_epochs(V, T, E)
    folds = 4
    clf = svm.SVC(kernel="linear", shrinking=False) if kind == "linear" else \
        svm.SVC(kernel="rbf", gamma="auto", shrinking=False)
    vs = VoxelSelector(labels, eps, folds, raw, device="cuda:0")
    assert vs._feature_kind(clf) == kind
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

    vs.run(clf)                               # warm-up: operands, scratch, module loads
    engine.svm_cv_f64 = timed_cv
    cv_ms.clear()
    lib.fcma_timing_enable(1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = vs.run(clf)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    gemm, stage = ctypes.c_double(), ctypes.c_double()
    passes = lib.fcma_timing_read(ctypes.byref(gemm), ctypes.byref(stage))
    lib.fcma_timing_enable(0)
    engine.svm_cv_f64 = orig
    acc = dict(res)
    pairs_g = E * (E + 1) / 2
    flops = 2.0 * V * V * pairs_g + (2.0 * V * V * E * (E - 1) / 2 if kind == "rbf" else 0.0)
    nbytes = 4.0 * V * E * V + 8.0 * V * E * E * (2 if kind == "rbf" else 1)
    st = stage.value / 1e3
    # host path on sampled voxels: the same GPU correlations, normalised as _voxel_scoring does, scikit-learn per voxel
    rng = np.random.default_rng(1)
    sample = np.sort(rng.choice(V, size=max(ncompare, ntime), replace=False))
    rows_op, cols_op = vs._operands()
    feats = []
    for v in sample:
        c = engine.corr_block(rows_op, cols_op, int(v), 1, layout=0).contiguous()
        feats.append(engine.within_subject_norm_(c, eps)[0].cpu().numpy())
    t0 = time.perf_counter()
    for k in range(ntime):
        host_acc((clf, feats[k], labels, folds))
    host_per_voxel = (time.perf_counter() - t0) / ntime
    cmp = sample[:ncompare]
    host = pool.map(host_acc, [(clf, feats[k], labels, folds) for k in range(ncompare)])
    same = sum(acc[int(v)] == h for v, h in zip(cmp, host))
    return {
        "V": V, "T": T, "E": E, "eps": eps, "kind": kind, "passes": passes,
        "run_s": round(wall, 3), "gemm_s": round(gemm.value / 1e3, 3), "kernel_pass_s": round(st, 3),
        "cv_s": round(sum(cv_ms) / 1e3, 3),
        "kernel_pass_GBps": round(nbytes / st / 1e9, 1), "kernel_pass_fp64_TFLOPs": round(flops / st / 1e12, 2),
        "kernel_pass_hbm_share": round(nbytes / HBM / st, 3),
        "kernel_pass_fp64_share": round((2.0 * V * V * pairs_g / FP64_TC +
                                         (flops - 2.0 * V * V * pairs_g) / FP64) / st, 3),
        "host_s_per_voxel": round(host_per_voxel, 4), "host_voxels_timed": ntime,
        "host_total_s_extrapolated": round(host_per_voxel * V, 1),
        "accuracies_compared": int(ncompare), "accuracies_identical": int(same),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voxels", type=int, default=50000)
    ap.add_argument("--T", type=int, default=200)
    ap.add_argument("--configs", default="32:8,64:8", help="E:eps,...")
    ap.add_argument("--kinds", default="linear,rbf")
    ap.add_argument("--compare", type=int, default=256)
    ap.add_argument("--time-voxels", type=int, default=16)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    a = ap.parse_args()
    _lib.require_device()
    print("card (name, power limit, max SM clock):", card(), flush=True)
    out = []
    with multiprocessing.get_context("spawn").Pool(max(1, min(16, os.cpu_count() or 1))) as pool:
        for cfg in a.configs.split(","):
            E, eps = (int(x) for x in cfg.split(":"))
            for kind in a.kinds.split(","):
                r = run_config(a.voxels, a.T, E, eps, kind, a.compare, a.time_voxels, pool)
                print(json.dumps(r), flush=True)
                out.append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": card(), "results": out}, f, indent=1)


if __name__ == "__main__":
    main()
