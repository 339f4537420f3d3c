#!/usr/bin/env python
"""Whole-brain activity-based searchlight (MVPAVoxelSelector) on one GPU; prints one JSON line.

Workload, generated from a seed: a 91 x 109 x 91 volume with an ellipsoid mask of about 2.3e5 voxels, E = 16, 32 and
64 epochs (8 per subject, folds = subjects), searchlight radius 1 and 2 (cube), ``SVC(kernel='linear', shrinking=False,
C=1)``, the classifier of the reference's example.  For each configuration:

* CUDA-event times of the kernel-matrix stage (k_searchlight_kernels) and of the cross-validation (fp64 SMO), summed
  over the batches, and the kernel stage's output bytes (M E^2 8) against the H100 SXM data-sheet HBM bandwidth;
* the end-to-end ``run()`` time (host clock, ends in a device synchronise);
* a parity sample: 256 random centres scored by the host path (the reference's per-centre ``cross_val_score``) against
  the GPU accuracies;
* the host path's time per centre on 500 centres, and its extrapolation to all centres (labelled as extrapolated).

The card's name and power limit are read in the same run.  Usage: ``python tools/mvpa_bench.py [--out FILE]``.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from sklearn import svm

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from brainiak_b200 import searchlight as slm  # noqa: E402
from brainiak_b200.fcma import engine  # noqa: E402
from brainiak_b200.fcma.mvpa_voxelselector import MVPAVoxelSelector  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
DIMS = (91, 109, 91)


def card():
    """Name and power limit of the device torch runs on, looked up in nvidia-smi by its UUID (torch's device index is not
    nvidia-smi's under CUDA_VISIBLE_DEVICES)."""
    uuid = "GPU-%s" % torch.cuda.get_device_properties(torch.cuda.current_device()).uuid
    q = subprocess.run(["nvidia-smi", "-i", uuid, "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, _, power = (q.stdout.strip() if q.returncode == 0 else "").partition(",")
    return {"name": name.strip() or torch.cuda.get_device_name(), "power_limit": power.strip() or "unknown",
            "uuid": uuid}


def volume(E, seed=0):
    rng = np.random.default_rng(seed)
    g = np.stack(np.meshgrid(*[np.arange(n) for n in DIMS], indexing="ij"))
    c = np.array(DIMS).reshape(3, 1, 1, 1) / 2.0
    ax = np.array([36.0, 43.0, 36.0]).reshape(3, 1, 1, 1)
    mask = (((g - c) / ax) ** 2).sum(0) <= 1.0
    labels = np.arange(E) % 2
    data = rng.standard_normal(DIMS + (E,), dtype=np.float32)
    data[40:46, 50:56, 40:46] += (0.5 * labels).astype(np.float32)
    return data, mask, labels


def stage_times(data, mask, labels, folds, r, shape, clf, centres):
    dev = torch.device("cuda")
    vol = torch.from_numpy(data).to(dev)
    mt = torch.from_numpy(mask.astype(np.uint8)).to(dev)
    st = torch.from_numpy(shape.astype(np.uint8)).to(dev)
    E = data.shape[3]
    svm_folds = engine.make_svm_folds(labels, folds)
    free, _ = torch.cuda.mem_get_info(dev)
    batch = max(1, min(1 << 16, (free // 4) // (E * E * 8)))
    t_k = t_cv = 0.0
    accs = []
    for b0 in range(0, len(centres), batch):
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        e0.record()
        K, Kp = engine.searchlight_kernels(vol, mt, r, st, centres[b0:b0 + batch], "linear")
        e1.record()
        accs.append(engine.svm_cv_f64(K, Kp, labels, folds, C=clf.C, tol=clf.tol, shrinking=clf.shrinking,
                                      folds=svm_folds))
        e2.record()
        torch.cuda.synchronize()
        t_k += e0.elapsed_time(e1) / 1e3
        t_cv += e1.elapsed_time(e2) / 1e3
        del K, Kp
    return t_k, t_cv, np.concatenate(accs)


def one(E, r):
    data, mask, labels = volume(E)
    folds = E // 8
    clf = svm.SVC(kernel="linear", shrinking=False, C=1)
    sl = slm.Searchlight(sl_rad=r, shape=slm.Cube)
    centres, nfeat = engine.searchlight_centres(mask, r, sl.shape, 0)
    # warm-up of every kernel and shape the timed window uses
    stage_times(data, mask, labels, folds, r, sl.shape, clf, centres[:4096])
    t_k, t_cv, acc = stage_times(data, mask, labels, folds, r, sl.shape, clf, centres)
    mvs = MVPAVoxelSelector(data, mask, labels, folds, sl)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    vol, results = mvs.run(clf)
    torch.cuda.synchronize()
    t_run = time.perf_counter() - t0
    run_acc = np.array([vol.reshape(-1)[c] for c in centres], dtype=np.float64)
    rng = np.random.RandomState(1)
    sample = np.sort(rng.choice(len(centres), size=256, replace=False))
    host = np.array(mvs._run_host(clf, centres[sample], sl.shape))
    t0 = time.perf_counter()
    mvs._run_host(clf, centres[:500], sl.shape)
    t_host = (time.perf_counter() - t0) / 500
    kbytes = len(centres) * E * E * 8
    return {
        "E": E, "sl_rad": r, "folds": folds, "centres": int(len(centres)), "mean_features": float(nfeat.mean()),
        "kernel_stage_s": round(t_k, 5), "cv_stage_s": round(t_cv, 5),
        "kernel_stage_bytes": kbytes, "kernel_stage_hbm_share": round(kbytes / t_k / HBM_BYTES_PER_S, 4),
        "run_s": round(t_run, 4), "run_matches_stages": bool(np.array_equal(run_acc, acc)),
        "parity_centres": 256, "parity_identical": int((host == acc[sample]).sum()),
        "host_s_per_centre": round(t_host, 6),
        "host_extrapolated_s": round(t_host * len(centres), 1),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--configs", default="16:1,32:1,32:2,64:1,64:2", help="E:sl_rad list")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mvpa_bench needs a CUDA device")
    res = {"bench": "mvpa_searchlight", "card": card(), "volume": list(DIMS),
           "configs": [one(int(e), int(r)) for e, r in (c.split(":") for c in args.configs.split(","))]}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
