#!/usr/bin/env python
"""Whole-brain activity-based searchlight (MVPAVoxelSelector) above 64 epochs on one GPU; prints one JSON line.

Workload: tools/mvpa_bench.py's seeded 91 x 109 x 91 volume (about 2.3e5 centres) at the shape of the reference's MVPA
example (examples/fcma/run_mvpa_voxel_selection.sh on the face-scene data: 18 subjects x 12 epochs = 216 epochs, 18
folds, searchlight radius 1 cube, ``SVC(kernel='linear', shrinking=False, C=1)``).  It reports:

* CUDA-event times of the kernel-matrix stage (k_searchlight_kernels_tiled) and of the cross-validation
  (fcma_svm_cv_solve_f64_wide), summed over the batches, and the kernel stage's output bytes (M E^2 8) against the H100
  SXM data-sheet HBM bandwidth;
* the end-to-end ``run()`` time (host clock, ends in a device synchronise);
* a parity sample: 256 random centres scored by the host path (the reference's per-centre ``cross_val_score``) against
  the GPU accuracies;
* the host path's time per centre, and its extrapolation to all centres (labelled as extrapolated);
* the A/B of the two kernel builders at E = 16, 32 and 64 (``--ab``): fcma_searchlight_kernels (k_searchlight_kernels)
  and fcma_searchlight_kernels_wide (k_searchlight_kernels_tiled) of the same library called alternately on all centres,
  linear and rbf, CUDA-event medians, outputs compared byte for byte.

The card's name and power limit are read in the same run.
Usage: ``python tools/mvpa_wide_bench.py [--E 216] [--folds 18] [--ab 16,32,64] [--out FILE]``.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch
from sklearn import svm

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from brainiak_b200 import searchlight as slm  # noqa: E402
from brainiak_b200.fcma import engine  # noqa: E402
from brainiak_b200.fcma.mvpa_voxelselector import MVPAVoxelSelector  # noqa: E402
from mvpa_bench import DIMS, HBM_BYTES_PER_S, card, volume  # noqa: E402


def stage_times(data, mask, labels, folds, r, shape, clf, centres):
    dev = torch.device("cuda")
    vol = torch.from_numpy(data).to(dev)
    mt = torch.from_numpy(mask.astype(np.uint8)).to(dev)
    st = torch.from_numpy(shape.astype(np.uint8)).to(dev)
    E = data.shape[3]
    svm_folds = engine.svm_folds_for(labels, folds, E)
    free, _ = torch.cuda.mem_get_info(dev)
    batch = max(1, min(1 << 16, (free // 4) // (E * E * 8)))
    t_k = t_cv = 0.0
    accs = []
    for b0 in range(0, len(centres), batch):
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        e0.record()
        K, Kp = engine.searchlight_kernels_wide(vol, mt, r, st, centres[b0:b0 + batch], "linear")
        e1.record()
        accs.append(engine.svm_cv_f64(K, Kp, labels, folds, C=clf.C, tol=clf.tol, shrinking=clf.shrinking,
                                      folds=svm_folds))
        e2.record()
        torch.cuda.synchronize()
        t_k += e0.elapsed_time(e1) / 1e3
        t_cv += e1.elapsed_time(e2) / 1e3
        del K, Kp
    return t_k, t_cv, np.concatenate(accs), batch


def example_shape(E, folds, r, nhost):
    data, mask, labels = volume(E)
    clf = svm.SVC(kernel="linear", shrinking=False, C=1)
    sl = slm.Searchlight(sl_rad=r, shape=slm.Cube)
    centres, nfeat = engine.searchlight_centres(mask, r, sl.shape, 0)
    # warm-up of every kernel and shape the timed window uses
    stage_times(data, mask, labels, folds, r, sl.shape, clf, centres[:4096])
    t_k, t_cv, acc, batch = stage_times(data, mask, labels, folds, r, sl.shape, clf, centres)
    print("stages: kernels %.3f s, cross-validation %.3f s, batch %d" % (t_k, t_cv, batch), file=sys.stderr, flush=True)
    mvs = MVPAVoxelSelector(data, mask, labels, folds, sl)
    assert mvs._gpu_kind(clf) == "linear"
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    vol, results = mvs.run(clf)
    torch.cuda.synchronize()
    t_run = time.perf_counter() - t0
    print("run(): %.3f s" % t_run, file=sys.stderr, flush=True)
    run_acc = np.array([vol.reshape(-1)[c] for c in centres], dtype=np.float64)
    rng = np.random.RandomState(1)
    sample = np.sort(rng.choice(len(centres), size=nhost, replace=False))
    t0 = time.perf_counter()
    host = np.array(mvs._run_host(clf, centres[sample], sl.shape))
    t_host = (time.perf_counter() - t0) / len(sample)
    kbytes = len(centres) * E * E * 8
    return {
        "E": E, "sl_rad": r, "folds": folds, "centres": int(len(centres)), "mean_features": float(nfeat.mean()),
        "batch_centres": int(batch),
        "kernel_stage_s": round(t_k, 4), "cv_stage_s": round(t_cv, 4),
        "kernel_stage_bytes": kbytes, "kernel_stage_hbm_share": round(kbytes / t_k / HBM_BYTES_PER_S, 4),
        "run_s": round(t_run, 3), "run_matches_stages": bool(np.array_equal(run_acc, acc)),
        "parity_centres": len(sample), "parity_identical": int((host == acc[sample]).sum()),
        "host_s_per_centre": round(t_host, 6), "host_extrapolated_s": round(t_host * len(centres), 1),
    }


def ab(E, r, reps):
    """k_searchlight_kernels against k_searchlight_kernels_tiled on all centres, called alternately."""
    data, mask, labels = volume(E)
    dev = torch.device("cuda")
    shape = slm.Cube(r).mask_
    centres, nfeat = engine.searchlight_centres(mask, r, shape, 0)
    vol = torch.from_numpy(data).to(dev)
    mt = torch.from_numpy(mask.astype(np.uint8)).to(dev)
    st = torch.from_numpy(shape.astype(np.uint8)).to(dev)
    gamma = 1.0 / nfeat.astype(np.float64)
    out = {"E": E, "sl_rad": r, "centres": int(len(centres))}
    for kind in ("linear", "rbf"):
        g = gamma if kind == "rbf" else None
        times = {"narrow": [], "tiled": []}
        fns = {"narrow": engine.searchlight_kernels, "tiled": engine.searchlight_kernels_wide}
        res = {}
        for i in range(reps + 1):                     # the first round is the warm-up
            for name in (("narrow", "tiled") if i % 2 == 0 else ("tiled", "narrow")):
                res.pop(name, None)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                res[name] = fns[name](vol, mt, r, st, centres, kind, g)
                e1.record()
                e1.synchronize()
                if i:
                    times[name].append(e0.elapsed_time(e1))
        same = all(torch.equal(a, b) for a, b in zip(res["narrow"], res["tiled"]))
        out[kind] = {"narrow_ms": times["narrow"], "tiled_ms": times["tiled"],
                     "narrow_median_ms": round(float(np.median(times["narrow"])), 3),
                     "tiled_median_ms": round(float(np.median(times["tiled"])), 3), "byte_identical": bool(same)}
        del res
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--E", type=int, default=216)
    ap.add_argument("--folds", type=int, default=18)
    ap.add_argument("--sl-rad", type=int, default=1)
    ap.add_argument("--host-centres", type=int, default=256)
    ap.add_argument("--ab", default="16,32,64", help="epoch counts of the kernel A/B ('' = none)")
    ap.add_argument("--ab-reps", type=int, default=6)
    ap.add_argument("--skip-example", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mvpa_wide_bench needs a CUDA device")
    res = {"bench": "mvpa_searchlight_wide", "card": card(), "volume": list(DIMS)}
    if args.ab:
        res["ab"] = [ab(int(e), args.sl_rad, args.ab_reps) for e in args.ab.split(",")]
    if not args.skip_example:
        res["example"] = example_shape(args.E, args.folds, args.sl_rad, args.host_centres)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
