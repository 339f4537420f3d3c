#!/usr/bin/env python
"""Leave-one-subject-out voxel selection: VoxelSelector.run_held_out (one kernel build, then every held-out subject's
compaction and cross validation) against the reference FCMA example's loop of one run() per held-out subject
(docs/examples/fcma/FCMA_script/fcma_voxel_selection_cv.py).

Shape of the example: V = 50 000 voxels, T = 15, 8 subjects x 20 epochs (E = 160), 7 inner folds,
SVC(kernel='precomputed', shrinking=False, C=1); ``--clf linear`` takes the feature route (fp64 kernels of the
normalised correlation vectors) instead.  Reported:
* run_held_out_s: the wall time of run_held_out() (after a small warm-up run at 2048 voxels);
* CUDA-event sums inside it: the kernel build, the compaction (engine.subset_kernels, with its achieved GB/s from the
  bytes the shapes give: E_keep^2 elements read and written per kernel) and the cross validation;
* the per-subject loop: run() of ``--loop-subjects`` held-out subjects in the same process, extrapolated to every subject
  (labelled as extrapolated);
* run_held_out()[s] against those run() lists over all voxels: equal lists, and the count of voxels with equal accuracy.
The card's name and power limit are printed in the same run.

    python tools/loso_bench.py [--voxels 50000] [--T 15] [--subjects 8] [--eps 20] [--clf precomputed|linear]
                               [--loop-subjects 2] [--out FILE]
"""
import argparse
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
from brainiak_b200.fcma.voxelselector import VoxelSelector, held_out_keep  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def timed(fn, sink, nbytes=None):
    """fn wrapped in CUDA events; the elapsed ms of every call go to sink (with the call's bytes when nbytes is given)."""
    def call(*a, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn(*a, **kw)
        e1.record()
        e1.synchronize()
        sink.append((e0.elapsed_time(e1), nbytes(*a, **kw) if nbytes else 0))
        return out
    return call


def subset_bytes(K, keep, **kw):
    return 2 * K.shape[0] * len(keep) ** 2 * K.element_size()


STAGES = {"precomputed": ("voxel_kernels", "svm_cv_precomputed"), "linear": ("feature_kernels_f64_wide", "svm_cv_f64")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voxels", type=int, default=50000)
    ap.add_argument("--T", type=int, default=15)
    ap.add_argument("--subjects", type=int, default=8)
    ap.add_argument("--eps", type=int, default=20)
    ap.add_argument("--clf", default="precomputed", choices=sorted(STAGES))
    ap.add_argument("--loop-subjects", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    a = ap.parse_args()
    _lib.require_device()
    print("card (name, power limit, max SM clock):", card(), flush=True)
    V, T, S, eps = a.voxels, a.T, a.subjects, a.eps
    E = S * eps
    clf = svm.SVC(kernel=a.clf, shrinking=False, C=1)
    raw, labels = synthetic.make_epochs(V, T, E)
    VoxelSelector(labels, eps, S - 1, [m[:, :2048] for m in raw], device="cuda:0").run_held_out(clf, subjects=[0])

    build_name, cv_name = STAGES[a.clf]
    sinks = {"build": [], "subset": [], "cv": []}
    orig = {n: getattr(engine, n) for n in (build_name, cv_name, "subset_kernels")}
    setattr(engine, build_name, timed(orig[build_name], sinks["build"]))
    setattr(engine, cv_name, timed(orig[cv_name], sinks["cv"]))
    engine.subset_kernels = timed(orig["subset_kernels"], sinks["subset"], subset_bytes)
    try:
        vs = VoxelSelector(labels, eps, S - 1, raw, device="cuda:0")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        held = vs.run_held_out(clf)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    finally:
        for n, f in orig.items():
            setattr(engine, n, f)
    sub_ms = sum(ms for ms, _ in sinks["subset"])
    sub_bytes = sum(b for _, b in sinks["subset"])

    loop_s, equal_lists, equal_accs = [], 0, 0
    for s in range(a.loop_subjects):
        keep = held_out_keep(E, eps, s)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = VoxelSelector([labels[i] for i in keep], eps, S - 1, [raw[i] for i in keep], device="cuda:0").run(clf)
        torch.cuda.synchronize()
        loop_s.append(time.perf_counter() - t0)
        equal_lists += int(res == held[s])
        mine = dict(held[s])
        equal_accs += sum(int(mine[v] == acc) for v, acc in res)
    per_run = sum(loop_s) / len(loop_s) if loop_s else float("nan")
    r = {
        "card": card(), "clf": a.clf, "V": V, "T": T, "E": E, "eps": eps, "subjects": S, "inner_folds": S - 1,
        "run_held_out_s": round(wall, 3),
        "build_s": round(sum(ms for ms, _ in sinks["build"]) / 1e3, 3),
        "subset_s": round(sub_ms / 1e3, 4), "subset_calls": len(sinks["subset"]),
        "subset_GBps": round(sub_bytes / (sub_ms * 1e-3) / 1e9, 1) if sub_ms > 0 else None,
        "cv_s": round(sum(ms for ms, _ in sinks["cv"]) / 1e3, 3),
        "loop_subjects_run": a.loop_subjects, "loop_run_s": [round(x, 3) for x in loop_s],
        "loop_all_subjects_s_extrapolated": round(per_run * S, 1),
        "speedup_vs_loop_extrapolated": round(per_run * S / wall, 2),
        "lists_identical": "%d of %d" % (equal_lists, a.loop_subjects),
        "accuracies_identical": "%d of %d" % (equal_accs, a.loop_subjects * V),
    }
    print(json.dumps(r), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(r, f, indent=1)


if __name__ == "__main__":
    main()
