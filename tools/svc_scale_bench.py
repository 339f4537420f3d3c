#!/usr/bin/env python
"""scikit-learn's default ``SVC()`` (rbf, gamma='scale': one gamma per item and fold) on the GPU, in both selectors.

Workloads:
* ``VoxelSelector.run(SVC())`` at V = V2 voxels (default 50 000) on synthetic epochs: E = 32 (T = 200, 8 epochs per
  subject, 4 folds) and E = 140 (T = 15, 20 epochs per subject, 7 folds);
* ``MVPAVoxelSelector.run(SVC())`` on tools/mvpa_bench.py's seeded 91 x 109 x 91 volume, radius-1 cube: E = 32 (8 folds)
  and E = 216 (18 folds, the shape of the reference's MVPA example).

For each run it reports the end-to-end ``run()`` time (host clock, ends in a device synchronise), the CUDA-event times
summed over the run of the stages -- builder (correlation GEMM, normalisation, G, D and the moments; searchlight: G, D and
the moments), fold gammas, per-fold rbf expansion, solver -- and the moments' share of the builder from a torch.profiler
trace of one block (the moments run inside the builder's pipeline call); the number of items scored on the host (the
variance check of engine.fold_gammas); and 256 sampled accuracies against the host path (scikit-learn per item, as the
reference does; ``--vs-compare`` takes fewer voxels, whose host path on 50 000 features costs over a second each).  The card's name and power limit are
read in the same run.

    python tools/svc_scale_bench.py [--voxels 50000] [--vs 32:200:8:4,140:15:20:7] [--mvpa 32:8,216:18] [--compare 256]
                                    [--vs-compare N] [--out FILE]
"""
import argparse
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
from brainiak_b200 import searchlight as slm  # noqa: E402
from brainiak_b200.fcma import engine, synthetic  # noqa: E402
from brainiak_b200.fcma.mvpa_voxelselector import MVPAVoxelSelector  # noqa: E402
from brainiak_b200.fcma.voxelselector import VoxelSelector  # noqa: E402
from feature_svc_bench import host_acc  # noqa: E402
from mvpa_bench import card, volume  # noqa: E402

STAGES = {"builder": ("feature_gram_wide", "searchlight_gram_wide"), "gammas": ("fold_gammas",),
          "expansion": ("rbf_fold_kernels",), "solver": ("_svm_correct",)}


class StageTimer:
    """Wraps the engine functions of each stage with CUDA events on the current stream (no synchronisation inside the
    run), and counts the items svm_cv_scale flags for the host."""

    def __init__(self):
        self.events = {k: [] for k in STAGES}
        self.flagged = 0
        self.saved = {}

    def __enter__(self):
        for stage, names in STAGES.items():
            for name in names:
                self.saved[name] = getattr(engine, name)
                setattr(engine, name, self._wrap(stage, self.saved[name]))
        self.saved["svm_cv_scale"] = orig_cv = engine.svm_cv_scale

        def counted(*a, **kw):
            out = orig_cv(*a, **kw)
            self.flagged += int(out[1].sum())
            return out
        engine.svm_cv_scale = counted
        return self

    def _wrap(self, stage, fn):
        def timed(*a, **kw):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = fn(*a, **kw)
            e1.record()
            self.events[stage].append((e0, e1))
            return out
        return timed

    def __exit__(self, *exc):
        for name, fn in self.saved.items():
            setattr(engine, name, fn)
        torch.cuda.synchronize()

    def seconds(self):
        return {k: round(sum(a.elapsed_time(b) for a, b in v) / 1e3, 3) for k, v in self.events.items()}


def profiled(fn, keys):
    """Kernel times (s) of one call of fn, by kernel name, from torch.profiler."""
    fn()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for key in keys:
            if key in ev.key:
                t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                out[key] = round(out.get(key, 0.0) + t / 1e6, 4)
    return out


def compare(acc, items, feats, labels, folds, pool):
    host = pool.map(host_acc, [(svm.SVC(), X, labels, folds) for X in feats])
    return sum(acc[i] == h for i, h in zip(items, host))


def run_vs(V, T, E, eps, folds, ncompare, pool):
    raw, labels = synthetic.make_epochs(V, T, E)
    clf = svm.SVC()
    VoxelSelector(labels, eps, folds, [m[:, :512] for m in raw], device="cuda:0").run(clf)      # warm-up, module loads
    vs = VoxelSelector(labels, eps, folds, raw, device="cuda:0")
    assert vs._scale_ok(clf)
    torch.cuda.synchronize()
    with StageTimer() as timer:
        t0 = time.perf_counter()
        res = vs.run(clf)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    rows_op, cols_op = vs._operands()
    rows = min(V, 2048)
    split = profiled(lambda: engine.feature_gram_wide(rows_op, cols_op, 0, rows, eps, work=vs._work),
                     ("k_corr", "k_block_within_subject_norm", "k_block_moments", "k_feature_gram_tiled"))
    print("VoxelSelector E=%d: run() %.1f s; comparing %d voxels with the host path" % (E, wall, ncompare), flush=True)
    acc = dict(res)
    sample = np.sort(np.random.default_rng(1).choice(V, size=ncompare, replace=False))
    feats = []
    for v in sample:
        c = engine.corr_block(rows_op, cols_op, int(v), 1, layout=0).contiguous()
        feats.append(engine.within_subject_norm_(c, eps)[0].cpu().numpy())
    same = compare(acc, [int(v) for v in sample], feats, labels, folds, pool)
    return {"selector": "VoxelSelector", "V": V, "T": T, "E": E, "eps": eps, "folds": folds, "run_s": round(wall, 3),
            "stage_s": timer.seconds(), "profiled_rows": rows, "profiled_kernel_s": split,
            "host_scored": timer.flagged, "accuracies_compared": int(ncompare), "accuracies_identical": int(same)}


def run_mvpa(E, folds, ncompare, pool):
    data, mask, labels = volume(E)
    sl = slm.Searchlight(sl_rad=1, shape=slm.Cube)
    clf = svm.SVC()
    small = np.zeros_like(mask)
    small[40:50, 50:60, 40:50] = mask[40:50, 50:60, 40:50]
    MVPAVoxelSelector(data, small, labels, folds, sl).run(clf)                                   # warm-up, module loads
    mvs = MVPAVoxelSelector(data, mask, labels, folds, sl)
    assert mvs._gpu_kind(clf) == "scale"
    torch.cuda.synchronize()
    with StageTimer() as timer:
        t0 = time.perf_counter()
        volres, _ = mvs.run(clf)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    print("MVPAVoxelSelector E=%d: run() %.1f s" % (E, wall), flush=True)
    shape = np.asarray(sl.shape).astype(bool)
    centres, _ = engine.searchlight_centres(mask, 1, shape, sl.min_active_voxels_proportion)
    dev = torch.device("cuda")
    vt = torch.from_numpy(np.ascontiguousarray(data)).to(dev)
    mt = torch.from_numpy(mask.astype(np.uint8)).to(dev)
    st = torch.from_numpy(shape.astype(np.uint8)).to(dev)
    cb = centres[:min(len(centres), 1 << 15)]
    split = profiled(lambda: engine.searchlight_gram_wide(vt, mt, 1, st, cb),
                     ("k_searchlight_kernels_tiled", "k_searchlight_moments"))
    del vt
    flat = volres.reshape(-1)
    sample = np.sort(np.random.default_rng(1).choice(centres, size=ncompare, replace=False))
    acc = {int(c): flat[c] for c in sample}
    feats = [mvs._features(int(c), shape) for c in sample]
    same = compare(acc, [int(c) for c in sample], feats, labels, folds, pool)
    return {"selector": "MVPAVoxelSelector", "dims": list(mask.shape), "centres": int(len(centres)), "E": E,
            "folds": folds, "run_s": round(wall, 3), "stage_s": timer.seconds(), "profiled_centres": int(len(cb)),
            "profiled_kernel_s": split, "host_scored": timer.flagged, "accuracies_compared": int(ncompare),
            "accuracies_identical": int(same)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voxels", type=int, default=50000)
    ap.add_argument("--vs", default="32:200:8:4,140:15:20:7", help="E:T:eps:folds,... ('' = none)")
    ap.add_argument("--mvpa", default="32:8,216:18", help="E:folds,... ('' = none)")
    ap.add_argument("--compare", type=int, default=256, help="items compared with the host path per run")
    ap.add_argument("--vs-compare", type=int, default=None, help="VoxelSelector runs only (default: --compare)")
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    a = ap.parse_args()
    _lib.require_device()
    print("card (name, power limit):", card(), flush=True)
    out = []
    with multiprocessing.get_context("spawn").Pool(max(1, min(32, os.cpu_count() or 1))) as pool:
        for cfg in filter(None, a.vs.split(",")):
            E, T, eps, folds = (int(x) for x in cfg.split(":"))
            out.append(run_vs(a.voxels, T, E, eps, folds, a.vs_compare or a.compare, pool))
            print(json.dumps(out[-1]), flush=True)
        for cfg in filter(None, a.mvpa.split(",")):
            E, folds = (int(x) for x in cfg.split(":"))
            out.append(run_mvpa(E, folds, a.compare, pool))
            print(json.dumps(out[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": card(), "results": out}, f, indent=1)


if __name__ == "__main__":
    main()
