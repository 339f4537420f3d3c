#!/usr/bin/env python
"""Generate tests/golden/vs_pre_w*.npz, the VoxelSelector fixtures for SVC(kernel='precomputed') above 64 epochs with an
epochs_per_subj that is not a power of two (the generic kernel-matrix pipeline: raw r, in-place normalisation, SIMT
SYRK), by running the UNMODIFIED reference VoxelSelector (oracle/_ref, built by oracle/build_ref.sh) single process
through oracle.reference.run_voxel_selection.

Each file stores a probe of the seeded synthetic inputs (the tests regenerate them from the seed), the labels, the
reference's voxel list and its accuracies in the list's order, and the reference's shrunk kernel matrices of a few
sampled voxels (planted ones included), taken from its own stages (oracle.reference.voxel_block_stages).

Run from the repo root where the reference tree exists:

    bash oracle/build_ref.sh && python tests/golden/make_golden_precomputed_wide.py
"""
import os
import sys

import numpy as np
from sklearn import svm

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, input_probe, reference, synthetic  # noqa: E402

# voxels whose shrunk kernels are stored: w1's planted voxels are 0 .. 7
SAMPLES = {"w1": (0, 5, 21, 47), "w2": (0, 9, 16, 23)}


def save(name, raw, raw2, labels, eps, folds):
    m = reference.load()
    clf = svm.SVC(kernel='precomputed', shrinking=False, C=1)
    vs = m.voxelselector.VoxelSelector(labels, eps, folds, raw, raw_data2=raw2, voxel_unit=13, process_num=0)
    res = reference.run_voxel_selection(vs, clf)
    vids = np.array(SAMPLES[name])
    kernels = np.stack([reference.voxel_block_stages(vs, (int(v), 1), clf)[2][0] for v in vids])
    out = dict(probe=input_probe(raw), labels=np.array(labels), eps=eps, num_folds=folds,
               clf="precomputed C=1 shrinking=False", vids=np.array([v for v, _ in res]),
               accs=np.array([a for _, a in res], dtype=np.float64), sample_vids=vids, sample_kernels=kernels)
    if raw2 is not None:
        out["probe2"] = input_probe(raw2)
    np.savez_compressed(os.path.join(OUT, "vs_pre_%s.npz" % name), **out)
    print(name, "top voxels", out["vids"][:10], "acc", out["accs"][:10])


def gen_precomputed_wide():
    # (w1) the inputs of vs_feat_w1: the reference FCMA script's epoch structure (7 subjects x 20 epochs = 140), 7 folds,
    # one mask of 48 voxels with 8 planted ones; dyadic, so every r is exact in any summation order
    raw, labels = synthetic.make_dyadic_epochs(48, 20, 140, seed=4242, informative=8)
    save("w1", raw, None, labels, 20, 7)
    # (w2) 100 epochs with eps 12: 8 subjects and 4 trailing raw epochs; three classes, 5 folds, two masks (24 row
    # voxels x 40 column voxels)
    d1, d2, _ = synthetic.make_two_masks(24, 40, 16, 100, seed=6262)
    save("w2", d1, d2, [e % 3 for e in range(100)], 12, 5)


if __name__ == "__main__":
    gen_precomputed_wide()
