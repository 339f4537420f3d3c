#!/usr/bin/env python
"""Generate tests/golden/loso_l*.npz, the leave-one-subject-out fixtures of VoxelSelector.run_held_out, by running the
UNMODIFIED reference VoxelSelector (oracle/_ref, built by oracle/build_ref.sh) single process through
oracle.reference.run_voxel_selection, once per held-out subject, as the reference's FCMA example does
(docs/examples/fcma/FCMA_script/fcma_voxel_selection_cv.py:69-79): the subject's epochs removed from the labels and the
epoch list (``subsampled_idx``), ``VoxelSelector(labels_s, eps, S - 1, raw_s)``, then the selection.

The inputs are seeded dyadic epochs (brainiak_b200.fcma.synthetic.make_dyadic_epochs: every correlation exact in fp32,
so every accuracy, chance-level voxels and ties included, is pinned); the tests regenerate them from the seed and each
file stores a probe of them, the labels and every subject's voxel list and accuracies in the list's order.

Run from the repo root where the reference tree exists:

    bash oracle/build_ref.sh && python tests/golden/make_golden_loso.py
"""
import os
import sys

import numpy as np
from sklearn import svm

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, input_probe, reference, synthetic  # noqa: E402


def loso_inputs(name):
    """(raw, raw2, labels, eps, clf) of fixture ``name``, regenerated from the seeds."""
    if name == "l1":
        # the example's structure: 8 subjects x 20 epochs = 160, one mask of 48 voxels with 8 planted ones; each
        # held-out run has 140 epochs (generic pipeline, wide solver)
        raw, labels = synthetic.make_dyadic_epochs(48, 20, 160, seed=7070, informative=8)
        return raw, None, labels, 20, svm.SVC(kernel='precomputed', shrinking=False, C=1)
    if name == "l2":
        # 8 subjects x 4 epochs = 32, 512 voxels: the full run and every held-out run take the symmetric pipeline
        raw, labels = synthetic.make_dyadic_epochs(512, 24, 32, seed=7171, informative=40)
        return raw, None, labels, 4, svm.SVC(kernel='precomputed', shrinking=False, C=1)
    if name == "l3":
        # two masks (20 row voxels x 36 column voxels), 6 subjects x 8 epochs = 48, three classes, linear SVC
        raw, _ = synthetic.make_dyadic_epochs(20, 16, 48, seed=7272, informative=5)
        raw2, _ = synthetic.make_dyadic_epochs(36, 16, 48, seed=7373, informative=6)
        labels = [e % 3 for e in range(48)]
        return raw, raw2, labels, 8, svm.SVC(kernel='linear', shrinking=False, C=1)
    raise ValueError(name)


def subsample(seq, eps, subject):
    """The example's subsampled list (fcma_voxel_selection_cv.py:69-75) without subject ``subject``."""
    start_idx = subject * eps
    subsampled_idx = list(set(range(len(seq))) - set(range(start_idx, start_idx + eps)))
    return [seq[i] for i in subsampled_idx]


def save(name):
    m = reference.load()
    raw, raw2, labels, eps, clf = loso_inputs(name)
    S = len(raw) // eps
    vids, accs = [], []
    for s in range(S):
        vs = m.voxelselector.VoxelSelector(subsample(labels, eps, s), eps, S - 1, subsample(raw, eps, s),
                                           raw_data2=None if raw2 is None else subsample(raw2, eps, s),
                                           voxel_unit=16, process_num=0)
        res = reference.run_voxel_selection(vs, clf)
        vids.append([v for v, _ in res])
        accs.append([a for _, a in res])
    out = dict(probe=input_probe(raw), labels=np.array(labels), eps=eps, vids=np.array(vids, dtype=np.int32),
               accs=np.array(accs, dtype=np.float64))
    if raw2 is not None:
        out["probe2"] = input_probe(raw2)
    np.savez_compressed(os.path.join(OUT, "loso_%s.npz" % name), **out)
    print(name, "subject 0 top voxels", out["vids"][0][:8], "acc", out["accs"][0][:8])


if __name__ == "__main__":
    for name in sys.argv[1:] or ["l1", "l2", "l3"]:
        save(name)
