#!/usr/bin/env python
"""Generate tests/golden/vs_feat_w*.npz, the VoxelSelector fixtures for SVC(kernel='linear' | 'rbf') on the correlation
vectors above 64 epochs, by running the UNMODIFIED reference VoxelSelector (oracle/_ref, built by oracle/build_ref.sh)
single process through oracle.reference.run_voxel_selection.

The inputs are seeded synthetic epochs (brainiak_b200.fcma.synthetic); at 140 and 256 epochs they do not fit the 1 MB a
fixture may take, so the tests regenerate them from the seed and each file stores a probe of them (as config1.npz does),
the reference's voxel list and its accuracies in the list's order.

Run from the repo root where the reference tree exists:

    bash oracle/build_ref.sh && python tests/golden/make_golden_feature_wide.py
"""
import os
import sys

import numpy as np
from sklearn import svm

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, input_probe, reference, synthetic  # noqa: E402


def save(name, raw, raw2, labels, eps, folds, clf_desc, clf, voxel_unit):
    m = reference.load()
    vs = m.voxelselector.VoxelSelector(labels, eps, folds, raw, raw_data2=raw2, voxel_unit=voxel_unit, process_num=0)
    res = reference.run_voxel_selection(vs, clf)
    out = dict(probe=input_probe(raw), labels=np.array(labels), eps=eps, num_folds=folds, clf=clf_desc,
               vids=np.array([v for v, _ in res]), accs=np.array([a for _, a in res], dtype=np.float64))
    if raw2 is not None:
        out["probe2"] = input_probe(raw2)
    np.savez_compressed(os.path.join(OUT, "vs_feat_%s.npz" % name), **out)
    print(name, "top voxels", out["vids"][:8], "acc", out["accs"][:8])


def gen_feature_wide():
    # (w1) the reference FCMA script's epoch structure: 7 subjects x 20 epochs = 140 epochs, 7 folds, linear SVC on the
    # correlation vectors, one mask of 48 voxels with 8 planted ones.  Dyadic inputs: the reference's sgemm and any other
    # summation order give the same r bit for bit, so every accuracy, chance-level voxels and ties included, is pinned.
    raw, labels = synthetic.make_dyadic_epochs(48, 20, 140, seed=4242, informative=8)
    save("w1", raw, None, labels, 20, 7, "linear C=1 shrinking=False",
         svm.SVC(kernel='linear', shrinking=False, C=1), voxel_unit=13)
    # (w2) 16 subjects x 16 epochs = 256 epochs, three classes, 16 folds, two masks (24 row voxels x 40 column voxels),
    # rbf with gamma='auto' (1 / 40)
    d1, d2, _ = synthetic.make_two_masks(24, 40, 16, 256, seed=5151)
    labels3 = [e % 3 for e in range(256)]
    save("w2", d1, d2, labels3, 16, 16, "rbf C=10 gamma=auto", svm.SVC(kernel='rbf', gamma='auto', C=10),
         voxel_unit=7)


if __name__ == "__main__":
    gen_feature_wide()
