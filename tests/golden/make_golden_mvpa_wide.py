#!/usr/bin/env python
"""Generate tests/golden/mvpa_w*.npz, the MVPAVoxelSelector fixtures above 64 epochs, by running the UNMODIFIED
reference MVPAVoxelSelector and Searchlight on small seeded inputs, single process, exactly as make_golden_mvpa.py does
(its one-rank mpi4py stub, pool_size=1, the same seeded volume with a planted blob and a ragged mask).

Run from the repo root where the reference tree exists (FCMA_REFERENCE_ROOT, default /root/reference):

    python tests/golden/make_golden_mvpa_wide.py
"""
import os
import sys

from sklearn import svm

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden_mvpa import save, synthetic  # noqa: E402  (loads the reference)


def gen_mvpa_wide():
    # (w1) the example's call (examples/fcma/run_mvpa_voxel_selection.sh on the face-scene data): 18 subjects x 12
    # epochs = 216 epochs, 18 folds, SVC(kernel='linear', shrinking=False, C=1), sl_rad 1 cube
    d, m, y = synthetic(16, (6, 7, 6), 216, 2)
    save("w1", d, m, y, 18, 1, "Cube", 0, "linear C=1 shrinking=False", svm.SVC(kernel='linear', shrinking=False, C=1))
    # (w2) 140 epochs, three classes, 7 folds, rbf, a radius-2 ball with min_active_voxels_proportion 0.2
    d, m, y = synthetic(17, (7, 8, 7), 140, 3)
    save("w2", d, m, y, 7, 2, "Ball", 0.2, "rbf C=10 gamma=auto", svm.SVC(kernel='rbf', C=10, gamma='auto'))


if __name__ == "__main__":
    gen_mvpa_wide()
