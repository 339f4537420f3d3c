#!/usr/bin/env python
"""Generate tests/golden/vs_scale_*.npz and mvpa_scale_*.npz, the fixtures of scikit-learn's default ``SVC()`` (rbf,
gamma='scale') and ``SVC(C=10, shrinking=False)``, by running the UNMODIFIED reference VoxelSelector (oracle/_ref,
built by oracle/build_ref.sh, single process through oracle.reference.run_voxel_selection) and the unmodified reference
MVPAVoxelSelector (loaded as make_golden_mvpa.py loads it, one-rank mpi4py stub, pool_size=1).

VoxelSelector inputs are dyadic epochs (synthetic.make_dyadic_epochs, as vs_feat_w1): every correlation is exact in
fp32, so the reference's sgemm and any other summation order give the same features bit for bit, and chance-level voxels
cannot be reordered by the GEMM.  They are regenerated from their seeds by the tests; each file stores a probe of them.
Each file holds the reference's voxel list (or result volume) and accuracies for both classifiers: ``*_default`` for
``SVC()``, ``*_c10`` for ``SVC(C=10, shrinking=False)``.

Run from the repo root where the reference tree exists:

    bash oracle/build_ref.sh && python tests/golden/make_golden_scale.py
"""
import os
import sys

import numpy as np
from sklearn import svm

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, input_probe, reference, synthetic  # noqa: E402

REF_VS = reference.load()      # before make_golden_mvpa installs its one-rank mpi4py stub (the VoxelSelector needs two)
from make_golden_mvpa import run_ref  # noqa: E402  (loads the reference searchlight)
from make_golden_mvpa import synthetic as mvpa_volume  # noqa: E402

CLFS = {"default": svm.SVC(), "c10": svm.SVC(C=10, shrinking=False)}


def vs_inputs(name):
    """The seeded inputs of vs_scale_<name>: (raw, raw2, labels, eps, folds); tests/test_gpu_svc_scale.py regenerates them."""
    if name == "s1":
        # 7 subjects x 20 epochs = 140 epochs (the reference FCMA script's structure), 7 folds, one mask of 48 voxels
        raw, labels = synthetic.make_dyadic_epochs(48, 20, 140, seed=6161, informative=8)
        return raw, None, labels, 20, 7
    # 4 subjects x 12 epochs = 48 epochs, three classes, 4 folds, two masks (24 row voxels x 40 column voxels)
    raw, _ = synthetic.make_dyadic_epochs(24, 16, 48, seed=7171, informative=6)
    raw2, _ = synthetic.make_dyadic_epochs(40, 16, 48, seed=8181, informative=10)
    return raw, raw2, [e % 3 for e in range(48)], 12, 4


def mvpa_inputs(name):
    """(data, mask, labels, folds) of mvpa_scale_<name>: sl_rad 1 cube."""
    if name == "s1":
        d, m, y = mvpa_volume(31, (7, 8, 6), 32, 2)
        return d, m, y, 4
    d, m, y = mvpa_volume(32, (6, 7, 6), 216, 3)
    return d, m, y, 18


def gen_vs(name):
    raw, raw2, labels, eps, folds = vs_inputs(name)
    m = REF_VS
    out = dict(probe=input_probe(raw), labels=np.array(labels), eps=eps, num_folds=folds)
    if raw2 is not None:
        out["probe2"] = input_probe(raw2)
    for key, clf in CLFS.items():
        vs = m.voxelselector.VoxelSelector(labels, eps, folds, raw, raw_data2=raw2, voxel_unit=11, process_num=0)
        res = reference.run_voxel_selection(vs, clf)
        out["vids_" + key] = np.array([v for v, _ in res])
        out["accs_" + key] = np.array([a for _, a in res], dtype=np.float64)
        print("vs", name, key, "top voxels", out["vids_" + key][:6], "acc", out["accs_" + key][:6])
    np.savez_compressed(os.path.join(OUT, "vs_scale_%s.npz" % name), **out)


def gen_mvpa(name):
    data, mask, labels, folds = mvpa_inputs(name)
    out = dict(data=data, mask=mask, labels=np.asarray(labels), num_folds=folds)
    for key, clf in CLFS.items():
        _, volf, ids, acc = run_ref(data, mask, labels, folds, 1, "Cube", 0, clf)
        out["volume_" + key], out["ids_" + key], out["acc_" + key] = volf, ids, acc
        print("mvpa", name, key, int(np.isfinite(volf).sum()), "centres, top", acc[:4])
    path = os.path.join(OUT, "mvpa_scale_%s.npz" % name)
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    for n in ("s1", "s2"):
        gen_vs(n)
        gen_mvpa(n)
