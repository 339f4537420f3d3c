#!/usr/bin/env python
"""Generate tests/golden/mvpa_*.npz by running the UNMODIFIED reference MVPAVoxelSelector and Searchlight
(src/brainiak/fcma/mvpa_voxelselector.py, src/brainiak/searchlight/searchlight.py of the reference tree) on small
seeded inputs, single process: mpi4py is replaced by a one-rank stub (rank 0, size 1, collectives that return their
argument) and the searchlight runs with pool_size=1, its serial branch.

Run from the repo root where the reference tree exists (FCMA_REFERENCE_ROOT, default /root/reference):

    python tests/golden/make_golden_mvpa.py

Each selector fixture stores the inputs, the result volume (NaN where the reference returns None) and the result list.
``mvpa_preproc.npz`` pins ``generate_epochs_info``, ``prepare_mvpa_data`` and ``prepare_searchlight_mvpa_data``
(src/brainiak/fcma/preprocessing.py of the reference, run unmodified) on the reference's two test subjects, together
with the reference's own expected outputs, and on a synthetic case with unequal epoch lengths and a constant voxel.
"""
import importlib.util
import os
import sys
import types

import numpy as np
from numpy.random import RandomState
from sklearn import svm
from sklearn.linear_model import LogisticRegression

OUT = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("FCMA_REFERENCE_ROOT", "/root/reference")


def _install_one_rank_mpi():
    mpi = types.ModuleType("mpi4py")
    MPI = types.ModuleType("mpi4py.MPI")

    class _Comm:
        rank, size = 0, 1

        def Get_rank(self):
            return 0

        def Get_size(self):
            return 1

        def bcast(self, obj, root=0):
            return obj

        def allreduce(self, obj):
            return obj

        def scatter(self, lst, root=0):
            return lst[0]

        def gather(self, obj, root=0):
            return [obj]

    MPI.COMM_WORLD = _Comm()
    mpi.MPI = MPI
    sys.modules["mpi4py"] = mpi
    sys.modules["mpi4py.MPI"] = MPI


def load_reference():
    """The reference's searchlight and mvpa_voxelselector modules, loaded from their files as a package
    ``brainiak`` with only what they import."""
    _install_one_rank_mpi()
    for k in [k for k in sys.modules if k == "brainiak" or k.startswith("brainiak.")]:
        del sys.modules[k]
    for name in ("brainiak", "brainiak.utils", "brainiak.searchlight", "brainiak.fcma"):
        pkg = types.ModuleType(name)
        pkg.__path__ = []
        sys.modules[name] = pkg
    utils = types.ModuleType("brainiak.utils.utils")
    utils.usable_cpu_count = lambda: len(os.sched_getaffinity(0))
    sys.modules["brainiak.utils.utils"] = utils
    # brainiak.image needs nibabel; preprocessing.py only calls mask_images, restated from image.py:107-187
    image = types.ModuleType("brainiak.image")
    image.mask_images = lambda images, mask, image_type=None: (
        (img.get_fdata().astype(image_type) if image_type is not None else img.get_fdata())[mask] for img in images)
    image.multimask_images = None
    sys.modules["brainiak.image"] = image
    mods = {}
    for name, rel in (("brainiak.searchlight.searchlight", "searchlight/searchlight.py"),
                      ("brainiak.fcma.mvpa_voxelselector", "fcma/mvpa_voxelselector.py"),
                      ("brainiak.fcma.preprocessing", "fcma/preprocessing.py")):
        spec = importlib.util.spec_from_file_location(name, os.path.join(REF, "src", "brainiak", rel))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        spec.loader.exec_module(mod)
        mods[name.rsplit(".", 1)[1]] = mod
    return mods["searchlight"], mods["mvpa_voxelselector"], mods["preprocessing"]


SL, MV, PP = load_reference()


def run_ref(data, mask, labels, folds, sl_rad, shape, p, clf):
    sl = SL.Searchlight(sl_rad=sl_rad, shape=getattr(SL, shape), min_active_voxels_proportion=p, pool_size=1)
    vol, results = MV.MVPAVoxelSelector(data, mask, labels, folds, sl).run(clf)
    volf = np.array([np.nan if v is None else float(v) for v in vol.ravel()]).reshape(vol.shape)
    ids = np.array([t[0] for t in results], dtype=np.int64)
    acc = np.array([float(t[1]) for t in results], dtype=np.float64)
    return vol, volf, ids, acc


def save(name, data, mask, labels, folds, sl_rad, shape, p, clf_spec, clf):
    _, volf, ids, acc = run_ref(data, mask, labels, folds, sl_rad, shape, p, clf)
    path = os.path.join(OUT, "mvpa_%s.npz" % name)
    np.savez_compressed(path, data=data, mask=mask, labels=np.asarray(labels), num_folds=folds, sl_rad=sl_rad,
                        shape=shape, min_active=p, clf=clf_spec, volume=volf, ids=ids, acc=acc)
    print(path, os.path.getsize(path), "bytes,", int(np.isfinite(volf).sum()), "centres")


def synthetic(seed, dims, E, nclass, blob_shift=0.6):
    """Seeded volume with a planted informative blob and a ragged mask that touches the faces."""
    prng = RandomState(seed)
    data = prng.randn(*dims, E).astype(np.float32)
    labels = np.arange(E) % nclass
    c = [d // 2 for d in dims]
    blob = np.zeros(dims, dtype=bool)
    blob[c[0] - 2:c[0] + 2, c[1] - 2:c[1] + 1, c[2] - 1:c[2] + 2] = True
    data[blob] += (np.float32(blob_shift) * labels.astype(np.float32))[None, :]
    mask = prng.rand(*dims) > 0.2
    mask[0, :, :] |= prng.rand(*dims[1:]) > 0.5
    mask[:, -1, :] |= prng.rand(dims[0], dims[2]) > 0.5
    return data.astype(np.float32), mask, labels


def gen_mvpa():
    # (a) the reference's own test input (tests/fcma/test_mvpa_voxel_selection.py:26-47), its expected output asserted
    prng = RandomState(1234567890)
    data = prng.rand(5, 5, 5, 8).astype(np.float32)
    mask = np.ones([5, 5, 5], dtype=bool)
    mask[0, 0, :] = False
    labels = [0, 1, 0, 1, 0, 1, 0, 1]
    clf = svm.SVC(kernel='rbf', C=10, gamma='auto')
    _, _, ids, acc = run_ref(data, mask, labels, 2, 1, "Cube", 0, clf)
    output = [int(8 * a) for a in acc if a > 0]
    expected = [6, 6, 5, 5, 5, 5, 5, 5, 5, 4, 4, 4, 4, 4, 4, 4, 4, 3, 3, 3, 3, 3, 2, 2, 2, 1]
    assert np.allclose(output, expected, atol=1), output
    save("a", data, mask, labels, 2, 1, "Cube", 0, "rbf C=10 gamma=auto", clf)

    # (b) the example's classifier (examples/fcma/mvpa_voxel_selection.py) on seeded volumes; the Ball of radius 2
    # covers 33 of 125 cube voxels, so min_active_voxels_proportion = 0.2 keeps some centres and drops others
    lin = "linear C=1 shrinking=False"
    d, m, y = synthetic(11, (10, 11, 9), 32, 2)
    save("b1", d, m, y, 4, 1, "Cube", 0, lin, svm.SVC(kernel='linear', shrinking=False, C=1))
    d, m, y = synthetic(12, (10, 11, 9), 64, 2)
    save("b2", d, m, y, 4, 2, "Ball", 0.2, lin, svm.SVC(kernel='linear', shrinking=False, C=1))
    d, m, y = synthetic(13, (10, 11, 9), 32, 3)
    save("b3", d, m, y, 4, 2, "Diamond", 0, lin, svm.SVC(kernel='linear', shrinking=False, C=1))
    d, m, y = synthetic(15, (9, 10, 8), 32, 2)
    save("b4", d, m, y, 4, 1, "Cube", 0.5, lin, svm.SVC(kernel='linear', shrinking=False, C=1))

    # (c) a classifier that is not an SVC: the host path
    d, m, y = synthetic(14, (6, 7, 6), 16, 2)
    save("c", d, m, y, 2, 1, "Cube", 0, "logistic", LogisticRegression())


class Image:
    """What the reference's preprocessing reads from a nibabel image."""

    def __init__(self, data, name):
        self.data, self.name = data, name

    def get_fdata(self):
        return self.data

    def get_filename(self):
        return self.name


def gen_preproc():
    sys.path.insert(0, OUT)
    from make_golden import read_nifti
    d = os.path.join(REF, "tests", "io", "data")
    mask = read_nifti(os.path.join(d, "mask.nii.gz")).astype(bool)
    subj = [read_nifti(os.path.join(d, "subject%d_bet.nii.gz" % s)) for s in (1, 2)]
    epochs = np.load(os.path.join(d, "epoch_labels.npy"))
    exp = os.path.join(REF, "tests", "fcma", "data")
    expected = np.load(os.path.join(exp, "expected_processed_data.npy"))
    expected_sl = np.load(os.path.join(exp, "expected_searchlight_processed_data.npy"))
    info = PP.generate_epochs_info(list(epochs))
    pd, labels = PP.prepare_mvpa_data([Image(v, "s%d" % i) for i, v in enumerate(subj)], list(epochs), mask)
    assert np.allclose(pd, expected)                      # the reference's own test (test_preprocessing.py:57-70)
    sd, sl_labels = PP.prepare_searchlight_mvpa_data([Image(v, "s%d" % i) for i, v in enumerate(subj)], list(epochs))
    assert np.allclose(sd, expected_sl)
    # synthetic: three subjects of unequal epoch lengths, one subject with a single epoch of a condition, a constant
    # voxel, and the reproducible voxel shuffle
    prng = RandomState(21)
    vols = [(prng.randn(5, 6, 4, 30) * 2 + 7).astype(np.float64) for _ in range(3)]
    for v in vols:
        v[2, 3, 1, :] = 4.0
    ep = np.zeros((3, 2, 3, 30), np.int8)
    for s in range(3):
        ep[s, 0, 0, 0:4 + s] = 1
        ep[s, 1, 0, 8:15] = 1
        ep[s, 0, 1, 16:19] = 1
        if s != 1:
            ep[s, 1, 1, 21:30 - s] = 1
    smask = prng.rand(5, 6, 4) > 0.3
    syn_info = PP.generate_epochs_info(list(ep))
    syn_pd, syn_labels = PP.prepare_mvpa_data([Image(v, "v") for v in vols], list(ep), smask)
    syn_sd, _ = PP.prepare_searchlight_mvpa_data([Image(v, "v") for v in vols], list(ep))
    syn_sd_rand, _ = PP.prepare_searchlight_mvpa_data([Image(v, "v") for v in vols], list(ep),
                                                       random=PP.RandomType.REPRODUCIBLE)
    path = os.path.join(OUT, "mvpa_preproc.npz")
    np.savez_compressed(path, mask=mask, subj=np.stack(subj), epochs=epochs, expected=expected,
                        expected_sl=expected_sl, info=np.array(info, dtype=np.int64), pd=pd, labels=labels, sd=sd,
                        sl_labels=sl_labels, vols=np.stack(vols), ep=ep, smask=smask,
                        syn_info=np.array(syn_info, dtype=np.int64), syn_pd=syn_pd, syn_labels=syn_labels,
                        syn_sd=syn_sd, syn_sd_rand=syn_sd_rand)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    gen_mvpa()
    gen_preproc()
