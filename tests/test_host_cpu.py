"""CPU-side checks: the C-ABI library loads and exports what include/fcma_b200.h declares, the host
logic behaves like the reference's, and nothing computes without a GPU (no silent fallback)."""
import ctypes
import os
import re

import numpy as np
import pytest
from sklearn import svm
from sklearn.base import clone
from sklearn.linear_model import LogisticRegression

from brainiak_b200 import _lib
from brainiak_b200.fcma import engine, synthetic
from brainiak_b200.fcma.classifier import Classifier
from brainiak_b200.fcma.voxelselector import VoxelSelector, shrink_kernels_

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _have_gpu():
    return _lib.device_count() > 0


def test_library_exports_every_declared_symbol():
    header = open(os.path.join(ROOT, "include", "fcma_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    declared = set(re.findall(r"\b(fcma_[a-z0-9_]+)\s*\(", header))
    assert len(declared) >= 20
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), "libfcma_b200.so does not export %s" % name
    # the ctypes signature table covers the header one to one
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    assert _lib.load().fcma_version() >= 100


def test_operand_geometry():
    lib = _lib.load()
    assert lib.fcma_operand_kp(_lib.PREC["bf16"], 200) == 208
    assert lib.fcma_operand_kp(_lib.PREC["tf32x3"], 200) == 200
    assert lib.fcma_operand_kp(_lib.PREC["tf32"], 12) == 16
    assert lib.fcma_operand_planes(_lib.PREC["bf16"]) == 1
    assert lib.fcma_operand_planes(_lib.PREC["bf16x3"]) == 2
    # K-major planes (rounded up to 256 B) + the exact self-correlation diagonal [E][V] fp32
    assert lib.fcma_operand_bytes(_lib.PREC["tf32x3"], 32, 200, 50000) == \
        2 * 32 * 50000 * 200 * 4 + 32 * 50000 * 4
    assert lib.fcma_operand_bytes(_lib.PREC["bf16"], 4, 50, 1000) == 4 * 1000 * 64 * 2 + 4 * 1000 * 4
    assert lib.fcma_operand_bytes(99, 4, 50, 1000) == 0
    assert lib.fcma_work_bytes_per_row(32, 50000) == 32 * 50176 * 4     # [E][ceil(V2/256)][rows][256]
    assert engine.fused_supported(32, 8) and engine.fused_supported(64, 64)
    assert not engine.fused_supported(32, 3) and not engine.fused_supported(65, 8)
    assert not engine.fused_supported(32, 64)


@pytest.mark.skipif(_have_gpu(), reason="checks the no-GPU behaviour")
def test_no_silent_cpu_fallback():
    lib = _lib.load()
    buf = np.zeros((2, 4, 8), np.float32)
    rc = lib.fcma_host_within_subject_norm(buf.ctypes.data_as(ctypes.c_void_p), 2, 4, 8, 2, 0)
    assert rc == _lib.FCMA_ENODEV and "sm_90" in _lib.last_error()
    rc = lib.fcma_within_subject_norm(None, 1, 1, 1, 1, None)
    assert rc == _lib.FCMA_ENODEV
    raw, labels = synthetic.make_epochs(16, 8, 4)
    vs = VoxelSelector(labels, 2, 2, raw)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        vs.run(svm.SVC(kernel="precomputed"))
    with pytest.raises(RuntimeError):
        vs._correlation_normalization(np.zeros((1, 4, 16), np.float32))
    from brainiak_b200.fcma.util import compute_correlation
    with pytest.raises(RuntimeError):
        compute_correlation(np.ones((2, 3), np.float32), np.ones((2, 3), np.float32))
    clf = Classifier(svm.SVC(kernel="precomputed"), epochs_per_subj=2)
    with pytest.raises(RuntimeError):
        clf.fit(list(zip(raw, raw)), labels)


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.FcmaLibraryMissing):
        _lib.load()


def test_resolve_precision_keeps_the_fp16_split_faithful():
    """'fp32' takes the fp16 hi/lo split only for |x| <= 8 and per-(epoch, voxel) norms >= 1/8 (or 0): below that the
    low plane goes subnormal and the split stops being fp32-faithful; tf32x3 otherwise.  CPU tensors, no device."""
    import torch
    rng = np.random.RandomState(3)
    g = rng.randn(4, 200, 64)
    unit = torch.from_numpy((g / np.linalg.norm(g, axis=1, keepdims=True)).astype(np.float32))
    res = engine.resolve_precision
    for s, want in ((8, "fp16x3"), (1, "fp16x3"), (0.25, "fp16x3"), (2.0 ** -4, "tf32x3"), (2.0 ** -8, "tf32x3"),
                    (2.0 ** -12, "tf32x3"), (2.0 ** -16, "tf32x3"), (2.0 ** -20, "tf32x3")):
        assert res("fp32", unit * s) == want, s
    big = unit.clone()
    big[1, 7, 3] = 8.5                                   # one element above the amax bound
    assert res("fp32", big) == "tf32x3"
    mixed = unit.clone()
    mixed[:, :, 10:18] *= 2.0 ** -14                     # normalised data with 8 voxels at a small scale
    assert res("fp32", mixed) == "tf32x3"
    one = unit.clone()
    one[2, :, 5] *= 2.0 ** -4                            # a single (epoch, voxel)
    assert res("fp32", one) == "tf32x3"
    tiny = unit.clone()
    tiny[0, :, 0] = 1e-30                                # squares underflow to a zero norm: still non-zero data
    assert res("fp32", tiny) == "tf32x3"
    zero = unit.clone()
    zero[:, :, :3] = 0                                   # all-zero voxels and (epoch, voxel) columns are exact
    zero[1, :, 10] = 0
    assert res("fp32", zero) == "fp16x3"
    assert res("fp32", torch.zeros(2, 5, 7)) == "fp16x3"
    # normalize=True: the packer's z-score makes every column unit-norm or zero, whatever the input scale
    assert res("fp32", unit * 2.0 ** -20, normalize=True) == "fp16x3"
    assert res("fp32", unit * 1e4, normalize=True) == "fp16x3"
    # explicit precisions are never changed
    for p in ("fp16x3", "tf32x3", "bf16x3", "tf32", "bf16"):
        assert res(p, unit * 2.0 ** -20) == p


def test_voxelselector_constructor_contract():
    raw, labels = synthetic.make_epochs(8, 6, 4)
    # voxelselector.py:130-134
    with pytest.raises(ValueError, match="same number"):
        VoxelSelector(labels, 2, 2, raw, raw_data2=raw[:3])
    # voxelselector.py:135-136
    with pytest.raises(ValueError, match="Zero processed voxels"):
        VoxelSelector(labels, 2, 2, [np.zeros((6, 0), np.float32)] * 4)
    with pytest.raises(ValueError):
        VoxelSelector(labels, 2, 2, raw, precision="fp8")
    vs = VoxelSelector(labels, 2, 2, raw, voxel_unit=3, process_num=0)
    assert vs.num_voxels == 8 and vs.num_voxels2 == 8 and not vs.use_multiprocessing
    assert vs.row_partition(10, 4) == [(0, 3), (3, 3), (6, 3), (9, 1)]
    assert sum(n for _, n in vs.row_partition(50000, 8)) == 50000
    assert vs.row_partition(3, 8)[3:] == [(3, 0)] * 5


def test_shrink_matches_reference_rule():
    from oracle import fcma_oracle as orc
    rng = np.random.RandomState(0)
    K = (rng.rand(7, 4, 4).astype(np.float32) + 0.5)
    K *= np.array([0.3, 5, 50, 99.9, 100, 4321, 1e6], np.float32)[:, None, None]
    K[:, 0, 0] = [0.3, 5, 50, 99.9, 100, 4321, 1e6]
    ref = K.copy()
    nds = [orc.shrink_(ref[i]) for i in range(7)]
    assert nds == [1, 1, 2, 2, 3, 4, 7]
    assert np.array_equal(shrink_kernels_(K.copy()), ref)


def test_classifier_is_a_cloneable_estimator():
    c = Classifier(svm.SVC(kernel="precomputed"), num_processed_voxels=7, epochs_per_subj=4)
    p = clone(c).get_params(deep=False)
    assert p["num_processed_voxels"] == 7 and p["epochs_per_subj"] == 4 and c.num_digits_ == 0
    # portion mode needs num_training_samples (classifier.py:399-409), checked before any GPU work
    raw, labels = synthetic.make_epochs(12, 6, 8)
    c = Classifier(svm.SVC(kernel="precomputed"), num_processed_voxels=4, epochs_per_subj=4)
    with pytest.raises(RuntimeError, match="portion by portion"):
        c.fit(list(zip(raw, raw)), labels)
    with pytest.raises(ValueError, match="smaller than"):
        c.fit(list(zip(raw, raw)), labels, num_training_samples=8)
    with pytest.raises(AssertionError):
        Classifier(LogisticRegression()).fit(list(zip(raw, raw)), labels[:3])


def test_host_shims_validate_like_cython_memoryviews():
    from brainiak_b200.fcma import cython_blas, fcma_extension
    with pytest.raises(RuntimeError, match="must be 3D"):
        fcma_extension.normalization(np.zeros((4, 4), np.float32), 2)
    a = np.zeros((4, 6), np.float64)
    with pytest.raises(ValueError):
        cython_blas.compute_self_corr_for_voxel_sel('N', 'T', 6, 2, 4, 1.0, a, 6, 0, a, 6, 0.0,
                                                    np.zeros((2, 1, 6), np.float32), 6, 0)


def test_svm_fold_descriptors_follow_sklearn_splits():
    """make_svm_folds: sklearn's own StratifiedKFold(shuffle=False) splits, training part ordered
    like libsvm's svm_group_classes (smaller label first = class +1, original order inside a class)."""
    from sklearn import model_selection
    labels = [3 if e % 3 else 7 for e in range(22)]          # unbalanced, labels other than 0/1
    folds, n_test = engine.make_svm_folds(labels, 3)
    skf = model_selection.StratifiedKFold(n_splits=3, shuffle=False)
    y = np.asarray(labels)
    for f, (tr, te) in enumerate(skf.split(np.zeros((22, 1)), y)):
        fd = folds[f]
        pos = [i for i in tr if y[i] == 3]
        neg = [i for i in tr if y[i] == 7]
        assert fd.n_train == len(tr) and fd.n_pos == len(pos) and fd.n_test == len(te) == n_test[f]
        assert list(fd.train_idx[:fd.n_train]) == pos + neg
        assert list(fd.test_idx[:fd.n_test]) == list(te)
        assert [bool(b) for b in fd.test_pos[:fd.n_test]] == [y[i] == 3 for i in te]
    assert ctypes.sizeof(folds[0]) == 592                    # layout of struct SvmFold in the library
    # more than two classes: one problem per (fold, class pair), libsvm's pair order, all held-out samples in each
    y3 = np.asarray([5, 1, 9, 1, 9, 5, 9, 5, 1, 5, 9, 1, 1, 5])
    mc = engine.make_svm_folds(y3, 2)
    assert list(mc.classes) == [1, 5, 9] and mc.pairs == [(0, 1), (0, 2), (1, 2)] and mc.nproblems == 6
    skf = model_selection.StratifiedKFold(n_splits=2, shuffle=False)
    for f, (tr, te) in enumerate(skf.split(np.zeros((len(y3), 1)), y3)):
        for q, (a, b) in enumerate(mc.pairs):
            fd = mc.structs[f * 3 + q]
            pos = [i for i in tr if y3[i] == mc.classes[a]]
            neg = [i for i in tr if y3[i] == mc.classes[b]]
            assert list(fd.train_idx[:fd.n_train]) == pos + neg and fd.n_pos == len(pos)
            assert list(fd.test_idx[:fd.n_test]) == list(te)
        assert list(mc.test_labels[f]) == list(np.searchsorted(mc.classes, y3[te]))
    with pytest.raises(ValueError):
        engine.make_svm_folds([0] * 8, 2)                    # a single class
    clf = svm.SVC(kernel="precomputed", shrinking=False)
    assert engine.svm_cv_supported(clf, [0, 1] * 8, 4, 16)
    # scikit-learn's default shrinking=True: restated as well (k_svm_cv_shrink); allow_shrinking=False keeps it on the host
    assert engine.svm_cv_supported(svm.SVC(kernel="precomputed"), [0, 1] * 8, 4, 16)
    assert not engine.svm_cv_supported(svm.SVC(kernel="precomputed"), [0, 1] * 8, 4, 16, allow_shrinking=False)
    assert engine.svm_cv_supported(clf, [0, 1, 2] * 4, 2, 12)                    # one-vs-one on the GPU
    assert not engine.svm_cv_supported(svm.SVC(kernel="precomputed", shrinking=False, break_ties=True,
                                               decision_function_shape="ovr"), [0, 1, 2] * 4, 2, 12)
    assert not engine.svm_cv_supported(clf, [0] * 12, 2, 12)
    assert not engine.svm_cv_supported(svm.SVC(kernel="linear"), [0, 1] * 8, 4, 16)
    assert not engine.svm_cv_supported(clf, [0, 1] * 40, 4, 80)


def test_sym_row_partition_covers_and_balances():
    """Shards of the symmetric pipeline: contiguous, 256-aligned cuts, equal trapezoid work within a few %."""
    from brainiak_b200.fcma import engine
    for V in (50000, 30000, 100000, 1000, 257):
        for W in (1, 2, 3, 4, 8):
            parts = engine.sym_row_partition(V, W)
            assert len(parts) == W and parts[0][0] == 0
            assert sum(n for _, n in parts) == V
            for r in range(1, W):
                assert parts[r][0] == parts[r - 1][0] + parts[r - 1][1]
                assert parts[r][0] % 256 == 0 or parts[r][0] == V
            if V >= 30000:
                work = [n * (V - s) - n * n / 2.0 for s, n in parts]
                assert max(work) / (sum(work) / W) < 1.08
    assert engine.sym_supported(32, 8) and not engine.sym_supported(32, 3)
    assert engine.sym_supported(32, 8, nb=512, start=0, V=1000)
    assert not engine.sym_supported(32, 8, nb=300, start=0, V=1000)
    assert engine.sym_supported(32, 8, nb=488, start=512, V=1000)


def test_bench_reference_arm_prints_one_json_line():
    """bench.py --impl reference (the reference's own CPU path, oracle/_ref or the oracle port) runs without a GPU and
    prints exactly one JSON line with the contract's keys."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--voxels", "1500",
                          "--steps", "1", "--warmup", "1"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [ln for ln in out.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "corr/s" and d["value"] > 0 and d["higher_is_better"] is True
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0 and d["gpu_launches"] == 0


def test_symmetric_pipeline_host_queries():
    """Host-only entry points of the symmetric pipeline (no device needed): which variant is taken and how many block
    rows a scratch buffer holds."""
    from brainiak_b200 import _lib
    lib = _lib.load()
    P = _lib.PREC
    F16 = _lib.FLAG_F16_INTERMEDIATE
    # column pass: E <= 32, power-of-two eps <= 32
    assert lib.fcma_sym_uses_column_pass(P["fp16x3"], 32, 8, 0) == 1
    assert lib.fcma_sym_uses_column_pass(P["tf32x3"], 16, 4, _lib.FLAG_MASK_SELF) == 1
    assert lib.fcma_sym_uses_column_pass(P["fp16x3"], 64, 8, 0) == 0          # E > 32: transposed copy + row pass
    assert lib.fcma_sym_uses_column_pass(P["fp16x3"], 32, 8, F16) == 1        # fp16 block: column pass as well
    assert lib.fcma_sym_uses_column_pass(P["bf16"], 32, 8, 0) == 1            # single-product modes imply the fp16 block
    assert lib.fcma_sym_uses_column_pass(P["bf16"], 48, 16, 0) == 0
    assert lib.fcma_sym_uses_column_pass(P["fp16x3"], 32, 3, 0) == 0          # eps not a power of two
    per_row = lib.fcma_work_bytes_per_row(32, 50000)
    assert per_row == 32 * 50176 * 4
    # the column-pass variant keeps only the block: twice the rows of the variant with a transposed copy
    assert lib.fcma_sym_rows_per_pass(P["fp16x3"], 32, 8, 0, 50000, 0, 4096 * per_row) == 4096
    assert lib.fcma_sym_rows_per_pass(P["fp16x3"], 64, 8, 0, 50000, 0, 4096 * lib.fcma_work_bytes_per_row(64, 50000)) == 2048
    assert lib.fcma_sym_rows_per_pass(P["fp16x3"], 32, 8, 0, 50000, 0, 300 * per_row) == 256
    assert lib.fcma_sym_rows_per_pass(P["fp16x3"], 32, 8, 0, 50000, 0, 100 * per_row) == 0     # too small
    # a shard that starts further right needs less scratch per row
    assert lib.fcma_sym_rows_per_pass(P["fp16x3"], 32, 8, 0, 50000, 25088, 4096 * per_row) > 8000


def test_sym_row_partition_is_min_max_over_whole_tiles():
    """Shards of the symmetric pipeline: contiguous, whole 256-row tiles (ragged tail only at V), covering [0, V) exactly
    once, and balanced: the bottleneck shard is within one tile's worth of work of the ideal share."""
    from brainiak_b200.fcma import engine

    def cost(V, s, n, pf=0.01):
        return ((1 - s / V) ** 2 - (1 - (s + n) / V) ** 2) + pf * (1 - s / V)
    for V, W in ((50000, 1), (50000, 2), (50000, 4), (50000, 8), (100000, 8), (30000, 3), (1536, 3), (1100, 2)):
        parts = engine.sym_row_partition(V, W)
        assert len(parts) == W and parts[0][0] == 0
        pos = 0
        for s, n in parts:
            assert s == pos and n >= 0
            assert n % 256 == 0 or s + n == V
            assert s % 256 == 0 or n == 0
            pos += n
        assert pos == V
        costs = [cost(V, s, n) for s, n in parts]
        ideal = sum(costs) / W
        one_tile = cost(V, 0, min(256, V))
        assert max(costs) <= ideal + one_tile + 1e-12
    # more ranks than tiles: the surplus ranks get empty shards at the end
    parts = engine.sym_row_partition(600, 4)
    assert sum(n for _, n in parts) == 600 and parts[-1][1] == 0


def test_epoch_partition_covers_all_epochs():
    from brainiak_b200.fcma.exchange import epoch_partition
    for E, W in ((32, 8), (64, 8), (10, 4), (3, 8), (16, 1)):
        p = epoch_partition(E, W)
        assert len(p) == W and p[0][0] == 0 and sum(n for _, n in p) == E
        assert all(p[r][0] + p[r][1] == p[r + 1][0] for r in range(W - 1))
        assert max(n for _, n in p) - min(n for _, n in p) <= 1


def test_epoch_groups_and_interleaved_shares_tile_the_epochs():
    """The grouped exchange: rank r uploads epochs r, r + W, ...; contiguous epoch groups complete one after the other,
    and every group contains epochs of (almost) every rank, so all PCIe links work on every group."""
    from brainiak_b200.fcma.exchange import epoch_groups
    for E, G in ((32, 4), (64, 4), (10, 4), (3, 4), (16, 1)):
        groups = epoch_groups(E, G)
        assert groups[0][0] == 0 and sum(n for _, n in groups) == E
        assert all(groups[k][0] + groups[k][1] == groups[k + 1][0] for k in range(len(groups) - 1))
        assert max(n for _, n in groups) - min(n for _, n in groups) <= 1
    for E, W in ((32, 8), (32, 2), (10, 4)):
        shares = [list(range(r, E, W)) for r in range(W)]
        assert sorted(e for sh in shares for e in sh) == list(range(E))
        for (e0, n) in epoch_groups(E, 4):
            owners = {e % W for e in range(e0, e0 + n)}
            assert len(owners) == min(W, n)


def test_one_vs_one_vote_is_libsvm_first_maximum():
    """engine._ovo_vote (torch ops, device-agnostic): decision bits of the k(k-1)/2 pair problems -> correct held-out samples per
    (voxel, fold), against a plain loop that votes as libsvm's svm_predict_values does (ties: smallest class index)."""
    import torch
    rng = np.random.RandomState(0)
    y = np.asarray([4, 8, 6, 2] * 5 + [2, 4])
    folds = engine.make_svm_folds(y, 2)
    k, npairs = len(folds.classes), len(folds.pairs)
    assert (k, npairs, folds.nproblems) == (4, 6, 12)
    nv = 50
    bits = rng.randint(0, 2 ** 11, size=(nv, folds.nproblems)).astype(np.int64)
    got = engine._ovo_vote(torch.from_numpy(bits), folds).numpy()
    for v in range(nv):
        for f in range(2):
            ok = 0
            for t in range(int(folds.n_test[f])):
                votes = [0] * k
                for q, (a, b) in enumerate(folds.pairs):
                    votes[a if (bits[v, f * npairs + q] >> t) & 1 else b] += 1
                pred = max(range(k), key=lambda c: (votes[c], -c))
                ok += int(pred == folds.test_labels[f][t])
            assert got[v, f] == ok
