"""CPU side of the wide SVM cross-validation (fcma_svm_cv_solve_wide, up to 256 epochs): the wide fold builder against
scikit-learn's splitter, the layout of its ctypes struct, the predicate's epoch limit and the one-vs-one vote over
several decision words."""
import ctypes

import numpy as np
import pytest
from sklearn import model_selection, svm

from brainiak_b200.fcma import engine


def _check_folds(folds, labels, num_folds, limit):
    y = np.asarray(labels)
    classes = np.unique(y)
    code = np.searchsorted(classes, y)
    pairs = [(a, b) for a in range(len(classes)) for b in range(a + 1, len(classes))]
    assert list(folds.pairs) == pairs and folds.nproblems == num_folds * len(pairs)
    splits = model_selection.StratifiedKFold(n_splits=num_folds, shuffle=False).split(np.zeros((len(y), 1)), y)
    for f, (tr, te) in enumerate(splits):
        assert folds.n_test[f] == len(te) and np.array_equal(folds.test_labels[f], code[te])
        for q, (a, b) in enumerate(pairs):
            fd = folds.structs[f * len(pairs) + q]
            order = [i for i in tr if code[i] == a] + [i for i in tr if code[i] == b]
            assert (fd.n_train, fd.n_pos, fd.n_test) == (len(order), int((code[tr] == a).sum()), len(te))
            assert list(fd.train_idx[:fd.n_train]) == order and not any(fd.train_idx[fd.n_train:limit])
            assert list(fd.test_idx[:fd.n_test]) == list(te)
            assert list(fd.test_pos[:fd.n_test]) == [int(code[i] == a) for i in te]


@pytest.mark.parametrize("E,nclass,num_folds", [(65, 2, 5), (140, 2, 7), (140, 3, 7), (256, 2, 16), (256, 4, 16),
                                                (200, 3, 2), (256, 2, 2)])
def test_wide_folds_follow_stratified_kfold(E, nclass, num_folds):
    """The wide builder's problems are StratifiedKFold(shuffle=False)'s splits in libsvm's one-vs-one order, with up to
    256 training and held-out samples (2 folds of 256 epochs: 128 of each)."""
    rng = np.random.RandomState(E + nclass)
    labels = rng.permutation(np.arange(E) % nclass) * 3 + 1          # label values other than 0 .. k-1
    folds = engine.make_svm_folds_wide(labels, num_folds)
    assert folds.wide and ctypes.sizeof(folds.structs) == folds.nproblems * 2320
    _check_folds(folds, labels, num_folds, 256)


@pytest.mark.parametrize("E,nclass", [(24, 2), (64, 3), (60, 4)])
def test_wide_folds_equal_narrow_folds(E, nclass):
    """Up to 64 epochs the wide builder describes the same problems as make_svm_folds, which keeps its 64 limit."""
    labels = np.arange(E) % nclass
    narrow, wide = engine.make_svm_folds(labels, 4), engine.make_svm_folds_wide(labels, 4)
    assert not narrow.wide and wide.wide and narrow.nproblems == wide.nproblems
    for a, b in zip(narrow.structs, wide.structs):
        assert (a.n_train, a.n_pos, a.n_test) == (b.n_train, b.n_pos, b.n_test)
        assert list(a.train_idx) == list(b.train_idx[:64]) and list(a.test_idx) == list(b.test_idx[:64])
        assert list(a.test_pos) == list(b.test_pos[:64])
    with pytest.raises(ValueError):
        engine.make_svm_folds(np.arange(100) % 2, 4)     # 75 training samples
    with pytest.raises(ValueError):
        engine.make_svm_folds_wide(np.arange(600) % 2, 2)     # 300 held-out samples
    assert engine.svm_folds_for(labels, 4, E).wide is False
    assert engine.svm_folds_for(np.arange(65) % 2, 4, 65).wide is True


def test_wide_fold_struct_layout():
    """_SvmFoldWide is the library's SvmFoldWide (static_assert in fcma_b200.cu, 2320 bytes in fcma_b200.h);
    _SvmFold keeps its 592 bytes."""
    W = engine._SvmFoldWide
    assert ctypes.sizeof(W) == 2320 and ctypes.sizeof(engine._SvmFold) == 592
    assert (W.n_train.offset, W.n_pos.offset, W.n_test.offset, W.pad.offset) == (0, 4, 8, 12)
    assert (W.train_idx.offset, W.test_idx.offset, W.test_pos.offset) == (16, 16 + 1024, 16 + 2048)


def test_predicate_epoch_limit():
    """The default keeps the 64-epoch answer; VoxelSelector's max_epochs=256 admits 65 .. 256 epochs."""
    clf = svm.SVC(kernel="precomputed", shrinking=False)
    for E, narrow, wide in ((64, True, True), (65, False, True), (256, False, True), (257, False, False)):
        labels = np.arange(E) % 2
        assert engine.svm_cv_supported(clf, labels, 4, E) is narrow, E
        assert engine.svm_cv_supported(clf, labels, 4, E, max_epochs=256) is wide, E
        assert engine.svm_cv_supported(svm.SVC(kernel="precomputed"), np.arange(E) % 3, 4, E, max_epochs=256) is wide
    assert not engine.svm_cv_supported(clf, np.arange(140) % 2, 65, 140, max_epochs=256)      # more than 64 folds


def test_vote_reads_every_word():
    """_ovo_vote on [nv, nproblems, 4] words gives what it gives on the single-word form for held-out sets up to 64,
    and reads sample t from bit t % 64 of word t // 64 beyond."""
    import torch
    rng = np.random.RandomState(3)
    labels = rng.permutation(np.arange(48) % 3)
    folds = engine.make_svm_folds(labels, 4)
    bits1 = torch.from_numpy(rng.randint(-2 ** 62, 2 ** 62, size=(5, folds.nproblems), dtype=np.int64))
    bits4 = torch.zeros((5, folds.nproblems, 4), dtype=torch.int64)
    bits4[:, :, 0] = bits1
    assert torch.equal(engine._ovo_vote(bits1, folds), engine._ovo_vote(bits4, folds))
    labels = rng.permutation(np.arange(256) % 3)
    folds = engine.make_svm_folds_wide(labels, 2)
    side = rng.rand(5, folds.nproblems, 128) < 0.5
    words = np.zeros((5, folds.nproblems, 4), np.uint64)
    for t in range(128):
        words[:, :, t // 64] |= side[:, :, t].astype(np.uint64) << np.uint64(t % 64)
    got = engine._ovo_vote(torch.from_numpy(words.view(np.int64)), folds).numpy()
    for f in range(2):
        votes = np.zeros((5, 128, 3), np.int64)
        for q, (a, b) in enumerate(folds.pairs):
            votes[:, :, a] += side[:, f * 3 + q]
            votes[:, :, b] += ~side[:, f * 3 + q]
        pred = votes.argmax(axis=2)
        assert np.array_equal(got[:, f], (pred == folds.test_labels[f][None, :]).sum(axis=1))
