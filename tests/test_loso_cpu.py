"""VoxelSelector.run_held_out without a device: argument validation, the held-out runs' epochs, labels and folds against
what the reference's FCMA example builds (fcma_voxel_selection_cv.py:69-79), the premise that holding a subject out
leaves the other subjects' z-scores and kernels unchanged (on the C oracle), and the loso_l* fixtures' input probes."""
import os
import sys

import numpy as np
import pytest
from sklearn import model_selection, svm

from brainiak_b200.fcma import engine, synthetic
from brainiak_b200.fcma.voxelselector import VoxelSelector, held_out_keep
from oracle import fcma_oracle as orc

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_golden_loso import loso_inputs, subsample  # noqa: E402
from test_generic_pipeline_cpu import kernel_pair_bound, ref_rho  # noqa: E402

PRE = svm.SVC(kernel='precomputed', shrinking=False, C=1)


def _vs(E, eps, V=6, **kw):
    raw, labels = synthetic.make_epochs(V, 8, E, seed=3)
    return VoxelSelector(labels, eps, 2, raw, **kw)


def _no_device(monkeypatch):
    """Any step that would touch the device fails the test."""
    def boom(*a, **k):
        raise AssertionError("the device was touched")
    monkeypatch.setattr(VoxelSelector, "_operands", boom)
    monkeypatch.setattr(VoxelSelector, "_score_cases", boom)


@pytest.mark.parametrize("E, eps, kw, msg", [
    (30, 4, {}, "whole subjects"),                       # 30 epochs are not whole subjects of 4
    (8, 4, {}, "at least 3 subjects"),
    (12, 4, {"subjects": [0, 3]}, "distinct indices"),
    (12, 4, {"subjects": [-1]}, "distinct indices"),
    (12, 4, {"subjects": [1, 1]}, "distinct indices"),
])
def test_run_held_out_refuses_before_the_device(monkeypatch, E, eps, kw, msg):
    _no_device(monkeypatch)
    vs = _vs(E, eps)
    with pytest.raises(ValueError, match=msg):
        vs.run_held_out(PRE, **kw)


@pytest.mark.parametrize("E, eps", [(160, 20), (32, 4), (48, 8), (12, 4), (15, 5)])
def test_keep_labels_and_folds_match_the_example(E, eps):
    """The keep list, labels_s and the fold problems are those the reference example builds for each held-out subject,
    and the default fold count is S - 1."""
    labels = [(e * 7 + 3) % 2 for e in range(E)]
    raw, _ = synthetic.make_epochs(5, 6, E, seed=1)
    vs = VoxelSelector(labels, eps, 2, raw)
    S = E // eps
    subjects, cases = vs.held_out_cases()
    assert subjects == list(range(S))
    for s, c in zip(subjects, cases):
        idx = subsample(list(range(E)), eps, s)
        assert list(c.keep) == idx == list(held_out_keep(E, eps, s))
        assert c.labels == subsample(labels, eps, s) and c.E == E - eps and c.num_folds == S - 1
        # the fold problems the GPU solves are StratifiedKFold(S - 1) on labels_s
        folds = engine.svm_folds_for(c.labels, c.num_folds, c.E)
        skf = model_selection.StratifiedKFold(n_splits=S - 1, shuffle=False)
        for f, (_, te) in enumerate(skf.split(np.zeros((len(c.labels), 1)), c.labels)):
            fd = folds.structs[f * len(folds.pairs)]
            assert list(fd.test_idx[:fd.n_test]) == list(te)
    subjects, cases = vs.held_out_cases(subjects=[S - 1, 0], num_folds=2)
    assert subjects == [S - 1, 0] and [c.num_folds for c in cases] == [2, 2]
    assert list(cases[1].keep) == list(range(eps, E))


@pytest.mark.parametrize("E, eps, s", [(32, 4, 0), (32, 4, 5), (60, 12, 4), (48, 16, 1)])
def test_premise_on_the_oracle(E, eps, s):
    """The within-subject z of the kept epochs is the same, bit for bit, computed with and without subject s; the full
    run's kernel sub-block agrees with the held-out run's kernels within the two fp32 chains' bound."""
    nb = 6
    # two masks: no self-correlation column (r = 1, which the bound's rule leaves out)
    raw, _ = synthetic.make_epochs(nb, 24, E, seed=11 + s)
    raw2, _ = synthetic.make_epochs(40, 24, E, seed=51 + s)
    keep = held_out_keep(E, eps, s)
    raw_s, raw2_s = [raw[i] for i in keep], [raw2[i] for i in keep]
    _, z_full, K_full = orc.voxel_block(raw, raw2, 0, nb, eps, shrink=False)
    _, z_sub, K_sub = orc.voxel_block(raw_s, raw2_s, 0, nb, eps, shrink=False)
    assert np.array_equal(z_full[:, keep], z_sub)
    for v in range(nb):
        _, bound = kernel_pair_bound(raw_s, raw2_s, v, eps, ref_rho)
        err = np.abs(K_full[v][np.ix_(keep, keep)].astype(np.float64) - K_sub[v].astype(np.float64))
        assert np.all(err <= bound[0].numpy()), (v, float(err.max()))


@pytest.mark.parametrize("name", ["l1", "l2", "l3"])
def test_fixture_probes_match(golden, name):
    g = golden("loso_" + name)
    raw, raw2, labels, eps, _ = loso_inputs(name)
    assert int(g["eps"]) == eps and list(g["labels"]) == list(labels)
    assert np.array_equal(np.stack([raw[e][:4, ::997][:, :16] for e in (0, len(raw) - 1)]), g["probe"])
    if raw2 is not None:
        assert np.array_equal(np.stack([raw2[e][:4, ::997][:, :16] for e in (0, len(raw2) - 1)]), g["probe2"])
    S = len(raw) // eps
    V = raw[0].shape[1]
    assert g["vids"].shape == (S, V) and g["accs"].shape == (S, V)
    for s in range(S):
        assert sorted(g["vids"][s]) == list(range(V))
