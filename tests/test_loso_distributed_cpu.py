"""gloo world-size 2 and 3 test of the host logic of VoxelSelector.run_held_out over several ranks: static row shards,
per-rank scoring of every held-out subject, one all-gather of the [subjects, rows] accuracy matrix, per-subject lists
on the master and {} elsewhere.  The device stage is replaced by a CPU scorer built from the oracle (the full run's
kernels, compacted per subject), so the plumbing runs without a device."""
import os
import socket

import pytest
import torch.distributed as dist
import torch.multiprocessing as mp
from sklearn import svm

from brainiak_b200.fcma import synthetic
from brainiak_b200.fcma.voxelselector import VoxelSelector, shrink_kernels_

CLF = svm.SVC(kernel="precomputed", shrinking=False, C=1)
V, T, E, EPS = 23, 16, 16, 4


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _cpu_score_cases(self, start, n, clf, cases):
    from oracle import fcma_oracle as orc
    _, _, K = orc.voxel_block(self.raw_data, self.raw_data2, start, n, self.epochs_per_subj, shrink=False)
    out = []
    for c in cases:
        Kc = c.take(K, (1, 2))
        shrink_kernels_(Kc)
        out.append(self._do_cross_validation(clf, Kc, (start, n), c.labels, c.num_folds))
    return out


def _inputs():
    return synthetic.make_epochs(V, T, E, informative=4, signal=1.5)


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        raw, labels = _inputs()
        VoxelSelector._score_cases = _cpu_score_cases
        vs = VoxelSelector(labels, EPS, 2, raw, process_num=0, master_rank=world - 1)
        out[rank] = vs.run_held_out(CLF, subjects=[3, 0, 2])
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("world", [2, 3])
def test_run_held_out_world_size_n_gloo(monkeypatch, world):
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    for r in range(world - 1):
        assert out[r] == {}
    res = out[world - 1]
    assert list(res) == [3, 0, 2]
    raw, labels = _inputs()
    monkeypatch.setattr(VoxelSelector, "_score_cases", _cpu_score_cases)
    serial = VoxelSelector(labels, EPS, 2, raw, process_num=0).run_held_out(CLF, subjects=[3, 0, 2])
    for s in (3, 0, 2):
        assert sorted(v for v, _ in res[s]) == list(range(V))
        assert [(v, float(a)) for v, a in res[s]] == [(v, float(a)) for v, a in serial[s]]
