"""The correlation GEMM stores the tiled block (fp32 or fp16) through shared memory with TMA bulk stores and the strided
block from registers.  Both routes store the same epilogue values, so the tiled block must equal the strided one bit
for bit, and it must cover exactly the elements the kernel writes: every row tile up to the 32-row chunk that holds the
last row, all 256 columns of every column tile, nothing in the rows after that chunk.

E = 64 puts 576 tiles on the persistent grid, so every CTA stores several tiles through the same staging slots."""
import numpy as np
import pytest
import torch

from brainiak_b200 import _lib
from brainiak_b200.fcma import engine, synthetic

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert _lib.device_count() > 0, "no sm_90 device"
    return torch.device("cuda:0")


def _detile(flat, row_tiles, col_tiles, E):
    """[row_tiles][col_tiles][E][256][256] -> [row_tiles*256, E, col_tiles*256], same dtype, on the host."""
    a = flat[:row_tiles * col_tiles * E * 65536].view(row_tiles, col_tiles, E, 256, 256)
    return a.permute(0, 3, 2, 1, 4).reshape(row_tiles * 256, E, col_tiles * 256).cpu()


@pytest.mark.parametrize("E", (6, 64))
@pytest.mark.parametrize("nb", (600, 545))
def test_tiled_block_equals_strided_block(dev, E, nb):
    V, T, eps, start = 700, 40, 4, 77
    raw, _ = synthetic.make_epochs(V, T, E, seed=4242)
    ep, T_e = engine.stack_epochs(raw, dev)
    op = engine.pack_epochs(ep, T_e, "fp32")
    work = engine.Workspace(E, V, 768, dev)
    rt, ct = -(-nb // 256), -(-V // 256)
    written = -(-nb // 32) * 32              # rows of the last row tile up to its last 32-row chunk

    work.buf.fill_(255)                      # NaN in fp32 and in fp16: unwritten elements show
    engine.voxel_kernels(op, op, start, nb, eps, flags=_lib.FLAG_STRIDED_BLOCK, work=work)
    torch.cuda.synchronize()
    ld = -(-V // 32) * 32
    strided = work.buf.view(torch.float32)[:nb * E * ld].view(nb, E, ld)[..., :V].cpu()
    assert not torch.isnan(strided).any()

    for half in (False, True):
        work.buf.fill_(255)
        engine.voxel_kernels(op, op, start, nb, eps, flags=_lib.FLAG_F16_INTERMEDIATE if half else 0, work=work)
        torch.cuda.synchronize()
        blk = _detile(work.buf.view(torch.float16 if half else torch.float32), rt, ct, E)
        want = strided.half() if half else strided
        got = blk[:nb, :, :V]
        assert torch.equal(got.view(torch.int16 if half else torch.int32), want.view(torch.int16 if half else torch.int32)), \
            "half=%s: tiled block != strided block at %s" % (half, np.argwhere((got != want).numpy())[:5].tolist())
        assert not torch.isnan(blk[:written]).any(), "half=%s: an element of a written 32-row chunk was not stored" % half
        assert torch.isnan(blk[written:]).all(), "half=%s: a row after the last 32-row chunk was stored" % half
