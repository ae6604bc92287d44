"""Row-sharded frames on real GPUs against the single-GPU frame, with both exchange paths of the C++
graph: peer-memory stores from the downsample kernel (default) and NCCL broadcasts + all-reduce.

The frame is split over 4 ranks where the machine has 4 GPUs, else over 2.  On a single GPU the two ranks
share it (see tests/sharded.py): every sharded step still runs, on one device."""
import pytest

from tests import common

pytestmark = pytest.mark.gpu


def _gpu_count():
    import torch

    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.parametrize("exchange", ["peer", "nccl"])
@pytest.mark.parametrize("fxaa", [0, 1])
def test_sharded_frame_is_bit_identical(cuda, fxaa, exchange):
    world = 4 if _gpu_count() >= 4 else 2
    rc, out, err = common.run_ranks("multi_gpu_worker.py", [1280, 768, 300, fxaa], world, {"GRB_SHARD_EXCHANGE": exchange}, 600)
    assert rc == 0, out[-3000:] + err[-3000:]
    assert out.count(f"sharded over {world} ranks == single GPU: True") == 3, out[-3000:]
    if exchange == "peer":
        assert "peer-memory exchange unavailable" not in out + err, "IPC works between the ranks: the peer path must be the one that ran"
