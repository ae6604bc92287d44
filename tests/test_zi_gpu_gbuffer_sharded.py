"""Row-sharded frames from G-buffers in device memory on the GPU: fed per rank (each rank's input rows only, every other
row poisoned) and from one rank that rasterised the whole frame (rank 0 or the last rank), with both exchange paths of
the C++ graph (peer-memory stores, NCCL broadcasts), against the unsharded host-fed frames."""
import pytest

from tests import common

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_device_fed_sharded_frames_are_bit_identical(cuda, exchange):
    """4 ranks (sharing GPUs where there are fewer); the configurations of sharded.config_args; per-rank and source-rank
    feeding; lighting stripes of 8 and 64 rows; a move_row_shards after the third frame; presenting from the last rank.
    6 frames each, a G-buffer that changes every frame and a moving camera; every assembled frame is the unsharded
    host-fed frame."""
    from tests.multi_gpu_gbuffer_worker import CONFIGS, FRAMES, RUNS

    rc, out, err = common.run_ranks("multi_gpu_gbuffer_worker.py", [320, 192, 120], 4, {"GRB_SHARD_EXCHANGE": exchange}, 1500)
    assert rc == 0, out[-3000:] + err[-3000:]
    assert out.count("device-fed sharded == host-fed single GPU: True") == len(CONFIGS) * len(RUNS) * FRAMES, out[-3000:]
    assert "host-fed single GPU: False" not in out
    if exchange == "peer":
        assert "peer-memory exchange unavailable" not in out + err, "IPC works between the ranks: the peer path must be the one that ran"
