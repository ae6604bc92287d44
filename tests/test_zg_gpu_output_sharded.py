"""Row-sharded frames rendered into caller-owned output images on the GPU: per-rank rings whose rows outside the band
stay untouched, and the presenting rank's ring filled by the present pass, with both exchange paths of the C++ graph
(peer-memory stores, NCCL broadcasts), against the unsharded host-fed frames."""
import pytest

from tests import common

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_ring_output_sharded_frames_are_bit_identical(cuda, exchange):
    """4 ranks (sharing GPUs where there are fewer); the configurations of sharded.config_args; per-rank rings with the
    rows outside each band poisoned before every acquire, presenting to rank 0 and to the last rank with a ring on that
    rank only; a move_row_shards after the third frame.  6 frames each; every assembled frame is the unsharded
    host-fed frame."""
    from tests.multi_gpu_output_worker import CONFIGS, FRAMES, RUNS

    rc, out, err = common.run_ranks("multi_gpu_output_worker.py", [320, 192, 120], 4, {"GRB_SHARD_EXCHANGE": exchange}, 1200)
    assert rc == 0, out[-3000:] + err[-3000:]
    assert out.count("ring output sharded == host-fed single GPU: True") == len(CONFIGS) * len(RUNS) * FRAMES, out[-3000:]
    assert "host-fed single GPU: False" not in out and "still poisoned" not in out, out[-3000:]
    if exchange == "peer":
        assert "peer-memory exchange unavailable" not in out + err, "IPC works between the ranks: the peer path must be the one that ran"
