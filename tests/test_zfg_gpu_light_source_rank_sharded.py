"""Row-sharded frames whose device light list and live count come from one rank (Viewer.set_light_source_rank): 4
ranks (sharing the GPUs there are), source rank 0 and the last rank, no AA and TAA High + FXAA with and without
lighting stripes, once with the G-buffer fed from the same rank; the count changes every frame (a drop from 6000 to 10,
a clamp past the capacity), every rank rebinds at another capacity between the same two frames, and the bands move
once.  Every assembled frame is the unsharded host-light frame of the first `live` lights, and every rank's light prep
is the source rank's.  The worker is tests/multi_gpu_light_source_worker.py."""
import pytest

from tests import common

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_device_lights_from_one_rank_sharded_frames_are_bit_identical(cuda, oracle, exchange):
    from tests.multi_gpu_light_source_worker import FRAMES, RUNS

    rc, out, err = common.run_ranks("multi_gpu_light_source_worker.py", [320, 192], 4, {"GRB_SHARD_EXCHANGE": exchange}, 900)
    assert rc == 0, out[-3000:] + err[-3000:]
    assert out.count("device lights from one rank sharded == host lights single GPU: True") == len(RUNS) * FRAMES, out[-3000:]
    assert out.count("light prep on every rank == the source rank's: True") == len(RUNS) * FRAMES, out[-3000:]
    assert ": False" not in out
    if exchange == "peer":
        assert "peer-memory exchange unavailable" not in out + err
