"""Row-sharded frames whose shadowed device light list comes from one rank by map id: 4 ranks (sharing the GPUs there
are), each with its own map pool of the same texels and its own table of them; source rank 0 and the last rank, no AA
and TAA High + FXAA with and without lighting stripes, once with the G-buffer fed from the same rank; the count changes
every frame, every rank rebinds at another capacity between the same two frames, and the bands move once.  Every
assembled frame is the unsharded host-light shadowed frame of the first `live` lights given table[id]; every rank's
light prep and shadow transforms are the source rank's, and its map pointers its own.  The worker is
tests/multi_gpu_light_shadow_ids_worker.py."""
import pytest

from tests import common

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_shadowed_device_lights_by_id_from_one_rank_are_bit_identical(cuda, oracle, exchange):
    from tests.multi_gpu_light_shadow_ids_worker import FRAMES, RUNS

    rc, out, err = common.run_ranks("multi_gpu_light_shadow_ids_worker.py", [320, 192], 4, {"GRB_SHARD_EXCHANGE": exchange}, 900)
    assert rc == 0, out[-3000:] + err[-3000:]
    assert out.count("sharded == host lights single GPU: True") == len(RUNS) * FRAMES, out[-3000:]
    assert out.count("on every rank == the source rank's: True") == len(RUNS) * FRAMES, out[-3000:]
    assert out.count("pointers to the same maps: True") == len(RUNS) * FRAMES, out[-3000:]
    assert ": False" not in out
    if exchange == "peer":
        assert "peer-memory exchange unavailable" not in out + err
