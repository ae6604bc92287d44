"""Row-sharded viewers whose band cuts move between frames without a re-bake (grbh_viewer_move_row_shards), and the
sharded row-cost measurement, against the unsharded viewer with both exchange paths of the C++ graph (peer-memory
stores, NCCL).  The worker is tests/multi_gpu_live_bands_worker.py."""
import pytest

from tests import common

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_moved_bands_keep_frames_bit_identical(cuda, exchange):
    """4 ranks (sharing GPUs where there are fewer); no AA, FXAA, SMAA Ultra, TAA High + FXAA, FSR 0.67 + RCAS, HDR10 +
    TAA, TAA High + FXAA presented from the last rank, and no AA on measured bands.  8 frames with a moving camera, the
    cuts moved after frames 2 and 5: every frame equals the unsharded one, including the two right after each move; the
    sharded row cost equals the unsharded one on every rank, and the bands cut from it agree on every rank."""
    from tests.multi_gpu_live_bands_worker import FRAMES, RUNS

    rc, out, err = common.run_ranks("multi_gpu_live_bands_worker.py", [640, 384, 200], 4, {"GRB_SHARD_EXCHANGE": exchange}, 1200)
    assert rc == 0, out[-3000:] + err[-3000:]
    assert out.count("live bands == single GPU: True") == len(RUNS) * FRAMES, out[-3000:]
    assert "live bands == single GPU: False" not in out
    measured_fixed = sum(1 for _, _, measure, layouts in RUNS if measure and layouts == "fixed")
    assert out.count("sharded row cost == single GPU on every rank: True") == 3 * measured_fixed, out[-3000:]
    measured_moves = sum(1 for *_, layouts in RUNS if layouts == "measured")
    assert out.count("measured bands identical on every rank: True") == 2 * measured_moves, out[-3000:]
    if exchange == "peer":
        assert "peer-memory exchange unavailable" not in out + err, "IPC works between the ranks: the peer path must be the one that ran"
