"""Row-sharded viewers lit in stripes (grbh_viewer_set_lighting_stripes) against the unsharded viewer, with both
exchange paths of the C++ graph (peer-memory stores, NCCL).  The worker is tests/multi_gpu_stripes_worker.py."""
import pytest

from tests import common

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_striped_frames_are_bit_identical(cuda, exchange):
    """4 ranks (sharing GPUs where there are fewer), stripes of 8 and 64 rows; no AA, FXAA on 16-row cuts, SMAA Ultra,
    TAA High + FXAA, HDR10 + TAA, tonemap-only, RGBA16F, and TAA High + FXAA presented from the last rank.  8 frames
    with a moving camera and the cuts moved after frame 3: every frame equals the unsharded one, and the striped row
    cost equals the unsharded one on every rank."""
    from tests.multi_gpu_stripes_worker import CONFIGS, FRAMES, STRIPES

    rc, out, err = common.run_ranks("multi_gpu_stripes_worker.py", [640, 384, 200], 4, {"GRB_SHARD_EXCHANGE": exchange}, 1500)
    assert rc == 0, out[-3000:] + err[-3000:]
    runs = len(CONFIGS) * len(STRIPES)
    assert out.count("striped == single GPU: True") == runs * FRAMES, out[-3000:]
    assert "striped == single GPU: False" not in out
    assert out.count("striped row cost == single GPU on every rank: True") == 2 * runs, out[-3000:]
    if exchange == "peer":
        assert "peer-memory exchange unavailable" not in out + err, "IPC works between the ranks: the peer path must be the one that ran"
