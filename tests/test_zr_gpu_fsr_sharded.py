"""FSR 1 upscaling on row-sharded frames on the GPU: whole sharded frames against the unsharded frame with both exchange
paths of the C++ graph (peer-memory stores, NCCL all-gathers), the render rows of every pass before FSR taken from
grbh_shard_plan_fsr."""
import pytest

from tests import common

pytestmark = pytest.mark.gpu
CONFIGS = 6


@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_sharded_fsr_frame_is_bit_identical(cuda, exchange):
    """4 ranks (sharing GPUs where there are fewer), 1280 x 768 display; scale 0.67 with RCAS and no AA, FXAA or TAA
    High + FXAA, 0.67 without RCAS and SMAA Ultra, 0.5 with RCAS and SMAA Low, 0.5 without RCAS and TAA Low; equal and
    narrow bands; 4 frames each."""
    world = 4
    rc, out, err = common.run_ranks("multi_gpu_fsr_worker.py", [1280, 768, 300], world, {"GRB_SHARD_EXCHANGE": exchange}, 900)
    assert rc == 0, out[-3000:] + err[-3000:]
    assert out.count(f"sharded over {world} ranks == single GPU: True") == CONFIGS * 2 * 4, out[-3000:]
    if exchange == "peer":
        assert "peer-memory exchange unavailable" not in out + err, "IPC works between the ranks: the peer path must be the one that ran"
