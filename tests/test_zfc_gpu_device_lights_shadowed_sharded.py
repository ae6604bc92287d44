"""Row-sharded frames with shadowed lights: host lights, and lights, shadow transforms and maps from device memory that
every rank binds its own copies of; with plain bands and with lighting stripes, on both exchange paths, against the
unsharded host-light shadowed frames.  The worker is tests/multi_gpu_shadowed_lights_worker.py."""
import pytest

from tests import common

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_shadowed_lights_sharded_frames_are_bit_identical(cuda, oracle, exchange):
    """4 ranks on 4 GPUs, else 2 sharing the GPUs there are; no AA and TAA High + FXAA; 4 frames with the lights, the
    maps and the camera changing; every assembled frame, of host and of device lights, is the unsharded host-light
    frame."""
    import torch

    from tests.multi_gpu_shadowed_lights_worker import CONFIGS, FRAMES, STRIPES

    world = 4 if torch.cuda.device_count() >= 4 else 2
    rc, out, err = common.run_ranks("multi_gpu_shadowed_lights_worker.py", [320, 192, 300], world, {"GRB_SHARD_EXCHANGE": exchange}, 900)
    assert rc == 0, out[-3000:] + err[-3000:]
    for kind in ("host", "device"):
        assert out.count(f"{kind} shadowed lights sharded == host lights single GPU: True") == len(CONFIGS) * len(STRIPES) * FRAMES, out[-3000:]
    assert "host lights single GPU: False" not in out
