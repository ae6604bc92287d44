"""Row-sharded frames whose lights come from device memory: every rank binds its own device copy of the same lights,
with plain bands and with lighting stripes, against the unsharded host-light frames."""
import pytest

from tests import common

pytestmark = pytest.mark.gpu


def test_device_lights_sharded_frames_are_bit_identical(cuda):
    """4 ranks on 4 GPUs, else sharing the GPUs there are; no AA and TAA High + FXAA; 4 frames with the lights and the
    camera moving; every assembled frame is the unsharded host-light frame."""
    import torch

    from tests.multi_gpu_lights_worker import CONFIGS, FRAMES, STRIPES

    world = 4 if torch.cuda.device_count() >= 4 else 2
    rc, out, err = common.run_ranks("multi_gpu_lights_worker.py", [320, 192, 600], world, {}, 900)
    assert rc == 0, out[-3000:] + err[-3000:]
    assert out.count("device lights sharded == host lights single GPU: True") == len(CONFIGS) * len(STRIPES) * FRAMES, out[-3000:]
    assert "host lights single GPU: False" not in out
