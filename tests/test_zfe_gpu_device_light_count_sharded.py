"""Row-sharded frames whose device light list has its length in device memory: every rank binds its own copy of the
list and of the count, with plain bands and with lighting stripes, unshadowed and shadowed, on both exchange paths,
against the unsharded host-light frames of the first `count` lights.  The worker is
tests/multi_gpu_light_count_worker.py."""
import pytest

from tests import common

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_counted_device_lights_sharded_frames_are_bit_identical(cuda, oracle, exchange):
    """4 ranks on 4 GPUs, else 2 sharing the GPUs there are; no AA and TAA High + FXAA, each with and without lighting
    stripes, and one shadowed run; the count and the camera change every frame (one count past the capacity); every
    assembled frame is the unsharded host-light frame of the first `count` lights."""
    import torch

    from tests.multi_gpu_light_count_worker import FRAMES, RUNS

    world = 4 if torch.cuda.device_count() >= 4 else 2
    rc, out, err = common.run_ranks("multi_gpu_light_count_worker.py", [320, 192, 600], world, {"GRB_SHARD_EXCHANGE": exchange}, 900)
    assert rc == 0, out[-3000:] + err[-3000:]
    assert out.count("counted device lights sharded == host lights single GPU: True") == len(RUNS) * FRAMES, out[-3000:]
    assert "host lights single GPU: False" not in out
