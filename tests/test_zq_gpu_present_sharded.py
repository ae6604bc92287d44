"""Presenting row-sharded frames from one rank on the GPU: the kernel that pushes a rank's band of the final image into
the presenting rank's frame slot (grb_present_rows_to_peer), and whole sharded frames read on the presenting rank
against the unsharded frame with both exchange paths of the C++ graph (peer-memory stores, NCCL all-gather)."""
import numpy as np
import pytest

from tests import common

pytestmark = pytest.mark.gpu
SENTINEL = 0x3C3C3C3C


@pytest.mark.parametrize("width,image_width", [(96, 96), (93, 93), (97, 100)])
def test_present_kernel_routes_own_rows(cuda, width, image_width):
    """Two allocations stand in for two ranks' frame slots and flag arrays; rank 1 presents.  Each call copies exactly
    its own rows into the presenting rank's slot and leaves every other byte (the other rows, the other rank's slot,
    the padding past the image width) at the sentinel; every flag array gets the epoch at the caller's index, and the
    scratch counter is reset.  Widths: a multiple of 4 texels (16-byte path), not a multiple of 4 (4-byte path), and
    not a multiple of 4 in a pitch that is (16-byte path with a scalar tail)."""
    import torch

    from granite_b200 import capi, harness

    h = 64
    rng = np.random.default_rng(width)
    srcs = [torch.from_numpy(rng.integers(0, 2**32, (h, image_width), dtype=np.uint32).view(np.int32)).cuda() for _ in range(2)]
    slots = [torch.full((h, image_width), SENTINEL, dtype=torch.int32, device="cuda") for _ in range(2)]
    flags = [torch.zeros(16, dtype=torch.int32, device="cuda") for _ in range(2)]
    counters = [torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(2)]
    bands = [(0, 27), (27, 64)]
    presenting = 1
    want = np.full((h, image_width), SENTINEL, np.int32)
    fmts = [capi.FORMAT_R8G8B8A8_SRGB, capi.FORMAT_A2B10G10R10_UNORM]

    for r in range(2):
        harness.present_rows_to_peer(srcs[r], slots[presenting], flags, r, 5, counters[r], bands[r], fmt=fmts[r], width=width)
        torch.cuda.synchronize()
        y0, y1 = bands[r]
        want[y0:y1, :width] = srcs[r].cpu().numpy()[y0:y1, :width]
        assert np.array_equal(slots[presenting].cpu().numpy(), want), f"after rank {r}: slot differs"
        assert (slots[1 - presenting].cpu().numpy() == SENTINEL).all(), "the other rank's slot was written"
        for f in flags:
            assert list(f.cpu().numpy()[:r + 1]) == [5] * (r + 1) and not f.cpu().numpy()[r + 1:].any()
    assert not counters[0].item() and not counters[1].item()  # the last CTA resets the scratch counter


@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_presented_sharded_frame_is_bit_identical(cuda, exchange):
    """4 ranks (sharing GPUs where there are fewer); no AA, FXAA, SMAA Ultra, TAA High + FXAA, FSR 0.67 + RCAS, HDR10 +
    TAA and tonemap-only without bloom; equal and narrow bands; presenting rank 0 and the last rank; one run that sleeps
    on the host before every read.  6 frames each with a moving camera; every frame the presenting rank returns is the
    unsharded frame, and the other ranks return their bands."""
    from tests.multi_gpu_present_worker import CONFIGS, FRAMES, RUNS

    rc, out, err = common.run_ranks("multi_gpu_present_worker.py", [640, 384, 200], 4, {"GRB_SHARD_EXCHANGE": exchange}, 1200)
    assert rc == 0, out[-3000:] + err[-3000:]
    assert out.count("tonemap-only sharded == single GPU: True") == 2 * FRAMES, out[-3000:]
    assert out.count("presented == single GPU: True") == len(CONFIGS) * len(RUNS) * FRAMES, out[-3000:]
    assert "presented == single GPU: False" not in out
    if exchange == "peer":
        assert "peer-memory exchange unavailable" not in out + err, "IPC works between the ranks: the peer path must be the one that ran"
