"""SMAA on row-sharded frames on the GPU: the edge kernel that stores its rows into the peers' edge images
(grb_smaa_edge_detection_to_peers), and whole sharded frames against the unsharded frame with both exchange paths
of the C++ graph (peer-memory stores, NCCL all-gather)."""
import numpy as np
import pytest

from tests import common
from tests.test_oracle_ref_smaa import smaa_test_image

pytestmark = pytest.mark.gpu
SENTINEL = 0xA5


def test_edge_kernel_routes_rows_to_peer_windows(cuda):
    """Two allocations stand in for two ranks' edge images and flag arrays.  Each call stores the texels of
    grb_smaa_edge_detection on the rows it produces into its own image and into the other image where that image's
    window holds the row; every other byte keeps the sentinel; both flag arrays get the epoch at the producer's index."""
    import torch

    from granite_b200 import harness

    w, h = 96, 64
    img = smaa_test_image(w, h, 5)
    color = harness.to_dev(img)
    ref = torch.zeros((h, w, 2), dtype=torch.uint8, device="cuda")
    harness.smaa_edge_detection(color, 3, ref)
    ref = ref.cpu().numpy()
    assert ref.any()
    images = [torch.full((h, w, 2), SENTINEL, dtype=torch.uint8, device="cuda") for _ in range(2)]
    flags = [torch.zeros(16, dtype=torch.int32, device="cuda") for _ in range(2)]
    counters = [torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(2)]
    windows = [(0, 40), (24, 64)]
    bands = [(0, 32), (32, 64)]

    def expect(produced):
        for q, (w0, w1) in enumerate(windows):
            want = np.full((h, w, 2), SENTINEL, np.uint8)
            for p in produced:
                y0, y1 = bands[p]
                if p != q:
                    y0, y1 = max(y0, w0), min(y1, w1)
                want[y0:y1] = ref[y0:y1]
            assert np.array_equal(images[q].cpu().numpy(), want), f"image {q} after producers {produced}"

    harness.smaa_edge_detection_to_peers(color, 3, images, flags, windows, 0, 7, counters[0], rows=bands[0])
    torch.cuda.synchronize()
    expect([0])
    for f in flags:
        assert f.cpu().numpy()[0] == 7 and not f.cpu().numpy()[1:].any()
    harness.smaa_edge_detection_to_peers(color, 3, images, flags, windows, 1, 7, counters[1], rows=bands[1])
    torch.cuda.synchronize()
    expect([0, 1])
    for f in flags:
        assert list(f.cpu().numpy()[:2]) == [7, 7] and not f.cpu().numpy()[2:].any()
    assert not counters[0].item() and not counters[1].item()  # the last CTA resets the scratch counter


@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_sharded_smaa_frame_is_bit_identical(cuda, exchange):
    """4 ranks (sharing GPUs where there are fewer), equal and narrow bands, presets Low and Ultra, 4 frames each."""
    world = 4
    rc, out, err = common.run_ranks("multi_gpu_smaa_worker.py", [1280, 768, 300], world, {"GRB_SHARD_EXCHANGE": exchange}, 900)
    assert rc == 0, out[-3000:] + err[-3000:]
    assert out.count(f"sharded over {world} ranks == single GPU: True") == 2 * 2 * 4, out[-3000:]
    assert out.count("weights near every border: True") == 4, out[-3000:]
    if exchange == "peer":
        assert "peer-memory exchange unavailable" not in out + err, "IPC works between the ranks: the peer path must be the one that ran"
