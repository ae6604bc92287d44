"""TAA on row-sharded frames on the GPU: the resolve kernel that stores its own history rows into every rank's history
image (grb_taa_resolve_to_peers), and whole sharded frames against the unsharded frame with both exchange paths of the
C++ graph (peer-memory stores, NCCL all-gather)."""
import numpy as np
import pytest

from tests import common

pytestmark = pytest.mark.gpu
SENTINEL16 = 0x5A5A
SENTINEL32 = 0x3C3C3C3C


def _inputs(rng, w, h):
    hdr = common.random_hdr(rng, w, h, scale=2.0)
    depth = rng.uniform(0.0005, 0.03, size=(h, w)).astype(np.float32)
    mv = np.zeros((h, w, 2), np.float16)
    m = rng.random((h, w)) < 0.2
    mv[m] = np.stack([rng.uniform(-2.0, 2.0, int(m.sum())) / w, rng.uniform(-0.5, 0.5, int(m.sum()))], -1).astype(np.float16)
    hist = np.concatenate([rng.uniform(0, 1, (h, w, 1)), rng.uniform(-0.5, 0.5, (h, w, 2)), np.ones((h, w, 1))], -1).astype(np.float16)
    reproj = np.array([[0.5, 0, 0, 0], [0, 0.5, 0, 0], [0.3, -0.2, 1, 0], [0.5 + 0.4 / w, 0.5 - 0.3 / h, 0, 1]], np.float32)
    return hdr, depth, mv.view(np.uint16), hist.view(np.uint16), reproj


@pytest.mark.parametrize("quality", [0, 2])
@pytest.mark.parametrize("with_history", [False, True])
def test_taa_kernel_routes_own_history_rows(cuda, quality, with_history):
    """Two allocations stand in for two ranks' history images and flag arrays.  Each call writes the colour of
    grb_taa_resolve on its TAA rows, stores the history of its own rows into both images, and leaves every other byte
    at the sentinel; both flag arrays get the epoch at the caller's index, and the scratch counter is reset."""
    import torch

    from granite_b200 import harness

    w, h = 96, 64
    hdr, depth, mv, hist, reproj = _inputs(np.random.default_rng(quality + 3 * with_history), w, h)
    args = [harness.to_dev(hdr), None, None, None, None]
    if with_history:
        args = [harness.to_dev(hdr), harness.to_dev(depth), harness.to_dev(mv.reshape(h, w, 2)).view(torch.int32).reshape(h, w),
                harness.to_dev(hist), reproj]
    ref_c = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    ref_h = harness.new_rgba16f(w, h)
    harness.taa_resolve(*args, quality, ref_c, ref_h)
    ref_c, ref_h = ref_c.cpu().numpy().view(np.uint32), ref_h.cpu().numpy().view(np.uint16)

    images = [torch.full((h, w, 4), SENTINEL16, dtype=torch.int16, device="cuda") for _ in range(2)]
    colours = [torch.full((h, w), SENTINEL32, dtype=torch.int32, device="cuda") for _ in range(2)]
    flags = [torch.zeros(16, dtype=torch.int32, device="cuda") for _ in range(2)]
    counters = [torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(2)]
    bands = [(0, 32), (32, 64)]
    taa_rows = [(0, 40), (23, 64)]

    for r in range(2):
        harness.taa_resolve_to_peers(*args, quality, colours[r], images, flags, r, 7, counters[r], rows=taa_rows[r], own=bands[r])
        torch.cuda.synchronize()
        got = colours[r].cpu().numpy().view(np.uint32)
        y0, y1 = taa_rows[r]
        assert np.array_equal(got[y0:y1], ref_c[y0:y1]), f"rank {r}: colour differs from grb_taa_resolve"
        assert (got[:y0] == SENTINEL32).all() and (got[y1:] == SENTINEL32).all(), f"rank {r}: colour written outside its rows"
        want = np.full((h, w, 4), SENTINEL16, np.uint16)
        for p in range(r + 1):
            want[bands[p][0]:bands[p][1]] = ref_h[bands[p][0]:bands[p][1]]
        for q in range(2):
            assert np.array_equal(images[q].cpu().numpy().view(np.uint16), want), f"image {q} after ranks 0..{r}"
        for f in flags:
            assert list(f.cpu().numpy()[:r + 1]) == [7] * (r + 1) and not f.cpu().numpy()[r + 1:].any()
    assert not counters[0].item() and not counters[1].item()  # the last CTA resets the scratch counter


@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_sharded_taa_frame_is_bit_identical(cuda, exchange):
    """4 ranks (sharing GPUs where there are fewer); TAA Low, High, High + FXAA, High with HDR10 output; equal and
    narrow bands; 6 frames each with a moving camera and large vertical motion vectors."""
    world = 4
    rc, out, err = common.run_ranks("multi_gpu_taa_worker.py", [1280, 768, 300], world, {"GRB_SHARD_EXCHANGE": exchange}, 900)
    assert rc == 0, out[-3000:] + err[-3000:]
    assert out.count(f"sharded over {world} ranks == single GPU: True") == 4 * 2 * 6, out[-3000:]
    assert out.count("motion vectors reach other bands from every rank: True") == 2, out[-3000:]
    if exchange == "peer":
        assert "peer-memory exchange unavailable" not in out + err, "IPC works between the ranks: the peer path must be the one that ran"
