"""Frames rendered into caller-owned output images on the GPU (grbh_viewer_set_output_images /
grbh_viewer_acquire_output): a ring of padded tensors bound as the backbuffer, against the host readback of a viewer
without a ring, bit for bit, with the ordering through the `acquired` and `rendered` events checked by a consumer that
lags behind the viewer."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FRAMES = 6
RING = 3
POISON = 0x5A5A5A5A
SLEEP_CYCLES = 10_000_000  # a few ms at the H100's clocks: longer than a frame at these sizes
CONFIGS = {
    "no AA": (318, dict()),
    "FXAA": (318, dict(post_aa=1)),
    "TAA High + FXAA": (320, dict(post_aa=100)),
    "SMAA Ultra": (318, dict(post_aa=6)),
    "FSR 0.67 + RCAS": (318, dict(resolution_scale=0.67, resolution_scale_sharpen=True)),
    "FSR 0.67": (320, dict(resolution_scale=0.67, resolution_scale_sharpen=False)),
    "RGBA16F": (320, dict(render_target_fp16=True)),
    "HDR10 + TAA": (318, dict(post_aa=10, hdr10_output=True)),
    "tonemap-only": (318, dict(hdr_bloom=False)),
    "pipelined_io + TAA": (320, dict(post_aa=10, pipelined_io=True)),
}
H = 184


def _frame_inputs(rw, rh, fp16):
    """One seeded G-buffer per frame at the render size: host arrays in host_gbuffer order (mv included)."""
    from granite_b200 import synth
    from tests import common, sharded

    out = []
    for i in range(FRAMES):
        s = synth.make_scene(rw, rh, seed=300 + i)
        em = common.random_hdr_f16(np.random.default_rng(i), rw, rh, scale=0.02, hot=0.001) if fp16 else s.emissive
        mv = sharded.motion_vectors(rw, rh, i).view(np.uint32).reshape(rh, rw)
        out.append([np.ascontiguousarray(a) for a in (s.albedo, s.normal, s.pbr, s.depth, em, mv)])
    return out


def _to_torch(a):
    import torch

    return torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else (a.view(np.int16) if a.dtype == np.uint16 else a))


def _setup(config):
    from granite_b200 import synth, viewer

    w, cfg = CONFIGS[config]
    probe = viewer.Viewer(w, H, cuda_device=-1, **cfg)
    rw, rh = probe.render_size()
    probe.close()
    scene = synth.make_scene(rw, rh)
    lights = synth.make_lights(120, spot_fraction=0.25, aspect=rw / rh)
    views = [synth.look_at_view((0.15 * i, 0.1 * i, 8.0 - 0.2 * i), (0.0, 0.0, 0.0)) for i in range(FRAMES)]
    return w, cfg, scene, lights, views, _frame_inputs(rw, rh, cfg.get("render_target_fp16", False))


def _reference(w, cfg, scene, lights, views, frames_in):
    """The frames of a viewer without a ring, read back to the host."""
    from granite_b200 import viewer
    from tests import sharded

    v = sharded.make_viewer(w, H, scene, lights, views[0], **cfg)
    outs = []
    for i in range(FRAMES):
        v.set_camera(scene.projection, views[i])
        v.render_frame(viewer.Viewer.host_gbuffer(*frames_in[i]))
        out = np.zeros((H, w), np.uint32)
        v.read_output(out)
        outs.append(out)
    v.close()
    return outs


@pytest.mark.parametrize("config", list(CONFIGS))
def test_ring_frames_equal_the_host_readback(cuda, config):
    """6 frames with a moving camera into a ring of 3 tensors, each row 10 or 12 texels wider than the image (a pitch of a
    multiple of 16 bytes) and the padding poisoned; even frames host-fed, odd frames from a padded device G-buffer.  A consumer stream waits on each frame's
    `rendered`, spins, copies the whole padded tensor, and records the image's `acquired` after the copy: without the
    viewer's wait on `acquired`, frame i + 3 would overwrite the image during the spin.  Every copy equals the host
    readback of a viewer without a ring bit for bit, and the padding keeps its poison.  read_output_async of the ring
    viewer reads the image each frame went into."""
    import torch

    from granite_b200 import viewer
    from tests import sharded

    w, cfg, scene, lights, views, frames_in = _setup(config)
    want = _reference(w, cfg, scene, lights, views, frames_in)

    pad = 12 if w % 4 == 0 else 10  # padded rows of a multiple of 16 bytes
    v = sharded.make_viewer(w, H, scene, lights, views[0], **cfg)
    ring_t = [torch.full((H, w + pad), POISON, dtype=torch.int32, device="cuda") for _ in range(RING)]
    v.set_output_images([t[:, :w] for t in ring_t])
    rw, rh = v.render_size()
    # the device G-buffer: padded tensors of the planes' element types, one set overwritten once `consumed` completes
    fp16 = cfg.get("render_target_fp16", False)
    padded = [torch.zeros((rh, rw + 8) + extra, dtype=dt, device="cuda")
              for dt, extra in [(torch.int32, ()), (torch.int32, ()), (torch.int16, ()), (torch.float32, ()),
                                (torch.int16, (4,)) if fp16 else (torch.int32, ()), (torch.int32, ())]]
    planes = [t[:, :rw] for t in padded]
    gb = v.device_gbuffer(*planes)
    ready, consumed = torch.cuda.Event(), torch.cuda.Event()

    consumer = torch.cuda.Stream()
    acquired = [torch.cuda.Event() for _ in range(RING)]
    rendered = [torch.cuda.Event() for _ in range(RING)]
    copies, readbacks = [], [torch.zeros((H, w), dtype=torch.int32, pin_memory=True) for _ in range(FRAMES)]
    for i in range(FRAMES):
        k = i % RING
        v.set_camera(scene.projection, views[i])
        v.acquire_output(k, acquired=acquired[k], rendered=rendered[k])
        if i % 2 == 0:
            v.render_frame(viewer.Viewer.host_gbuffer(*frames_in[i]))
        else:
            consumed.synchronize()
            for t, a in zip(planes, frames_in[i]):
                t.copy_(_to_torch(a))
            ready.record()
            v.render_frame_device(gb, ready=ready, consumed=consumed)
        v.read_output_async(readbacks[i])
        with torch.cuda.stream(consumer):
            consumer.wait_event(rendered[k])
            torch.cuda._sleep(SLEEP_CYCLES)
            copies.append(ring_t[k].clone())
            acquired[k].record(consumer)
    v.wait_outputs(0)
    consumer.synchronize()
    for i in range(FRAMES):
        got = copies[i].cpu().numpy().view(np.uint32)
        assert np.array_equal(got[:, :w], want[i]), f"{config} frame {i}: {int((got[:, :w] != want[i]).sum())} pixels differ from the host readback"
        assert (got[:, w:] == POISON).all(), f"{config} frame {i}: the padding lost its poison"
        assert np.array_equal(readbacks[i].numpy().view(np.uint32), want[i]), f"{config} frame {i}: read_output_async differs"
    v.close()


def test_ring_lifecycle_and_refusals(cuda):
    """On a device viewer: a frame without an acquire and an index past the ring are refused, and so is memory that is
    not device memory of the viewer's device (pinned and pageable host memory).  Replacing the ring, and going back to the graph-owned image (an empty ring), keep every frame equal to the
    viewer without a ring."""
    import torch

    from granite_b200 import capi, viewer
    from tests import sharded

    w, cfg, scene, lights, views, frames_in = _setup("FXAA")
    want = _reference(w, cfg, scene, lights, views, frames_in)
    v = sharded.make_viewer(w, H, scene, lights, views[0], **cfg)
    pitch = (w * 4 + 15) // 16 * 16

    host = torch.zeros((H, pitch // 4), dtype=torch.int32, pin_memory=True)
    pageable = np.zeros(H * pitch // 4 + 4, np.int32)
    page_base = (pageable.ctypes.data + 15) // 16 * 16
    for ptr in (host.data_ptr(), page_base):
        arr = (capi.GrbImage * 1)(capi.GrbImage(ptr, w, H, pitch, capi.FORMAT_R8G8B8A8_SRGB))
        assert viewer.lib().grbh_viewer_set_output_images(v._h, arr, 1) < 0
        assert "is not device memory of the viewer's device" in viewer.lib().grbh_last_error().decode()

    ring_a = [torch.full((H, pitch // 4), POISON, dtype=torch.int32, device="cuda") for _ in range(2)]
    v.set_output_images([t[:, :w] for t in ring_a])
    with pytest.raises(capi.GrbError, match="index 2 is out of range: the ring holds 2 images"):
        v.acquire_output(2)
    v.set_camera(scene.projection, views[0])
    with pytest.raises(capi.GrbError, match="grbh_viewer_acquire_output must precede every frame"):
        v.render_frame(viewer.Viewer.host_gbuffer(*frames_in[0]))
    with pytest.raises(capi.GrbError, match="grbh_viewer_acquire_output must precede every frame"):
        v.render_frame_device(None)

    def frame(i, index=None):
        if index is not None:
            v.acquire_output(index)
        v.set_camera(scene.projection, views[i])
        v.render_frame(viewer.Viewer.host_gbuffer(*frames_in[i]))
        out = np.zeros((H, w), np.uint32)
        v.read_output(out)
        assert np.array_equal(out, want[i]), f"frame {i} differs"

    frame(0, 0)
    assert np.array_equal(ring_a[0].cpu().numpy().view(np.uint32)[:, :w], want[0])
    frame(1, 1)
    assert np.array_equal(ring_a[1].cpu().numpy().view(np.uint32)[:, :w], want[1])
    v.set_output_images([])  # back to the graph-owned image: no acquire needed
    frame(2)
    assert np.array_equal(ring_a[0].cpu().numpy().view(np.uint32)[:, :w], want[0]), "a frame without a ring wrote into the old ring"
    ring_b = [torch.full((H, pitch // 4 + 4), POISON, dtype=torch.int32, device="cuda")]
    v.set_output_images([t[:, :w] for t in ring_b])
    frame(3, 0)
    frame(4, 0)
    got = ring_b[0].cpu().numpy().view(np.uint32)
    assert np.array_equal(got[:, :w], want[4]) and (got[:, w:] == POISON).all()
    v.set_output_images([t[:, :w] for t in ring_a])  # replacing the ring: a pending acquire is dropped
    frame(5, 1)
    assert np.array_equal(ring_a[1].cpu().numpy().view(np.uint32)[:, :w], want[5])
    v.close()
