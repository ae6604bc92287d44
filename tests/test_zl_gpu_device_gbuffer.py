"""G-buffers in device memory on the GPU: the row copy into the attachments (grb_gbuffer_copy_rows), the push of each
rank's rows into its G-buffer slot (grb_gbuffer_rows_to_peers), and whole frames rendered from a device G-buffer
(grbh_viewer_render_frame_device) against the frames of the host-fed viewer, bit for bit."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
SENTINEL = 0xA5


def _fmts(fp16):
    from granite_b200 import capi

    return [capi.FORMAT_R16G16B16A16_SFLOAT if fp16 else capi.FORMAT_B10G11R11_UFLOAT, capi.FORMAT_R8G8B8A8_SRGB, capi.FORMAT_A2B10G10R10_UNORM,
            capi.FORMAT_R8G8_UNORM, capi.FORMAT_D32_SFLOAT, capi.FORMAT_R16G16_SFLOAT]


def _byte_planes(rng, w, pitch_texels, h, fp16, fill=None):
    """Six planes as (h, pitch) uint8 tensors and the GrbGBufferPlanes over their first w texels: random bytes, or
    `fill` everywhere."""
    import torch

    from granite_b200 import capi

    tensors, g = [], capi.GrbGBufferPlanes()
    for p, fmt in enumerate(_fmts(fp16)):
        t = capi.TEXEL_BYTES[fmt]
        a = rng.integers(0, 256, (h, pitch_texels * t), dtype=np.uint8) if fill is None else np.full((h, pitch_texels * t), fill, np.uint8)
        tensors.append(torch.from_numpy(a).cuda())
        g.plane[p] = capi.GrbImage(tensors[-1].data_ptr(), w, h, pitch_texels * t, fmt)
    return tensors, g


@pytest.mark.parametrize("fp16", [False, True], ids=["b10g11r11", "rgba16f"])
@pytest.mark.parametrize("width,pitch_texels,ranges", [
    (96, 96, [(0, 3), (5, 6), (10, 20), (40, 41)]),
    (93, 93, [(0, 3), (5, 6), (10, 20), (40, 41)]),
    (97, 100, [(0, 3), (5, 6), (10, 20), (40, 41), (47, 48)]),
    (96, 96, [(y, y + 1) for y in range(0, 300, 2)] + [(301, 303), (280, 290)]),  # more ranges than one launch takes
])
def test_copy_rows_writes_only_the_listed_rows(cuda, fp16, width, pitch_texels, ranges):
    """Sentinel-filled destinations: after the copy every listed row of every plane holds the source's bytes over the
    image width, and every other byte (the other rows, the padding past the width) is still the sentinel.  Widths: 16-byte
    rows on every plane (96), rows of no 16-byte multiple (93: texel path), and 97 texels in a pitch of 100 (16-byte
    rows on the 4- and 8-byte planes with a texel tail, the texel path on the 2-byte pbr plane)."""
    import torch

    from granite_b200 import capi, harness

    h = max(y1 for _, y1 in ranges) + 1
    rng = np.random.default_rng(width + pitch_texels + int(fp16))
    src_t, src = _byte_planes(rng, width, pitch_texels, h, fp16)
    dst_t, dst = _byte_planes(rng, width, pitch_texels, h, fp16, fill=SENTINEL)
    harness.gbuffer_copy_rows(src, dst, ranges)
    torch.cuda.synchronize()
    for p, fmt in enumerate(_fmts(fp16)):
        row = width * capi.TEXEL_BYTES[fmt]
        want = np.full(dst_t[p].shape, SENTINEL, np.uint8)
        s = src_t[p].cpu().numpy()
        for y0, y1 in ranges:
            want[y0:y1, :row] = s[y0:y1, :row]
        assert np.array_equal(dst_t[p].cpu().numpy(), want), f"plane {capi.GBUFFER_PLANES[p]} differs"
    # absent planes: a set of motion vectors only
    mv = capi.GrbGBufferPlanes()
    mv.plane[5] = src.plane[5]
    mv_dst_t = torch.full_like(dst_t[5], SENTINEL)
    mv_dst = capi.GrbGBufferPlanes()
    mv_dst.plane[5] = capi.GrbImage(mv_dst_t.data_ptr(), width, h, dst.plane[5].row_pitch, capi.FORMAT_R16G16_SFLOAT)
    harness.gbuffer_copy_rows(mv, mv_dst, ranges[:2])
    torch.cuda.synchronize()
    want = np.full(mv_dst_t.shape, SENTINEL, np.uint8)
    for y0, y1 in ranges[:2]:
        want[y0:y1, :width * 4] = src_t[5].cpu().numpy()[y0:y1, :width * 4]
    assert np.array_equal(mv_dst_t.cpu().numpy(), want)


@pytest.mark.parametrize("width,pitch_texels", [(96, 96), (93, 93), (97, 100)])
def test_rows_to_peers_routes_each_ranks_rows(cuda, width, pitch_texels):
    """Two allocations stand in for two ranks' G-buffer slots; rank 1 is the source.  Each rank's slot receives exactly
    its listed rows of every plane at their place in the slot layout, every other byte stays the sentinel; every flag
    array gets the epoch at the caller's index; the scratch counter is reset.  Then rank 0's credit (grb_peer_publish)
    raises its word and writes nothing."""
    import torch

    from granite_b200 import capi, harness

    h = 40
    rng = np.random.default_rng(width)
    src_t, src = _byte_planes(rng, width, pitch_texels, h, True)
    _, size = harness.gbuffer_slot_layout(src)
    slots = [torch.full((size,), SENTINEL, dtype=torch.uint8, device="cuda") for _ in range(2)]
    flags = [torch.zeros(16, dtype=torch.int32, device="cuda") for _ in range(2)]
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    rows = [[(0, 5), (9, 12), (30, 40)], [(4, 20)]]
    harness.gbuffer_rows_to_peers(src, slots, flags, rows, 1, 5, counter)
    torch.cuda.synchronize()
    for q in range(2):
        planes, _ = harness.gbuffer_slot_layout(src, slots[q].data_ptr())
        want = np.full(size, SENTINEL, np.uint8)
        for p, fmt in enumerate(_fmts(True)):
            row = width * capi.TEXEL_BYTES[fmt]
            off = planes.plane[p].data - slots[q].data_ptr()
            s = src_t[p].cpu().numpy()
            for y0, y1 in rows[q]:
                want[off + y0 * row:off + y1 * row] = s[y0:y1, :row].reshape(-1)
        assert np.array_equal(slots[q].cpu().numpy(), want), f"rank {q}'s slot differs"
    for f in flags:
        assert list(f.cpu().numpy()) == [0, 5] + [0] * 14
    assert counter.item() == 0
    before = [s.clone() for s in slots]
    harness.peer_publish(flags, 0, 6, counter)
    torch.cuda.synchronize()
    for f in flags:
        assert list(f.cpu().numpy()) == [6, 5] + [0] * 14
    assert counter.item() == 0 and all(torch.equal(a, b) for a, b in zip(before, slots))


FRAMES = 6
CONFIGS = {
    "no AA": dict(),
    "TAA High + FXAA": dict(post_aa=100),
    "SMAA Ultra": dict(post_aa=6),
    "FSR 0.67 + RCAS": dict(resolution_scale=0.67, resolution_scale_sharpen=True),
    "RGBA16F": dict(render_target_fp16=True),
    "HDR10 + TAA": dict(post_aa=10, hdr10_output=True),
    "pipelined_io + TAA": dict(post_aa=10, pipelined_io=True),
}


def _frame_inputs(rw, rh, fp16):
    """One seeded G-buffer per frame at the render size (the scene's emissive, or an RGBA16F one): lists of host arrays in
    host_gbuffer order (albedo, normal, pbr, depth, emissive, mv)."""
    from granite_b200 import synth
    from tests import common, sharded

    out = []
    for i in range(FRAMES):
        scene = synth.make_scene(rw, rh, seed=100 + i)
        em = common.random_hdr_f16(np.random.default_rng(i), rw, rh, scale=0.02, hot=0.001) if fp16 else scene.emissive
        mv = sharded.motion_vectors(rw, rh, i).view(np.uint32).reshape(rh, rw)
        out.append([np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, em, mv)])
    return out


@pytest.mark.parametrize("config", list(CONFIGS))
def test_device_gbuffer_frames_equal_host_fed_frames(cuda, config):
    """6 frames with a moving camera and a G-buffer that changes every frame, then one resident frame (NULL).  The device
    G-buffer lives in padded tensors (each row 24 texels wider than the image): one set, overwritten with the next
    frame's G-buffer once the viewer's `consumed` event of the last frame has completed, its copy ordered before the frame
    by `ready`.  Every frame equals the host-fed viewer's frame bit for bit."""
    import torch

    from granite_b200 import synth, viewer
    from tests import sharded

    w, h, pad = 320, 192, 24
    cfg = CONFIGS[config]
    probe = viewer.Viewer(w, h, cuda_device=-1, **cfg)
    rw, rh = probe.render_size()
    probe.close()
    fp16 = cfg.get("render_target_fp16", False)
    frames_in = _frame_inputs(rw, rh, fp16)
    scene = synth.make_scene(rw, rh)
    lights = synth.make_lights(120, spot_fraction=0.25, aspect=rw / rh)
    views = [synth.look_at_view((0.15 * i, 0.1 * i, 8.0 - 0.2 * i), (0.0, 0.0, 0.0)) for i in range(FRAMES + 1)]

    def run(device):
        v = sharded.make_viewer(w, h, scene, lights, views[0], **cfg)
        outs = []
        if device:
            # (rh, rw + pad) tensors of the planes' element types; the G-buffer is the first rw texels of each row
            shapes = [(torch.int32, ()), (torch.int32, ()), (torch.int16, ()), (torch.float32, ()), (torch.int16, (4,)) if fp16 else (torch.int32, ()),
                      (torch.int32, ())]
            padded = [torch.zeros((rh, rw + pad) + extra, dtype=dt, device="cuda") for dt, extra in shapes]
            views_ = [t[:, :rw] for t in padded]
            gb = v.device_gbuffer(*views_)
            ready, consumed = torch.cuda.Event(), torch.cuda.Event()
        for i in range(len(views)):
            v.set_camera(scene.projection, views[i])
            if i == FRAMES:
                v.render_frame_device(None) if device else v.render_frame(None)
            elif device:
                consumed.synchronize()
                for t, a in zip(views_, frames_in[i]):
                    t.copy_(torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else (a.view(np.int16) if a.dtype == np.uint16 else a)))
                ready.record()
                v.render_frame_device(gb, ready=ready, consumed=consumed)
            else:
                v.render_frame(viewer.Viewer.host_gbuffer(*frames_in[i]))
            out = np.zeros((h, w), np.uint32)
            v.read_output(out)
            outs.append(out)
        v.close()
        return outs

    if cfg.get("pipelined_io"):
        views = views[:FRAMES]  # pipelined_io needs a G-buffer every frame: no resident frame
    want, got = run(False), run(True)
    for i, (a, b) in enumerate(zip(want, got)):
        assert np.array_equal(a, b), f"{config} frame {i}: {int((a != b).sum())} pixels differ from the host-fed frame"


def test_pipelined_io_needs_a_device_gbuffer_every_frame(cuda):
    """pipelined_io refuses a frame without a G-buffer on the device path too."""
    from granite_b200 import capi, synth
    from tests import sharded

    w, h = 64, 48
    scene = synth.make_scene(w, h)
    v = sharded.make_viewer(w, h, scene, synth.make_lights(8, aspect=w / h), scene.view, pipelined_io=True)
    with pytest.raises(capi.GrbError, match="pipelined_io"):
        v.render_frame_device(None)
    v.close()
