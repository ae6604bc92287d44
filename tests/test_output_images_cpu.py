"""Rings of caller-owned output images, without a GPU: the refusals of grbh_viewer_set_output_images,
grbh_viewer_acquire_output and grbh_viewer_render_frame that a host-only viewer
(cuda_device = -1) reaches, each matched by its message.  Every host check comes before any CUDA call, so the images
are plain addresses that nothing dereferences."""
import pytest

BASE = 0x7F0000000000  # 16-byte aligned; never dereferenced


@pytest.fixture(scope="module")
def viewer():
    from granite_b200 import build, viewer

    build.build_all()
    return viewer


def _images(specs):
    """(GrbImage array, count) from (data, width, height, row_pitch, format) tuples."""
    from granite_b200 import capi

    arr = (capi.GrbImage * max(len(specs), 1))(*[capi.GrbImage(*s) for s in specs])
    return arr, len(specs)


def _set(viewer, v, specs, null=False, count=None):
    arr, n = _images(specs)
    rc = viewer.lib().grbh_viewer_set_output_images(v._h, None if null else arr, n if count is None else count)
    return rc, viewer.lib().grbh_last_error().decode()


def _refused(viewer, v, specs, match, **kw):
    rc, msg = _set(viewer, v, specs, **kw)
    assert rc < 0, f"accepted; expected a refusal matching {match!r}"
    assert match in msg, msg


def _ring(w, h, n=3, pitch=None, fmt=43):
    pitch = pitch if pitch is not None else (w * 4 + 15) // 16 * 16
    return [(BASE + i * pitch * h, w, h, pitch, fmt) for i in range(n)]


def test_ring_argument_checks(viewer):
    from granite_b200 import capi

    w, h = 100, 48  # 400-byte rows: a multiple of 16
    v = viewer.Viewer(w, h, cuda_device=-1)
    srgb = capi.FORMAT_R8G8B8A8_SRGB
    _refused(viewer, v, _ring(w, h), "bad arguments", count=-1)
    _refused(viewer, v, _ring(w, h), "images NULL", null=True)
    _refused(viewer, v, [(0, w, h, 400, srgb)], "has no memory")
    _refused(viewer, v, [(BASE, w - 1, h, 400, srgb)], "is 99 x 48; the display size is 100 x 48")
    _refused(viewer, v, [(BASE, w, h + 1, 400, srgb)], "is 100 x 49; the display size is 100 x 48")
    _refused(viewer, v, [(BASE, w, h, 400, capi.FORMAT_R8G8B8A8_UNORM)], "the viewer's output format is 43")
    _refused(viewer, v, [(BASE, w, h, 400, capi.FORMAT_A2B10G10R10_UNORM)], "the viewer's output format is 43")
    _refused(viewer, v, [(BASE, w, h, 384, srgb)], "row_pitch 384 must be a multiple of 16 bytes and at least width x 4 (400)")
    _refused(viewer, v, [(BASE, w, h, 408, srgb)], "row_pitch 408 must be a multiple of 16")
    _refused(viewer, v, [(BASE + 4, w, h, 400, srgb)], "not 16-byte aligned")
    _refused(viewer, v, [(BASE + 8, w, h, 416, srgb)], "not 16-byte aligned")
    # overlaps: the second image starts inside the first one's last row; two images share a base; a pitched image whose
    # padding holds a second one still overlaps by span
    _refused(viewer, v, [(BASE, w, h, 400, srgb), (BASE + 400 * (h - 1) + 384, w, h, 400, srgb)], "output images 0 and 1 overlap")
    _refused(viewer, v, [(BASE, w, h, 400, srgb), (BASE + 4096 * h, w, h, 400, srgb), (BASE, w, h, 416, srgb)], "output images 0 and 2 overlap")
    _refused(viewer, v, [(BASE, w, h, 800, srgb), (BASE + 400, w, h, 800, srgb)], "output images 0 and 1 overlap")
    # images that touch end to start do not overlap: they reach the device check
    _refused(viewer, v, [(BASE, w, h, 400, srgb), (BASE + 400 * h, w, h, 400, srgb)], "host-only viewer")
    # an image that passes every host check reaches the device check; count 0 needs no device
    _refused(viewer, v, _ring(w, h, 1), "host-only viewer (cuda_device < 0) has no device")
    assert _set(viewer, v, [])[0] == 0
    v.close()


def test_display_size_and_format_follow_the_config(viewer):
    """The ring has the display size under FSR 1, and the HDR10 swapchain format with hdr10_output."""
    from granite_b200 import capi

    w, h = 128, 72
    fsr = viewer.Viewer(w, h, cuda_device=-1, resolution_scale=0.67)
    rw, rh = fsr.render_size()
    assert (rw, rh) != (w, h)
    _refused(viewer, fsr, _ring(rw, rh, 1), f"is {rw} x {rh}; the display size is {w} x {h}")
    _refused(viewer, fsr, _ring(w, h, 1), "host-only viewer")
    fsr.close()
    hdr = viewer.Viewer(w, h, cuda_device=-1, post_aa=viewer.AA_TAA_HIGH, hdr10_output=True)
    _refused(viewer, hdr, _ring(w, h, 1, fmt=capi.FORMAT_R8G8B8A8_SRGB), "the viewer's output format is 64 (A2B10G10R10_UNORM_PACK32: HDR10 output)")
    _refused(viewer, hdr, _ring(w, h, 1, fmt=capi.FORMAT_A2B10G10R10_UNORM), "host-only viewer")
    hdr.close()


def test_acquire_and_frames(viewer):
    """An acquire needs a ring and an index within it; a host-only viewer never holds one, so a frame reaches the
    checks behind the acquire rule."""
    v = viewer.Viewer(64, 48, cuda_device=-1)
    L = viewer.lib()
    for index in (0, 2, -1):
        assert L.grbh_viewer_acquire_output(v._h, index, None, None) < 0
        assert "no output images are set" in L.grbh_last_error().decode()
    with pytest.raises(Exception, match="not baked"):
        v.render_frame(None)
    assert L.grbh_viewer_acquire_output(None, 0, None, None) < 0
    assert L.grbh_viewer_set_output_images(None, None, 0) < 0
    v.close()


@pytest.mark.parametrize("present", [0, 3])
def test_only_the_presenting_rank_holds_a_ring(viewer, present):
    """On a presenting layout every other rank's ring is refused; the presenting rank's reaches the device check."""
    w, h = 64, 128
    bands = [(0, 32), (32, 64), (64, 96), (96, 128)]
    for rank in range(4):
        v = viewer.Viewer(w, h, cuda_device=-1)
        v.set_row_shards(bands, rank)
        v.set_present_rank(present)
        if rank == present:
            _refused(viewer, v, _ring(w, h, 2), "host-only viewer")
        else:
            _refused(viewer, v, _ring(w, h, 2), f"rank {rank} does not present (grbh_viewer_set_present_rank {present})")
            assert _set(viewer, v, [])[0] == 0  # dropping a ring is always allowed
        v.close()
    # without a presenting rank every rank may hold one
    v = viewer.Viewer(w, h, cuda_device=-1)
    v.set_row_shards(bands, 1)
    _refused(viewer, v, _ring(w, h, 2), "host-only viewer")
    v.close()


def test_python_wrapper(viewer):
    """Viewer.acquire_output without events, and Viewer.set_output_images([]) (back to the graph-owned image)."""
    v = viewer.Viewer(32, 16, cuda_device=-1)
    with pytest.raises(Exception, match="no output images are set"):
        v.acquire_output(0)
    v.set_output_images([])
    v.close()
