"""G-buffers in device memory, without a GPU: the argument checks of grb_gbuffer_copy_rows, grb_gbuffer_slot_layout and
grb_gbuffer_rows_to_peers (every check comes before any CUDA call, so host pointers stand in for device memory), the
refusals of grbh_viewer_render_frame_device and grbh_viewer_set_gbuffer_source_rank that a host-only viewer reaches, and
grbh_viewer_get_input_rows against the row plans of grbh_shard_plan*."""
import ctypes as C

import numpy as np
import pytest

OK, ERR_ARG = 0, -1


@pytest.fixture(scope="module")
def viewer():
    from granite_b200 import build, viewer

    build.build_all()
    return viewer


def _lib():
    from granite_b200 import capi

    L = C.CDLL(capi.LIB_PATH)
    L.grb_last_error_string.restype = C.c_char_p
    return L


def _msg(L):
    return (L.grb_last_error_string() or b"").decode()


def _planes(keep, w, h, fp16=False, mv=True, pitch_pad=0):
    """A GrbGBufferPlanes over host arrays (never dereferenced by a refused call)."""
    from granite_b200 import capi

    fmts = [capi.FORMAT_R16G16B16A16_SFLOAT if fp16 else capi.FORMAT_B10G11R11_UFLOAT, capi.FORMAT_R8G8B8A8_SRGB, capi.FORMAT_A2B10G10R10_UNORM,
            capi.FORMAT_R8G8_UNORM, capi.FORMAT_D32_SFLOAT, capi.FORMAT_R16G16_SFLOAT]
    g = capi.GrbGBufferPlanes()
    for p, fmt in enumerate(fmts):
        if p == 5 and not mv:
            continue
        t = capi.TEXEL_BYTES[fmt]
        pitch = w * t + pitch_pad * t
        a = np.zeros(pitch * h // 8 + 2, np.uint64)
        keep.append(a)
        g.plane[p] = capi.GrbImage(a.ctypes.data, w, h, pitch, fmt)
    return g


def test_copy_rows_argument_checks(viewer):
    from granite_b200 import capi

    L = _lib()
    keep = []
    w, h = 24, 16
    src, dst = _planes(keep, w, h), _planes(keep, w, h)
    rows = (capi.GrbRows * 2)(capi.GrbRows(0, 4), capi.GrbRows(8, 16))

    def call(s=src, d=dst, r=rows, n=2):
        return L.grb_gbuffer_copy_rows(None if s is None else C.byref(s), None if d is None else C.byref(d), r, n, None)

    def changed(g, p, **kw):
        c = capi.GrbGBufferPlanes.from_buffer_copy(g)
        for k, v in kw.items():
            setattr(c.plane[p], k, v)
        return c

    assert call(s=None) == ERR_ARG and "grb_gbuffer_copy_rows" in _msg(L)
    assert call(d=None) == ERR_ARG
    assert call(r=None) == ERR_ARG
    assert call(n=-1) == ERR_ARG
    # no plane at all
    assert call(s=capi.GrbGBufferPlanes(), d=capi.GrbGBufferPlanes()) == ERR_ARG and "no plane" in _msg(L)
    # a texel size that does not fit the plane: 8-byte albedo, 4-byte pbr, 2-byte depth
    for p, fmt in ((1, capi.FORMAT_R16G16B16A16_SFLOAT), (3, capi.FORMAT_D32_SFLOAT), (4, capi.FORMAT_R8G8_UNORM), (0, 12345)):
        assert call(s=changed(src, p, format=fmt)) == ERR_ARG and "does not fit" in _msg(L)
    # pitch too small, not a multiple of the texel, misaligned base, empty size
    assert call(s=changed(src, 1, row_pitch=w * 4 - 4)) == ERR_ARG and "row pitch" in _msg(L)
    assert call(d=changed(dst, 3, row_pitch=w * 2 + 1)) == ERR_ARG and "row pitch" in _msg(L)
    assert call(s=changed(src, 0, row_pitch=w * 4 + 2)) == ERR_ARG
    assert call(s=changed(src, 4, data=src.plane[4].data + 2)) == ERR_ARG and "aligned" in _msg(L)
    assert call(s=changed(src, 2, width=0)) == ERR_ARG
    assert call(s=changed(src, 2, height=0)) == ERR_ARG
    # planes of different sizes within a set, and sets that disagree
    assert call(s=changed(src, 2, width=w - 1)) == ERR_ARG and "differs in size" in _msg(L)
    assert call(s=changed(src, 5, data=None)) == ERR_ARG and "same planes" in _msg(L)
    assert call(s=changed(src, 0, format=capi.FORMAT_R16G16B16A16_SFLOAT, row_pitch=w * 8)) == ERR_ARG and "formats" in _msg(L)
    assert call(d=changed(dst, 1, format=capi.FORMAT_R8G8B8A8_UNORM)) == ERR_ARG and "formats" in _msg(L)
    assert call(d=changed(dst, 2, data=src.plane[2].data)) == ERR_ARG and "same image" in _msg(L)
    # ranges outside the image
    for bad in ((-1, 4), (6, 4), (8, h + 1)):
        assert call(r=(capi.GrbRows * 1)(capi.GrbRows(*bad)), n=1) == ERR_ARG and "range" in _msg(L)
    assert not any(a.any() for a in keep), "a refused call wrote something"


def test_slot_layout(viewer):
    from granite_b200 import capi, harness

    keep = []
    w, h = 93, 7
    g = _planes(keep, w, h, fp16=True, pitch_pad=3)
    slot, size = harness.gbuffer_slot_layout(g, 0x10000)
    texels = [8, 4, 4, 2, 4, 4]
    at = 0
    for p, t in enumerate(texels):
        assert slot.plane[p].data == 0x10000 + at and slot.plane[p].row_pitch == w * t
        assert (slot.plane[p].width, slot.plane[p].height, slot.plane[p].format) == (w, h, g.plane[p].format)
        at = (at + w * t * h + 255) // 256 * 256
    assert size == at
    # absent planes take no room; without a base only the size comes back
    g.plane[5].data = None
    g.plane[2].data = None
    slot, size2 = harness.gbuffer_slot_layout(g)
    assert not slot.plane[2].data and not slot.plane[5].data and not slot.plane[0].data
    assert size2 == sum((w * t * h + 255) // 256 * 256 for p, t in enumerate(texels) if p not in (2, 5))
    with pytest.raises(capi.GrbError, match="no plane"):
        harness.gbuffer_slot_layout(capi.GrbGBufferPlanes())


def test_rows_to_peers_argument_checks(viewer):
    from granite_b200 import capi

    L = _lib()
    keep = [np.zeros(64, np.uint32) for _ in range(4)]
    w, h = 32, 16
    src = _planes(keep, w, h)
    slots = (C.c_void_p * 2)(keep[0].ctypes.data, keep[1].ctypes.data)
    flags = (C.c_void_p * 2)(keep[2].ctypes.data, keep[3].ctypes.data)
    counter = C.c_void_p(keep[2].ctypes.data + 32)
    rows = (capi.GrbRows * 3)(capi.GrbRows(0, 4), capi.GrbRows(8, 12), capi.GrbRows(4, 16))

    def call(s=src, sl=slots, fl=flags, r=rows, counts=(2, 1), n=2, k=0, ctr=counter):
        cnt = None if counts is None else (C.c_int32 * len(counts))(*counts)
        return L.grb_gbuffer_rows_to_peers(None if s is None else C.byref(s), sl, fl, r, cnt, n, k, C.c_uint32(1), ctr, None)

    assert call(s=None) == ERR_ARG and "grb_gbuffer_rows_to_peers" in _msg(L)
    assert call(counts=None) == ERR_ARG
    assert call(fl=None) == ERR_ARG
    assert call(ctr=None) == ERR_ARG
    assert call(fl=(C.c_void_p * 2)(keep[2].ctypes.data, None)) == ERR_ARG and "null peer" in _msg(L)
    assert call(sl=(C.c_void_p * 2)(keep[0].ctypes.data, None)) == ERR_ARG and "null peer pointer" in _msg(L)
    assert call(n=0) == ERR_ARG and "peer_count" in _msg(L)
    assert call(n=9, counts=(0,) * 9) == ERR_ARG
    assert call(k=2) == ERR_ARG and "flag_index" in _msg(L)
    assert call(k=-1) == ERR_ARG
    assert call(counts=(2, -1)) == ERR_ARG and "negative" in _msg(L)
    # no slots, also with no rows listed (the credit is grb_peer_publish); rows listed without a list
    assert call(sl=None) == ERR_ARG and "grb_gbuffer_rows_to_peers: null pointer" in _msg(L)
    assert call(sl=None, r=None, counts=(0, 0)) == ERR_ARG and "grb_gbuffer_rows_to_peers: null pointer" in _msg(L)
    assert call(r=None) == ERR_ARG and "row list" in _msg(L)
    # a bad plane, a range outside the image
    bad = capi.GrbGBufferPlanes.from_buffer_copy(src)
    bad.plane[3].row_pitch = w * 2 - 2
    assert call(s=bad) == ERR_ARG and "row pitch" in _msg(L)
    assert call(r=(capi.GrbRows * 3)(capi.GrbRows(0, 4), capi.GrbRows(8, 12), capi.GrbRows(4, h + 1))) == ERR_ARG and "range" in _msg(L)
    assert not any(a.any() for a in keep), "a refused call wrote something"


def _device_gbuffer(viewer, keep, w, h, fp16=False, mv=True, **override):
    """A GrbhDeviceGBuffer over host arrays: the viewer refuses it before it touches any memory."""
    from granite_b200 import capi

    g = _planes(keep, w, h, fp16=fp16, mv=mv)
    d = viewer.GrbhDeviceGBuffer(*[g.plane[p] for p in range(6)])
    for name, fields in override.items():
        for k, v in fields.items():
            setattr(getattr(d, name), k, v)
    return d


def test_render_frame_device_refusals(viewer):
    from granite_b200 import capi

    keep = []
    v = viewer.Viewer(64, 48, post_aa=viewer.AA_TAA_HIGH, cuda_device=-1)
    fsr = viewer.Viewer(64, 48, resolution_scale=0.67, cuda_device=-1)
    fp16 = viewer.Viewer(64, 48, render_target_fp16=True, cuda_device=-1)
    try:
        def refused(vw, gb, match):
            with pytest.raises(capi.GrbError, match=match):
                vw.render_frame_device(gb)

        refused(v, _device_gbuffer(viewer, keep, 64, 48, mv=False), "mv plane is missing")
        for name in ("emissive", "albedo", "normal", "pbr", "depth"):
            refused(v, _device_gbuffer(viewer, keep, 64, 48, **{name: dict(data=None)}), f"the {name} plane is missing")
        refused(v, _device_gbuffer(viewer, keep, 64, 47), r"64 x 47; the viewer renders at 64 x 48")
        refused(v, _device_gbuffer(viewer, keep, 63, 48), "renders at 64 x 48")
        refused(v, _device_gbuffer(viewer, keep, 64, 48, albedo=dict(row_pitch=64 * 4 - 4)), "albedo plane's row_pitch 252")
        refused(v, _device_gbuffer(viewer, keep, 64, 48, pbr=dict(row_pitch=64 * 2 + 1)), "multiple of its texel size")
        refused(v, _device_gbuffer(viewer, keep, 64, 48, depth=dict(format=capi.FORMAT_R16G16_SFLOAT)), "depth plane has format")
        # the emissive format follows render_target_fp16
        refused(v, _device_gbuffer(viewer, keep, 64, 48, fp16=True), "emissive plane has format")
        refused(fp16, _device_gbuffer(viewer, keep, 64, 48), "emissive plane has format")
        # FSR 1: the render size, not the display size
        refused(fsr, _device_gbuffer(viewer, keep, 64, 48, mv=False), "renders at 43 x 33")
        # a G-buffer that passes every check, and NULL, reach the device check
        refused(v, _device_gbuffer(viewer, keep, 64, 48, pbr=dict(row_pitch=64 * 2 + 6)), "host-only viewer")
        refused(fsr, _device_gbuffer(viewer, keep, 43, 33, mv=False), "host-only viewer")
        refused(fp16, _device_gbuffer(viewer, keep, 64, 48, fp16=True, mv=False), "host-only viewer")
        refused(v, None, "host-only viewer")
        assert not any(a.any() for a in keep)
    finally:
        for x in (v, fsr, fp16):
            x.close()


def test_gbuffer_source_rank(viewer):
    from granite_b200 import capi

    keep = []
    v = viewer.Viewer(64, 128, cuda_device=-1)
    try:
        v.set_gbuffer_source_rank(0)  # unsharded: one band, and 0 changes nothing
        v.set_gbuffer_source_rank(-1)
        for bad in (1, -2):
            with pytest.raises(capi.GrbError, match="grbh_viewer_set_gbuffer_source_rank"):
                v.set_gbuffer_source_rank(bad)
        v.set_row_shards([(0, 32), (32, 64), (64, 128)], 1)
        for r in (-1, 0, 1, 2):
            v.set_gbuffer_source_rank(r)
        for bad in (3, -2):
            with pytest.raises(capi.GrbError, match=r"within \[0, 3\)"):
                v.set_gbuffer_source_rank(bad)
        # the source rank keeps a band
        with pytest.raises(capi.GrbError, match="G-buffer source rank 2 would have no band"):
            v.set_row_shards([(0, 64), (64, 128)], 1)
        # rank 1 is not the source: it passes NULL, and the host path is refused on every rank
        gb = _device_gbuffer(viewer, keep, 64, 128, mv=False)
        with pytest.raises(capi.GrbError, match="every other rank passes NULL"):
            v.render_frame_device(gb)
        with pytest.raises(capi.GrbError, match="grbh_viewer_render_frame_device"):
            v.render_frame(None)
        with pytest.raises(capi.GrbError, match="host-only viewer"):
            v.render_frame_device(None)
        v.set_gbuffer_source_rank(1)
        with pytest.raises(capi.GrbError, match="this rank is the G-buffer source rank"):
            v.render_frame_device(None)
        with pytest.raises(capi.GrbError, match="host-only viewer"):
            v.render_frame_device(gb)
        with pytest.raises(capi.GrbError, match="G-buffer source rank"):
            v.render_frame(None)
        v.set_gbuffer_source_rank(-1)
        with pytest.raises(capi.GrbError, match="not baked"):
            v.render_frame(None)
    finally:
        v.close()
    p = viewer.Viewer(64, 128, cuda_device=-1, pipelined_io=True)
    try:
        p.set_row_shards([(0, 64), (64, 128)], 0)
        with pytest.raises(capi.GrbError, match="pipelined_io"):
            p.set_gbuffer_source_rank(0)
        p.set_gbuffer_source_rank(-1)
    finally:
        p.close()


LAYOUTS = {2: [(0, 64), (64, 200)], 3: [(0, 48), (48, 112), (112, 200)], 4: [(0, 32), (32, 96), (96, 160), (160, 200)]}
CONFIGS = {"no AA": {}, "FXAA": dict(post_aa=1), "SMAA Ultra": dict(post_aa=6), "TAA High": dict(post_aa=10), "TAA High + FXAA": dict(post_aa=100)}


@pytest.mark.parametrize("world", sorted(LAYOUTS))
@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_input_rows_follow_the_plan(viewer, world, config):
    w, h = 96, 200
    bands = LAYOUTS[world]
    post_aa = CONFIGS[config].get("post_aa", viewer.AA_NONE)
    fxaa = post_aa in (viewer.AA_FXAA, viewer.AA_TAA_HIGH_PLUS_FXAA)
    taa = post_aa in (viewer.AA_TAA_HIGH, viewer.AA_TAA_HIGH_PLUS_FXAA)
    for rank in range(world):
        v = viewer.Viewer(w, h, cuda_device=-1, **CONFIGS[config])
        try:
            assert v.input_rows() == [(0, h)]  # unsharded: the whole image
            v.set_row_shards(bands, rank)
            if taa:
                want = viewer.shard_plan_taa(w, h, bands, rank, fxaa)["lighting"]
            elif post_aa == viewer.AA_SMAA_ULTRA:
                want = viewer.shard_plan_smaa(w, h, bands, rank, 3)["lighting"]
            else:
                want = viewer.shard_plan(w, h, bands, rank, fxaa)["lighting"]
            assert v.input_rows() == [want]
            for stripe in (8, 16, 64):
                v.set_lighting_stripes(stripe)
                assert v.input_rows() == viewer.shard_plan_stripes(w, h, bands, rank, stripe, post_aa)["upload"]
            v.set_lighting_stripes(0)
            # the rows follow the bands as they move
            moved = [(0, 16), (16, bands[1][1])] + list(bands[2:])
            v.set_row_shards(moved, rank)
            want = viewer.shard_plan_taa(w, h, moved, rank, fxaa)["lighting"] if taa else (
                viewer.shard_plan_smaa(w, h, moved, rank, 3)["lighting"] if post_aa == viewer.AA_SMAA_ULTRA else viewer.shard_plan(w, h, moved, rank, fxaa)["lighting"])
            assert v.input_rows() == [want]
        finally:
            v.close()


@pytest.mark.parametrize("post_aa", [0, 1, 6, 100])
def test_input_rows_with_fsr(viewer, post_aa):
    w, h = 160, 240
    bands = [(0, 64), (64, 128), (128, 176), (176, 240)]
    for rank in range(len(bands)):
        v = viewer.Viewer(w, h, cuda_device=-1, post_aa=post_aa, resolution_scale=0.67, resolution_scale_sharpen=True)
        try:
            rw, rh = v.render_size()
            assert (rw, rh) == (108, 161)
            assert v.input_rows() == [(0, rh)]
            v.set_row_shards(bands, rank)
            want = viewer.shard_plan_fsr(w, h, rw, rh, bands, rank, post_aa, True)["lighting"]
            assert v.input_rows() == [want]
            assert 0 <= want[0] < want[1] <= rh
        finally:
            v.close()
