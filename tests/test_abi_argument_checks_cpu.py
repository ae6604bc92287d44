"""The C ABI's error behaviour without a GPU: every entry point validates its arguments BEFORE it touches CUDA, returns a
negative GrbResult and leaves a message in grb_last_error_string() -- no exception, no abort crosses the boundary
(include/granite_b200.h, SURVEY 8(b) error conventions).  Exercised here for the entry points added in round 2."""
import ctypes as C

import numpy as np
import pytest

OK, ERR_ARG, ERR_FORMAT = 0, -1, -2


@pytest.fixture(scope="module")
def lib():
    from granite_b200 import build, capi

    build.build_all()
    L = C.CDLL(capi.LIB_PATH)
    L.grb_last_error_string.restype = C.c_char_p
    return L


def _image(capi, arr, fmt, w=None, h=None):
    h_, w_ = arr.shape[:2]
    w, h = w or w_, h or h_
    return capi.GrbImage(arr.ctypes.data, w, h, w * capi.TEXEL_BYTES[fmt], fmt)


def _msg(lib):
    return (lib.grb_last_error_string() or b"").decode()


def test_fsr_argument_checks(lib):
    from granite_b200 import capi

    lo, hi = np.zeros((8, 8), np.uint32), np.zeros((12, 12), np.uint32)
    rows, f = capi.GrbRows(0, 0), C.c_float
    a, b = _image(capi, lo, capi.FORMAT_R8G8B8A8_UNORM), _image(capi, hi, capi.FORMAT_R8G8B8A8_UNORM)
    wrong = _image(capi, hi, capi.FORMAT_B10G11R11_UFLOAT)
    assert lib.grb_fsr_upscale(C.byref(a), C.byref(wrong), rows, None) == ERR_FORMAT and "grb_fsr_upscale" in _msg(lib)
    assert lib.grb_fsr_upscale(None, C.byref(b), rows, None) == ERR_FORMAT
    assert lib.grb_fsr_upscale(C.byref(a), C.byref(a), rows, None) == ERR_FORMAT  # out must not alias the input
    assert lib.grb_fsr_sharpen(C.byref(a), C.byref(b), f(0.5), rows, None) == ERR_FORMAT  # sizes differ
    b2 = _image(capi, np.zeros((12, 12), np.uint32), capi.FORMAT_R8G8B8A8_SRGB)
    assert lib.grb_fsr_sharpen(C.byref(b), C.byref(b2), f(-1.0), rows, None) == ERR_ARG and "stops" in _msg(lib)
    assert lib.grb_fsr_sharpen(C.byref(b), C.byref(b2), f(float("nan")), rows, None) == ERR_ARG
    con = np.zeros(16, np.float32)
    assert lib.grb_fsr_easu_constants(0, 8, 12, 12, con.ctypes.data_as(C.c_void_p)) == ERR_ARG
    assert lib.grb_fsr_easu_constants(8, 8, 12, 12, None) == ERR_ARG
    assert lib.grb_fsr_easu_constants(8, 8, 12, 12, con.ctypes.data_as(C.c_void_p)) == OK and con[0] == np.float32(8.0) / np.float32(12.0)


def test_decal_binning_argument_checks(lib):
    from granite_b200 import capi

    p = capi.GrbClusterParameters()
    p.resolution_xy[0], p.resolution_xy[1] = 128, 64
    buf = np.zeros(64, np.float32)
    ptr = buf.ctypes.data_as(C.c_void_p)
    assert lib.grb_cluster_decal_binning(None, ptr, 1, ptr, ptr, None) == ERR_ARG
    assert lib.grb_cluster_decal_binning(C.byref(p), ptr, 4097, ptr, ptr, None) == ERR_ARG and "4096" in _msg(lib)
    assert lib.grb_cluster_decal_binning(C.byref(p), ptr, -1, ptr, ptr, None) == ERR_ARG
    assert lib.grb_cluster_decal_binning(C.byref(p), None, 3, ptr, ptr, None) == ERR_ARG
    assert lib.grb_cluster_decal_binning(C.byref(p), None, 0, None, None, None) == OK  # no decals: nothing to launch (clusterer.cpp:1394-1395)
    p.resolution_xy[0] = 0
    assert lib.grb_cluster_decal_binning(C.byref(p), ptr, 1, ptr, ptr, None) == ERR_ARG


def test_shadowed_and_fp16_lighting_argument_checks(lib):
    from granite_b200 import capi

    w, h = 16, 8
    g = capi.GrbGBuffer()
    keep = [np.zeros((h, w), np.uint32), np.zeros((h, w), np.uint32), np.zeros((h, w), np.uint16), np.zeros((h, w), np.float32)]
    g.albedo = _image(capi, keep[0], capi.FORMAT_R8G8B8A8_SRGB)
    g.normal = _image(capi, keep[1], capi.FORMAT_A2B10G10R10_UNORM)
    g.pbr = _image(capi, keep[2], capi.FORMAT_R8G8_UNORM)
    g.depth = _image(capi, keep[3], capi.FORMAT_D32_SFLOAT)
    cam, params, bufs = capi.GrbCamera(), capi.GrbClusterParameters(), capi.GrbClusterBuffers()
    params.num_lights = 4
    hdr = _image(capi, np.zeros((h, w), np.uint32), capi.FORMAT_B10G11R11_UFLOAT)
    rows = capi.GrbRows(0, 0)
    assert lib.grb_deferred_lighting_shadowed(C.byref(g), C.byref(cam), C.byref(params), C.byref(bufs), None, C.byref(hdr), rows, None) == ERR_ARG
    assert "shadows" in _msg(lib)
    sh = capi.GrbLightShadows(None, None, 512)
    assert lib.grb_deferred_lighting_shadowed(C.byref(g), C.byref(cam), C.byref(params), C.byref(bufs), C.byref(sh), C.byref(hdr), rows, None) == ERR_ARG
    t = np.zeros((4, 16), np.float32)
    table = np.zeros(4, np.uint64)
    sh = capi.GrbLightShadows(t.ctypes.data, table.ctypes.data, 0)
    assert lib.grb_deferred_lighting_shadowed(C.byref(g), C.byref(cam), C.byref(params), C.byref(bufs), C.byref(sh), C.byref(hdr), rows, None) == ERR_ARG
    # an HDR target that is neither B10G11R11 nor RGBA16F; an emissive image whose format differs from the target's
    bad = _image(capi, np.zeros((h, w), np.uint32), capi.FORMAT_R8G8B8A8_UNORM)
    assert lib.grb_deferred_lighting(C.byref(g), C.byref(cam), C.byref(params), C.byref(bufs), C.byref(bad), rows, None) == ERR_FORMAT
    hdr16 = _image(capi, np.zeros((h, w, 4), np.uint16), capi.FORMAT_R16G16B16A16_SFLOAT)
    g.emissive = _image(capi, np.zeros((h, w), np.uint32), capi.FORMAT_B10G11R11_UFLOAT)
    params.num_lights = 0
    dummy = np.zeros(16, np.uint32)
    bufs.cluster_range = dummy.ctypes.data  # never dereferenced on the host
    assert lib.grb_deferred_lighting(C.byref(g), C.byref(cam), C.byref(params), C.byref(bufs), C.byref(hdr16), rows, None) == ERR_FORMAT
    assert "emissive" in _msg(lib)


def test_post_passes_reject_unknown_hdr_formats(lib):
    from granite_b200 import capi

    w, h = 16, 8
    rows, f = capi.GrbRows(0, 0), C.c_float
    bad = _image(capi, np.zeros((h, w), np.uint32), capi.FORMAT_R8G8B8A8_UNORM)
    t = _image(capi, np.zeros((h // 2, w // 2, 4), np.uint16), capi.FORMAT_R16G16B16A16_SFLOAT)
    out = _image(capi, np.zeros((h, w), np.uint32), capi.FORMAT_R8G8B8A8_SRGB)
    assert lib.grb_bloom_threshold(C.byref(bad), None, C.byref(t), rows, None) == ERR_FORMAT
    assert lib.grb_tonemap(C.byref(bad), C.byref(t), None, f(1.0), C.byref(out), rows, None) == ERR_FORMAT
    oc = _image(capi, np.zeros((h, w), np.uint32), capi.FORMAT_B10G11R11_UFLOAT)
    oh = _image(capi, np.zeros((h, w, 4), np.uint16), capi.FORMAT_R16G16B16A16_SFLOAT)
    assert lib.grb_taa_resolve(C.byref(bad), None, None, None, None, 2, C.byref(oc), C.byref(oh), rows, None) == ERR_FORMAT
    hdr16 = _image(capi, np.zeros((h, w, 4), np.uint16), capi.FORMAT_R16G16B16A16_SFLOAT)
    assert lib.grb_taa_resolve(C.byref(hdr16), None, None, None, None, 3, C.byref(oc), C.byref(oh), rows, None) == ERR_ARG  # quality 0..2


def test_fog_accumulate_argument_checks(lib):
    a, b = np.zeros(64, np.uint16), np.zeros(64, np.uint16)
    pa, pb = a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p)
    assert lib.grb_fog_accumulate(None, 2, 2, 2, pb, None) == ERR_ARG
    assert lib.grb_fog_accumulate(pa, 0, 2, 2, pb, None) == ERR_ARG
    assert lib.grb_fog_accumulate(pa, 2, 2, 2, pa, None) == ERR_ARG and "distinct" in _msg(lib)
    assert lib.grb_fog_accumulate(C.c_void_p(a.ctypes.data + 2), 2, 2, 2, pb, None) == ERR_ARG  # misaligned


def test_fog_light_density_argument_checks(lib):
    from granite_b200 import capi

    g = capi.GrbFogParameters(8, 4, 4, 0, 0.157, 0.5, 1.0)
    cam, params, bufs = capi.GrbCamera(), capi.GrbClusterParameters(), capi.GrbClusterBuffers()
    m, v3, buf = np.zeros(16, np.float32), np.zeros(3, np.float32), np.zeros(1024, np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    args = lambda fog, out: (C.byref(fog), C.byref(cam), p(m), p(m), C.byref(params), C.byref(bufs), p(v3), p(v3), p(m), p(buf), out, None)  # noqa: E731
    assert lib.grb_fog_light_density(*args(g, None)) == ERR_ARG
    assert lib.grb_fog_light_density(*args(g, p(buf))) == ERR_ARG and "cluster" in _msg(lib)  # cluster_range is null
    bad = capi.GrbFogParameters(8, 4, 0, 0, 0.157, 0.5, 1.0)
    assert lib.grb_fog_light_density(*args(bad, p(buf))) == ERR_ARG
    bad = capi.GrbFogParameters(8, 4, 4, -1, 0.157, 0.5, 1.0)
    assert lib.grb_fog_light_density(*args(bad, p(buf))) == ERR_ARG
    bad = capi.GrbFogParameters(8, 4, 4, 0, 0.0, 0.5, 1.0)
    assert lib.grb_fog_light_density(*args(bad, p(buf))) == ERR_ARG


def test_bloom_to_peers_argument_checks(lib):
    """Both bloom d0 exchanges refuse a flag_index outside 0..peer_count-1 (word peer_count onwards of a flag array may
    hold the scratch counter), a null peer pointer and a peer_count outside 1..GRB_MAX_PEERS, and write nothing."""
    from granite_b200 import capi

    keep = [np.zeros((16, 32), np.uint32), np.zeros((8, 16, 4), np.uint16)] + [np.zeros((4, 8, 4), np.uint16) for _ in range(8)] + \
           [np.zeros(16, np.uint32) for _ in range(8)]
    hdr = _image(capi, keep[0], capi.FORMAT_B10G11R11_UFLOAT)
    t = _image(capi, keep[1], capi.FORMAT_R16G16B16A16_SFLOAT)
    d0 = capi.GrbImage(None, 8, 4, 8 * 8, capi.FORMAT_R16G16B16A16_SFLOAT)
    images = (C.c_void_p * 8)(*[a.ctypes.data for a in keep[2:10]])
    flags = (C.c_void_p * 8)(*[a.ctypes.data for a in keep[10:]])
    counter = C.c_void_p(keep[10].ctypes.data + 32)

    def head(im=images, fl=flags, n=2, k=0):
        return lib.grb_bloom_threshold_downsample_to_peers(C.byref(hdr), None, C.byref(d0), im, fl, n, k, C.c_uint32(1), counter, capi.GrbRows(0, 4), None)

    def down(im=images, fl=flags, n=2, k=0):
        return lib.grb_bloom_downsample_to_peers(C.byref(t), C.byref(d0), im, fl, n, k, C.c_uint32(1), counter, capi.GrbRows(0, 4), None)

    null_image = (C.c_void_p * 8)(keep[2].ctypes.data, None)
    null_flags = (C.c_void_p * 8)(None, keep[11].ctypes.data)
    for call, name in ((head, "grb_bloom_threshold_downsample_to_peers"), (down, "grb_bloom_downsample_to_peers")):
        assert call(k=2) == ERR_ARG and name in _msg(lib) and "flag_index" in _msg(lib)
        assert call(n=8, k=8) == ERR_ARG
        assert call(k=-1) == ERR_ARG
        assert call(im=null_image) == ERR_ARG and "null peer" in _msg(lib)
        assert call(fl=null_flags) == ERR_ARG and "null peer" in _msg(lib)
        assert call(im=None) == ERR_ARG
        assert call(n=0) == ERR_ARG and "peer_count" in _msg(lib)
        assert call(n=9) == ERR_ARG and "peer_count" in _msg(lib)
    assert all(a.sum() == 0 for a in keep[2:])


def test_peer_publish_argument_checks(lib):
    """grb_peer_publish (the flags-only publish of a receiving rank's credit) refuses null flag arrays, a null flag array
    among them, a null counter, a peer_count of 0 or GRB_MAX_PEERS + 1 (9) and a flag_index of -1 or peer_count, each
    before any CUDA call, with its message, and writes nothing."""
    keep = [np.zeros(16, np.uint32) for _ in range(9)]
    flags = (C.c_void_p * 9)(*[a.ctypes.data for a in keep])
    counter = C.c_void_p(keep[0].ctypes.data + 32)

    def call(fl=flags, n=2, k=0, ctr=counter):
        return lib.grb_peer_publish(fl, n, k, C.c_uint32(1), ctr, None)

    peers = "grb_peer_publish: null pointer, peer_count outside 1..GRB_MAX_PEERS or flag_index outside 0..peer_count-1"
    for bad in (dict(fl=None), dict(ctr=None), dict(n=0), dict(n=9), dict(k=-1), dict(k=2), dict(n=8, k=8)):
        assert call(**bad) == ERR_ARG and peers in _msg(lib), bad
    assert call(fl=(C.c_void_p * 2)(keep[0].ctypes.data, None)) == ERR_ARG and "grb_peer_publish: null peer flag array" in _msg(lib)
    assert not any(a.any() for a in keep), "a refused call wrote something"


def test_lighting_rejects_misaligned_lights(lib):
    """Every lighting form reads the light records as float4, so a light table that is not 16-byte aligned is refused
    before any CUDA call, by the lighting pass and by its row-cost estimate."""
    from granite_b200 import capi

    w, h = 16, 8
    g = capi.GrbGBuffer()
    keep = [np.zeros((h, w), np.uint32), np.zeros((h, w), np.uint32), np.zeros((h, w), np.uint16), np.zeros((h, w), np.float32)]
    g.albedo = _image(capi, keep[0], capi.FORMAT_R8G8B8A8_SRGB)
    g.normal = _image(capi, keep[1], capi.FORMAT_A2B10G10R10_UNORM)
    g.pbr = _image(capi, keep[2], capi.FORMAT_R8G8_UNORM)
    g.depth = _image(capi, keep[3], capi.FORMAT_D32_SFLOAT)
    hdr = _image(capi, np.zeros((h, w), np.uint32), capi.FORMAT_B10G11R11_UFLOAT)
    cam, params, bufs = capi.GrbCamera(), capi.GrbClusterParameters(), capi.GrbClusterBuffers()
    params.num_lights, params.num_lights_32 = 4, 1
    table = np.zeros(64, np.uint32)
    base = (table.ctypes.data + 15) // 16 * 16
    bufs.type_mask = bufs.bitmask = bufs.cluster_range = base
    rows = capi.GrbRows(0, 0)
    cost = np.zeros(4, np.uint32)
    for off in (4, 8, 12):
        bufs.lights = base + off
        assert lib.grb_deferred_lighting(C.byref(g), C.byref(cam), C.byref(params), C.byref(bufs), C.byref(hdr), rows, None) == ERR_ARG
        assert "16-byte" in _msg(lib)
        assert lib.grb_deferred_lighting_blocks(C.byref(g), C.byref(cam), C.byref(params), C.byref(bufs), C.byref(hdr), rows, None) == ERR_ARG
        assert lib.grb_deferred_lighting_scheduled(C.byref(g), C.byref(cam), C.byref(params), C.byref(bufs), C.byref(hdr), rows, None, None) == ERR_ARG
        assert lib.grb_lighting_row_cost(C.byref(g.depth), C.byref(cam), C.byref(params), C.byref(bufs), rows,
                                         cost.ctypes.data_as(C.c_void_p), None) == ERR_ARG
        assert "16-byte" in _msg(lib)
    assert cost.sum() == 0
