"""Presenting row-sharded frames from one rank, without a GPU: the argument checks of grb_present_rows_to_peer (every
check comes before any CUDA call, so host pointers stand in for device memory), and the host-only checks of
grbh_viewer_set_present_rank and of grbh_viewer_set_row_shards against the presenting rank."""
import ctypes as C

import numpy as np
import pytest

OK, ERR_ARG = 0, -1


@pytest.fixture(scope="module")
def viewer():
    from granite_b200 import build, viewer

    build.build_all()
    return viewer


def test_present_rows_to_peer_argument_checks(viewer):
    from granite_b200 import capi

    L = C.CDLL(capi.LIB_PATH)
    L.grb_last_error_string.restype = C.c_char_p
    w, h = 32, 16
    keep = [np.zeros((h, w), np.uint32), np.zeros((h, w), np.uint32), np.zeros(16, np.uint32), np.zeros(16, np.uint32)]
    src = capi.GrbImage(keep[0].ctypes.data, w, h, w * 4, capi.FORMAT_R8G8B8A8_SRGB)
    dst = C.c_void_p(keep[1].ctypes.data)
    flags = (C.c_void_p * 2)(keep[2].ctypes.data, keep[3].ctypes.data)
    counter = C.c_void_p(keep[2].ctypes.data + 32)

    def call(s=C.byref(src), d=dst, fl=flags, n=2, k=0, ctr=counter, own=(0, 8)):
        return L.grb_present_rows_to_peer(s, d, fl, n, k, C.c_uint32(1), ctr, capi.GrbRows(*own), None)

    def msg():
        return (L.grb_last_error_string() or b"").decode()

    def image(fmt=capi.FORMAT_R8G8B8A8_SRGB, data=keep[0].ctypes.data, width=w, height=h, pitch=w * 4):
        return C.byref(capi.GrbImage(data, width, height, pitch, fmt))

    # null pointers
    assert call(s=None) == ERR_ARG and "grb_present_rows_to_peer" in msg()
    assert call(s=image(data=None)) == ERR_ARG
    assert call(d=None) == ERR_ARG
    assert call(fl=None) == ERR_ARG
    assert call(ctr=None) == ERR_ARG
    assert call(fl=(C.c_void_p * 2)(keep[2].ctypes.data, None)) == ERR_ARG and "null peer flag" in msg()
    # peer_count and flag_index
    assert call(n=0) == ERR_ARG and "peer_count" in msg()
    assert call(n=9) == ERR_ARG
    assert call(k=2) == ERR_ARG and "flag_index" in msg()
    assert call(k=-1) == ERR_ARG
    # own rows: empty, or outside the image
    assert call(own=(0, 0)) == ERR_ARG and "own rows" in msg()
    assert call(own=(8, 8)) == ERR_ARG
    assert call(own=(6, 4)) == ERR_ARG
    assert call(own=(-1, 4)) == ERR_ARG
    assert call(own=(8, h + 1)) == ERR_ARG
    # texel size other than 4 bytes, and bad geometry
    for fmt in (capi.FORMAT_R16G16B16A16_SFLOAT, capi.FORMAT_R8G8_UNORM, capi.FORMAT_R8_UNORM, 12345):
        assert call(s=image(fmt=fmt)) == ERR_ARG and "4-byte texels" in msg()
    assert call(s=image(pitch=w * 4 - 4)) == ERR_ARG
    assert call(s=image(width=0)) == ERR_ARG
    assert call(s=image(height=0)) == ERR_ARG
    # dst equal to the source
    assert call(d=C.c_void_p(keep[0].ctypes.data)) == ERR_ARG and "distinct" in msg()
    # no refused call wrote anything
    assert keep[1].sum() == 0 and keep[2].sum() == 0 and keep[3].sum() == 0


def test_set_present_rank_range(viewer):
    v = viewer.Viewer(64, 128, cuda_device=-1)
    try:
        v.set_present_rank(0)  # unsharded: one band, and 0 changes nothing
        v.set_present_rank(-1)
        for bad in (1, -2):
            with pytest.raises(Exception, match="grbh_viewer_set_present_rank"):
                v.set_present_rank(bad)
        v.set_row_shards([(0, 32), (32, 64), (64, 128)], 1)
        for r in (-1, 0, 1, 2):
            v.set_present_rank(r)
        for bad in (3, 4, -2, -100):
            with pytest.raises(Exception, match=r"within \[0, 3\)"):
                v.set_present_rank(bad)
    finally:
        v.close()


def test_set_row_shards_keeps_a_band_for_the_presenting_rank(viewer):
    v = viewer.Viewer(64, 128, cuda_device=-1)
    try:
        v.set_row_shards([(0, 32), (32, 64), (64, 96), (96, 128)], 0)
        v.set_present_rank(3)
        with pytest.raises(Exception, match="presenting rank 3 would have no band"):
            v.set_row_shards([(0, 64), (64, 128)], 0)
        with pytest.raises(Exception, match="presenting rank 3"):
            v.set_row_shards([], 0)
        v.set_row_shards([(0, 16), (16, 32), (32, 64), (64, 100), (100, 128)], 4)  # still has a band
        v.set_present_rank(-1)
        v.set_row_shards([(0, 64), (64, 128)], 1)
        v.set_present_rank(0)
        v.set_row_shards([], 0)  # rank 0 always has a band
    finally:
        v.close()
