"""Moving the band cuts of a row-sharded viewer, without a GPU: every refusal of grbh_viewer_move_row_shards that needs no
device is reached on a host-only viewer (cuda_device = -1) after set_row_shards, before the "not baked" check, and a
refused layout changes nothing (the same layout still reaches "not baked" afterwards)."""
import ctypes as C

import pytest


@pytest.fixture(scope="module")
def viewer():
    from granite_b200 import build, viewer

    build.build_all()
    return viewer


def _rows(bands):
    from granite_b200 import capi

    return (capi.GrbRows * max(len(bands), 1))(*[capi.GrbRows(a, b) for a, b in bands])


def test_move_refuses_an_unsharded_viewer(viewer):
    v = viewer.Viewer(64, 128, cuda_device=-1)
    try:
        with pytest.raises(Exception, match="not row-sharded"):
            v.move_row_shards([(0, 64), (64, 128)])
        v.set_row_shards([(0, 128)], 0)  # one band is not a sharded frame either
        with pytest.raises(Exception, match="not row-sharded"):
            v.move_row_shards([(0, 128)])
    finally:
        v.close()


def test_move_refuses_another_band_count(viewer):
    v = viewer.Viewer(64, 128, cuda_device=-1)
    try:
        v.set_row_shards([(0, 32), (32, 64), (64, 128)], 1)
        for bands in ([(0, 64), (64, 128)], [(0, 32), (32, 64), (64, 96), (96, 128)]):
            with pytest.raises(Exception, match=f"{len(bands)} bands for a viewer of 3"):
                v.move_row_shards(bands)
    finally:
        v.close()


def test_move_refuses_bands_that_do_not_tile_the_frame(viewer):
    v = viewer.Viewer(64, 128, cuda_device=-1)
    try:
        v.set_row_shards([(0, 32), (32, 64), (64, 128)], 0)
        for bands in ([(8, 32), (32, 64), (64, 128)],     # does not start at 0
                      [(0, 32), (40, 64), (64, 128)],     # gap
                      [(0, 40), (32, 64), (64, 128)],     # overlap
                      [(0, 32), (32, 32), (32, 128)],     # empty band
                      [(64, 128), (0, 32), (32, 64)]):    # out of order
            with pytest.raises(Exception, match="tile the frame in order"):
                v.move_row_shards(bands)
        for bands in ([(0, 32), (32, 64), (64, 120)], [(0, 32), (32, 64), (64, 136)]):
            with pytest.raises(Exception, match=r"cover rows \[0, 128\)"):
                v.move_row_shards(bands)
    finally:
        v.close()


def test_move_refuses_an_fsr_layout_without_render_rows(viewer):
    """At FSR 0.5, 8-row display bands put two cuts into one 8-row unit of the render image: a rank would produce no
    render rows, as grbh_viewer_set_row_shards refuses too."""
    v = viewer.Viewer(64, 128, cuda_device=-1, resolution_scale=0.5)
    try:
        v.set_row_shards([(0, 32), (32, 64), (64, 96), (96, 128)], 2)
        with pytest.raises(Exception, match="produces no render rows"):
            v.move_row_shards([(0, 8), (8, 16), (16, 24), (24, 128)])
        with pytest.raises(Exception, match="not baked"):  # a layout with render rows for every rank gets further
            v.move_row_shards([(0, 16), (16, 48), (48, 96), (96, 128)])
    finally:
        v.close()


def test_move_refuses_null_arguments(viewer):
    v = viewer.Viewer(64, 128, cuda_device=-1)
    try:
        v.set_row_shards([(0, 64), (64, 128)], 0)
        L = viewer.lib()
        good = _rows([(0, 64), (64, 128)])
        for args in ((None, good, 2), (v._h, None, 2), (v._h, good, 0), (v._h, good, C.c_int32(-1))):
            assert L.grbh_viewer_move_row_shards(*args) < 0
            assert "grbh_viewer_move_row_shards: bad arguments" in L.grbh_last_error().decode()
    finally:
        v.close()


def test_move_of_a_valid_layout_needs_a_baked_viewer(viewer):
    v = viewer.Viewer(64, 128, cuda_device=-1)
    try:
        v.set_row_shards([(0, 32), (32, 64), (64, 96), (96, 128)], 3)
        v.set_present_rank(3)
        for bands in ([(0, 48), (48, 64), (64, 112), (112, 128)], [(0, 32), (32, 64), (64, 96), (96, 128)]):
            with pytest.raises(Exception, match="viewer not baked"):
                v.move_row_shards(bands)
        # a refused layout left the viewer as it was: the 4-band layout of set_row_shards still stands
        with pytest.raises(Exception, match="tile the frame"):
            v.move_row_shards([(0, 48), (40, 64), (64, 112), (112, 128)])
        with pytest.raises(Exception, match="viewer not baked"):
            v.move_row_shards([(0, 16), (16, 32), (32, 48), (48, 128)])
    finally:
        v.close()
