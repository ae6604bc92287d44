"""SMAA on row-sharded frames without a GPU: the C++ shard plan's SMAA rows (granite_b200/host/shard_plan.cpp through
grbh_shard_plan_smaa) drive an emulated sharded chain of the CPU oracle's SMAA passes, and the assembled frame must
equal the unsharded one bit for bit.  Each emulated rank sees real data only where the plan says it has some: its
colour on its tonemap rows, the edges other ranks push to it on its edge window, its own weights on its weight rows;
everything else is junk.  Also: the routing of edge rows between ranks, and the argument checks of the new entry
points."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.test_oracle_ref_smaa import smaa_test_image

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
H = 512
STEPS = (4, 8, 16, 32)
OK, ERR_ARG, ERR_FORMAT = 0, -1, -2


@pytest.fixture(scope="module")
def viewer():
    from granite_b200 import build, viewer

    build.build_all()
    return viewer


@pytest.fixture(scope="module")
def luts():
    f = np.load(os.path.join(GOLDEN, "refsmaa_160x96.npz"))
    return np.ascontiguousarray(f["area"]), np.ascontiguousarray(f["search"])


def partitions(world):
    """Equal 64-row bands, and narrow 8-row-aligned bands (a window then spans several ranks)."""
    from granite_b200 import viewer

    rng = np.random.default_rng(world)
    cuts = np.cumsum(rng.choice([8, 16, 24, 40], size=world - 1))
    narrow = [(int(a), int(b)) for a, b in zip([0, *cuts], [*cuts, H])]
    return {"equal": viewer.band_partition(H, world), "narrow": narrow}


def strips_image(bands):
    """3-px bright vertical strips on a dark background whose ends lie 1.. rows outside each band border: for every
    border B and distance d, one strip from inside the lower band up to B - d, one from inside the upper band down to
    B + d - 1.  Distances cover the first rows and every preset's search reach."""
    dists = sorted({1, 2, 3} | {2 * s + k for s in STEPS for k in range(-1, 7)})
    borders = [b[1] for b in bands[:-1]]
    w = 6 * 2 * len(dists) * len(borders)
    img = np.full((H, w, 4), 25, np.uint8)
    img[..., 3] = 255
    x = 0
    for b in borders:
        for d in dists:
            img[max(b - d, 0):min(b + 12, H), x:x + 3, :3] = 230
            img[max(b - 12, 0):min(b + d, H), x + 6:x + 9, :3] = 230
            x += 12
    return np.ascontiguousarray(img).view(np.uint32).reshape(H, w)


def sharded_smaa(oracle, viewer, img, area, search, q, bands, shrink=(0, 0)):
    """The chain every rank runs, on the CPU oracle.  Returns (assembled output, weights equal on every rank's weight
    rows).  shrink: rows taken off the top / bottom of every edge window (to show that the plan's window is needed)."""
    h, w = img.shape
    rng = np.random.default_rng(q)
    plans = [viewer.shard_plan_smaa(w, h, bands, r, q) for r in range(len(bands))]
    ref_w = oracle.smaa_weights(oracle.smaa_edge(img, q), area, search, q)
    produced = []
    for p in plans:
        col = rng.integers(0, 2**32, img.shape, dtype=np.uint32)  # colour rows this rank never tonemaps
        t0, t1 = p["tonemap"]
        col[t0:t1] = img[t0:t1]
        produced.append((col, oracle.smaa_edge(col, q, rows=p["edges"])))
    out = np.zeros_like(img)
    weights_ok = True
    for p, (col, _) in zip(plans, produced):
        edges = rng.integers(0, 256, (h, w, 2), dtype=np.uint8)
        win0, win1 = p["edge_window"][0] + shrink[0], p["edge_window"][1] - shrink[1]
        for other, (_, e) in zip(plans, produced):  # the rows the producers push into this rank's window
            y0, y1 = max(other["edges"][0], win0), min(other["edges"][1], win1)
            if y1 > y0:
                edges[y0:y1] = e[y0:y1]
        wgt = rng.integers(0, 2**32, (h, w), dtype=np.uint32)
        w0, w1 = p["weights"]
        wgt[w0:w1] = oracle.smaa_weights(edges, area, search, q, rows=p["weights"])[w0:w1]
        weights_ok &= bool(np.array_equal(wgt[w0:w1], ref_w[w0:w1]))
        b0, b1 = p["blend"]
        out[b0:b1] = oracle.smaa_blend(col, wgt, rows=p["blend"])[b0:b1]
    return out, weights_ok


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("layout", ["equal", "narrow"])
def test_sharded_smaa_equals_unsharded(oracle, viewer, luts, world, layout):
    area, search = luts
    bands = partitions(world)[layout]
    for name, img in (("test image", smaa_test_image(160, H, world)), ("strips", strips_image(bands))):
        for q in range(4):
            ref = oracle.smaa_blend(img, oracle.smaa_weights(oracle.smaa_edge(img, q), area, search, q))
            out, weights_ok = sharded_smaa(oracle, viewer, img, area, search, q, bands)
            assert weights_ok, f"{name}, preset {q}: weights differ on a rank's weight rows"
            assert np.array_equal(out, ref), f"{name}, preset {q}: sharded frame differs from the unsharded one"


def test_smaller_window_changes_the_frame(oracle, viewer, luts):
    """The plan's window is needed: without its last nominal row at either end (one row inside its rounding guard row,
    shard_plan.hpp), the Ultra weights on the strips image change for some rank."""
    area, search = luts
    for side in ((2, 0), (0, 2)):
        bitten = False
        for world in (2, 4, 8):
            for bands in partitions(world).values():
                img = strips_image(bands)
                ref = oracle.smaa_blend(img, oracle.smaa_weights(oracle.smaa_edge(img, 3), area, search, 3))
                out, weights_ok = sharded_smaa(oracle, viewer, img, area, search, 3, bands, shrink=side)
                bitten |= not weights_ok or not np.array_equal(out, ref)
        assert bitten, f"shrinking the edge window by {side} rows (top, bottom) changed nothing"


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_edge_rows_routing(viewer, world):
    """Every row of every rank's edge window is produced by exactly one rank, and the producer stores it to that rank
    (grb_smaa_edge_detection_to_peers: its own copy, and every rank whose window holds the row)."""
    for bands in partitions(world).values():
        for q in range(4):
            plans = [viewer.shard_plan_smaa(1280, H, bands, r, q) for r in range(world)]
            assert [p["edges"] for p in plans] == [tuple(b) for b in bands]
            for r, p in enumerate(plans):
                w0, w1 = p["edge_window"]
                assert 0 <= w0 <= p["weights"][0] and p["weights"][1] <= w1 <= H
                reach = 2 * STEPS[q]
                assert w0 == max(p["weights"][0] - reach - 2, 0) and w1 == min(p["weights"][1] + reach + 4, H)
                for y in range(w0, w1):
                    producers = [k for k, o in enumerate(plans) if o["edges"][0] <= y < o["edges"][1]]
                    assert len(producers) == 1
                    k = producers[0]
                    targets = [t for t, o in enumerate(plans) if t == k or o["edge_window"][0] <= y < o["edge_window"][1]]
                    assert r in targets


def test_unsharded_and_other_plans_unchanged(viewer):
    """One band: whole images.  Without SMAA the plan is what it was (the SMAA rows do not touch it)."""
    p = viewer.shard_plan_smaa(640, 360, [], 0, 3)
    assert all(v == (0, 360) for v in p.values())
    bands = viewer.band_partition(H, 4)
    for r in range(4):
        plain = viewer.shard_plan(1280, H, bands, r, False)
        assert plain["tonemap"] == plain["own"] == bands[r]
        smaa = viewer.shard_plan_smaa(1280, H, bands, r, 0)
        assert smaa["tonemap"] == (max(bands[r][0] - 3, 0), min(bands[r][1] + 2, H))
        assert smaa["lighting"][0] <= smaa["tonemap"][0] and smaa["tonemap"][1] <= smaa["lighting"][1]


def test_shard_plan_smaa_argument_checks(viewer):
    from granite_b200 import capi

    L = viewer.lib()
    bands = (capi.GrbRows * 2)(capi.GrbRows(0, 64), capi.GrbRows(64, 128))
    out = (capi.GrbRows * 6)()
    assert L.grbh_shard_plan_smaa(64, 128, bands, 2, 0, 4, out) < 0 and b"grbh_shard_plan_smaa" in L.grbh_last_error()
    assert L.grbh_shard_plan_smaa(64, 128, bands, 2, 2, 0, out) < 0
    assert L.grbh_shard_plan_smaa(64, 128, bands, 2, 0, 0, None) < 0
    assert L.grbh_shard_plan_smaa(0, 128, bands, 2, 0, 0, out) < 0
    assert L.grbh_shard_plan_smaa(64, 128, bands, 2, 1, 3, out) == 0 and (out[2].y0, out[2].y1) == (64, 128)


def test_edge_to_peers_argument_checks(viewer):
    """Every check comes before any CUDA call: host pointers stand in for device memory."""
    from granite_b200 import capi

    L = C.CDLL(capi.LIB_PATH)
    L.grb_last_error_string.restype = C.c_char_p
    w, h = 32, 16
    keep = [np.zeros((h, w), np.uint32), np.zeros((h, w, 2), np.uint8), np.zeros((h, w, 2), np.uint8), np.zeros(16, np.uint32), np.zeros(16, np.uint32)]
    color = capi.GrbImage(keep[0].ctypes.data, w, h, w * 4, capi.FORMAT_R8G8B8A8_UNORM)
    layout = capi.GrbImage(None, w, h, w * 2, capi.FORMAT_R8G8_UNORM)
    images = (C.c_void_p * 2)(keep[1].ctypes.data, keep[2].ctypes.data)
    flags = (C.c_void_p * 2)(keep[3].ctypes.data, keep[4].ctypes.data)
    wins = (capi.GrbRows * 2)(capi.GrbRows(0, 12), capi.GrbRows(4, 16))
    counter = C.c_void_p(keep[3].ctypes.data + 32)

    def call(col=C.byref(color), q=3, lay=C.byref(layout), im=images, fl=flags, wi=wins, n=2, k=0, ctr=counter):
        return L.grb_smaa_edge_detection_to_peers(col, q, lay, im, fl, wi, n, k, C.c_uint32(1), ctr, capi.GrbRows(0, 8), None)

    def msg():
        return (L.grb_last_error_string() or b"").decode()

    assert call(col=None) == ERR_ARG and "grb_smaa_edge_detection_to_peers" in msg()
    assert call(lay=None) == ERR_ARG
    assert call(im=None) == ERR_ARG
    assert call(fl=None) == ERR_ARG
    assert call(wi=None) == ERR_ARG
    assert call(ctr=None) == ERR_ARG
    assert call(n=0) == ERR_ARG and "peer_count" in msg()
    assert call(n=9) == ERR_ARG
    assert call(k=2) == ERR_ARG and "flag_index" in msg()
    assert call(k=-1) == ERR_ARG
    assert call(im=(C.c_void_p * 2)(keep[1].ctypes.data, None)) == ERR_ARG and "null peer" in msg()
    assert call(fl=(C.c_void_p * 2)(None, keep[4].ctypes.data)) == ERR_ARG
    assert call(wi=(capi.GrbRows * 2)(capi.GrbRows(0, 12), capi.GrbRows(4, 17))) == ERR_ARG and "window" in msg()
    assert call(wi=(capi.GrbRows * 2)(capi.GrbRows(-1, 12), capi.GrbRows(4, 16))) == ERR_ARG
    assert call(wi=(capi.GrbRows * 2)(capi.GrbRows(8, 4), capi.GrbRows(4, 16))) == ERR_ARG
    assert call(q=4) == ERR_FORMAT
    wrong = capi.GrbImage(None, w, h, w * 4, capi.FORMAT_R8G8B8A8_UNORM)
    assert call(lay=C.byref(wrong)) == ERR_FORMAT and "R8G8_UNORM" in msg()
    small = capi.GrbImage(None, w, h - 1, w * 2, capi.FORMAT_R8G8_UNORM)
    assert call(lay=C.byref(small)) == ERR_FORMAT
    hdr = capi.GrbImage(keep[0].ctypes.data, w, h, w * 4, capi.FORMAT_B10G11R11_UFLOAT)
    assert call(col=C.byref(hdr)) == ERR_FORMAT
