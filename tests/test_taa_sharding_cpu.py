"""TAA on row-sharded frames without a GPU: the C++ shard plan's TAA rows (granite_b200/host/shard_plan.cpp through
grbh_shard_plan_taa) drive an emulated sharded chain of the CPU oracle's TAA resolve over several frames, and the
assembled colour and history must equal the unsharded ones bit for bit.  Each emulated rank has real HDR, depth and
motion vectors only on its lighting rows (junk elsewhere), resolves its TAA rows, and reads a history assembled from
every rank's own rows of the previous frame -- what the peer stores (grb_taa_resolve_to_peers) or the all-gather
deliver.  The motion vectors send a share of the pixels up to half the image height away, so most ranks read history
rows that other ranks produced.  Also: the argument checks of the new entry points."""
import ctypes as C

import numpy as np
import pytest

from tests import common

W, H = 48, 512
FRAMES = 3
OK, ERR_ARG, ERR_FORMAT = 0, -1, -2


@pytest.fixture(scope="module")
def viewer():
    from granite_b200 import build, viewer

    build.build_all()
    return viewer


def partitions(world):
    """Equal 64-row bands, and narrow 8-row-aligned bands."""
    from granite_b200 import viewer

    rng = np.random.default_rng(world)
    cuts = np.cumsum(rng.choice([8, 16, 24, 40], size=world - 1))
    narrow = [(int(a), int(b)) for a, b in zip([0, *cuts], [*cuts, H])]
    return {"equal": viewer.band_partition(H, world), "narrow": narrow}


def frame_inputs(frame):
    """HDR, depth, mv and reprojection of one frame.  The camera moves every frame (the reprojection's translation
    changes); 15 % of the pixels have a motion vector of up to half the image height (and a few columns), the rest
    zero, which takes the reprojection path."""
    rng = np.random.default_rng(100 + frame)
    hdr = common.random_hdr(rng, W, H, scale=2.0)
    depth = rng.uniform(0.0005, 0.03, (H, W)).astype(np.float32)
    depth[rng.random((H, W)) < 0.1] = 0.0
    mv = np.zeros((H, W, 2), np.float16)
    moving = rng.random((H, W)) < 0.15
    n = int(moving.sum())
    mv[moving] = np.stack([rng.uniform(-4.0, 4.0, n) / W, rng.uniform(-0.5, 0.5, n)], -1).astype(np.float16)
    reproj = np.array([[0.5, 0, 0, 0], [0, 0.5, 0, 0], [0.3, -0.2, 1, 0],
                       [0.5 + (0.4 + 0.7 * frame) / W, 0.5 - (0.3 + 1.1 * frame) / H, 0, 1]], np.float32)
    return hdr, depth, mv.view(np.uint16), reproj


def junk_except(real, rows, rng):
    """`real` on rows [y0, y1), random bits elsewhere (what a rank holds where nothing was uploaded or computed)."""
    out = rng.integers(0, 256, real.nbytes, dtype=np.uint8).view(real.dtype).reshape(real.shape)
    out[rows[0]:rows[1]] = real[rows[0]:rows[1]]
    return out


def unsharded(oracle, q):
    colours, histories, hist = [], [], None
    for f in range(FRAMES):
        hdr, depth, mv, reproj = frame_inputs(f)
        c, hist = oracle.taa_resolve(hdr, depth, mv, hist, reproj, q)
        colours.append(c)
        histories.append(hist)
    return colours, histories


def sharded(oracle, viewer, bands, q, fxaa=False, lighting_cut=(0, 0), history_window=None):
    """The chain every rank runs, frame by frame.  Returns per frame (colour assembled from every rank's TAA rows
    -- equal where they overlap, else None --, history assembled from every rank's own rows).
    lighting_cut: rows taken off the top / bottom of every rank's lighting rows.  history_window: deliver only the
    history rows within that many rows of a rank's own band (junk beyond)."""
    plans = [viewer.shard_plan_taa(W, H, bands, r, fxaa) for r in range(len(bands))]
    rng = np.random.default_rng(q)
    out, own_hist = [], None
    for f in range(FRAMES):
        hdr, depth, mv, reproj = frame_inputs(f)
        colour = np.zeros((H, W), np.uint32)
        written = np.zeros(H, bool)
        consistent = True
        next_hist = []
        for r, p in enumerate(plans):
            lit = (p["lighting"][0] + lighting_cut[0], p["lighting"][1] - lighting_cut[1])
            hist = None
            if own_hist is not None:
                hist = rng.integers(0, 2**16, (H, W, 4), dtype=np.uint16)
                lo, hi = (0, H) if history_window is None else (p["own"][0] - history_window, p["own"][1] + history_window)
                for k, pk in enumerate(plans):  # the rows each rank produced last frame land in this rank's copy
                    y0, y1 = max(pk["own"][0], lo), min(pk["own"][1], hi)
                    if y1 > y0:
                        hist[y0:y1] = own_hist[k][y0:y1]
            c, h = oracle.taa_resolve(junk_except(hdr, lit, rng), junk_except(depth, lit, rng), junk_except(mv.reshape(H, W, 2), lit, rng),
                                      hist, reproj, q, rows=p["taa"])
            t0, t1 = p["taa"]
            consistent &= bool(np.array_equal(colour[t0:t1][written[t0:t1]], c[t0:t1][written[t0:t1]]))
            colour[t0:t1] = c[t0:t1]
            written[t0:t1] = True
            next_hist.append(h)
        own_hist = next_hist
        assembled = np.zeros((H, W, 4), np.uint16)
        for p, h in zip(plans, own_hist):
            assembled[p["own"][0]:p["own"][1]] = h[p["own"][0]:p["own"][1]]
        out.append((colour if consistent and written.all() else None, assembled))
    return out


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("layout", ["equal", "narrow"])
@pytest.mark.parametrize("fxaa", [False, True])
def test_taa_plan(viewer, world, layout, fxaa):
    """The TAA rows are the lighting rows of the plan without TAA; the lighting rows are the TAA rows +- 1, clamped;
    the history rows a rank produces are its own rows, so the ranks' history rows tile the image."""
    bands = partitions(world)[layout]
    for r, band in enumerate(bands):
        plain = viewer.shard_plan(1280, H, bands, r, fxaa)
        p = viewer.shard_plan_taa(1280, H, bands, r, fxaa)
        assert p["own"] == tuple(band) == plain["own"]
        assert p["taa"] == plain["lighting"]
        assert p["lighting"] == (max(p["taa"][0] - 1, 0), min(p["taa"][1] + 1, H))
    assert all(v == (0, H) for v in viewer.shard_plan_taa(1280, H, [], 0, fxaa).values())
    assert all(v == (0, H) for v in viewer.shard_plan_taa(1280, H, [(0, H)], 0, fxaa).values())


def test_existing_plans_unchanged(viewer):
    """grbh_shard_plan keeps its output: its lighting rows are what the TAA rows are now."""
    bands = viewer.band_partition(H, 4)
    for r in range(4):
        plain = viewer.shard_plan(1280, H, bands, r, True)
        assert plain["tonemap"] == (max(bands[r][0] - 6, 0), min(bands[r][1] + 6, H))
        assert plain["lighting"] == viewer.shard_plan_taa(1280, H, bands, r, True)["taa"]


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("layout", ["equal", "narrow"])
@pytest.mark.parametrize("fxaa", [False, True])
def test_sharded_taa_equals_unsharded(oracle, viewer, world, layout, fxaa):
    bands = partitions(world)[layout]
    for q in range(3):
        ref_c, ref_h = unsharded(oracle, q)
        for f, (colour, hist) in enumerate(sharded(oracle, viewer, bands, q, fxaa)):
            assert colour is not None, f"quality {q} frame {f}: ranks disagree on rows they both resolve"
            assert np.array_equal(colour, ref_c[f]), f"quality {q} frame {f}: sharded colour differs from the unsharded one"
            assert np.array_equal(hist, ref_h[f]), f"quality {q} frame {f}: assembled history differs from the unsharded one"


def test_motion_reaches_other_bands(viewer):
    """The inputs are a real test of the exchange: on every frame with history, pixels of every rank read history
    rows (at v - mv) that lie in another rank's band."""
    bands = partitions(4)["equal"]
    for f in range(1, FRAMES):
        _, _, mv, _ = frame_inputs(f)
        mvy = mv.reshape(H, W, 2).view(np.float16)[..., 1].astype(np.float32)
        ys = np.arange(H)[:, None] + 0.5 - mvy * H
        for y0, y1 in bands:
            src = ys[y0:y1][mvy[y0:y1] != 0]
            assert ((src < y0 - 2) | (src >= y1 + 2)).sum() > 100


def test_fewer_rows_change_the_frame(oracle, viewer):
    """The plan's rows are needed: one lighting row fewer at either end, or a history exchange limited to +-64 rows
    around each band, changes the colour or the history of some frame."""
    for q in (0, 2):
        ref_c, ref_h = unsharded(oracle, q)

        def differs(**kw):
            for layout in ("equal", "narrow"):
                for f, (colour, hist) in enumerate(sharded(oracle, viewer, partitions(4)[layout], q, **kw)):
                    if colour is None or not np.array_equal(colour, ref_c[f]) or not np.array_equal(hist, ref_h[f]):
                        return True
            return False

        assert differs(lighting_cut=(1, 0)), f"quality {q}: one lighting row fewer at the top changed nothing"
        assert differs(lighting_cut=(0, 1)), f"quality {q}: one lighting row fewer at the bottom changed nothing"
        assert differs(history_window=64), f"quality {q}: a +-64-row history exchange changed nothing"


def test_shard_plan_taa_argument_checks(viewer):
    from granite_b200 import capi

    L = viewer.lib()
    bands = (capi.GrbRows * 2)(capi.GrbRows(0, 64), capi.GrbRows(64, 128))
    out = (capi.GrbRows * 3)()
    assert L.grbh_shard_plan_taa(64, 128, bands, 2, 2, 0, out) < 0 and b"grbh_shard_plan_taa" in L.grbh_last_error()
    assert L.grbh_shard_plan_taa(64, 128, bands, 2, -1, 0, out) < 0
    assert L.grbh_shard_plan_taa(64, 128, bands, 2, 0, 0, None) < 0
    assert L.grbh_shard_plan_taa(0, 128, bands, 2, 0, 0, out) < 0
    assert L.grbh_shard_plan_taa(64, 0, bands, 2, 0, 0, out) < 0
    assert L.grbh_shard_plan_taa(64, 128, None, 2, 0, 0, out) < 0
    assert L.grbh_shard_plan_taa(64, 128, bands, 2, 1, 1, out) == 0 and (out[0].y0, out[0].y1) == (64, 128)


def test_taa_to_peers_argument_checks(viewer):
    """Every check comes before any CUDA call: host pointers stand in for device memory."""
    from granite_b200 import capi

    L = C.CDLL(capi.LIB_PATH)
    L.grb_last_error_string.restype = C.c_char_p
    w, h = 32, 16
    keep = [np.zeros((h, w), np.uint32) for _ in range(3)] + [np.zeros((h, w, 4), np.uint16) for _ in range(3)] + \
           [np.zeros((h, w), np.float32), np.zeros(16, np.uint32), np.zeros(16, np.uint32), np.eye(4, dtype=np.float32)]
    hdr = capi.GrbImage(keep[0].ctypes.data, w, h, w * 4, capi.FORMAT_B10G11R11_UFLOAT)
    mv = capi.GrbImage(keep[1].ctypes.data, w, h, w * 4, capi.FORMAT_R16G16_SFLOAT)
    oc = capi.GrbImage(keep[2].ctypes.data, w, h, w * 4, capi.FORMAT_B10G11R11_UFLOAT)
    hist = capi.GrbImage(keep[3].ctypes.data, w, h, w * 8, capi.FORMAT_R16G16B16A16_SFLOAT)
    layout = capi.GrbImage(None, w, h, w * 8, capi.FORMAT_R16G16B16A16_SFLOAT)
    depth = capi.GrbImage(keep[6].ctypes.data, w, h, w * 4, capi.FORMAT_D32_SFLOAT)
    images = (C.c_void_p * 2)(keep[4].ctypes.data, keep[5].ctypes.data)
    flags = (C.c_void_p * 2)(keep[7].ctypes.data, keep[8].ctypes.data)
    reproj = keep[9].ctypes.data_as(C.c_void_p)
    counter = C.c_void_p(keep[7].ctypes.data + 32)

    def call(hd=C.byref(hdr), dp=C.byref(depth), m=C.byref(mv), hs=C.byref(hist), rp=reproj, q=2, o=C.byref(oc), lay=C.byref(layout), im=images,
             fl=flags, n=2, k=0, ctr=counter, rows=(0, 8), own=(0, 8)):
        return L.grb_taa_resolve_to_peers(hd, dp, m, hs, rp, q, o, lay, im, fl, n, k, C.c_uint32(1), ctr, capi.GrbRows(*rows), capi.GrbRows(*own), None)

    def msg():
        return (L.grb_last_error_string() or b"").decode()

    assert call(hd=None) == ERR_FORMAT and "grb_taa_resolve_to_peers" in msg()
    assert call(o=None) == ERR_FORMAT
    assert call(lay=None) == ERR_FORMAT
    wrong = capi.GrbImage(None, w, h, w * 8, capi.FORMAT_B10G11R11_UFLOAT)
    assert call(lay=C.byref(wrong)) == ERR_FORMAT and "history layout" in msg()
    small = capi.GrbImage(None, w, h - 1, w * 8, capi.FORMAT_R16G16B16A16_SFLOAT)
    assert call(lay=C.byref(small)) == ERR_FORMAT
    narrow_pitch = capi.GrbImage(None, w, h, w * 8 - 8, capi.FORMAT_R16G16B16A16_SFLOAT)
    assert call(lay=C.byref(narrow_pitch)) == ERR_FORMAT
    assert call(o=C.byref(hist)) == ERR_FORMAT
    assert call(dp=None) == ERR_ARG and "depth" in msg()
    assert call(m=None) == ERR_ARG
    assert call(rp=None) == ERR_ARG
    assert call(hs=C.byref(capi.GrbImage(keep[3].ctypes.data, w, h, w * 4, capi.FORMAT_B10G11R11_UFLOAT))) == ERR_ARG
    assert call(q=3) == ERR_ARG and "quality" in msg()
    assert call(q=-1) == ERR_ARG
    assert call(im=None) == ERR_ARG and "peer_count" in msg()
    assert call(fl=None) == ERR_ARG
    assert call(ctr=None) == ERR_ARG
    assert call(n=0) == ERR_ARG and "peer_count" in msg()
    assert call(n=9) == ERR_ARG
    assert call(k=2) == ERR_ARG and "flag_index" in msg()
    assert call(k=-1) == ERR_ARG
    assert call(im=(C.c_void_p * 2)(keep[4].ctypes.data, None)) == ERR_ARG and "null peer" in msg()
    assert call(fl=(C.c_void_p * 2)(None, keep[8].ctypes.data)) == ERR_ARG
    assert call(im=(C.c_void_p * 2)(keep[4].ctypes.data, keep[3].ctypes.data)) == ERR_ARG and "distinct" in msg()
    assert call(own=(4, 12)) == ERR_ARG and "own rows" in msg()
    assert call(own=(-1, 4)) == ERR_ARG
    assert call(own=(6, 4)) == ERR_ARG
    assert call(rows=(0, 0), own=(8, 17)) == ERR_ARG
    assert call(rows=(4, 8), own=(0, 0)) == ERR_ARG  # {0, 0} = the whole image, which is not inside rows
