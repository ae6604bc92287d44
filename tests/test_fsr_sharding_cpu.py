"""FSR 1 upscaling on row-sharded frames without a GPU: the C++ shard plan's FSR rows (granite_b200/host/shard_plan.cpp
through grbh_shard_plan_fsr) drive an emulated sharded chain of the CPU oracle -- the post-AA pass at the render size
(none, FXAA, or SMAA with the edge rows every rank produces pushed into the other ranks' windows), EASU on the plan's
EASU rows, RCAS on the band -- and the assembled display frame must equal the unsharded one bit for bit.  Each
emulated rank holds real tonemapped rows only where the plan says it computes them; every other row is junk.  Also:
a TAA chain driven by the same plan, the plan without upscale, the rows of the EASU window being needed, the refusal
of layouts in which a rank produces no render rows, and the argument checks of the new entry point."""
import os

import numpy as np
import pytest

from tests import test_taa_sharding_cpu as taa_cpu
from tests.test_oracle_ref_smaa import smaa_test_image

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
WD, HD = 96, 512  # display size
SCALES = (0.5, 0.67, 0.75, 0.77)


@pytest.fixture(scope="module")
def viewer():
    from granite_b200 import build, viewer

    build.build_all()
    return viewer


@pytest.fixture(scope="module")
def luts():
    f = np.load(os.path.join(GOLDEN, "refsmaa_160x96.npz"))
    return np.ascontiguousarray(f["area"]), np.ascontiguousarray(f["search"])


def post_aa_modes(viewer):
    return [("none", viewer.AA_NONE), ("FXAA", viewer.AA_FXAA)] + [(f"SMAA {q}", viewer.AA_SMAA_LOW + q) for q in range(4)]


def render_size(w, h, scale):
    """The viewer's render size: ceil(scale * size), computed in fp32."""
    return (max(int(np.ceil(np.float32(scale) * np.float32(w))), 1), max(int(np.ceil(np.float32(scale) * np.float32(h))), 1))


def partitions(viewer, world, h):
    """Equal 64-row bands, and narrow 8-row-aligned bands of 16 .. 40 rows (a window then spans several ranks; 8-row
    bands would leave a rank without render rows at scale 0.5)."""
    rng = np.random.default_rng(world)
    cuts = np.cumsum(rng.choice([16, 24, 40], size=world - 1))
    narrow = [(int(a), int(b)) for a, b in zip([0, *cuts], [*cuts, h])]
    return {"equal": viewer.band_partition(h, world), "narrow": narrow}


def smaa_quality(viewer, aa):
    return aa - viewer.AA_SMAA_LOW if viewer.AA_SMAA_LOW <= aa <= viewer.AA_SMAA_ULTRA else None


def unsharded(oracle, viewer, img, display, aa, rcas, luts):
    q = smaa_quality(viewer, aa)
    if aa == viewer.AA_FXAA:
        img = oracle.fxaa(img)
    elif q is not None:
        img = oracle.smaa_blend(img, oracle.smaa_weights(oracle.smaa_edge(img, q), *luts, q))
    up = oracle.fsr_upscale(img, display, target_srgb=not rcas)
    return oracle.fsr_sharpen(up, 0.5, srgb=True) if rcas else up


def sharded(oracle, viewer, img, display, aa, rcas, bands, luts, window_cut=(0, 0)):
    """The chain every rank runs, on the CPU oracle; returns the display frame assembled from every rank's band.
    window_cut: rows of the final render-resolution image taken off the top / bottom of every rank's EASU window."""
    hr, wr = img.shape
    wd, hd = display
    q = smaa_quality(viewer, aa)
    rng = np.random.default_rng(aa + 10 * rcas)
    plans = [viewer.shard_plan_fsr(wd, hd, wr, hr, bands, r, aa, rcas) for r in range(len(bands))]

    def junk(shape, dtype=np.uint32):
        return rng.integers(0, np.iinfo(dtype).max, shape, dtype=dtype, endpoint=True)

    cols = []
    for p in plans:  # the tonemap output: real on the plan's tonemap rows only
        col = junk(img.shape)
        t0, t1 = p["tonemap"]
        col[t0:t1] = img[t0:t1]
        cols.append(col)
    if q is not None:  # every rank detects edges on the render rows it produces
        produced = [oracle.smaa_edge(col, q, rows=p["smaa_edges"]) for p, col in zip(plans, cols)]
    out = np.zeros((hd, wd), np.uint32)
    for p, col in zip(plans, cols):
        f0, f1 = p["easu_window"]
        if aa == viewer.AA_NONE:
            fin = col
        elif aa == viewer.AA_FXAA:
            fin = oracle.fxaa(col, rows=p["fxaa"])
        else:
            edges = junk((hr, wr, 2), np.uint8)
            win0, win1 = p["smaa_edge_window"]
            for other, e in zip(plans, produced):  # the rows the producers push into this rank's window
                y0, y1 = max(other["smaa_edges"][0], win0), min(other["smaa_edges"][1], win1)
                if y1 > y0:
                    edges[y0:y1] = e[y0:y1]
            wgt = junk((hr, wr))
            w0, w1 = p["smaa_weights"]
            wgt[w0:w1] = oracle.smaa_weights(edges, *luts, q, rows=(w0, w1))[w0:w1]
            fin = oracle.smaa_blend(col, wgt, rows=(f0, f1))
        final = junk((hr, wr))
        f0, f1 = f0 + window_cut[0], f1 - window_cut[1]
        final[f0:f1] = fin[f0:f1]
        e0, e1 = p["easu"]
        up = oracle.fsr_upscale(final, display, target_srgb=not rcas, rows=(e0, e1))
        if rcas:
            upscaled = junk((hd, wd))
            upscaled[e0:e1] = up[e0:e1]
            up = oracle.fsr_sharpen(upscaled, 0.5, srgb=True, rows=p["own"])
        b0, b1 = p["own"]
        out[b0:b1] = up[b0:b1]
    return out


def check_chain(oracle, viewer, luts, hd, bands, label):
    for scale in SCALES:
        wr, hr = render_size(WD, hd, scale)
        img = smaa_test_image(wr, hr, len(bands))
        for name, aa in post_aa_modes(viewer):
            for rcas in (True, False):
                ref = unsharded(oracle, viewer, img, (WD, hd), aa, rcas, luts)
                out = sharded(oracle, viewer, img, (WD, hd), aa, rcas, bands, luts)
                assert np.array_equal(out, ref), f"{label}, scale {scale}, {name}, RCAS {rcas}: sharded frame differs from the unsharded one"


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("layout", ["equal", "narrow"])
def test_sharded_fsr_equals_unsharded(oracle, viewer, luts, world, layout):
    check_chain(oracle, viewer, luts, HD, partitions(viewer, world, HD)[layout], f"{world} ranks, {layout} bands")


@pytest.mark.parametrize("layout", ["equal", "narrow"])
def test_sharded_fsr_display_height_not_a_multiple_of_8(oracle, viewer, luts, layout):
    hd = 500
    check_chain(oracle, viewer, luts, hd, partitions(viewer, 3, hd)[layout], f"height {hd}, {layout} bands")


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("layout", ["equal", "narrow"])
def test_fsr_plan_rows(viewer, world, layout):
    """The render rows the ranks produce tile the render image in 8-row units; the EASU rows are the band (+-1 with
    RCAS); the final render-resolution image, the tonemap and the TAA rows cover what their consumers read."""
    bands = partitions(viewer, world, HD)[layout]
    for scale in SCALES:
        wr, hr = render_size(WD, HD, scale)
        for _, aa in post_aa_modes(viewer) + [("TAA", viewer.AA_TAA_HIGH_PLUS_FXAA)]:
            for rcas in (True, False):
                plans = [viewer.shard_plan_fsr(WD, HD, wr, hr, bands, r, aa, rcas) for r in range(world)]
                cuts = [p["render_own"][0] for p in plans] + [hr]
                assert cuts[0] == 0 and all(a < b for a, b in zip(cuts, cuts[1:])) and all(c % 8 == 0 for c in cuts[:-1])
                assert [p["render_own"][1] for p in plans] == cuts[1:]
                for r, p in enumerate(plans):
                    b0, b1 = bands[r]
                    assert p["own"] == (b0, b1)
                    assert p["easu"] == ((max(b0 - 1, 0), min(b1 + 1, HD)) if rcas else (b0, b1))
                    assert cuts[r] == 8 * (b0 * hr // (8 * HD))
                    t0, t1 = p["tonemap"]
                    w0, w1 = p["easu_window"]
                    assert 0 <= t0 <= w0 < w1 <= t1 <= hr
                    x0, x1 = p["fxaa"]
                    assert x1 == w1 and x0 == w0 // 16 * 16  # FXAA's 16-row tiles start where they start unsharded
                    if aa == viewer.AA_FXAA:
                        assert (t0, t1) == (max(x0 - 6, 0), min(x1 + 6, hr))
                    assert p["taa"][0] <= min(t0, p["render_own"][0]) and max(t1, p["render_own"][1]) <= p["taa"][1]
                    if aa == viewer.AA_TAA_HIGH_PLUS_FXAA:
                        assert p["lighting"] == (max(p["taa"][0] - 1, 0), min(p["taa"][1] + 1, hr))


def test_sharded_taa_with_fsr(oracle, viewer):
    """TAA High + FXAA + FSR at scale 0.5 (render 48 x 512 for a 96 x 1024 display), 3 frames: every rank resolves
    its TAA rows from real data on its lighting rows only and from the history assembled from every rank's produced
    render rows of the last frame; the colour on its TAA rows and the assembled history equal the unsharded ones."""
    q, wd, hd = 2, 2 * taa_cpu.W, 2 * taa_cpu.H
    assert render_size(wd, hd, 0.5) == (taa_cpu.W, taa_cpu.H)
    ref_c, ref_h = taa_cpu.unsharded(oracle, q)
    for world in (2, 4, 8):
        for layout, bands in partitions(viewer, world, hd).items():
            plans = [viewer.shard_plan_fsr(wd, hd, taa_cpu.W, taa_cpu.H, bands, r, viewer.AA_TAA_HIGH_PLUS_FXAA, True) for r in range(world)]
            rng = np.random.default_rng(world)
            own_hist = None
            for f in range(taa_cpu.FRAMES):
                hdr, depth, mv, reproj = taa_cpu.frame_inputs(f)
                hists = []
                for r, p in enumerate(plans):
                    lit = p["lighting"]
                    hist = None
                    if own_hist is not None:
                        hist = rng.integers(0, 2**16, (taa_cpu.H, taa_cpu.W, 4), dtype=np.uint16)
                        for k, pk in enumerate(plans):
                            y0, y1 = pk["render_own"]
                            hist[y0:y1] = own_hist[k][y0:y1]
                    c, h = oracle.taa_resolve(taa_cpu.junk_except(hdr, lit, rng), taa_cpu.junk_except(depth, lit, rng),
                                              taa_cpu.junk_except(mv.reshape(taa_cpu.H, taa_cpu.W, 2), lit, rng), hist, reproj, q, rows=p["taa"])
                    t0, t1 = p["taa"]
                    assert np.array_equal(c[t0:t1], ref_c[f][t0:t1]), f"{world} ranks, {layout}, frame {f}, rank {r}: colour differs"
                    hists.append(h)
                own_hist = hists
                assembled = np.zeros_like(ref_h[f])
                for p, h in zip(plans, own_hist):
                    y0, y1 = p["render_own"]
                    assembled[y0:y1] = h[y0:y1]
                assert np.array_equal(assembled, ref_h[f]), f"{world} ranks, {layout}, frame {f}: assembled history differs"


def test_no_upscale_is_the_existing_plan(viewer):
    """Render size = display size: the rows of grbh_shard_plan / _smaa / _taa, and the produced rows are the band."""
    for world in (2, 4, 8):
        for bands in partitions(viewer, world, HD).values():
            for r, band in enumerate(bands):
                for rcas in (True, False):
                    for fxaa in (False, True):
                        plain = viewer.shard_plan(WD, HD, bands, r, fxaa)
                        p = viewer.shard_plan_fsr(WD, HD, WD, HD, bands, r, viewer.AA_FXAA if fxaa else viewer.AA_NONE, rcas)
                        assert p["own"] == p["easu"] == p["easu_window"] == p["render_own"] == tuple(band)
                        assert (p["tonemap"], p["taa"], p["lighting"]) == (plain["tonemap"], plain["lighting"], plain["lighting"])
                        taa = viewer.shard_plan_taa(WD, HD, bands, r, fxaa)
                        p = viewer.shard_plan_fsr(WD, HD, WD, HD, bands, r, viewer.AA_TAA_HIGH_PLUS_FXAA if fxaa else viewer.AA_TAA_LOW, rcas)
                        assert (p["render_own"], p["taa"], p["lighting"]) == (taa["own"], taa["taa"], taa["lighting"])
                    for q in range(4):
                        smaa = viewer.shard_plan_smaa(WD, HD, bands, r, q)
                        p = viewer.shard_plan_fsr(WD, HD, WD, HD, bands, r, viewer.AA_SMAA_LOW + q, rcas)
                        assert p["render_own"] == tuple(band)
                        assert (p["smaa_blend"], p["smaa_weights"], p["smaa_edges"], p["smaa_edge_window"], p["tonemap"], p["lighting"]) == \
                            (smaa["blend"], smaa["weights"], smaa["edges"], smaa["edge_window"], smaa["tonemap"], smaa["lighting"])
    assert all(v == (0, HD) for v in viewer.shard_plan_fsr(WD, HD, WD, HD, [], 0, viewer.AA_SMAA_HIGH, True).values())
    whole = viewer.shard_plan_fsr(WD, HD, 48, 256, [(0, HD)], 0, viewer.AA_FXAA, True)
    assert whole["own"] == whole["easu"] == (0, HD) and all(whole[k] == (0, 256) for k in list(whole)[2:])


def strips_image(w, h):
    """Two-row horizontal strips, alternately dark and bright, with a different colour in every strip: the content
    changes at every strip border."""
    rng = np.random.default_rng(7)
    img = np.zeros((h, w, 4), np.uint8)
    img[..., 3] = 255
    for y in range(0, h, 2):
        img[y:y + 2, :, :3] = rng.integers(0, 80, 3) + (160 if (y // 2) % 2 else 0)
    img[:, ::5, :3] = 128
    return np.ascontiguousarray(img).view(np.uint32).reshape(h, w)


def test_easu_window_is_needed(oracle, viewer, luts):
    """The EASU window has no spare row: without its first or its last row (junk there instead), some rank's band of
    the display frame changes on the strips image."""
    for cut in ((1, 0), (0, 1)):
        for rcas in (True, False):
            bitten = False
            for scale in (0.5, 0.67):
                wr, hr = render_size(WD, HD, scale)
                img = strips_image(wr, hr)
                ref = unsharded(oracle, viewer, img, (WD, HD), viewer.AA_NONE, rcas, luts)
                for world in (2, 4):
                    for bands in partitions(viewer, world, HD).values():
                        out = sharded(oracle, viewer, img, (WD, HD), viewer.AA_NONE, rcas, bands, luts, window_cut=cut)
                        bitten |= not np.array_equal(out, ref)
            assert bitten, f"taking {cut} rows (top, bottom) off the EASU window changed nothing (RCAS {rcas})"


def test_layout_without_render_rows_is_refused(viewer):
    """8-row display bands at scale 0.5 give a rank no 8-row unit of the render image: the plan and the viewer refuse
    the layout (no boundary is moved); the same layout without upscale, and wider bands with it, are accepted."""
    from granite_b200 import capi

    bands = [(0, 8), (8, 16), (16, HD)]
    wr, hr = render_size(WD, HD, 0.5)
    with pytest.raises(capi.GrbError, match="no render rows"):
        viewer.shard_plan_fsr(WD, HD, wr, hr, bands, 0)
    with pytest.raises(capi.GrbError, match="no render rows"):
        viewer.shard_plan_fsr(WD, HD, wr, hr, bands, 2, viewer.AA_SMAA_ULTRA, False)  # every rank refuses the layout
    v = viewer.Viewer(WD, HD, cuda_device=-1, resolution_scale=0.5)
    try:
        with pytest.raises(capi.GrbError, match="grbh_viewer_set_row_shards.*no render rows"):
            v.set_row_shards(bands, 0)
        v.set_row_shards([(0, 16), (16, 32), (32, HD)], 1)
    finally:
        v.close()
    v = viewer.Viewer(WD, HD, cuda_device=-1)
    try:
        v.set_row_shards(bands, 0)
    finally:
        v.close()


def test_shard_plan_fsr_argument_checks(viewer):
    from granite_b200 import capi

    L = viewer.lib()
    bands = (capi.GrbRows * 2)(capi.GrbRows(0, 64), capi.GrbRows(64, 128))
    out = (capi.GrbRows * 12)()

    def call(w=64, h=128, rw=32, rh=64, b=bands, n=2, r=0, aa=0, rcas=1, o=out):
        return L.grbh_shard_plan_fsr(w, h, rw, rh, b, n, r, aa, rcas, o)

    assert call(r=2) < 0 and b"grbh_shard_plan_fsr" in L.grbh_last_error()
    assert call(r=-1) < 0
    assert call(o=None) < 0
    assert call(b=None) < 0
    assert call(n=-1) < 0
    assert call(w=0) < 0
    assert call(h=0) < 0
    assert call(rw=0) < 0
    assert call(rh=0) < 0
    assert call(rw=65) < 0
    assert call(rh=129) < 0
    for aa in (2, 7, 11, 99, 101, -1):
        assert call(aa=aa) < 0, f"post_aa {aa}"
    for aa in (0, 1, 3, 4, 5, 6, 8, 9, 10, 100):
        assert call(aa=aa) == 0, f"post_aa {aa}"
    assert call(r=1) == 0 and (out[0].y0, out[0].y1) == (64, 128) and (out[3].y0, out[3].y1) == (32, 64)
    assert call(b=None, n=0, r=5) == 0 and (out[2].y0, out[2].y1) == (0, 64)
