"""Lighting in stripes on row-sharded frames, without a GPU.  The stripe plan (granite_b200/host/shard_plan.cpp through
grbh_shard_plan_stripes) must give every row of the image to exactly one rank's stripes, and route to each rank every
row of its lighting rows that it does not light itself.  An emulated striped frame -- each rank lights only its stripes
with the CPU oracle, receives the rows the other ranks push to it and runs its band's post chain -- must equal the
unsharded frame bit for bit.  Also: the argument checks of grb_deferred_lighting_stripes and grb_hdr_rows_to_peers,
which refuse before any CUDA call."""
import ctypes as C

import numpy as np
import pytest

from tests import common

H = 512
OK, ERR_ARG = 0, -1


@pytest.fixture(scope="module")
def viewer():
    from granite_b200 import build, viewer

    build.build_all()
    return viewer


def layouts(viewer, world):
    """Equal bands, and narrow 8-row-aligned bands at the top."""
    rng = np.random.default_rng(world)
    cuts = np.cumsum(rng.choice([8, 16, 24, 40], size=world - 1))
    return {"equal": viewer.band_partition(H, world), "narrow": [(int(a), int(b)) for a, b in zip([0, *cuts], [*cuts, H])]}


def row_set(ranges):
    s = np.zeros(H, bool)
    for a, b in ranges:
        assert 0 <= a < b <= H
        s[a:b] = True
    return s


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("stripe_rows", [8, 16, 64])
@pytest.mark.parametrize("post_aa", ["AA_NONE", "AA_FXAA", "AA_SMAA_ULTRA", "AA_TAA_HIGH_PLUS_FXAA"])
def test_stripe_plan(viewer, world, stripe_rows, post_aa):
    aa = getattr(viewer, post_aa)
    cluster_rows = 64
    for name, bands in layouts(viewer, world).items():
        plans = [viewer.shard_plan_stripes(1280, H, bands, r, stripe_rows, aa, cluster_rows) for r in range(world)]
        lighting = [viewer.shard_plan_fsr(1280, H, 1280, H, bands, r, aa)["lighting"] for r in range(world)]
        # the ranks' stripes tile [0, H) exactly once, rank r holding the stripes k with k mod world == r
        count = sum(row_set(p["lit"]).astype(int) for p in plans)
        assert (count == 1).all(), name
        for r, p in enumerate(plans):
            assert p["lit"] == [(y, min(y + stripe_rows, H)) for y in range(r * stripe_rows, H, world * stripe_rows)]
        for q in range(world):
            L = row_set([lighting[q]])
            pushed = np.zeros(H, bool)
            for r, p in enumerate(plans):
                rows = row_set(p["push"][q])
                assert not (rows & ~L).any(), f"{name}: rank {r} pushes rows outside rank {q}'s lighting rows"
                assert not (rows & ~row_set(p["lit"])).any(), f"{name}: rank {r} pushes rows it does not light"
                pushed |= rows
            assert plans[q]["push"][q] == []
            lit_q = row_set(plans[q]["lit"])
            # every lighting row of q is lit by q or pushed to q; what q receives is exactly what it does not light
            assert not (L & ~(lit_q | pushed)).any(), f"{name}: rank {q} misses lighting rows"
            assert np.array_equal(row_set(plans[q]["receive"]), L & ~lit_q)
            assert np.array_equal(row_set(plans[q]["upload"]), L | lit_q)
            # binning covers the tile row of every pixel row of the stripes (clustering.frag's rounding, in fp32)
            y = np.nonzero(lit_q)[0]
            tile = np.floor((y.astype(np.float32) + np.float32(0.5)) / np.float32(H) * np.float32(cluster_rows)).astype(int)
            tiles = np.zeros(cluster_rows, bool)
            for a, b in plans[q]["tile_rows"]:
                assert 0 <= a < b <= cluster_rows
                tiles[a:b] = True
            assert tiles[tile].all(), f"{name}: rank {q} does not bin a tile row its stripes read"
            assert all(a[1] < b[0] for a, b in zip(plans[q]["tile_rows"], plans[q]["tile_rows"][1:]))  # merged, in order


def test_stripe_plan_unsharded(viewer):
    for bands in ([], [(0, H)]):
        p = viewer.shard_plan_stripes(640, H, bands, 0, 16)
        assert p["lit"][0] == (0, 16) and row_set(p["lit"]).all()
        assert p["receive"] == [] and p["upload"] == [(0, H)] and p["push"] == [[]]


@pytest.mark.parametrize("stripe_rows", [0, -8, 4, 12, 20])
def test_stripe_plan_refuses_stripe_heights(viewer, stripe_rows):
    from granite_b200 import capi

    with pytest.raises(capi.GrbError, match="positive multiple of 8"):
        viewer.shard_plan_stripes(640, H, viewer.band_partition(H, 2), 0, stripe_rows)
    with pytest.raises(capi.GrbError, match="bad arguments"):
        viewer.shard_plan_stripes(640, H, viewer.band_partition(H, 2), 2, 16)


@pytest.mark.parametrize("world,stripe_rows", [(2, 8), (3, 16), (4, 64), (6, 8)])
@pytest.mark.parametrize("fxaa", [False, True])
def test_emulated_striped_frame(oracle, viewer, monkeypatch, world, stripe_rows, fxaa):
    """test_sharding_gloo's emulated ranks, with the lighting pass replaced by what a rank of a striped frame holds in
    HDR-main: its own stripes lit, the rows the other ranks pushed to it, and zero everywhere else."""
    from tests import test_sharding_gloo as gloo

    W, Hg = gloo.W, gloo.H
    scene, cam, lights, prep = common.build_case(oracle, W, Hg, gloo.N_LIGHTS, 0.25)
    clus, full, _, f, ldr_fxaa = gloo._reference_frame(oracle, scene, cam, prep)
    expect = ldr_fxaa if fxaa else f.ldr
    bands = gloo._bands_for(world, False)
    aa = viewer.AA_FXAA if fxaa else viewer.AA_NONE
    plans = [viewer.shard_plan_stripes(W, Hg, bands, r, stripe_rows, aa) for r in range(world)]
    # each rank lights only its stripes: junk elsewhere, so that a row taken from the wrong rank shows
    rng = np.random.default_rng(stripe_rows)
    hdr_by_rank = []
    for p in plans:
        hdr = rng.integers(0, 2**32, full.shape, dtype=np.uint32)
        for a, b in p["lit"]:
            hdr[a:b] = oracle.deferred_lighting(scene, cam, prep, clus, rows=(a, b))[a:b]
        hdr_by_rank.append(hdr)

    current = [0]

    def striped_hdr(scene, cam, prep, clus, rows=None):
        q = current[0]
        hdr = np.zeros_like(full)
        for a, b in plans[q]["lit"]:
            hdr[a:b] = hdr_by_rank[q][a:b]
        for r, p in enumerate(plans):
            for a, b in p["push"][q]:
                hdr[a:b] = hdr_by_rank[r][a:b]
        return hdr

    monkeypatch.setattr(oracle, "deferred_lighting", striped_hdr)
    contributions = {}

    def hooks(rank, stage):
        def gather(img, rows_per_rank):
            if stage == 0:
                contributions[("d0", rank)] = img
                return img
            out = np.zeros_like(img)
            for r, (a, b) in enumerate(rows_per_rank):
                out[a:b] = contributions[("d0", r)][a:b]
            return out

        def reduce(grid):
            if stage <= 1:
                contributions[("grid", rank)] = grid
                return grid
            return sum(contributions[("grid", r)] for r in range(world))
        return gather, reduce

    # the collection passes of the two exchanges, then the frame (as test_sharding_gloo.test_emulated_many_ranks)
    for stage in (0, 1, 2):
        for r in range(world):
            g, rd = hooks(r, stage)
            current[0] = r
            try:
                plan, out = gloo._sharded_rank(r, world, bands, fxaa, g, rd)
            except AssertionError:
                if stage == 2:
                    raise
                continue
            if stage == 2:
                a, b = plan["own"]
                assert np.array_equal(out[a:b], expect[a:b]), f"rank {r}"


def _lighting_args(capi, h=8, w=16):
    g = capi.GrbGBuffer()
    keep = [np.zeros((h, w), np.uint32), np.zeros((h, w), np.uint32), np.zeros((h, w), np.uint16), np.zeros((h, w), np.float32),
            np.zeros((h, w), np.uint32), np.zeros(16, np.uint32)]
    g.albedo = capi.GrbImage(keep[0].ctypes.data, w, h, w * 4, capi.FORMAT_R8G8B8A8_SRGB)
    g.normal = capi.GrbImage(keep[1].ctypes.data, w, h, w * 4, capi.FORMAT_A2B10G10R10_UNORM)
    g.pbr = capi.GrbImage(keep[2].ctypes.data, w, h, w * 2, capi.FORMAT_R8G8_UNORM)
    g.depth = capi.GrbImage(keep[3].ctypes.data, w, h, w * 4, capi.FORMAT_D32_SFLOAT)
    hdr = capi.GrbImage(keep[4].ctypes.data, w, h, w * 4, capi.FORMAT_B10G11R11_UFLOAT)
    bufs = capi.GrbClusterBuffers()
    bufs.cluster_range = keep[5].ctypes.data  # never dereferenced on the host
    return g, hdr, bufs, keep


def test_lighting_stripes_argument_checks(viewer):
    from granite_b200 import capi

    L = capi.lib()
    g, hdr, bufs, keep = _lighting_args(capi)
    cam, params = capi.GrbCamera(), capi.GrbClusterParameters()
    call = lambda s, shadows=None, image=hdr: L.grb_deferred_lighting_stripes(C.byref(g), C.byref(cam), C.byref(params), C.byref(bufs), shadows,
                                                                              C.byref(image), s, None, None)
    for bad in [(-4, 8, 16), (0, 0, 16), (0, 6, 16), (0, 8, 4)]:
        assert call(capi.GrbStripes(*bad)) == ERR_ARG and "grb_deferred_lighting_stripes" in L.grb_last_error_string().decode()
    params.num_lights = 4
    sh = capi.GrbLightShadows(None, None, 512)
    assert call(capi.GrbStripes(0, 8, 16), C.byref(sh)) == ERR_ARG and "resolution" in L.grb_last_error_string().decode()
    params.num_lights = 0
    wrong = capi.GrbImage(keep[4].ctypes.data, 16, 8, 64, capi.FORMAT_R8G8B8A8_UNORM)
    assert call(capi.GrbStripes(0, 8, 16), image=wrong) == -2
    assert call(capi.GrbStripes(8, 8, 16)) == OK  # a set below the image's last row: nothing to light, nothing launched


def test_hdr_rows_to_peers_argument_checks(viewer):
    from granite_b200 import capi

    L = capi.lib()
    h, w = 32, 16
    src, slot = np.zeros((h, w), np.uint32), np.zeros((h, w), np.uint32)
    flags, counter = np.zeros(2, np.uint32), np.zeros(1, np.uint32)
    hdr = capi.GrbImage(src.ctypes.data, w, h, w * 4, capi.FORMAT_B10G11R11_UFLOAT)
    images = (C.c_void_p * 2)(src.ctypes.data, slot.ctypes.data)
    fl = (C.c_void_p * 2)(flags.ctypes.data, flags.ctypes.data)
    rows = (capi.GrbRows * 2)(capi.GrbRows(0, 16), capi.GrbRows(16, 32))
    good = capi.GrbStripes(0, 8, 16)
    cnt = counter.ctypes.data

    def call(image=hdr, imgs=images, flg=fl, rws=rows, n=2, idx=0, c=cnt, s=good):
        return L.grb_hdr_rows_to_peers(C.byref(image) if image is not None else None, imgs, flg, rws, n, idx, 1, c, s, None)

    msg = lambda: L.grb_last_error_string().decode()
    assert call(image=None) == ERR_ARG and "null" in msg()
    assert call(rws=None) == ERR_ARG
    assert call(imgs=None) == ERR_ARG and "peer_count" in msg()
    assert call(flg=None) == ERR_ARG
    assert call(c=None) == ERR_ARG
    assert call(n=0) == ERR_ARG and call(n=9) == ERR_ARG
    assert call(idx=2) == ERR_ARG and call(idx=-1) == ERR_ARG
    assert call(imgs=(C.c_void_p * 2)(src.ctypes.data, None)) == ERR_ARG and "null peer pointer" in msg()
    rgba8 = capi.GrbImage(src.ctypes.data, w, h, w * 4, capi.FORMAT_R8G8_UNORM)
    assert call(image=rgba8) == ERR_ARG and "4- or 8-byte" in msg()
    tall = capi.GrbImage(src.ctypes.data, w, 65536, w * 4, capi.FORMAT_B10G11R11_UFLOAT)
    assert call(image=tall) == ERR_ARG and "65535" in msg()
    for bad in [(-1, 8, 16), (0, 0, 16), (0, 8, 4)]:
        assert call(s=capi.GrbStripes(*bad)) == ERR_ARG and "stripes" in msg()
    for bad in [(0, 33), (-1, 4), (9, 8)]:
        assert call(rws=(capi.GrbRows * 2)(capi.GrbRows(0, 16), capi.GrbRows(*bad))) == ERR_ARG and "peer_rows" in msg()
    assert call(imgs=(C.c_void_p * 2)(src.ctypes.data, src.ctypes.data)) == ERR_ARG and "distinct" in msg()
    assert not slot.any() and not flags.any() and not counter.any()  # nothing was written


def test_viewer_lighting_stripes_refusals(viewer):
    """grbh_viewer_set_lighting_stripes refuses a stripe height that is not a multiple of 8 and any stripes under FSR 1,
    and accepts 0 (off) and multiples of 8, on a sharded viewer and on an unsharded one (where it changes nothing)."""
    from granite_b200 import capi

    v = viewer.Viewer(64, 128, cuda_device=-1)
    for bad in (-8, 4, 12):
        with pytest.raises(capi.GrbError, match="multiple of 8"):
            v.set_lighting_stripes(bad)
    v.set_lighting_stripes(16)  # unsharded: accepted
    v.set_row_shards([(0, 64), (64, 128)], 0)
    for ok in (8, 64, 0):
        v.set_lighting_stripes(ok)
    v.close()
    fsr = viewer.Viewer(64, 128, cuda_device=-1, resolution_scale=0.5)
    with pytest.raises(capi.GrbError, match="FSR 1"):
        fsr.set_lighting_stripes(16)
    fsr.set_lighting_stripes(0)
    fsr.close()
