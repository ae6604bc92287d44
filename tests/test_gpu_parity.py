"""GPU parity: every C-ABI entry point against the CPU oracle on identical seeded inputs.

Bar (BASELINE.json north_star): bit-exact for cluster bitmasks / ranges / indices; <= 1 ULP of
the STORED format per channel elsewhere (B10G11R11 code, fp16 ulp, 8-bit LSB).  Kernels with no
transcendental in them are additionally required to be bit-exact.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import cluster_cases, common

pytestmark = pytest.mark.gpu

CONFIGS = [
    pytest.param(256, 256, 16, 0.0, id="C1-256x256-16pt"),
    pytest.param(640, 360, 300, 0.25, id="small-300-25pct-spots"),
    pytest.param(1920, 1080, 1024, 0.0, id="C2-1080p-1024pt"),
]
# the benchmarked configuration (BASELINE config 3): 100-230 candidate lights per pixel in the dense rows
C3 = pytest.param(3840, 2160, 4096, 0.0, id="C3-4K-4096pt")


def _cluster(cuda, oracle, cam, prep):
    from granite_b200 import harness

    dev = harness.ClusterDevice(prep.records, prep.model, prep.type_mask, prep.z_ranges, prep.params, prep.res)
    gcam = harness.camera_struct(cam)
    dev.build(gcam)
    torch.cuda.synchronize()
    return dev, gcam


# the default view at the configurations above, and the geometry cases of tests/cluster_cases.py (turned cameras,
# lights at and behind the eye, a finite far plane, a tall wide-angle view)
_GEOMETRY = [pytest.param(name, id=name) for name in cluster_cases.CASES]


def _config(p):
    return pytest.param(p.values, id=p.id)


def _lights_case(oracle, case):
    """(cam, prep) of a default-view configuration (w, h, n, spots) or a named geometry case."""
    if isinstance(case, str):
        _, cam, _, prep = cluster_cases.build(oracle, case)
        return cam, prep
    w, h, n, spots = case
    cam, _, prep = common.build_lights_case(oracle, w / h, n, spots)  # the clusterer does not read the G-buffer
    return cam, prep


@pytest.mark.parametrize("case", [_config(p) for p in CONFIGS + [pytest.param(3840, 2160, 4096, 0.25, id="C3-4096-25pct-spots")]] + _GEOMETRY)
def test_cluster_build_bit_exact(cuda, oracle, case):
    cam, prep = _lights_case(oracle, case)
    ref = oracle.cluster_build(cam, prep)
    dev, _ = _cluster(cuda, oracle, cam, prep)
    cluster_cases.assert_cluster_equal(dev.download(), ref, prep)


@pytest.mark.parametrize("case", [_config(p) for p in CONFIGS + [C3]] + _GEOMETRY)
def test_cluster_indices_bit_exact(cuda, oracle, case):
    if isinstance(case, str):
        scene, cam, _, prep = cluster_cases.build(oracle, case)
    else:
        scene, cam, _, prep = common.build_case(oracle, *case)
    clus = oracle.cluster_build(cam, prep)
    _, tile, zi, _ = oracle.deferred_lighting(scene, cam, prep, clus, want_indices=True)
    got_t, got_z = cluster_cases.debug_cluster_indices(cam, prep, scene.depth)
    assert np.array_equal(got_t, tile)
    assert np.array_equal(got_z, zi)


@pytest.mark.parametrize("w,h,n,spots", [pytest.param(640, 360, 300, 0.25, id="small-300-25pct-spots"), pytest.param(322, 190, 100, 0.0, id="ragged-322x190")])
def test_lighting_row_cost_is_the_cluster_walk(cuda, oracle, w, h, n, spots):
    """grb_lighting_row_cost charges 700 + 45 words + 29 union lights + 89 lights in reach per 16x4
    block; recomputed here from the oracle's cluster (indices, bitmask, ranges) in numpy."""
    from granite_b200 import capi, harness

    scene, cam, lights, prep = common.build_case(oracle, w, h, n, spots)
    clus = oracle.cluster_build(cam, prep)
    _, tile, zi, _ = oracle.deferred_lighting(scene, cam, prep, clus, want_indices=True)
    dev, gcam = _cluster(cuda, oracle, cam, prep)
    depth = harness.to_dev(scene.depth)
    groups = (h + 3) // 4
    out = torch.full((groups,), 12345, dtype=torch.int32, device="cuda")
    img = capi.image(depth, capi.FORMAT_D32_SFLOAT)
    capi.check(capi.lib().grb_lighting_row_cost(C.byref(img), C.byref(gcam), C.byref(dev.params), C.byref(dev.buffers), capi.rows(),
                                                C.c_void_p(out.data_ptr()), capi.stream_ptr()), "grb_lighting_row_cost")
    got = out.cpu().numpy().astype(np.int64)

    # world positions in float64 (the radius test is the only non-integer step)
    ivp = np.asarray(list(cam.inv_view_projection), np.float64).reshape(4, 4).T
    ys, xs = np.mgrid[0:h, 0:w]
    clip = np.stack([2 * (xs + 0.5) / w - 1, 2 * (ys + 0.5) / h - 1, scene.depth.astype(np.float64), np.ones((h, w))], -1) @ ivp.T
    pos = clip[..., :3] / clip[..., 3:4]
    lpos = prep.records["position"].astype(np.float64)
    inv_r = prep.records["inv_radius"].astype(np.float64)
    n32 = prep.n32
    bitmask = clus.bitmask.reshape(-1, n32)
    want = np.zeros(groups, np.int64)
    borderline = 0
    for g in range(groups):
        for bx in range(0, w, 16):
            sl = (slice(4 * g, min(4 * g + 4, h)), slice(bx, min(bx + 16, w)))
            lit = scene.depth[sl] != 0
            total = 700
            if lit.any():
                t, z, P = tile[sl][lit], zi[sl][lit], pos[sl][lit]
                rx, ry = clus.range[z, 0].astype(np.int64), clus.range[z, 1].astype(np.int64)
                lo, hi = int((rx >> 5).min()), min(int((ry >> 5).max()), n32 - 1)
                for i in range(lo, hi + 1):
                    total += 45
                    first = np.clip(rx, 32 * i, 32 * i + 32) - 32 * i
                    last = np.clip(np.maximum(ry + 1, rx), 32 * i, 32 * i + 32) - 32 * i  # exclusive
                    own = bitmask[t, i].astype(np.int64)
                    inrange = ((rx >> 5) <= i) & ((ry >> 5) >= i)
                    rm = np.where(last - first >= 32, 0xFFFFFFFF, ((1 << np.maximum(last - first, 0)) - 1) << first)
                    own = np.where(inrange, own & rm, 0)
                    union = int(np.bitwise_or.reduce(own))
                    for b in range(32):
                        if not (union >> b) & 1:
                            continue
                        li = 32 * i + b
                        d2 = ((P - lpos[li]) ** 2).sum(-1) * inv_r[li] ** 2
                        has = ((own >> b) & 1) == 1
                        near = has & (d2 < 1.0)
                        borderline += int((has & (np.abs(d2 - 1.0) < 1e-5)).any())
                        total += 29 + (89 if near.any() else 0)
            want[g] += total
    # a light whose radius passes within rounding of a pixel may be counted either way
    assert np.abs(got - want).sum() <= 89 * borderline, (np.abs(got - want).sum(), borderline)
    assert got.sum() > 700 * groups * ((w + 15) // 16)


@pytest.mark.parametrize("w,h,n,spots", CONFIGS + [C3, pytest.param(3840, 2160, 4096, 0.25, id="C3-4K-4096-25pct-spots")])
def test_deferred_lighting_parity(cuda, oracle, w, h, n, spots):
    from granite_b200 import harness

    scene, cam, lights, prep = common.build_case(oracle, w, h, n, spots)
    clus = oracle.cluster_build(cam, prep)
    ref = oracle.deferred_lighting(scene, cam, prep, clus)
    dev, gcam = _cluster(cuda, oracle, cam, prep)
    gb = harness.GBufferDevice(scene)
    hdr = gb.emissive.clone()
    harness.deferred_lighting(gb, gcam, dev, hdr)
    got = harness.to_host(hdr, np.uint32)
    sky = scene.depth == 0
    assert np.array_equal(got[sky], scene.emissive[sky]), "sky pixels must keep the attachment value"
    assert common.max_code_diff_r11g11b10(got, ref) <= 1
    exact = float((got == ref).mean())
    print(f"lighting exact-match fraction: {exact:.5f}")
    assert exact > 0.97
    # the work schedule (rows by falling cost, fed back from the previous launch) only reorders the
    # pixel blocks: every launch on the same schedule buffer reproduces the unscheduled frame
    sched = harness.lighting_schedule(h)
    for _ in range(3):
        hdr_s = gb.emissive.clone()
        harness.deferred_lighting(gb, gcam, dev, hdr_s, schedule=sched)
        assert torch.equal(hdr, hdr_s)
    head = sched[:4].cpu().numpy()
    assert head[2] == 1 and head[1] == (h + 3) // 4, "the kernel publishes the next schedule"
    order = sched[4 + (h + 3) // 4: 4 + 2 * ((h + 3) // 4)].cpu().numpy()
    assert np.array_equal(np.sort(order), np.arange((h + 3) // 4)), "a permutation of the block rows"
    # row sharding is bit-invariant
    hdr2 = gb.emissive.clone()
    cut = (h // 3) & ~3
    harness.deferred_lighting(gb, gcam, dev, hdr2, rows=(0, cut))
    harness.deferred_lighting(gb, gcam, dev, hdr2, rows=(cut, h))
    assert torch.equal(hdr, hdr2)


@pytest.mark.parametrize("w,h", [(256, 256), (1920, 1080), (1001, 517)])
@pytest.mark.parametrize("dynamic", [True, False])
def test_bloom_threshold(cuda, oracle, w, h, dynamic):
    from granite_b200 import harness

    rng = np.random.default_rng(w * 7 + h)
    hdr = common.random_hdr(rng, w, h)
    ow, oh = oracle.pyramid_sizes(w, h)[0]
    lum = np.array([0.3, 2.0 ** 0.3, 2.0 ** -0.3], np.float32) if dynamic else None
    ref = oracle.bloom_threshold(hdr, lum, (ow, oh))
    out = harness.new_rgba16f(ow, oh)
    harness.bloom_threshold(harness.to_dev(hdr), harness.to_dev(lum) if dynamic else None, out)
    got = harness.to_host(out, np.uint16)
    assert np.array_equal(got[..., :3], ref[..., :3]), "rgb has no transcendental: must be bit-exact"
    assert common.f16_ulp_diff(got[..., 3], ref[..., 3]).max() <= 1  # log2


@pytest.mark.parametrize("w,h", [(256, 256), (1920, 1080), (3840, 2160), (136, 72)])
@pytest.mark.parametrize("dynamic", [True, False])
def test_bloom_threshold_downsample_fused(cuda, oracle, w, h, dynamic):
    """K7 + first K8 in one kernel (threshold tile in shared memory, TMA-loaded HDR tiles): within 1 fp16
    ulp of the two separate passes, with and without materialising the threshold image, and on a row band."""
    from granite_b200 import harness

    rng = np.random.default_rng(w * 11 + h)
    hdr = common.random_hdr(rng, w, h)
    (tw, th), (dw, dh) = oracle.pyramid_sizes(w, h)[:2]
    lum = np.array([0.3, 2.0 ** 0.3, 2.0 ** -0.3], np.float32) if dynamic else None
    ref_t = oracle.bloom_threshold(hdr, lum, (tw, th))
    hdr_t, lum_t = harness.to_dev(hdr), harness.to_dev(lum) if dynamic else None
    d0, t = harness.new_rgba16f(dw, dh), harness.new_rgba16f(tw, th)
    harness.bloom_threshold_downsample(hdr_t, lum_t, d0, t)
    got_t = harness.to_host(t, np.uint16)
    common.assert_f16_close(got_t, ref_t, "fused threshold vs oracle", min_identical=0.99, abs_floor=2.0 ** -18)  # log2 of a luminance within an ulp of 1
    # d0 is computed from the fused kernel's OWN threshold tile: compare with the oracle's downsample of it
    ref_d0 = oracle.bloom_downsample(got_t, (dw, dh))
    got_d0 = harness.to_host(d0, np.uint16)
    common.assert_f16_close(got_d0, ref_d0, "fused d0")
    d0b = harness.new_rgba16f(dw, dh)
    harness.bloom_threshold_downsample(hdr_t, lum_t, d0b)  # threshold image not materialised
    assert np.array_equal(harness.to_host(d0b, np.uint16), got_d0)
    band = (dh // 3, dh // 3 + 21)
    d0c = harness.new_rgba16f(dw, dh)
    harness.bloom_threshold_downsample(hdr_t, lum_t, d0c, rows=band)
    got = harness.to_host(d0c, np.uint16)
    assert np.array_equal(got[band[0]:band[1]], got_d0[band[0]:band[1]])
    assert not got[:band[0]].any() and not got[band[1]:].any(), "rows outside the band must not be written"


@pytest.mark.parametrize("w_in,h_in,w,h", [(128, 128, 64, 64), (960, 540, 480, 270), (1920, 1080, 960, 540), (240, 135, 120, 68), (33, 17, 17, 9), (64, 36, 32, 18)])
@pytest.mark.parametrize("feedback", [False, True])
def test_bloom_downsample_bit_exact(cuda, oracle, w_in, h_in, w, h, feedback):
    from granite_b200 import harness

    rng = np.random.default_rng(w_in + 3 * h_in + feedback)
    src = common.random_rgba16f(rng, w_in, h_in)
    hist = common.random_rgba16f(rng, w, h) if feedback else None
    lerp = float(np.float32(1.0 - 0.001 ** (1 / 60)))
    ref = oracle.bloom_downsample(src, (w, h), hist, lerp)
    out = harness.new_rgba16f(w, h)
    harness.bloom_downsample(harness.to_dev(src), out, harness.to_dev(hist) if feedback else None, lerp)
    full = harness.to_host(out, np.uint16)
    # exact 2:1 steps run the TMA tile kernel, whose packed multiply-adds are contracted by ptxas
    # (grb_post_tiles.cu): 1 fp16 ulp on ~5e-5 of the texels; other shapes are bit-exact
    tiled = (w_in == 2 * w and h_in == 2 * h and w * h >= 200000)  # smaller levels stay on the generic kernels
    if tiled:
        common.assert_f16_close(full, ref, "downsample")
    else:
        assert np.array_equal(full, ref)
    if h >= 9:  # a row band (row-sharded frames): same texels, nothing outside the band
        band = (h // 3, h // 3 + max(h // 4, 2))
        out2 = harness.new_rgba16f(w, h)
        harness.bloom_downsample(harness.to_dev(src), out2, harness.to_dev(hist) if feedback else None, lerp, rows=band)
        got = harness.to_host(out2, np.uint16)
        assert np.array_equal(got[band[0]:band[1]], full[band[0]:band[1]]) and not got[:band[0]].any() and not got[band[1]:].any()


@pytest.mark.parametrize("w_in,h_in,w,h", [(8, 8, 16, 16), (120, 68, 240, 135), (480, 270, 960, 540), (9, 5, 17, 9), (30, 17, 60, 34)])
def test_bloom_upsample_bit_exact(cuda, oracle, w_in, h_in, w, h):
    from granite_b200 import harness

    rng = np.random.default_rng(w_in * 5 + h_in)
    src = common.random_rgba16f(rng, w_in, h_in)
    ref = oracle.bloom_upsample(src, (w, h))
    out = harness.new_rgba16f(w, h)
    harness.bloom_upsample(harness.to_dev(src), out)
    full = harness.to_host(out, np.uint16)
    if w == 2 * w_in and h == 2 * h_in and w * h >= 200000:
        common.assert_f16_close(full, ref, "upsample")
    else:
        assert np.array_equal(full, ref)
    for band in ((h // 3, h // 3 + max(h // 4, 2)), (h // 3 + 1, h - 1)):  # even and odd first rows
        out2 = harness.new_rgba16f(w, h)
        harness.bloom_upsample(harness.to_dev(src), out2, rows=band)
        got = harness.to_host(out2, np.uint16)
        common.assert_f16_close(got[band[0]:band[1]], ref[band[0]:band[1]], "upsample band")
        assert not got[:band[0]].any() and not got[band[1]:].any()


@pytest.mark.parametrize("w0,h0", [(960, 540), (480, 270), (64, 36), (33, 17)])
@pytest.mark.parametrize("feedback,dynamic", [(True, True), (False, False), (False, True)])
def test_bloom_tail_fused_bit_exact(cuda, oracle, w0, h0, feedback, dynamic):
    """d1, d2, d3 (+history), luminance, u2, u1 in one cooperative launch: every level bit for bit the
    oracle's (the kernel uses the unfused arithmetic), the log-average exact, its exp2 within 4 ulps."""
    import math

    from granite_b200 import harness

    rng = np.random.default_rng(w0 + 7 * h0 + feedback)
    d0 = common.random_rgba16f(rng, w0, h0)
    sz = [(w0, h0)]
    for _ in range(3):
        sz.append((int(math.ceil(sz[-1][0] * 0.5)), int(math.ceil(sz[-1][1] * 0.5))))
    if sz[3][0] < 2 or sz[3][1] < 2:
        pytest.skip("d3 too small for the luminance grid")
    hist = common.random_rgba16f(rng, *sz[3]) if feedback else None
    lerp_d3, lerp_lum = float(np.float32(1.0 - 0.001 ** (1 / 60))), float(np.float32(1.0 - 0.5 ** (1 / 60)))
    lum0 = np.array([0.3, 2.0 ** 0.3, 2.0 ** -0.3], np.float32)
    d1 = oracle.bloom_downsample(d0, sz[1])
    d2 = oracle.bloom_downsample(d1, sz[2])
    d3 = oracle.bloom_downsample(d2, sz[3], hist, lerp_d3)
    lum_ref = oracle.luminance(d3, lum0, lerp_lum)
    u2 = oracle.bloom_upsample(d3, sz[2])
    u1 = oracle.bloom_upsample(u2, sz[1])
    t = {k: harness.new_rgba16f(*s_) for k, s_ in (("d1", sz[1]), ("d2", sz[2]), ("d3", sz[3]), ("u2", sz[2]), ("u1", sz[1]))}
    lum_t = harness.to_dev(lum0.copy()) if dynamic else None
    harness.bloom_tail(harness.to_dev(d0), t["d1"], t["d2"], t["d3"], harness.to_dev(hist) if feedback else None, lerp_d3, lum_t, lerp_lum, t["u2"], t["u1"])
    for k, ref in (("d1", d1), ("d2", d2), ("d3", d3), ("u2", u2), ("u1", u1)):
        assert np.array_equal(harness.to_host(t[k], np.uint16), ref), k
    if dynamic:
        lum = lum_t.cpu().numpy()
        assert lum.view(np.uint32)[0] == lum_ref.view(np.uint32)[0]
        assert common.f32_ulp_diff(lum[1:], lum_ref[1:]).max() <= 4


@pytest.mark.parametrize("w0,h0,rows,ctas", [(960, 540, None, 0), (960, 540, (128, 280), 16), (66, 37, (3, 30), 2), (480, 270, None, 1)])
def test_bloom_tail_with_u0_and_cta_cap(cuda, oracle, w0, h0, rows, ctas):
    """grb_bloom_tail_ex: the last upsample u0 (rows of it) inside the same launch, and the launch capped to a few
    CTAs (the form the frame uses beside the next lighting pass): every level bit for bit the oracle's."""
    import math

    from granite_b200 import harness

    rng = np.random.default_rng(w0 * 3 + h0)
    d0 = common.random_rgba16f(rng, w0, h0)
    sz = [(w0, h0)]
    for _ in range(3):
        sz.append((int(math.ceil(sz[-1][0] * 0.5)), int(math.ceil(sz[-1][1] * 0.5))))
    hist = common.random_rgba16f(rng, *sz[3])
    lerp_d3, lerp_lum = float(np.float32(1.0 - 0.001 ** (1 / 60))), float(np.float32(1.0 - 0.5 ** (1 / 60)))
    lum0 = np.array([0.3, 2.0 ** 0.3, 2.0 ** -0.3], np.float32)
    d1 = oracle.bloom_downsample(d0, sz[1])
    d2 = oracle.bloom_downsample(d1, sz[2])
    d3 = oracle.bloom_downsample(d2, sz[3], hist, lerp_d3)
    lum_ref = oracle.luminance(d3, lum0, lerp_lum)
    u2 = oracle.bloom_upsample(d3, sz[2])
    u1 = oracle.bloom_upsample(u2, sz[1])
    u0 = oracle.bloom_upsample(u1, sz[0])
    t = {k: harness.new_rgba16f(*s_) for k, s_ in (("d1", sz[1]), ("d2", sz[2]), ("d3", sz[3]), ("u2", sz[2]), ("u1", sz[1]), ("u0", sz[0]))}
    lum_t = harness.to_dev(lum0.copy())
    harness.bloom_tail(harness.to_dev(d0), t["d1"], t["d2"], t["d3"], harness.to_dev(hist), lerp_d3, lum_t, lerp_lum, t["u2"], t["u1"], u0_t=t["u0"],
                       u0_rows=rows, max_ctas=ctas)
    for k, ref in (("d1", d1), ("d2", d2), ("d3", d3), ("u2", u2), ("u1", u1)):
        assert np.array_equal(harness.to_host(t[k], np.uint16), ref), k
    got = harness.to_host(t["u0"], np.uint16)
    y0, y1 = rows if rows else (0, h0)
    assert np.array_equal(got[y0:y1], u0[y0:y1]), "u0"
    assert not got[:y0].any() and not got[y1:].any()
    lum = lum_t.cpu().numpy()
    assert lum.view(np.uint32)[0] == lum_ref.view(np.uint32)[0] and common.f32_ulp_diff(lum[1:], lum_ref[1:]).max() <= 4


@pytest.mark.parametrize("w,h", [(8, 8), (60, 34), (120, 68), (61, 35)])
def test_luminance(cuda, oracle, w, h):
    from granite_b200 import harness

    rng = np.random.default_rng(w + h)
    d3 = common.random_rgba16f(rng, w, h, -6.0, 6.0)
    lum0 = np.array([0.25, 2.0 ** 0.25, 2.0 ** -0.25], np.float32)
    lerp = float(np.float32(1.0 - 0.5 ** (1 / 60)))
    ref, grid = oracle.luminance(d3, lum0, lerp, want_grid=True)
    d3_t = harness.to_dev(d3)
    lum_t = harness.to_dev(lum0.copy())
    harness.luminance(d3_t, lum_t, lerp)
    got = lum_t.cpu().numpy()
    assert got[0].view(np.uint32) == ref[0].view(np.uint32), "average log luminance (pure add/mul) must be bit-exact"
    assert common.f32_ulp_diff(got[1:], ref[1:]).max() <= 4  # exp2
    # sharded form: grid rows from two "ranks", summed (x + 0 is exact), then finalised
    sx, sy = w // 2, h // 2
    g0 = torch.zeros(sy * sx, dtype=torch.float32, device="cuda")
    g1 = torch.zeros(sy * sx, dtype=torch.float32, device="cuda")
    cut = sy // 2
    harness.luminance_grid(d3_t, g0, rows=(0, cut))
    harness.luminance_grid(d3_t, g1, rows=(cut, sy))
    gsum = g0 + g1
    assert np.array_equal(gsum.cpu().numpy().reshape(sy, sx).view(np.uint32), grid.view(np.uint32))
    lum_t2 = harness.to_dev(lum0.copy())
    harness.luminance_finalize(gsum, sx, sy, lum_t2, lerp)
    assert torch.equal(lum_t, lum_t2)


@pytest.mark.parametrize("w,h", [(256, 256), (1920, 1080), (1001, 517)])
@pytest.mark.parametrize("dynamic", [True, False])
def test_tonemap(cuda, oracle, w, h, dynamic):
    from granite_b200 import harness

    rng = np.random.default_rng(w + 11 * h)
    hdr = common.random_hdr(rng, w, h)
    bw, bh = oracle.pyramid_sizes(w, h)[1]
    bloom = common.random_rgba16f(rng, bw, bh, 0.0, 0.5)
    lum = np.array([-0.7, 2.0 ** -0.7, 2.0 ** 0.7], np.float32) if dynamic else None
    ref = oracle.tonemap(hdr, bloom, lum, 1.25)
    out = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    harness.tonemap(harness.to_dev(hdr), harness.to_dev(bloom), harness.to_dev(lum) if dynamic else None, out, exposure=1.25)
    got = harness.to_host(out, np.uint32)
    d = common.rgba8_channel_diff(got, ref)
    assert d.max() <= 1
    print(f"tonemap exact fraction {float((got == ref).mean()):.6f}")
    assert (got == ref).mean() > 0.999


@pytest.mark.parametrize("w,h", [(256, 256), (1280, 720), (333, 177), (3840, 2160)])
@pytest.mark.parametrize("srgb", [True, False])
def test_fxaa(cuda, oracle, w, h, srgb):
    from granite_b200 import harness

    rng = np.random.default_rng(w - h)
    # blocky image with edges so the directional taps are exercised
    base = rng.integers(0, 256, size=(h // 8 + 1, w // 8 + 1, 4), dtype=np.uint8)
    img = np.kron(base, np.ones((8, 8, 1), np.uint8))[:h, :w].copy()
    img = (img.astype(np.int32) + rng.integers(-6, 7, size=img.shape)).clip(0, 255).astype(np.uint8)
    img32 = np.ascontiguousarray(img).view(np.uint32)[..., 0]
    ref = oracle.fxaa(img32, srgb)
    out = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    harness.fxaa(harness.to_dev(img32), out, target_srgb=srgb)
    got = harness.to_host(out, np.uint32)
    d = common.rgba8_channel_diff(got, ref)
    # The tile kernel works in 0..255 units with FMA and folds decode_srgb / re-encode: 1 code, rarely.
    # FXAA itself is discontinuous -- it outputs rgbA or rgbB depending on lumaB < lumaMin || lumaB > lumaMax --
    # so when lumaB equals a neighbour's luma to within fp32 rounding (about 1 pixel in 1e5 of this blocky
    # test image) any re-associated evaluation may take the other branch; those pixels are counted apart.
    flips = (d > 1).reshape(h, w, 4).any(-1)
    print(f"fxaa identical fraction {float((d == 0).mean()):.6f}, branch flips {int(flips.sum())} of {h * w} pixels")
    assert flips.mean() <= 1e-4
    assert (d == 0).mean() > 0.995  # rounding ties at x.5 of the folded sRGB round trip on this blocky image


@pytest.mark.parametrize("w,h,rows", [(96, 64, None), (333, 177, (10, 150)), (1921, 1080, None), (3840, 2160, None)])
def test_pq10_encode(cuda, oracle, w, h, rows):
    """HDR10 output encoding (pq10_encode.frag, hdr.cpp:595-658) vs the oracle, whose codes equal the reference
    shader's bit for bit (tests/test_oracle_ref_post_shaders.py).  Odd widths take the unaligned load / store path."""
    from granite_b200 import harness
    from tests.test_oracle_ref_post_shaders import pq_inputs

    rng = np.random.default_rng(w + 7 * h)
    hdr, ui = pq_inputs(rng, w, h)
    m = oracle.rec709_to_display_primaries(oracle.BT2020_PRIMARIES)
    for max_light in (1000.0, 4000.0):
        ref = oracle.pq10_encode(hdr, ui, m, 500.0, 400.0, max_light, rows=rows)
        out = torch.zeros((h, w), dtype=torch.int32, device="cuda")
        harness.pq10_encode(harness.to_dev(hdr), harness.to_dev(ui), m, 500.0, 400.0, max_light, out, rows=rows)
        got = harness.to_host(out, np.uint32)
        d = common.a2b10g10r10_channel_diff(got, ref)
        print(f"pq10 {w}x{h} max_light {max_light}: identical {float((d == 0).mean()):.6f}, max code diff {int(d.max())}")
        assert d.max() <= 1 and (d == 0).mean() > 0.99
        if rows:  # nothing outside the band is written
            assert not got[: rows[0]].any() and not got[rows[1]:].any()


def _taa_inputs(rng, w, h):
    hdr = common.random_hdr(rng, w, h, scale=2.0)
    depth = rng.uniform(0.0005, 0.03, size=(h, w)).astype(np.float32)
    depth[rng.random((h, w)) < 0.1] = 0.0
    mv = np.zeros((h, w, 2), np.float16)
    m = rng.random((h, w)) < 0.1
    mv[m] = (rng.uniform(-2.0, 2.0, size=(int(m.sum()), 2)) / np.array([w, h])).astype(np.float16)
    hist = np.concatenate([rng.uniform(0, 1, (h, w, 1)), rng.uniform(-0.5, 0.5, (h, w, 2)), np.ones((h, w, 1))], -1).astype(np.float16)
    # reproj = T*S*VP_prev*invVP_cur for a slightly moved camera: near-identity in UV space
    reproj = np.array([[0.5, 0, 0, 0], [0, 0.5, 0, 0], [0.3, -0.2, 1, 0], [0.5 + 0.4 / w, 0.5 - 0.3 / h, 0, 1]], np.float32)
    return hdr, depth, mv.view(np.uint16), hist.view(np.uint16), reproj


@pytest.mark.parametrize("w,h,quality", [(w, h, q) for (w, h) in [(256, 256), (1280, 720), (333, 177)] for q in (0, 1, 2)] + [(3840, 2160, 2)])
def test_taa_resolve_bit_exact(cuda, oracle, w, h, quality):
    from granite_b200 import harness

    rng = np.random.default_rng(w * 3 + h + quality)
    hdr, depth, mv, hist, reproj = _taa_inputs(rng, w, h)
    hdr_t = harness.to_dev(hdr)
    oc = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    oh = harness.new_rgba16f(w, h)
    # first frame: no history
    ref_c, ref_h = oracle.taa_resolve(hdr, depth, mv, None, reproj, quality)
    harness.taa_resolve(hdr_t, None, None, None, None, quality, oc, oh)
    assert np.array_equal(harness.to_host(oc, np.uint32), ref_c)
    assert np.array_equal(harness.to_host(oh, np.uint16), ref_h)
    # steady state
    ref_c, ref_h = oracle.taa_resolve(hdr, depth, mv, hist, reproj, quality)
    harness.taa_resolve(hdr_t, harness.to_dev(depth), harness.to_dev(mv.reshape(h, w, 2)).view(torch.int32).reshape(h, w),
                        harness.to_dev(hist), reproj, quality, oc, oh)
    got_c, got_h = harness.to_host(oc, np.uint32), harness.to_host(oh, np.uint16)
    assert np.array_equal(got_c, ref_c)
    assert np.array_equal(got_h, ref_h)


def test_error_reporting(cuda):
    from granite_b200 import capi

    bad = capi.GrbImage(None, 0, 0, 0, 0)
    rc = capi.lib().grb_bloom_upsample(C.byref(bad), C.byref(bad), capi.rows(), capi.stream_ptr())
    assert rc == -2
    assert b"R16G16B16A16_SFLOAT" in capi.lib().grb_last_error_string()


def test_peer_wait_timeout_reaches_the_error_string(cuda, monkeypatch):
    """A rank that never publishes its band must not go unnoticed: the bounded spin writes a device
    error word and the NEXT entry point on the device returns GRB_ERR_CUDA naming the rank."""
    from granite_b200 import capi

    monkeypatch.setenv("GRB_PEER_WAIT_SPINS", "200")
    flags = torch.zeros(8, dtype=torch.int32, device="cuda")
    flags[0] = 7  # rank 0 has published epoch 7, rank 1 never does
    L = capi.lib()
    L.grb_peer_wait.argtypes = [C.c_void_p, C.c_int32, C.c_uint32, C.c_void_p]
    assert L.grb_peer_wait(C.c_void_p(flags.data_ptr()), 2, 7, capi.stream_ptr()) == 0
    torch.cuda.synchronize()
    bad = capi.GrbImage(None, 0, 0, 0, 0)
    img = torch.zeros((8, 8, 4), dtype=torch.int16, device="cuda")
    ok = capi.image(img, capi.FORMAT_R16G16B16A16_SFLOAT)
    rc = L.grb_bloom_upsample(C.byref(ok), C.byref(ok), capi.rows(), capi.stream_ptr())
    assert rc == -3, rc  # GRB_ERR_CUDA
    msg = L.grb_last_error_string()
    assert b"timed out waiting for rank 1" in msg, msg
    # reported once: the device is usable again
    assert L.grb_bloom_upsample(C.byref(ok), C.byref(ok), capi.rows(), capi.stream_ptr()) == 0
