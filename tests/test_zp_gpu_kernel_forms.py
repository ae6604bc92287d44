"""The post chain's other kernel forms and run-time switches against the oracle.

The launchers choose between several kernels by shape (tile / 4-pixel / generic tonemap, the generic luminance
reduction above 8192 grid samples, the unfused pyramid when the fused tail refuses a shape) or by a GRB_* switch.
Each case here asserts that it reaches the form it names -- the selection condition on its inputs, a return code,
or the switch a child process reports -- and holds that form to the bar its code states.

Most switches are read once per process (`static const bool ... = getenv(...)`), so those cases run
tests/kernel_forms_worker.py in a child process with the switch set, and compare its files with the oracle or with
the same case run under the default environment.  GRB_NO_ASYNC_CLUSTER / GRB_NO_ASYNC_POST are read when a viewer
bakes its graph, so they are set in-process."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from granite_b200 import synth
from tests import common
from tests.kernel_forms_worker import CHAIN_FRAMES, CHAIN_SIZES, PYRAMID, SWITCHES, blocky_image

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LUM_FAST_MAX_SAMPLES = 8192  # kLumFastMaxSamples (grb_post.cu): larger grids take luminance_kernel, and the fused tail refuses them
TILE_MIN_TEXELS = 200000     # launch_tent_tiled (grb_post_tiles.cu): smaller levels stay on the generic kernels
LERP_D3 = float(np.float32(1.0 - 0.001 ** (1 / 60)))
LERP_LUM = float(np.float32(1.0 - 0.5 ** (1 / 60)))


def _halve(s):
    return int(math.ceil(s[0] * 0.5)), int(math.ceil(s[1] * 0.5))


def _tiled(in_wh, out_wh):
    """Whether grb_bloom_downsample / grb_bloom_upsample take the tile kernel for this step."""
    exact = (in_wh[0] == 2 * out_wh[0] and in_wh[1] == 2 * out_wh[1]) or (out_wh[0] == 2 * in_wh[0] and out_wh[1] == 2 * in_wh[1])
    return exact and out_wh[0] * out_wh[1] >= TILE_MIN_TEXELS


def _assert_lum(got, ref):
    assert got.view(np.uint32)[0] == ref.view(np.uint32)[0], "average log luminance (pure add/mul) must be bit-exact"
    assert common.f32_ulp_diff(got[1:], ref[1:]).max() <= 4  # exp2


# ------------------------------------------------------------------------------------------------ tonemap forms
def _tonemap_form(w, h, bw, bh, fp16):
    """grb_tonemap's choice for 16-byte aligned, unpadded images (grb_post.cu, launch_tonemap_fast)."""
    if fp16:
        return "generic-rgba16f"
    if w % 4 == 0 and bw * 4 == w:
        return "tile" if bh * 4 == h else "4px"
    return "generic"


@pytest.mark.parametrize("w,h,fp16,form", [pytest.param(256, 256, False, "tile", id="tile-256x256"),
                                           pytest.param(1280, 718, False, "4px", id="4px-1280x718"),
                                           pytest.param(1001, 517, False, "generic", id="generic-1001x517"),
                                           pytest.param(640, 360, True, "generic-rgba16f", id="rgba16f-640x360")])
@pytest.mark.parametrize("dynamic", [True, False], ids=["dynamic", "static"])
@pytest.mark.parametrize("srgb", [True, False], ids=["srgb", "unorm"])
def test_tonemap_forms(cuda, oracle, w, h, fp16, form, dynamic, srgb):
    """Every tonemap kernel x exposure x target: at most 1 code per channel and > 99.9 % of pixels identical, as in
    test_tonemap; a band with an odd first row gives the whole-image call's pixels and writes nothing else."""
    from granite_b200 import harness

    rng = np.random.default_rng(w + 11 * h + fp16)
    hdr = common.random_hdr_f16(rng, w, h) if fp16 else common.random_hdr(rng, w, h)
    bw, bh = oracle.pyramid_sizes(w, h)[1]
    assert _tonemap_form(w, h, bw, bh, fp16) == form
    bloom = common.random_rgba16f(rng, bw, bh, 0.0, 0.5)
    lum = np.array([-0.7, 2.0 ** -0.7, 2.0 ** 0.7], np.float32) if dynamic else None
    ref = oracle.tonemap(hdr, bloom, lum, 1.25, target_srgb=srgb)
    hdr_t, bloom_t, lum_t = harness.to_dev(hdr), harness.to_dev(bloom), harness.to_dev(lum) if dynamic else None
    out = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    harness.tonemap(hdr_t, bloom_t, lum_t, out, exposure=1.25, srgb=srgb)
    got = harness.to_host(out, np.uint32)
    d = common.rgba8_channel_diff(got, ref)
    print(f"tonemap {form} {w}x{h}: exact fraction {float((got == ref).mean()):.6f}, max code diff {int(d.max())}")
    assert d.max() <= 1
    assert (got == ref).mean() > 0.999
    y0 = (h // 3) | 1
    y1 = y0 + h // 4
    band = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    harness.tonemap(hdr_t, bloom_t, lum_t, band, exposure=1.25, srgb=srgb, rows=(y0, y1))
    got_b = harness.to_host(band, np.uint32)
    assert np.array_equal(got_b[y0:y1], got[y0:y1])
    assert not got_b[:y0].any() and not got_b[y1:].any(), "rows outside the band must not be written"


# ------------------------------------------------------------------------------- luminance above the fast grid
@pytest.mark.parametrize("w,h", [(364, 364), (482, 272)])
def test_luminance_generic_kernel(cuda, oracle, w, h):
    """A d3 whose (w/2)(h/2) grid exceeds the fast kernel's shared memory runs luminance_kernel."""
    from granite_b200 import harness

    assert (w // 2) * (h // 2) > LUM_FAST_MAX_SAMPLES
    rng = np.random.default_rng(w * 3 + h)
    d3 = common.random_rgba16f(rng, w, h, -6.0, 6.0)
    lum0 = np.array([0.25, 2.0 ** 0.25, 2.0 ** -0.25], np.float32)
    ref = oracle.luminance(d3, lum0, LERP_LUM)
    lum_t = harness.to_dev(lum0.copy())
    harness.luminance(harness.to_dev(d3), lum_t, LERP_LUM)
    _assert_lum(lum_t.cpu().numpy(), ref)


@pytest.mark.parametrize("w0,h0,d3_wh", [(2905, 2905, (364, 364)), (3849, 2169, (482, 272))])
def test_bloom_tail_refuses_large_luminance_grid(cuda, oracle, w0, h0, d3_wh):
    """grb_bloom_tail_ex with a luminance buffer refuses a d3 above the fast grid (GRB_ERR_UNSUPPORTED_FORMAT) and
    writes nothing; the separate calls the frame then makes (hdr.cpp) give the oracle's levels bit for bit.  The
    odd sizes keep every step off the tile kernels, so each level is the generic kernel the fused tail would use."""
    from granite_b200 import capi, harness

    sz = [(w0, h0)]
    for _ in range(3):
        sz.append(_halve(sz[-1]))
    assert sz[3] == d3_wh and (d3_wh[0] // 2) * (d3_wh[1] // 2) > LUM_FAST_MAX_SAMPLES
    assert not any(_tiled(a, b) for a, b in zip(sz[:3], sz[1:])) and not any(_tiled(a, b) for a, b in zip(sz[3:0:-1], sz[2::-1]))
    rng = np.random.default_rng(w0 + h0)
    # alpha (log2 luminance) averages to 0.5, inside the [-3, 2] clamp, so the luminance result depends on every sample
    d0 = common.random_rgba16f(rng, w0, h0, -2.0, 3.0)
    hist = common.random_rgba16f(rng, *sz[3], -2.0, 3.0)
    lum0 = np.array([0.3, 2.0 ** 0.3, 2.0 ** -0.3], np.float32)
    sentinel = 0x7E00  # an fp16 NaN no level can produce from these inputs
    t = {k: torch.full((s_[1], s_[0], 4), sentinel, dtype=torch.int16, device="cuda")
         for k, s_ in (("d1", sz[1]), ("d2", sz[2]), ("d3", sz[3]), ("u2", sz[2]), ("u1", sz[1]), ("u0", sz[0]))}
    lum_sentinel = np.array([1.5, 2.5, 3.5], np.float32)
    lum_t = harness.to_dev(lum_sentinel.copy())
    d0_t, hist_t = harness.to_dev(d0), harness.to_dev(hist)
    with pytest.raises(capi.GrbError, match=r"grb_bloom_tail_ex failed \(-2\)"):  # GRB_ERR_UNSUPPORTED_FORMAT
        harness.bloom_tail(d0_t, t["d1"], t["d2"], t["d3"], hist_t, LERP_D3, lum_t, LERP_LUM, t["u2"], t["u1"], u0_t=t["u0"], max_ctas=16)
    torch.cuda.synchronize()
    for k, v in t.items():
        assert bool((v == sentinel).all()), f"{k} written by a refused launch"
    assert np.array_equal(lum_t.cpu().numpy(), lum_sentinel), "luminance written by a refused launch"

    # hdr.cpp's fallback: three downsamples, the luminance, two upsamples and the exact u0
    lum_t = harness.to_dev(lum0.copy())
    harness.bloom_downsample(d0_t, t["d1"])
    harness.bloom_downsample(t["d1"], t["d2"])
    harness.bloom_downsample(t["d2"], t["d3"], hist_t, LERP_D3)
    harness.luminance(t["d3"], lum_t, LERP_LUM)
    harness.bloom_upsample(t["d3"], t["u2"])
    harness.bloom_upsample(t["u2"], t["u1"])
    harness.bloom_upsample_exact(t["u1"], t["u0"])
    ref = {"d1": oracle.bloom_downsample(d0, sz[1])}
    ref["d2"] = oracle.bloom_downsample(ref["d1"], sz[2])
    ref["d3"] = oracle.bloom_downsample(ref["d2"], sz[3], hist, LERP_D3)
    ref["u2"] = oracle.bloom_upsample(ref["d3"], sz[2])
    ref["u1"] = oracle.bloom_upsample(ref["u2"], sz[1])
    ref["u0"] = oracle.bloom_upsample(ref["u1"], sz[0])
    for k, r in ref.items():
        assert np.array_equal(harness.to_host(t[k], np.uint16), r), k
    assert -3.0 < float(ref["d3"][..., 3].view(np.float16).astype(np.float32).mean()) < 2.0, "the log-average must not sit at the clamp"
    _assert_lum(lum_t.cpu().numpy(), oracle.luminance(ref["d3"], lum0, LERP_LUM))


# ------------------------------------------------------------------------------------ grb_bloom_upsample_exact
@pytest.mark.parametrize("w_in,h_in,w,h", [pytest.param(480, 270, 960, 540, id="tile-shape-480x270"), pytest.param(241, 135, 481, 269, id="odd-241x135")])
def test_bloom_upsample_exact(cuda, oracle, w_in, h_in, w, h):
    """The u0 a frame computes without the fused tail: the generic kernel at every size, bit for bit the oracle's,
    also at the 2:1 shape where grb_bloom_upsample takes the tile kernel, and on a band with an odd first row."""
    from granite_b200 import harness

    if (w_in, h_in) == (480, 270):
        assert _tiled((w_in, h_in), (w, h)), "grb_bloom_upsample takes the tile kernel at this shape"
    rng = np.random.default_rng(w_in * 13 + h_in)
    src = common.random_rgba16f(rng, w_in, h_in)
    ref = oracle.bloom_upsample(src, (w, h))
    src_t = harness.to_dev(src)
    out = harness.new_rgba16f(w, h)
    harness.bloom_upsample_exact(src_t, out)
    assert np.array_equal(harness.to_host(out, np.uint16), ref)
    y0, y1 = (h // 3) | 1, h - 1
    band = harness.new_rgba16f(w, h)
    harness.bloom_upsample_exact(src_t, band, rows=(y0, y1))
    got = harness.to_host(band, np.uint16)
    assert np.array_equal(got[y0:y1], ref[y0:y1])
    assert not got[:y0].any() and not got[y1:].any(), "rows outside the band must not be written"


@pytest.mark.parametrize("w0,h0", [(960, 540), (66, 37)])
def test_bloom_upsample_exact_equals_fused_tail_u0(cuda, oracle, w0, h0):
    """hdr.cpp computes u0 with grb_bloom_upsample_exact when the fused tail does not run, as "the arithmetic the
    fused tail uses": on the same u1 both give the same texels."""
    from granite_b200 import harness

    sz = [(w0, h0)]
    for _ in range(3):
        sz.append(_halve(sz[-1]))
    rng = np.random.default_rng(w0 * 5 + h0)
    d0 = common.random_rgba16f(rng, w0, h0)
    t = {k: harness.new_rgba16f(*s_) for k, s_ in (("d1", sz[1]), ("d2", sz[2]), ("d3", sz[3]), ("u2", sz[2]), ("u1", sz[1]), ("u0", sz[0]))}
    lum_t = harness.to_dev(np.array([0.3, 2.0 ** 0.3, 2.0 ** -0.3], np.float32))
    harness.bloom_tail(harness.to_dev(d0), t["d1"], t["d2"], t["d3"], None, LERP_D3, lum_t, LERP_LUM, t["u2"], t["u1"], u0_t=t["u0"], max_ctas=16)
    u0 = harness.new_rgba16f(*sz[0])
    harness.bloom_upsample_exact(t["u1"], u0)
    assert torch.equal(u0, t["u0"])
    assert np.array_equal(harness.to_host(u0, np.uint16), oracle.bloom_upsample(harness.to_host(t["u1"], np.uint16), sz[0]))


# ------------------------------------------------------------------------------- switches, one child process each
def _run_worker(case, out_dir, **switches):
    """tests/kernel_forms_worker.py <case> in a child process whose GRB_* switches are exactly `switches`."""
    env = {k: v for k, v in os.environ.items() if k not in SWITCHES}
    env.update(switches)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-m", "tests.kernel_forms_worker", case, str(out_dir)]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"worker {case} {switches} exited with {r.returncode}:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    seen = next(line for line in r.stdout.splitlines() if line.startswith("switches:"))
    assert seen.split()[1:] == [f"{k}={switches[k]}" for k in SWITCHES if k in switches], seen
    return out_dir


def test_post_exact_fxaa_and_tonemap(cuda, oracle, tmp_path):
    """GRB_POST_EXACT=1: grb_fxaa runs fxaa_kernel (grb_post.cu, -fmad=false): bit for bit the oracle on a UNORM target
    (no transcendental there); decode_srgb's powf allows 1 code on an sRGB target, with test_fxaa's branch-flip bound.
    grb_tonemap at 256x256 (1/4 bloom both ways) then runs tonemap4_kernel: the tonemap bar."""
    f = np.load(_run_worker("post_exact", tmp_path, GRB_POST_EXACT="1") / "post_exact.npz")
    for w, h in ((333, 177), (1280, 720)):
        img = f[f"fxaa_{w}x{h}_in"]
        assert np.array_equal(img, blocky_image(w, h))
        assert np.array_equal(f[f"fxaa_{w}x{h}_unorm"], oracle.fxaa(img, False)), f"fxaa {w}x{h} UNORM"
        got, ref = f[f"fxaa_{w}x{h}_srgb"], oracle.fxaa(img, True)
        d = common.rgba8_channel_diff(got, ref).reshape(h, w, 4)
        flips = (d > 1).any(-1)
        print(f"exact fxaa {w}x{h} sRGB: identical {float((d == 0).mean()):.6f}, branch flips {int(flips.sum())}")
        assert flips.mean() <= 1e-4  # every other pixel within 1 code
        assert (d == 0).mean() > 0.999
    hdr, bloom, lum = f["tonemap_hdr"], f["tonemap_bloom"], f["tonemap_lum"]
    assert _tonemap_form(256, 256, bloom.shape[1], bloom.shape[0], False) == "tile"  # the tile kernel's shape, refused under the switch
    for dynamic in (True, False):
        for srgb in (True, False):
            got = f[f"tonemap_{'dynamic' if dynamic else 'static'}_{'srgb' if srgb else 'unorm'}"]
            ref = oracle.tonemap(hdr, bloom, lum if dynamic else None, 1.25, target_srgb=srgb)
            assert common.rgba8_channel_diff(got, ref).max() <= 1
            assert (got == ref).mean() > 0.999


def test_post_no_tiles_chain_is_bit_exact(cuda, oracle, tmp_path):
    """GRB_POST_NO_TILES=1: no tile kernel and no fused threshold + downsample, so the frame's d0, d2 and u0 are the
    generic kernels': rgb bit for bit the oracle's (given the frame's own luminance), alpha within the log2 bound of
    the threshold.  The luminance itself: log-average bit-exact, exp2 within 4 ulps."""
    _run_worker("chain", tmp_path, GRB_POST_NO_TILES="1")
    for w, h in CHAIN_SIZES:
        f = np.load(tmp_path / f"chain_{w}x{h}.npz")
        hdr = f["hdr"]
        lum, d3_hist = np.zeros(3, np.float32), None
        for i in range(CHAIN_FRAMES):
            assert np.array_equal(f[f"{i}/HDR-main"], hdr)
            ref = oracle.hdr_chain(hdr, lum, d3_hist)
            got_lum = f[f"{i}/average-luminance"]
            _assert_lum(got_lum, ref.lum)
            for name, r in (("downsample-0", ref.d0), ("downsample-2", ref.d2), ("upsample-0", ref.u0)):
                got = f[f"{i}/{name}"]
                assert np.array_equal(got[..., :3], r[..., :3]), f"{w}x{h} frame {i}: {name} rgb"
                common.assert_f16_close(got[..., 3], r[..., 3], f"{w}x{h} frame {i}: {name} alpha", min_identical=0.99, abs_floor=2.0 ** -18)
            # the next frame starts from the device's own state, so each frame isolates that frame's kernels
            lum, d3_hist = got_lum, f[f"{i}/downsample-3"]


@pytest.fixture(scope="module")
def default_chain(tmp_path_factory):
    return _run_worker("chain", tmp_path_factory.mktemp("chain-default"))


@pytest.mark.parametrize("switch", [{"GRB_BLOOM_NO_FUSED_TAIL": "1"}, {"GRB_BLOOM_TAIL_CTAS": "1"}, {"GRB_BLOOM_TAIL_CTAS": "132"}],
                         ids=["no-fused-tail", "tail-ctas-1", "tail-ctas-132"])
def test_bloom_tail_switches_keep_the_frame(cuda, tmp_path, default_chain, switch):
    """The unfused pyramid (separate calls + grb_bloom_upsample_exact) and the fused tail capped to 1 or 132 CTAs give the
    default frame bit for bit: the frame, every pyramid level and average-luminance, 3 frames with d3 history and
    dynamic exposure, at 640x360 and 3840x2160."""
    _run_worker("chain", tmp_path, **switch)
    for w, h in CHAIN_SIZES:
        got, ref = np.load(tmp_path / f"chain_{w}x{h}.npz"), np.load(default_chain / f"chain_{w}x{h}.npz")
        for i in range(CHAIN_FRAMES):
            for name in ("frame", "average-luminance") + PYRAMID:
                assert np.array_equal(got[f"{i}/{name}"].view(np.uint8), ref[f"{i}/{name}"].view(np.uint8)), f"{w}x{h} frame {i}: {name}"


def test_zrange_scan_is_bit_exact(cuda, oracle, tmp_path):
    """GRB_ZRANGE_SCAN=1: the reference's per-slice z-range scan; cluster-range and cluster-bitmask bit for bit the oracle's."""
    f = np.load(_run_worker("zrange", tmp_path, GRB_ZRANGE_SCAN="1") / "zrange.npz")
    cam, _, prep = common.build_lights_case(oracle, 640 / 360, 300, 0.25)
    ref = oracle.cluster_build(cam, prep)
    assert np.array_equal(f["range"], ref.range)
    assert np.array_equal(f["bitmask"], ref.bitmask)


# ----------------------------------------------------------------- host switches read when a viewer bakes its graph
def _taa_fxaa_frames(w, h, n_frames):
    from granite_b200 import viewer

    scene, lights = synth.make_scene(w, h), synth.make_lights(100, aspect=w / h)
    v = viewer.Viewer(w, h, post_aa=viewer.AA_TAA_HIGH_PLUS_FXAA)
    v.set_camera(scene.projection, scene.view)
    v.set_directional(scene.dir_color, scene.dir_direction)
    v.set_lights(lights)
    v.bake()
    assert v.pass_names() == ["gbuffer", "clustering-bindless", "lighting", "mv", "taa-resolve", "bloom-compute", "tonemap", "fxaa"]
    frames = []
    for i in range(n_frames):
        rng = np.random.default_rng(100 + i)  # new motion vectors every frame
        mv = np.zeros((h, w, 2), np.float16)
        m = rng.random((h, w)) < 0.1
        mv[m] = (rng.uniform(-2, 2, size=(int(m.sum()), 2)) / np.array([w, h])).astype(np.float16)
        keep = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, scene.emissive)]
        keep.append(np.ascontiguousarray(mv).view(np.uint32)[..., 0])
        v.render_frame(viewer.Viewer.host_gbuffer(*keep))
        out = np.zeros((h, w), np.uint32)
        v.read_output(out)
        frames.append((out, v.download_image("HDR-resolved")))
    v.close()
    return frames


@pytest.mark.parametrize("switches", [("GRB_NO_ASYNC_CLUSTER",), ("GRB_NO_ASYNC_POST",), ("GRB_NO_ASYNC_CLUSTER", "GRB_NO_ASYNC_POST")],
                         ids=["cluster", "post", "both"])
def test_single_stream_frames_equal_async_frames(cuda, monkeypatch, switches):
    """GRB_NO_ASYNC_CLUSTER / GRB_NO_ASYNC_POST put the cluster build and the post chain on the main stream: 4 frames of
    TAA High + FXAA at 640x360, with new motion vectors every frame, equal the default (asynchronous) viewer's bit for
    bit, output and HDR-resolved."""
    w, h, n = 640, 360, 4
    for k in ("GRB_NO_ASYNC_CLUSTER", "GRB_NO_ASYNC_POST"):
        monkeypatch.delenv(k, raising=False)
    ref = _taa_fxaa_frames(w, h, n)
    for k in switches:
        monkeypatch.setenv(k, "1")
    got = _taa_fxaa_frames(w, h, n)
    for i, ((out, res), (ref_out, ref_res)) in enumerate(zip(got, ref)):
        assert np.array_equal(res, ref_res), f"frame {i}: HDR-resolved"
        assert np.array_equal(out, ref_out), f"frame {i}: output"
