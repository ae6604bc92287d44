"""Graph-level GPU parity: whole frames through the C++ host layer (RenderGraph + pass builders +
viewer harness, libgranite_b200_host.so) against the oracle pipeline, over several frames so the
cross-frame state (d3 history, adapted luminance, TAA history) is exercised."""
import os

import numpy as np
import pytest

from granite_b200 import synth
from tests import common

pytestmark = pytest.mark.gpu


def _oracle_frames(oracle, scene, cam, prep, n_frames, dynamic=True, bloom=True, exposure=1.0):
    clus = oracle.cluster_build(cam, prep)
    hdr = oracle.deferred_lighting(scene, cam, prep, clus)
    lum = np.zeros(3, np.float32)  # graph buffers start zeroed (render_graph.cpp:2587)
    d3_hist = None
    frames = []
    for _ in range(n_frames):
        if bloom:
            f = oracle.hdr_chain(hdr, lum, d3_hist, frame_time=1.0 / 60.0, exposure=exposure, dynamic_exposure=dynamic)
            if dynamic:
                lum = f.lum
            d3_hist = f.d3
        else:
            h, w = hdr.shape
            zero = np.zeros((-(-h // 4), -(-w // 4), 4), np.uint16)
            f = type("F", (), {})()
            f.ldr = oracle.tonemap(hdr, zero, None, exposure)
        f.hdr = hdr
        frames.append(f)
    return clus, frames


def _make_viewer(scene, lights, **kw):
    from granite_b200 import viewer

    v = viewer.Viewer(scene.width, scene.height, **kw)
    v.set_camera(scene.projection, scene.view)
    v.set_directional(scene.dir_color, scene.dir_direction)
    v.set_lights(lights)
    v.bake()
    return v


def _host_gb(scene, mv=None):
    from granite_b200 import viewer

    keep = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, scene.emissive)]
    if mv is not None:
        keep.append(np.ascontiguousarray(mv))
    return viewer.Viewer.host_gbuffer(*keep), keep


def test_config1_single_tonemap_pass(cuda, oracle):
    """BASELINE config 1: 256x256, 16 point lights, tonemap only (no bloom, exposure 1)."""
    scene, lights = synth.make_scene(256, 256), synth.make_lights(16, aspect=1.0)
    v = _make_viewer(scene, lights, hdr_bloom=False, dynamic_exposure=False)
    cam, prep = common.build_case_for_viewer(oracle, v, scene, lights)
    clus, frames = _oracle_frames(oracle, scene, cam, prep, 1, dynamic=False, bloom=False)
    assert v.pass_names() == ["gbuffer", "clustering-bindless", "lighting", "bloom-disabled", "tonemap"]
    gb, keep = _host_gb(scene)
    v.render_frame(gb)
    out = np.zeros((256, 256), np.uint32)
    assert v.read_output(out) == (0, 256)
    assert common.max_code_diff_r11g11b10(v.download_image("HDR-main"), frames[0].hdr) <= 1
    assert common.rgba8_channel_diff(out, frames[0].ldr).max() <= 1
    assert (out == frames[0].ldr).mean() > 0.995
    v.close()


@pytest.mark.parametrize("aa", ["none", "taa"])
def test_hdr10_output_frames(cuda, oracle, aa):
    """HDR10 swapchain (scene_viewer_application.cpp:1233-1288): lighting (+ TAA) -> "ui" -> "pq10", no bloom / tonemap.
    The encoder is checked on the HDR image the device itself produced (that image has its own tests)."""
    from granite_b200 import viewer

    w, h = 640, 360
    scene, lights = synth.make_scene(w, h), synth.make_lights(200, aspect=w / h)
    v = _make_viewer(scene, lights, post_aa=viewer.AA_TAA_HIGH if aa == "taa" else viewer.AA_NONE, hdr10_output=True, hdr10_max_cll=1000.0)
    names = v.pass_names()
    assert names[-2:] == ["ui", "pq10"] and "tonemap" not in names and "bloom-compute" not in names
    m = oracle.rec709_to_display_primaries(oracle.BT2020_PRIMARIES)
    assert common.f32_ulp_diff(viewer.rec709_to_display_primaries(oracle.BT2020_PRIMARIES).reshape(4, 4)[:3, :3].reshape(-1),
                               np.asarray(m, np.float32).reshape(4, 4)[:3, :3].reshape(-1)).max() <= 2
    mv = np.zeros((h, w), np.uint32) if aa == "taa" else None
    gb, keep = _host_gb(scene, mv)
    for frame in range(3):
        v.render_frame(gb)
        out = np.zeros((h, w), np.uint32)
        assert v.read_output(out) == (0, h)
        src = v.download_image("HDR-resolved" if aa == "taa" else "HDR-main")
        ui = v.download_image("ui-temporary")
        assert np.all(ui == 0xFF000000)
        ref = oracle.pq10_encode(src, ui, viewer.rec709_to_display_primaries(oracle.BT2020_PRIMARIES), 500.0, 400.0, 1000.0)
        d = common.a2b10g10r10_channel_diff(out, ref)
        assert d.max() <= 1 and (d == 0).mean() > 0.99, f"frame {frame}"
        assert (out >> 30).min() == 3
    v.close()


@pytest.mark.parametrize("w,h,n,spots", [(640, 360, 300, 0.25), (1920, 1080, 1024, 0.0), (3840, 2160, 4096, 0.0)])
def test_full_chain_frames(cuda, oracle, w, h, n, spots):
    scene, lights = synth.make_scene(w, h), synth.make_lights(n, spot_fraction=spots, aspect=w / h)
    v = _make_viewer(scene, lights)
    cam, prep = common.build_case_for_viewer(oracle, v, scene, lights)
    clus, frames = _oracle_frames(oracle, scene, cam, prep, 3)
    assert v.pass_names() == ["gbuffer", "clustering-bindless", "lighting", "bloom-compute", "tonemap"]
    gb, keep = _host_gb(scene)
    out = np.zeros((h, w), np.uint32)
    for i, f in enumerate(frames):
        v.render_frame(gb if i == 0 else None)  # frames 1.. run on the resident G-buffer
        v.read_output(out)
        if i == 0:
            # the clusterer's device buffers are the oracle's, bit for bit
            p, b = v.cluster()
            n32 = p.num_lights_32
            bm = v.download_buffer("cluster-bitmask", np.uint32, 128 * 64 * n32).reshape(64, 128, n32)
            assert np.array_equal(bm, clus.bitmask)
            assert np.array_equal(v.download_buffer("cluster-range", np.uint32).reshape(-1, 2), clus.range)
            got_hdr = v.download_image("HDR-main")
            assert common.max_code_diff_r11g11b10(got_hdr, f.hdr) <= 1
        # pyramid / luminance / output: the lighting differs from the oracle by <= 1 code on a few
        # pixels, which the chain then propagates; bound the deviation instead of bit-comparing
        got_d3 = v.download_image("downsample-3").view(np.float16).astype(np.float32)
        ref_d3 = f.d3.view(np.float16).astype(np.float32)
        assert np.abs(got_d3 - ref_d3).max() <= 2e-2 * max(1.0, np.abs(ref_d3).max())
        lum = v.download_buffer("average-luminance", np.float32, 3)
        assert abs(lum[0] - f.lum[0]) < 2e-4
        d = common.rgba8_channel_diff(out, f.ldr)
        assert d.max() <= 2, f"frame {i}"
        assert (d <= 1).mean() > 0.9999 and (out == f.ldr).mean() > 0.99, f"frame {i}"
    v.close()


def test_chain_is_bit_exact_given_identical_hdr(cuda, oracle):
    """Feed the ORACLE's HDR image through the graph's post chain (emissive = that image, no lights,
    black directional light, sky everywhere): every level must then match the oracle bit for bit
    except the log2 alpha of the threshold (<= 1 fp16 ulp) and what descends from it."""
    w, h = 640, 360
    os.environ["GRB_BLOOM_KEEP_THRESHOLD"] = "1"
    scene, cam, lights, prep = common.build_case(oracle, w, h, 50)
    clus = oracle.cluster_build(cam, prep)
    hdr = oracle.deferred_lighting(scene, cam, prep, clus)
    sky = synth.Scene(w, h, scene.projection, scene.view, scene.albedo, scene.normal, scene.pbr, np.zeros_like(scene.depth), hdr)
    v = _make_viewer(sky, synth.make_lights(0))
    gb, keep = _host_gb(sky)
    lum = np.zeros(3, np.float32)
    d3_hist = None
    out = np.zeros((h, w), np.uint32)
    for i in range(3):
        f = oracle.hdr_chain(hdr, lum, d3_hist)
        lum, d3_hist = f.lum, f.d3
        v.render_frame(gb if i == 0 else None)
        v.read_output(out)
        assert np.array_equal(v.download_image("HDR-main"), hdr)
        t = v.download_image("threshold")  # materialised because GRB_BLOOM_KEEP_THRESHOLD is set below
        common.assert_f16_close(t, f.t, "threshold", min_identical=0.99, abs_floor=2.0 ** -18)
        # the tile kernels are within 1 fp16 ulp per level; a handful of texels may carry 2 through three levels
        for name, ref, ulps in [("downsample-0", f.d0, 1), ("downsample-2", f.d2, 2), ("upsample-0", f.u0, 2)]:
            got = v.download_image(name)
            d = common.f16_ulp_diff(got[..., :3], ref[..., :3])
            assert d.max() <= ulps and (d == 0).mean() > 0.97, name
        d = common.rgba8_channel_diff(out, f.ldr)
        assert d.max() <= 1 and (d == 0).mean() > 0.999
    os.environ.pop("GRB_BLOOM_KEEP_THRESHOLD", None)
    v.close()


@pytest.mark.parametrize("w,h,n", [(640, 360, 100), (3840, 2160, 4096)])
def test_taa_fxaa_chain(cuda, oracle, w, h, n):
    """BASELINE config 5 wiring: TAA (quality 2) before the HDR chain, FXAA after it, with history
    (3 frames; the second case is config 5 itself: 3840x2160, 4096 lights)."""
    from granite_b200 import viewer

    scene, lights = synth.make_scene(w, h), synth.make_lights(n, aspect=w / h)
    rng = np.random.default_rng(5)
    mv = np.zeros((h, w, 2), np.float16)
    m = rng.random((h, w)) < 0.1
    mv[m] = (rng.uniform(-2, 2, size=(int(m.sum()), 2)) / np.array([w, h])).astype(np.float16)
    mv32 = np.ascontiguousarray(mv).view(np.uint32)[..., 0]
    v = _make_viewer(scene, lights, post_aa=viewer.AA_TAA_HIGH_PLUS_FXAA)
    assert v.pass_names() == ["gbuffer", "clustering-bindless", "lighting", "mv", "taa-resolve", "bloom-compute", "tonemap", "fxaa"]
    gb, keep = _host_gb(scene, mv32)
    hist = None
    lum = np.zeros(3, np.float32)
    d3_hist = None
    out = np.zeros((h, w), np.uint32)
    cameras = []
    for i in range(3):
        v.render_frame(gb)
        v.read_output(out)
        # The frame is clustered and lit with the JITTERED projection of this frame
        # (scene_viewer_application.cpp:1431-1432); the history is reprojected with the unjittered
        # matrices (temporal.cpp:239-243).  Both are taken from the host layer (its mat4 inverse differs
        # from the oracle's by an ulp, and matrices are inputs of the path).
        cam, prep = common.build_case_for_viewer(oracle, v, scene, lights)
        cameras.append(np.array(list(cam.view_projection), np.float32))
        clus = oracle.cluster_build(cam, prep)
        hdr = oracle.deferred_lighting(scene, cam, prep, clus)
        got_hdr = v.download_image("HDR-main")
        assert common.max_code_diff_r11g11b10(got_hdr, hdr) <= 1, f"frame {i}"
        reproj = v.taa_reprojection()
        # oracle continues from the GPU's own lit image so TAA/FXAA parity is isolated from lighting ulps
        res_c, res_h = oracle.taa_resolve(got_hdr, scene.depth, mv.view(np.uint16), hist, reproj, 2)
        hist = res_h
        f = oracle.hdr_chain(res_c, lum, d3_hist)
        lum, d3_hist = f.lum, f.d3
        ldr = oracle.fxaa(f.ldr, True)
        got_res = v.download_image("HDR-resolved")
        # 1 code, or 2^-16 absolute for the nearly black pixels of a real frame (a code is 1e-6 there)
        common.assert_r11g11b10_close(got_res, res_c, f"frame {i}: HDR-resolved", min_identical=0.97)
        d = common.rgba8_channel_diff(out, ldr)
        assert (d <= 1).mean() > 0.999, f"frame {i}"
    # the 16-phase jitter moves the projection every frame
    assert not np.array_equal(cameras[0], cameras[1]) and not np.array_equal(cameras[1], cameras[2])
    v.close()


def test_pipelined_io_frames_equal_serial_frames(cuda):
    """Uploads on the side stream into ping-pong images + asynchronous readbacks must give the
    same frames as the plain upload -> compute -> readback sequence."""
    import torch

    w, h = 640, 360
    scene, lights = synth.make_scene(w, h), synth.make_lights(200, spot_fraction=0.25, aspect=w / h)
    gb, keep = _host_gb(scene)
    ref = []
    v = _make_viewer(scene, lights)
    for _ in range(4):
        v.render_frame(gb)
        out = np.zeros((h, w), np.uint32)
        v.read_output(out)
        ref.append(out)
    v.close()
    vp = _make_viewer(scene, lights, pipelined_io=True)
    outs = [torch.zeros((h, w), dtype=torch.int32).pin_memory() for _ in range(4)]
    for i in range(4):
        vp.render_frame(gb)
        vp.read_output_async(outs[i])
        vp.wait_outputs(1)
    vp.wait_outputs(0)
    for i in range(4):
        assert np.array_equal(outs[i].numpy().view(np.uint32), ref[i]), f"frame {i}"
    with pytest.raises(Exception):
        vp.render_frame(None)
    vp.close()
