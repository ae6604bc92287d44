""""renderTargetFp16" on the GPU: lighting into, and bloom threshold / tonemap / TAA out of, an R16G16B16A16_SFLOAT HDR-main
(the fp16 instantiations of the generic kernels, through the C ABI) against the oracle, and a viewer frame with
render_target_fp16.  Sorted after the other GPU tests.  Also verified without
a GPU: the oracle's fp16 paths against the reference's own shaders with the shims' HDR
sampler / blend in that format (tests/test_oracle_ref_fp16_hdr.py); the kernels' B10G11R11 instantiations (same source, the
texel decode apart) are the ones the other GPU tests run."""
import numpy as np
import pytest

from tests import common
from tests import lighting_ref64 as R

pytestmark = pytest.mark.gpu


def _f16_code_diff(a, b):
    """fp16 bit patterns of non-negative finite values are ordered like the values."""
    return np.abs(a.astype(np.int32) - b.astype(np.int32))


@pytest.mark.parametrize("w,h,n,spots", [pytest.param(160, 96, 300, 0.25, id="160x96-300-25pct-spots"), pytest.param(1920, 1080, 1024, 0.0, id="C2-1080p-1024")])
def test_cuda_lighting_into_fp16_hdr(cuda, oracle, w, h, n, spots):
    import torch

    from granite_b200 import harness
    from tests.test_gpu_parity import _cluster

    scene, cam, lights, prep = common.build_case(oracle, w, h, n, spots)
    clus = oracle.cluster_build(cam, prep)
    rng = np.random.default_rng(w + n)
    em16 = common.random_hdr_f16(rng, w, h, scale=0.02, hot=0.001)
    ref = oracle.deferred_lighting_fp16(scene, cam, prep, clus, em16)
    dev, gcam = _cluster(cuda, oracle, cam, prep)
    gb = harness.GBufferDevice(scene)
    hdr = harness.to_dev(em16)
    harness.deferred_lighting(gb, gcam, dev, hdr)
    torch.cuda.synchronize()
    got = harness.to_host(hdr, np.uint16)
    sky = scene.depth == 0
    assert np.array_equal(got[sky], em16[sky]) and np.array_equal(got[..., 3], em16[..., 3])
    d = _f16_code_diff(got[..., :3], ref[..., :3])
    exact = float((d.max(-1) == 0).mean())
    print(f"fp16 lighting: max code diff {int(d.max())}, exact pixels {exact:.4f}")
    assert d.max() <= 2 and (d <= 1).mean() > 0.9999 and exact > 0.8
    share = R.assert_meets_bar(got, R.reference(oracle, scene, cam, prep, clus, emissive=em16, fmt=R.RGBA16F), f"fp16 {w}x{h}")
    print(f"fp16 lighting: within the float64 bar; it admits one code on {share:.4f} of the lit channels")
    # row bands are bit-invariant
    cut = (h // 3) & ~3
    hdr2 = harness.to_dev(em16)
    harness.deferred_lighting(gb, gcam, dev, hdr2, rows=(0, cut))
    harness.deferred_lighting(gb, gcam, dev, hdr2, rows=(cut, h))
    assert torch.equal(hdr, hdr2)


@pytest.mark.parametrize("w,h", [(256, 256), (1001, 517), (1920, 1080)])
def test_cuda_post_passes_over_fp16_hdr(cuda, oracle, w, h):
    import torch

    from granite_b200 import harness
    from tests.test_gpu_parity import _taa_inputs

    rng = np.random.default_rng(w * 5 + h)
    hdr = common.random_hdr_f16(rng, w, h)
    hdr_t = harness.to_dev(hdr)
    lum = np.array([0.3, 2.0 ** 0.3, 2.0 ** -0.3], np.float32)
    # K7: rgb has no transcendental
    ow, oh = oracle.pyramid_sizes(w, h)[0]
    out = harness.new_rgba16f(ow, oh)
    harness.bloom_threshold(hdr_t, harness.to_dev(lum), out)
    got, ref = harness.to_host(out, np.uint16), oracle.bloom_threshold(hdr, lum, (ow, oh))
    assert np.array_equal(got[..., :3], ref[..., :3]) and common.f16_ulp_diff(got[..., 3], ref[..., 3]).max() <= 1
    # K11
    bw, bh = oracle.pyramid_sizes(w, h)[1]
    bloom = common.random_rgba16f(rng, bw, bh, 0.0, 0.5)
    ldr = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    harness.tonemap(hdr_t, harness.to_dev(bloom), harness.to_dev(lum), ldr, exposure=1.25)
    got, ref = harness.to_host(ldr, np.uint32), oracle.tonemap(hdr, bloom, lum, 1.25)
    assert common.rgba8_channel_diff(got, ref).max() <= 1 and (got == ref).mean() > 0.999
    # K13: the exact kernel, first frame and steady state
    _, depth, mv, hist, reproj = _taa_inputs(rng, w, h)
    hdr2 = common.random_hdr_f16(rng, w, h, scale=2.0)
    oc, ohist = torch.zeros((h, w), dtype=torch.int32, device="cuda"), harness.new_rgba16f(w, h)
    ref_c, ref_h = oracle.taa_resolve(hdr2, depth, mv, None, reproj, 2)
    harness.taa_resolve(harness.to_dev(hdr2), None, None, None, None, 2, oc, ohist)
    assert np.array_equal(harness.to_host(oc, np.uint32), ref_c) and np.array_equal(harness.to_host(ohist, np.uint16), ref_h)
    for q in (0, 1, 2):
        ref_c, ref_h = oracle.taa_resolve(hdr2, depth, mv, hist, reproj, q)
        harness.taa_resolve(harness.to_dev(hdr2), harness.to_dev(depth), harness.to_dev(mv.reshape(h, w, 2)).view(torch.int32).reshape(h, w),
                            harness.to_dev(hist), reproj, q, oc, ohist)
        assert np.array_equal(harness.to_host(oc, np.uint32), ref_c) and np.array_equal(harness.to_host(ohist, np.uint16), ref_h)


def test_viewer_frame_with_fp16_render_target(cuda, oracle):
    """Whole frame through the host layer with render_target_fp16: the G-buffer's emissive is RGBA16F, HDR-main RGBA16F, the
    bloom chain takes the unfused threshold + downsample pair (the TMA tile kernel reads B10G11R11 only)."""
    from granite_b200 import capi, synth, viewer

    w, h = 640, 360
    scene, lights = synth.make_scene(w, h), synth.make_lights(200, spot_fraction=0.2, aspect=w / h)
    v = viewer.Viewer(w, h, render_target_fp16=True)
    v.set_camera(scene.projection, scene.view)
    v.set_directional(scene.dir_color, scene.dir_direction)
    v.set_lights(lights)
    v.bake()
    em16 = common.random_hdr_f16(np.random.default_rng(2), w, h, scale=0.02, hot=0.001)
    keep = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, em16)]
    gb = viewer.Viewer.host_gbuffer(*keep)
    cam, prep = common.build_case_for_viewer(oracle, v, scene, lights)
    clus = oracle.cluster_build(cam, prep)
    hdr_ref = oracle.deferred_lighting_fp16(scene, cam, prep, clus, em16)
    ref64 = R.reference(oracle, scene, cam, prep, clus, emissive=em16, fmt=R.RGBA16F)
    lum, d3 = np.zeros(3, np.float32), None
    out = np.zeros((h, w), np.uint32)
    for i in range(2):
        v.render_frame(gb)
        v.read_output(out)
        img = v.image("HDR-main")
        assert img.format == capi.FORMAT_R16G16B16A16_SFLOAT
        hdr_dev = v.download_image("HDR-main")
        d = _f16_code_diff(hdr_dev[..., :3], hdr_ref[..., :3])
        assert d.max() <= 2 and (d.max(-1) == 0).mean() > 0.8
        share = R.assert_meets_bar(hdr_dev, ref64, f"viewer fp16 frame {i}")
        print(f"viewer fp16 frame {i}: within the float64 bar; it admits one code on {share:.4f} of the lit channels")
        # the post chain is checked on the HDR image the device itself produced
        f = oracle.hdr_chain(hdr_dev, lum, d3)
        lum, d3 = f.lum, f.d3
        dd = common.rgba8_channel_diff(out, f.ldr)
        assert (dd <= 1).mean() > 0.999, f"frame {i}"
    v.close()
