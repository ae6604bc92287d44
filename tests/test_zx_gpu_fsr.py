"""FSR 1 on the GPU (granite_b200/csrc/grb_fsr.cu through the C ABI, and a viewer frame with resolution_scale < 1) against the
oracle and the reference-shader fixture.  Sorted after the other GPU tests.  Also verified
without a GPU: their source, compiled for the CPU, bit for
bit against the oracle (tests/test_fsr_kernel_source_cpu.py), and the oracle bit for bit against the reference's two shaders
(tests/test_oracle_ref_fsr.py).  What this file adds on hardware: the launch configuration and CUDA's powf in the sRGB
stores (<= 1 code where a target is sRGB; UNORM targets must be exact)."""
import os

import numpy as np
import pytest

from tests import common
from tests.test_oracle_ref_smaa import smaa_test_image

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _gpu_upscale(img, wo, ho, srgb=False, rows=None):
    import torch

    from granite_b200 import harness

    out = torch.zeros((ho, wo), dtype=torch.int32, device="cuda")
    harness.fsr_upscale(harness.to_dev(img), out, target_srgb=srgb, rows=rows)
    torch.cuda.synchronize()
    return harness.to_host(out, np.uint32)


def _gpu_sharpen(img, stops=0.5, srgb=True, rows=None):
    import torch

    from granite_b200 import harness

    out = torch.zeros(img.shape, dtype=torch.int32, device="cuda")
    harness.fsr_sharpen(harness.to_dev(img), out, sharpness_stops=stops, srgb=srgb, rows=rows)
    torch.cuda.synchronize()
    return harness.to_host(out, np.uint32)


def _close_srgb(a, b):
    d = common.rgba8_channel_diff(a, b)
    assert d.max() <= 1 and (d == 0).mean() > 0.995  # CUDA powf vs glibc in the sRGB encode / decode


def test_cuda_fsr_vs_reference_shader_fixture(cuda):
    f = np.load(os.path.join(GOLDEN, "reffsr_160x96_to_240x144.npz"))
    img = np.ascontiguousarray(f["color"])
    up = _gpu_upscale(img, 240, 144)
    assert np.array_equal(up, f["upscaled_unorm"])
    _close_srgb(_gpu_upscale(img, 240, 144, srgb=True), f["upscaled_srgb"])
    assert np.array_equal(_gpu_sharpen(up, srgb=False), f["sharpened_unorm"])
    _close_srgb(_gpu_sharpen(up, srgb=True), f["sharpened_srgb"])


@pytest.mark.parametrize("w,h,wo,ho", [(333, 177, 500, 266), (1280, 720, 1920, 1080), (2880, 1620, 3840, 2160)])
def test_cuda_fsr_vs_oracle(cuda, oracle, w, h, wo, ho):
    img = smaa_test_image(w, h, w + h)
    up = _gpu_upscale(img, wo, ho)
    up_o = oracle.fsr_upscale(img, (wo, ho))
    assert np.array_equal(up, up_o)
    assert np.array_equal(_gpu_sharpen(up, srgb=False), oracle.fsr_sharpen(up_o, srgb=False))
    _close_srgb(_gpu_sharpen(up, srgb=True), oracle.fsr_sharpen(up_o, srgb=True))
    # a row band writes its rows only, with the values of the whole image
    band = _gpu_upscale(img, wo, ho, rows=(16, ho - 24))
    assert np.array_equal(band[16:ho - 24], up[16:ho - 24]) and not band[:16].any() and not band[ho - 24:].any()


def test_viewer_frame_with_fsr_upscaling(cuda, oracle):
    """Whole frame through the host layer at "resolutionScale" 0.75: lighting -> bloom -> tonemap at 480 x 270, then
    post-scale-output-scale / -sharpen to 640 x 360 (host/post/aa.cpp).  The two FSR passes are checked on the tonemapped
    image the device itself produced."""
    from granite_b200 import synth, viewer

    W, H = 640, 360
    v = viewer.Viewer(W, H, resolution_scale=0.75, resolution_scale_sharpen=True)
    w, h = v.render_size()
    assert (w, h) == (480, 270)
    scene, lights = synth.make_scene(w, h), synth.make_lights(200, aspect=w / h)
    v.set_camera(scene.projection, scene.view)
    v.set_directional(scene.dir_color, scene.dir_direction)
    v.set_lights(lights)
    v.bake()
    assert v.pass_names()[-2:] == ["post-scale-output-scale", "post-scale-output-sharpen"]
    keep = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, scene.emissive)]
    gb = viewer.Viewer.host_gbuffer(*keep)
    for _ in range(2):
        v.render_frame(gb)
        out = np.zeros((H, W), np.uint32)
        assert v.read_output(out) == (0, H)
        ldr = v.download_image("tonemapped")
        assert ldr.shape == (h, w)
        up = oracle.fsr_upscale(ldr, (W, H))
        assert np.array_equal(v.download_image("post-scale-output-scale"), up)
        _close_srgb(out, oracle.fsr_sharpen(up, 0.5, srgb=True))
    v.close()
