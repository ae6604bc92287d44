"""SMAA on the GPU (granite_b200/csrc/grb_smaa.cu through the C ABI) against the oracle and against the
reference-shader fixture.  Sorted last.  Also verified without a GPU: their source, compiled for the CPU and compared bit for bit with
the oracle and the reference shaders (tests/test_smaa_kernel_source_cpu.py); what this file adds on hardware is the
launch configuration, the vector loads and CUDA's powf in the sRGB round trip of the blend pass."""
import os

import numpy as np
import pytest

from tests import common
from tests.test_oracle_ref_smaa import smaa_test_image

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _gpu_smaa(img, area, search, q, srgb=True, rows=None):
    import torch

    from granite_b200 import harness

    h, w = img.shape
    color = harness.to_dev(img)
    edges = torch.zeros((h, w, 2), dtype=torch.uint8, device="cuda")
    weights = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    out = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    harness.smaa_edge_detection(color, q, edges, rows=rows)
    harness.smaa_blend_weights(edges, harness.to_dev(np.ascontiguousarray(area)), harness.to_dev(np.ascontiguousarray(search).reshape(16, 64)), q, weights, rows=rows)
    harness.smaa_neighborhood_blend(color, weights, out, target_srgb=srgb, rows=rows)
    torch.cuda.synchronize()
    return edges.cpu().numpy(), harness.to_host(weights, np.uint32), harness.to_host(out, np.uint32)


def test_cuda_smaa_vs_reference_shader_fixture(cuda):
    f = np.load(os.path.join(GOLDEN, "refsmaa_160x96.npz"))
    for q in range(4):
        e, wg, out = _gpu_smaa(np.ascontiguousarray(f["color"]), f["area"], f["search"], q)
        assert np.array_equal(e, f[f"q{q}_edges"]), f"edges q{q}"
        assert np.array_equal(wg, f[f"q{q}_weights"]), f"weights q{q}"
        d = common.rgba8_channel_diff(out, f[f"q{q}_out"])
        assert d.max() <= 1 and (d == 0).mean() > 0.995, f"blend q{q}"  # CUDA powf vs glibc in decode_srgb


@pytest.mark.parametrize("w,h", [(333, 177), (1920, 1080), (3840, 2160)])
def test_cuda_smaa_vs_oracle(cuda, oracle, w, h):
    f = np.load(os.path.join(GOLDEN, "refsmaa_160x96.npz"))
    img = smaa_test_image(w, h, w + h)
    q = 3 if w < 3000 else 2
    e, wg, out = _gpu_smaa(img, f["area"], f["search"], q)
    e_o = oracle.smaa_edge(img, q)
    assert np.array_equal(e, e_o)
    w_o = oracle.smaa_weights(e_o, f["area"], f["search"], q)
    assert np.array_equal(wg, w_o)
    d = common.rgba8_channel_diff(out, oracle.smaa_blend(img, w_o))
    assert d.max() <= 1 and (d == 0).mean() > 0.995
    # a row band of the last pass writes its rows only, with the values of the whole image (its inputs being complete)
    import torch

    from granite_b200 import harness

    band = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    harness.smaa_neighborhood_blend(harness.to_dev(img), harness.to_dev(wg), band, target_srgb=True, rows=(16, h - 24))
    band = harness.to_host(band, np.uint32)
    assert np.array_equal(band[16:h - 24], out[16:h - 24]) and not band[:16].any() and not band[h - 24:].any()


def test_viewer_frame_with_smaa(cuda, oracle):
    """Whole frame through the host layer: lighting -> bloom -> tonemap -> smaa-edge / smaa-weights / smaa-blend
    (host/post/smaa.cpp).  The three SMAA passes are checked on the tonemapped image the device itself produced."""
    from granite_b200 import synth, viewer

    f = np.load(os.path.join(GOLDEN, "refsmaa_160x96.npz"))
    w, h = 640, 360
    scene, lights = synth.make_scene(w, h), synth.make_lights(200, aspect=w / h)
    v = viewer.Viewer(w, h, post_aa=viewer.AA_SMAA_HIGH)
    v.set_camera(scene.projection, scene.view)
    v.set_directional(scene.dir_color, scene.dir_direction)
    v.set_lights(lights)
    v.set_smaa_lookup_textures(f["area"], f["search"])
    v.bake()
    assert v.pass_names()[-3:] == ["smaa-edge", "smaa-weights", "smaa-blend"]
    keep = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, scene.emissive)]
    gb = viewer.Viewer.host_gbuffer(*keep)
    for _ in range(2):
        v.render_frame(gb)
        out = np.zeros((h, w), np.uint32)
        assert v.read_output(out) == (0, h)
        ldr = v.download_image("tonemapped")
        e = oracle.smaa_edge(ldr, 2)
        assert np.array_equal(np.ascontiguousarray(v.download_image("smaa-edge")).view(np.uint8).reshape(h, w, 2), e)
        wg = oracle.smaa_weights(e, f["area"], f["search"], 2)
        assert np.array_equal(v.download_image("smaa-weights"), wg)
        d = common.rgba8_channel_diff(out, oracle.smaa_blend(ldr, wg))
        assert d.max() <= 1 and (d == 0).mean() > 0.995
    v.close()
