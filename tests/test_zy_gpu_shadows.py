"""Shadowed positional lights on the GPU (grb_deferred_lighting_shadowed through the C ABI, and a viewer frame with
clustered_lights_shadows) against the oracle and the reference-shader fixture.  Sorted after the other GPU tests.
Also verified without a GPU:
the comparison samplers' source, compiled for the CPU, bit for bit against the oracle (tests/test_shadow_source_cpu.py);
the oracle against the reference's own shadowed clustering.frag (tests/test_oracle_ref_light_shadows.py); the host
clusterer's shadow transforms against the reference's math.  What this file adds on hardware: the shadow branch inside
the warp-uniform light walk of the generic lighting kernel, the pointer table, the upload."""
import os

import numpy as np
import pytest

from tests import common
from tests.test_oracle_ref_light_shadows import shadow_case

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _device_shadows(transforms, maps):
    import torch

    held = [None if m is None else torch.from_numpy(np.ascontiguousarray(m).view(np.int16)).cuda() for m in maps]
    table = torch.tensor([0 if t is None else t.data_ptr() for t in held] or [0], dtype=torch.int64, device="cuda")
    t = torch.from_numpy(np.ascontiguousarray(transforms if len(transforms) else np.zeros((1, 16), np.float32))).cuda()
    return t, table, held


def _gpu_shadowed(cuda, oracle, scene, cam, prep, transforms, maps, res, rows=None, pcf_wide=False):
    import torch

    from granite_b200 import harness
    from tests.test_gpu_parity import _cluster

    dev, gcam = _cluster(cuda, oracle, cam, prep)
    gb = harness.GBufferDevice(scene)
    hdr = gb.emissive.clone()
    t, table, held = _device_shadows(transforms, maps)
    harness.deferred_lighting_shadowed(gb, gcam, dev, t, table, res, hdr, rows=rows, pcf_wide=pcf_wide)
    torch.cuda.synchronize()
    return harness.to_host(hdr, np.uint32)


def _compare(got, ref, floor):
    assert common.max_code_diff_r11g11b10(got, ref) <= 1
    exact = float((got == ref).mean())
    print(f"shadowed lighting exact-match fraction: {exact:.5f}")
    assert exact > floor


@pytest.mark.parametrize("w,h,n,spots,res", [pytest.param(160, 96, 300, 0.25, 32, id="160x96-300-25pct-spots-res32"),
                                             pytest.param(641, 359, 300, 0.5, 64, id="641x359-300-50pct-spots-res64"),
                                             pytest.param(1920, 1080, 1024, 0.25, 128, id="C2-1080p-1024-res128")])
def test_cuda_shadowed_lighting_vs_oracle(cuda, oracle, w, h, n, spots, res):
    scene, cam, prep, clus, transforms, maps = shadow_case(oracle, w, h, n, spots, res)
    ref = oracle.deferred_lighting_shadowed(scene, cam, prep, clus, transforms, maps, res)
    got = _gpu_shadowed(cuda, oracle, scene, cam, prep, transforms, maps, res)
    sky = scene.depth == 0
    assert np.array_equal(got[sky], scene.emissive[sky]), "sky pixels must keep the attachment value"
    _compare(got, ref, 0.97)
    assert (ref != oracle.deferred_lighting(scene, cam, prep, clus)).mean() > 0.001, "the case must actually shadow pixels"
    # no maps at all == the unshadowed pass of the same kernel family
    none = _gpu_shadowed(cuda, oracle, scene, cam, prep, transforms, [None] * prep.n, res)
    _compare(none, oracle.deferred_lighting(scene, cam, prep, clus), 0.97)
    # row bands are bit-invariant
    cut = (h // 3) & ~3
    a = _gpu_shadowed(cuda, oracle, scene, cam, prep, transforms, maps, res, rows=(0, cut))
    b = _gpu_shadowed(cuda, oracle, scene, cam, prep, transforms, maps, res, rows=(cut, h))
    assert np.array_equal(a[:cut], got[:cut]) and np.array_equal(b[cut:], got[cut:])


def test_cuda_wide_pcf_vs_oracle(cuda, oracle):
    """SHADOW_MAP_PCF_KERNEL_WIDE: the 6 x 6 kernel of the spot lights (its exp2 is CUDA's on hardware: lighting bar)."""
    scene, cam, prep, clus, transforms, maps = shadow_case(oracle, 320, 180, 300, 0.6, 64)
    ref = oracle.deferred_lighting_shadowed(scene, cam, prep, clus, transforms, maps, 64, pcf_wide=True)
    _compare(_gpu_shadowed(cuda, oracle, scene, cam, prep, transforms, maps, 64, pcf_wide=True), ref, 0.97)


def test_cuda_shadowed_lighting_vs_reference_shader_fixture(cuda, oracle):
    f = np.load(os.path.join(GOLDEN, "reflight_shadows_160x96_300.npz"))
    scene, cam, prep, clus, transforms, maps = shadow_case(oracle, 160, 96, 300, 0.25, 32)
    assert np.array_equal(scene.depth, f["depth"]) and np.array_equal(transforms, f["transforms"])
    _compare(_gpu_shadowed(cuda, oracle, scene, cam, prep, transforms, maps, 32), f["ref_hdr"], 0.97)


def test_viewer_frame_with_shadowed_lights(cuda, oracle):
    """Whole frame through the host layer: the clusterer computes and uploads the shadow transforms and the map
    pointers in its own sorted order; HDR-main is compared with the oracle's shadowed pass."""
    import torch

    from granite_b200 import synth, viewer

    w, h, res = 640, 360, 64
    scene, lights = synth.make_scene(w, h), synth.make_lights(200, spot_fraction=0.3, aspect=w / h)
    v = viewer.Viewer(w, h, light_shadows=True, shadow_resolution=res)
    v.set_camera(scene.projection, scene.view)
    v.set_directional(scene.dir_color, scene.dir_direction)
    v.set_lights(lights)
    cam, prep = common.build_case_for_viewer(oracle, v, scene, lights)
    # the synthetic lights come sorted front to back, so cluster order = input order minus the culled ones
    keep = oracle.visible_lights(cam, lights)
    assert int(keep.sum()) == prep.n
    maps = common.make_shadow_maps(prep, res)
    held = [None if m is None else torch.from_numpy(np.ascontiguousarray(m).view(np.int16)).cuda() for m in maps]
    by_input, k = [], 0
    for visible in keep:
        by_input.append(0 if (not visible or held[k] is None) else held[k].data_ptr())
        k += 1 if visible else 0
    v.set_light_shadow_maps(by_input)
    v.bake()
    keep = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, scene.emissive)]
    v.render_frame(viewer.Viewer.host_gbuffer(*keep))
    out = np.zeros((h, w), np.uint32)
    v.read_output(out)
    clus = oracle.cluster_build(cam, prep)
    transforms = oracle.shadow_transforms(prep)
    assert np.array_equal(v.shadow_transforms(), transforms)
    ref = oracle.deferred_lighting_shadowed(scene, cam, prep, clus, transforms, maps, res)
    _compare(v.download_image("HDR-main"), ref, 0.97)
    v.close()
