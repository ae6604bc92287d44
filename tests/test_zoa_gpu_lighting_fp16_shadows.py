"""The lighting kernel's RGBA16F and shadowed instantiations against the float64 reference (tests/lighting_ref64.py):
deferred_lighting_kernel<false, true> (grb_deferred_lighting into an RGBA16F HDR-main) on the dense, grazing, odd-width,
partial-block, overflow and subnormal cases, and deferred_lighting_kernel<true, true> (grb_deferred_lighting_shadowed
into RGBA16F) on narrow and wide PCF, on spot footprints past the map's edge and on the cube edge cases, directly and in a viewer frame with light_shadows and
render_target_fp16.  Each is also compared with the fp32 oracle.  The bar's own claims (the oracle meets it, each
deliberate store or sampler error misses it, the cases reach their branches) are pinned on the CPU in
tests/test_lighting_ref64_cpu.py."""
import numpy as np
import pytest
import torch

from granite_b200 import synth
from tests import common
from tests import lighting_ref64 as R
from tests.test_lighting_ref64_cpu import shadowed_case

pytestmark = pytest.mark.gpu

SENTINEL16 = 0x2AB5


def _device(scene, cam, prep):
    from tests.test_zo_gpu_lighting_forms import _device as device

    return device(scene, cam, prep)


def _fp16_case(oracle, name):
    if name == "overflow":
        return R.fp16_overflow_case(oracle)
    if name == "subnormal":
        return R.fp16_subnormal_case(oracle)
    if name == "dense-256x144":
        scene, cam, _, prep = R.dense_case(oracle)
    elif name == "grazing-640x360":
        scene, cam, _, prep, _, _ = R.grazing_case(oracle)
    else:
        w, h = {"odd-641x359": (641, 359), "partial-block-328x184": (328, 184)}[name]
        scene, cam, _, prep = common.build_case(oracle, w, h, 300, 0.25)
    h, w = scene.depth.shape
    em = common.random_hdr_f16(np.random.default_rng(w + prep.n), w, h, scale=0.02, hot=0.001)
    return scene, cam, prep, oracle.cluster_build(cam, prep), em


def _oracle_codes(got, want, what):
    """At most one fp16 code from the oracle per channel; returns the share of identical pixels."""
    d = np.abs(got[..., :3].astype(np.int32) - want[..., :3].astype(np.int32))
    assert d.max() <= 1, f"{what}: {int((d > 1).sum())} channels more than one code from the oracle"
    return float((d.max(-1) == 0).mean())


@pytest.mark.parametrize("name", ["dense-256x144", "grazing-640x360", "odd-641x359", "partial-block-328x184", "overflow", "subnormal"])
def test_fp16_lighting_meets_the_float64_bar(cuda, oracle, name):
    """grb_deferred_lighting into RGBA16F: the generic kernel's <false, true> instantiation."""
    from granite_b200 import harness

    scene, cam, prep, clus, em = _fp16_case(oracle, name)
    gb, dev, gcam = _device(scene, cam, prep)
    hdr = harness.to_dev(em)
    harness.deferred_lighting(gb, gcam, dev, hdr)
    torch.cuda.synchronize()
    got = harness.to_host(hdr, np.uint16)
    share = R.assert_meets_bar(got, R.reference(oracle, scene, cam, prep, clus, emissive=em, fmt=R.RGBA16F), f"fp16 {name}")
    exact = _oracle_codes(got, oracle.deferred_lighting_fp16(scene, cam, prep, clus, em), f"fp16 {name}")
    print(f"fp16 {name}: within the float64 bar (one code admitted on {share:.4f} of the lit channels); {exact:.5f} of the pixels equal the oracle's")
    c = R.codes(got[scene.depth != 0])
    if name == "overflow":
        assert (c == R.half_code(np.inf)).sum() >= 50
    if name == "subnormal":
        assert ((c > 0) & (c < 0x400)).mean() > 0.95


def _shadowed16(gb, gcam, dev, shadows, hdr, rows=None):
    from granite_b200 import harness
    from tests.test_zy_gpu_shadows import _device_shadows

    transforms, maps, res, wide = shadows
    t, table, held = _device_shadows(transforms, maps)
    harness.deferred_lighting_shadowed(gb, gcam, dev, t, table, res, hdr, rows=rows, pcf_wide=wide)
    torch.cuda.synchronize()
    return harness.to_host(hdr, np.uint16)


@pytest.mark.parametrize("case", ["narrow-160x96-res32", "wide-320x180-res64", "spot-edge-narrow-res8", "spot-edge-wide-res8", "cube-res3", "cube-res48"])
def test_shadowed_fp16_lighting(cuda, oracle, case):
    """grb_deferred_lighting_shadowed into RGBA16F: the <true, true> instantiation, against the float64 bar and the
    oracle; row bands are bit-identical to the whole image; with a separate emissive and a sentinel-filled target,
    a band writes every pixel of its rows (sky pixels copied) and leaves the other rows alone."""
    from granite_b200 import capi, harness

    scene, cam, prep, clus, shadows = shadowed_case(oracle, case)
    h, w = scene.depth.shape
    em = common.random_hdr_f16(np.random.default_rng(w + prep.n), w, h, scale=0.02, hot=0.001)
    gb, dev, gcam = _device(scene, cam, prep)
    got = _shadowed16(gb, gcam, dev, shadows, harness.to_dev(em))
    share = R.assert_meets_bar(got, R.reference(oracle, scene, cam, prep, clus, emissive=em, fmt=R.RGBA16F, shadows=shadows), f"shadowed fp16 {case}")
    exact = _oracle_codes(got, oracle.deferred_lighting_fp16(scene, cam, prep, clus, em, shadows=shadows), f"shadowed fp16 {case}")
    print(f"shadowed fp16 {case}: within the float64 bar (one code admitted on {share:.4f} of the lit channels); {exact:.5f} of the pixels equal the oracle's")
    assert not np.array_equal(got, oracle.deferred_lighting_fp16(scene, cam, prep, clus, em)), "the maps must shadow pixels"
    cut = (h // 3) & ~3
    hdr = harness.to_dev(em)
    _shadowed16(gb, gcam, dev, shadows, hdr, rows=(0, cut))
    assert np.array_equal(_shadowed16(gb, gcam, dev, shadows, hdr, rows=(cut, h)), got)
    em_t = harness.to_dev(em)
    gb.struct.emissive = capi.image(em_t, capi.FORMAT_R16G16B16A16_SFLOAT)
    y0, y1 = 5, h - 7
    out = _shadowed16(gb, gcam, dev, shadows, torch.full((h, w, 4), SENTINEL16, dtype=torch.int16, device="cuda"), rows=(y0, y1))
    assert (scene.depth[y0:y1] == 0).any(), "the band must hold sky pixels"
    assert np.array_equal(out[y0:y1], got[y0:y1])
    assert (out[:y0] == SENTINEL16).all() and (out[y1:] == SENTINEL16).all()


def test_viewer_frame_with_shadowed_lights_into_fp16(cuda, oracle):
    """A viewer frame with light_shadows and render_target_fp16: HDR-main against the float64 bar and the oracle's
    shadowed RGBA16F pass, as test_zy_gpu_shadows.py::test_viewer_frame_with_shadowed_lights does for B10G11R11."""
    from granite_b200 import capi, viewer

    w, h, res = 640, 360, 64
    scene, lights = synth.make_scene(w, h), synth.make_lights(200, spot_fraction=0.3, aspect=w / h)
    v = viewer.Viewer(w, h, light_shadows=True, shadow_resolution=res, render_target_fp16=True)
    v.set_camera(scene.projection, scene.view)
    v.set_directional(scene.dir_color, scene.dir_direction)
    v.set_lights(lights)
    cam, prep = common.build_case_for_viewer(oracle, v, scene, lights)
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
    em = common.random_hdr_f16(np.random.default_rng(5), w, h, scale=0.02, hot=0.001)
    planes = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, em)]
    v.render_frame(viewer.Viewer.host_gbuffer(*planes))
    assert v.image("HDR-main").format == capi.FORMAT_R16G16B16A16_SFLOAT
    got = v.download_image("HDR-main")
    clus = oracle.cluster_build(cam, prep)
    transforms = oracle.shadow_transforms(prep)
    assert np.array_equal(v.shadow_transforms(), transforms)
    shadows = (transforms, maps, res, False)
    share = R.assert_meets_bar(got, R.reference(oracle, scene, cam, prep, clus, emissive=em, fmt=R.RGBA16F, shadows=shadows), "viewer fp16 shadowed")
    exact = _oracle_codes(got, oracle.deferred_lighting_fp16(scene, cam, prep, clus, em, shadows=shadows), "viewer fp16 shadowed")
    print(f"viewer fp16 shadowed frame: within the float64 bar (one code admitted on {share:.4f} of the lit channels); {exact:.5f} of the pixels equal the oracle's")
    v.close()
