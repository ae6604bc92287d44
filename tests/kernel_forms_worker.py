"""Child process for tests/test_zp_gpu_kernel_forms.py: runs one case on cuda:0 under the GRB_* switches of its
environment (most are read once per process) and writes what it computed to .npz files in <out_dir>.  It compares
nothing itself; the parent compares the files with the oracle or with the same case run under the default
environment.

    python -m tests.kernel_forms_worker <case> <out_dir>

Cases:
  post_exact  grb_fxaa on a blocky image (333x177, 1280x720; sRGB and UNORM targets) and grb_tonemap at 256x256
              (dynamic / static exposure; sRGB and UNORM targets), inputs saved beside the outputs
  chain       the viewer's post chain on a fixed HDR image (the oracle's lit frame as emissive, no lights, sky
              everywhere) at 640x360 and 3840x2160, 3 frames: the frame, every pyramid level and average-luminance
  zrange      grb_cluster_build for 300 lights (25 % spots) at the 640x360 aspect: cluster-bitmask and cluster-range
  lighting    grb_deferred_lighting on the 640x360 / 300 lights / 25 % spots case
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SWITCHES = ("GRB_POST_EXACT", "GRB_POST_NO_TILES", "GRB_BLOOM_NO_FUSED_TAIL", "GRB_BLOOM_TAIL_CTAS", "GRB_ZRANGE_SCAN", "GRB_LIGHTING_V2",
            "GRB_LIGHTING_1PX")
LIGHTING_CASE = (640, 360, 300, 0.25)
CHAIN_SIZES = ((640, 360), (3840, 2160))
CHAIN_FRAMES = 3
PYRAMID = ("downsample-0", "downsample-1", "downsample-2", "downsample-3", "upsample-2", "upsample-1", "upsample-0")


def blocky_image(w, h):
    """The FXAA input of tests/test_gpu_parity.py::test_fxaa: 8x8 blocks with noise, so the directional taps see edges."""
    rng = np.random.default_rng(w - h)
    base = rng.integers(0, 256, size=(h // 8 + 1, w // 8 + 1, 4), dtype=np.uint8)
    img = np.kron(base, np.ones((8, 8, 1), np.uint8))[:h, :w].copy()
    img = (img.astype(np.int32) + rng.integers(-6, 7, size=img.shape)).clip(0, 255).astype(np.uint8)
    return np.ascontiguousarray(img).view(np.uint32)[..., 0]


def tonemap_inputs(w, h):
    from oracle import pyoracle as oracle
    from tests import common

    rng = np.random.default_rng(w + 11 * h)
    hdr = common.random_hdr(rng, w, h)
    bw, bh = oracle.pyramid_sizes(w, h)[1]
    return hdr, common.random_rgba16f(rng, bw, bh, 0.0, 0.5), np.array([-0.7, 2.0 ** -0.7, 2.0 ** 0.7], np.float32)


def post_exact(out_dir):
    from granite_b200 import harness

    res = {}
    for w, h in ((333, 177), (1280, 720)):
        img = blocky_image(w, h)
        res[f"fxaa_{w}x{h}_in"] = img
        for srgb in (True, False):
            out = torch.zeros((h, w), dtype=torch.int32, device="cuda")
            harness.fxaa(harness.to_dev(img), out, target_srgb=srgb)
            res[f"fxaa_{w}x{h}_{'srgb' if srgb else 'unorm'}"] = harness.to_host(out, np.uint32)
    w, h = 256, 256
    hdr, bloom, lum = tonemap_inputs(w, h)
    res.update(tonemap_hdr=hdr, tonemap_bloom=bloom, tonemap_lum=lum)
    for dynamic in (True, False):
        for srgb in (True, False):
            out = torch.zeros((h, w), dtype=torch.int32, device="cuda")
            harness.tonemap(harness.to_dev(hdr), harness.to_dev(bloom), harness.to_dev(lum) if dynamic else None, out, exposure=1.25, srgb=srgb)
            res[f"tonemap_{'dynamic' if dynamic else 'static'}_{'srgb' if srgb else 'unorm'}"] = harness.to_host(out, np.uint32)
    np.savez(os.path.join(out_dir, "post_exact.npz"), **res)


def chain_hdr(oracle, w, h):
    """The oracle's lit frame for the scene of tests/test_gpu_graph.py::test_chain_is_bit_exact_given_identical_hdr."""
    from tests import common

    scene, cam, lights, prep = common.build_case(oracle, w, h, 50)
    return scene, oracle.deferred_lighting(scene, cam, prep, oracle.cluster_build(cam, prep))


def chain(out_dir):
    from granite_b200 import synth, viewer
    from oracle import pyoracle as oracle

    oracle.build(ref=False)
    for w, h in CHAIN_SIZES:
        scene, hdr = chain_hdr(oracle, w, h)
        sky = synth.Scene(w, h, scene.projection, scene.view, scene.albedo, scene.normal, scene.pbr, np.zeros_like(scene.depth), hdr)
        v = viewer.Viewer(w, h)
        v.set_camera(sky.projection, sky.view)
        v.set_directional(sky.dir_color, sky.dir_direction)
        v.set_lights(synth.make_lights(0))
        v.bake()
        keep = [np.ascontiguousarray(a) for a in (sky.albedo, sky.normal, sky.pbr, sky.depth, sky.emissive)]
        gb = viewer.Viewer.host_gbuffer(*keep)
        res = {"hdr": hdr}
        for i in range(CHAIN_FRAMES):
            v.render_frame(gb if i == 0 else None)
            out = np.zeros((h, w), np.uint32)
            v.read_output(out)
            res[f"{i}/frame"] = out
            res[f"{i}/HDR-main"] = v.download_image("HDR-main")
            for name in PYRAMID:
                res[f"{i}/{name}"] = v.download_image(name)
            res[f"{i}/average-luminance"] = v.download_buffer("average-luminance", np.float32, 3)
        v.close()
        np.savez(os.path.join(out_dir, f"chain_{w}x{h}.npz"), **res)


def zrange(out_dir):
    from granite_b200 import harness
    from oracle import pyoracle as oracle
    from tests import common

    oracle.build(ref=False)
    cam, _, prep = common.build_lights_case(oracle, 640 / 360, 300, 0.25)
    dev = harness.ClusterDevice(prep.records, prep.model, prep.type_mask, prep.z_ranges, prep.params, prep.res)
    dev.build(harness.camera_struct(cam))
    torch.cuda.synchronize()
    got = dev.download()
    np.savez(os.path.join(out_dir, "zrange.npz"), bitmask=got.bitmask, range=got.range)


def lighting_device_case(oracle):
    """Scene, device G-buffer, device cluster (built by grb_cluster_build) and camera of LIGHTING_CASE."""
    from granite_b200 import harness
    from tests import common

    scene, cam, _, prep = common.build_case(oracle, *LIGHTING_CASE)
    dev = harness.ClusterDevice(prep.records, prep.model, prep.type_mask, prep.z_ranges, prep.params, prep.res)
    gcam = harness.camera_struct(cam)
    dev.build(gcam)
    return scene, harness.GBufferDevice(scene), dev, gcam


def lighting(out_dir):
    from granite_b200 import harness
    from oracle import pyoracle as oracle

    oracle.build(ref=False)
    _, gb, dev, gcam = lighting_device_case(oracle)
    hdr = gb.emissive.clone()
    harness.deferred_lighting(gb, gcam, dev, hdr)
    np.savez(os.path.join(out_dir, "lighting.npz"), default=harness.to_host(hdr, np.uint32))


def main():
    case, out_dir = sys.argv[1], sys.argv[2]
    seen = " ".join(f"{k}={os.environ[k]}" for k in SWITCHES if k in os.environ)
    print(f"switches: {seen}", flush=True)
    torch.cuda.set_device(0)
    from granite_b200 import capi

    capi.lib()
    capi.init()
    {"post_exact": post_exact, "chain": chain, "zrange": zrange, "lighting": lighting}[case](out_dir)
    torch.cuda.synchronize()
    print(f"{case}: done", flush=True)


if __name__ == "__main__":
    main()
