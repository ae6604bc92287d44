"""Volumetric-decal binning on the GPU (granite_b200/csrc/grb_decal.cu through the C ABI, and a viewer frame with
volumetric_decals) against the oracle.  Sorted after the other GPU tests.  Also verified without
a GPU: the kernels' source compiled for the CPU, bit for bit with the oracle,
and the oracle bit for bit with the reference's shader (tests/test_decal_cpu.py)."""
import ctypes as C

import numpy as np
import pytest

from tests import common
from tests.test_decal_cpu import _camera, make_decals

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,res", [(1, (16, 8)), (33, (128, 64)), (300, (128, 64)), (4096, (128, 64))])
def test_cuda_decal_binning_vs_oracle(cuda, oracle, n, res):
    import torch

    from granite_b200 import capi, harness

    cam = _camera(oracle)
    mvps = oracle.decal_mvps(cam, make_decals(n))
    rx, ry = res
    params = capi.GrbClusterParameters()
    params.resolution_xy[0], params.resolution_xy[1] = rx, ry
    params.inv_resolution_xy[0], params.inv_resolution_xy[1] = float(np.float32(1.0 / rx)), float(np.float32(1.0 / ry))
    d_mvps = harness.to_dev(mvps)
    boxes = torch.zeros((n, 4), dtype=torch.float32, device="cuda")
    bm = torch.zeros((ry, rx, (n + 31) // 32), dtype=torch.int32, device="cuda")
    capi.check(capi.lib().grb_cluster_decal_binning(C.byref(params), C.c_void_p(d_mvps.data_ptr()), n, C.c_void_p(boxes.data_ptr()), C.c_void_p(bm.data_ptr()),
                                                    capi.stream_ptr()), "grb_cluster_decal_binning")
    torch.cuda.synchronize()
    assert np.array_equal(harness.to_host(bm, np.uint32), oracle.decal_binning(res, mvps))


def test_viewer_frame_with_decals(cuda, oracle):
    from granite_b200 import synth, viewer

    w, h = 640, 360
    scene, lights = synth.make_scene(w, h), synth.make_lights(64, aspect=w / h)
    v = viewer.Viewer(w, h, volumetric_decals=True)
    v.set_camera(scene.projection, scene.view)
    v.set_directional(scene.dir_color, scene.dir_direction)
    v.set_lights(lights)
    v.set_decals(make_decals(150, seed=8, aspect=w / h))
    v.bake()
    keep = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, scene.emissive)]
    v.render_frame(viewer.Viewer.host_gbuffer(*keep))
    out = np.zeros((h, w), np.uint32)
    v.read_output(out)
    mvps, zr = v.decal_prep()
    n = len(mvps)
    assert n > 20
    n32 = (n + 31) // 32
    bm = v.download_buffer("cluster-bitmask-decal", np.uint32, 128 * 64 * n32).reshape(64, 128, n32)
    assert np.array_equal(bm, oracle.decal_binning((128, 64), mvps))
    rng_ = v.download_buffer("cluster-range-decal", np.uint32, 4096 * 2).reshape(4096, 2)
    want = np.zeros((4096, 2), np.uint32)
    oracle.lib().orc_z_range(zr.ctypes.data_as(C.c_void_p), n, 4096, want.ctypes.data_as(C.c_void_p))
    assert np.array_equal(rng_, want)
    v.close()
