"""Volumetric fog accumulation on the GPU (granite_b200/csrc/grb_fog.cu through the C ABI) against the oracle.  Sorted after the
other GPU tests.  Also verified without a GPU: the
kernel's source compiled for the CPU, bit for bit with the oracle, and the oracle against the reference's shader
(tests/test_fog_cpu.py).  On hardware exp2f is CUDA's: the stored fp16 values may differ by one ulp."""
import ctypes as C

import numpy as np
import pytest

from tests.test_fog_cpu import make_density

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("w,h,d", [(33, 17, 7), (160, 92, 64), (320, 180, 128)])
def test_cuda_fog_accumulate_vs_oracle(cuda, oracle, w, h, d):
    import torch

    from granite_b200 import capi, harness

    light = make_density(w, h, d, seed=2)
    dev = harness.to_dev(light)
    fog = torch.zeros((d, h, w, 4), dtype=torch.int16, device="cuda")
    capi.check(capi.lib().grb_fog_accumulate(C.c_void_p(dev.data_ptr()), w, h, d, C.c_void_p(fog.data_ptr()), capi.stream_ptr()), "grb_fog_accumulate")
    torch.cuda.synchronize()
    got, ref = harness.to_host(fog, np.uint16), oracle.fog_accumulate(light)
    diff = np.abs(got.astype(np.int32) - ref.astype(np.int32))
    assert diff.max() <= 1 and (diff == 0).mean() > 0.999, (int(diff.max()), float((diff == 0).mean()))


@pytest.mark.parametrize("w,h,d,n", [(40, 23, 16, 300), (160, 92, 64, 1024)])
def test_cuda_fog_light_density_vs_oracle(cuda, oracle, w, h, d, n):
    """fog_light_density.comp (base variant) on the device; exp2f / sqrtf are CUDA's: one fp16 code."""
    import torch

    from granite_b200 import capi, harness
    from tests import common
    from tests.test_fog_cpu import DIR_COLOR, DIR_DIRECTION
    from tests.test_gpu_parity import _cluster

    cam, lights, prep = common.build_lights_case(oracle, 16.0 / 9.0, n, 0.25)
    clus = oracle.cluster_build(cam, prep)
    fp = oracle.fog_params(w, h, d, z_range=80.0, density=0.5, in_scatter=1.25, dither_offset=1)
    lut = np.random.default_rng(17).integers(0, 2 ** 32, (3, 128, 128), dtype=np.uint64).astype(np.uint32)
    ref = oracle.fog_light_density(fp, cam, prep, clus, DIR_COLOR, DIR_DIRECTION, lut)
    dev, gcam = _cluster(cuda, oracle, cam, prep)
    g = capi.GrbFogParameters(fp.width, fp.height, fp.depth, fp.dither_offset, fp.slice_z_log2_scale, fp.density_mod, fp.in_scatter_strength)
    t = lambda a, dt: harness.to_dev(np.ascontiguousarray(a, dt))  # noqa: E731
    proj, inv_proj = t(list(cam.projection), np.float32), t(list(cam.inv_projection), np.float32)
    ext, lut_d = t(oracle.fog_slice_extents(fp), np.float32), harness.to_dev(lut)
    out = torch.zeros((d, h, w, 4), dtype=torch.int16, device="cuda")
    dc, dd = (C.c_float * 3)(*DIR_COLOR), (C.c_float * 3)(*DIR_DIRECTION)
    hp, hip = np.array(list(cam.projection), np.float32), np.array(list(cam.inv_projection), np.float32)
    capi.check(capi.lib().grb_fog_light_density(C.byref(g), C.byref(gcam), hp.ctypes.data_as(C.c_void_p), hip.ctypes.data_as(C.c_void_p), C.byref(dev.params),
                                                C.byref(dev.buffers), dc, dd, C.c_void_p(ext.data_ptr()), C.c_void_p(lut_d.data_ptr()), C.c_void_p(out.data_ptr()),
                                                capi.stream_ptr()), "grb_fog_light_density")
    torch.cuda.synchronize()
    got = harness.to_host(out, np.uint16)
    diff = np.abs(got.astype(np.int32) - ref.astype(np.int32))
    assert diff.max() <= 1 and (diff == 0).mean() > 0.99, (int(diff.max()), float((diff == 0).mean()))
    # the two passes chained: the accumulated fog of the device's own density volume
    fog = torch.zeros_like(out)
    capi.check(capi.lib().grb_fog_accumulate(C.c_void_p(out.data_ptr()), w, h, d, C.c_void_p(fog.data_ptr()), capi.stream_ptr()), "grb_fog_accumulate")
    torch.cuda.synchronize()
    d2 = np.abs(harness.to_host(fog, np.uint16).astype(np.int32) - oracle.fog_accumulate(got).astype(np.int32))
    assert d2.max() <= 1 and (d2 == 0).mean() > 0.999
