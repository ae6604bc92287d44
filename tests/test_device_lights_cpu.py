"""Device light prep without a GPU: the per-light functions of granite_b200/csrc/grb_light_prep.cuh compiled for the CPU
(tests/cpp/cuda_host_emul.h) against the host prep (Viewer.light_prep on a host-only viewer), and the argument checks of
grbh_viewer_set_lights_device that refuse before any CUDA call."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import device_lights_cases as cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built():
    from granite_b200 import build

    return build.build_all()


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emu") / "libemu_light_prep.so")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    cmd = ["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-x", "c++", f"-I{cuda}/include",
           os.path.join(ROOT, "tests", "cpp", "emulate_light_prep.cpp"), "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(out)


class GrbLightList(C.Structure):
    _fields_ = [("count", C.c_int32), ("color", C.c_void_p), ("position", C.c_void_p), ("is_point", C.c_void_p), ("rotation", C.c_void_p),
                ("inner_cone", C.c_void_p), ("outer_cone", C.c_void_p), ("cutoff_range", C.c_float)]


class GrbLightPrepView(C.Structure):
    _fields_ = [("camera_position", C.c_float * 3), ("camera_front", C.c_float * 3), ("planes", C.c_float * 24), ("z_slice_extent", C.c_float),
                ("z_max_index", C.c_int32), ("frustum_culling", C.c_int32)]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def prep_view(oracle, v, res_z=4096):
    """The camera terms LightClusterer::refresh_bindless_prepare hands the device prep, from the viewer's camera."""
    cam, _, _ = v.camera()
    ivp = np.array(list(cam.inv_view_projection), np.float32)
    planes = np.zeros(24, np.float32)
    oracle.lib().orc_frustum_planes(_p(ivp), _p(planes))
    view = GrbLightPrepView()
    view.camera_position[:] = list(cam.camera_position)
    view.camera_front[:] = list(cam.camera_front)
    view.planes[:] = planes.tolist()
    view.z_slice_extent = float(min(np.float32(0.5), np.float32(cam.z_far) / np.float32(res_z)))
    view.z_max_index = res_z - 1
    view.frustum_culling = 1
    return view


def emulate(emu, lights, view, cutoff=1e10):
    """Every input light through the device prep's per-light functions: visibility, key, radix code, record, model row,
    Z range."""
    n = len(lights.color)
    arrs = [np.ascontiguousarray(a, t) for a, t in ((lights.color, np.float32), (lights.position, np.float32), (lights.is_point, np.uint8),
                                                    (lights.rot, np.float32), (lights.inner_cone, np.float32), (lights.outer_cone, np.float32))]
    ll = GrbLightList(n, *[_p(a) for a in arrs], cutoff)
    from granite_b200 import capi

    vis, keys, radix = np.zeros(n, np.uint8), np.zeros(n, np.float32), np.zeros(n, np.uint32)
    recs, model, zr = np.zeros(max(n, 1), capi.LIGHT_DTYPE), np.zeros((max(n, 1), 12), np.float32), np.zeros((max(n, 1), 2), np.uint32)
    emu.emu_light_prep(C.byref(ll), C.byref(view), _p(vis), _p(keys), _p(radix), _p(recs), _p(model), _p(zr))
    return vis.astype(bool), keys, radix, recs[:n], model[:n], zr[:n]


@pytest.mark.parametrize("name", cases.HOST_PREP_CASES + cases.TIE_CASES)
def test_per_light_functions_give_the_host_prep_bytes(built, oracle, emu, name):
    """Kept lights, their order (a stable sort of the emitted 33-bit radix keys), records, model rows, type mask and
    Z ranges byte for byte the host prep's; visibility the oracle's; keys dot(position, front) in fp32."""
    from granite_b200 import viewer
    from tests import common

    w, h, proj, view_m, lights, _ = cases.case(oracle, name)
    v = viewer.Viewer(w, h, cuda_device=-1)
    v.set_camera(proj, view_m)
    v.set_lights(lights)
    k, recs, model, tmask, zr = v.light_prep()
    view = prep_view(oracle, v)
    vis, keys, radix, e_recs, e_model, e_zr = emulate(emu, lights, view)

    cam = common.oracle_camera_from_viewer(oracle, v)
    if len(lights.color):
        assert np.array_equal(vis, oracle.visible_lights(cam, lights))
    f = np.array(list(cam.camera_front), np.float32)
    p = lights.position.astype(np.float32)
    expect_keys = (p[:, 0] * f[0] + p[:, 1] * f[1]) + p[:, 2] * f[2]
    assert keys.view(np.uint32).tolist() == expect_keys.view(np.uint32).tolist()
    # -0 and +0 share a code; otherwise the codes order like the floats
    assert np.array_equal(radix[keys == 0], np.full((keys == 0).sum(), 0x80000000, np.uint32))
    o = np.argsort(keys, kind="stable")
    assert np.all(np.diff(radix[o].astype(np.int64)) >= 0)

    sort_key = radix.astype(np.uint64) | ((~vis).astype(np.uint64) << np.uint64(32))
    order = np.argsort(sort_key, kind="stable")[: min(int(vis.sum()), 4096)]
    assert len(order) == k
    assert e_recs[order].tobytes() == recs.tobytes()
    assert np.array_equal(e_model[order].view(np.uint32), model.view(np.uint32))
    assert np.array_equal(e_zr[order] if k else np.array([[0xFFFFFFFF, 0]], np.uint32), zr)
    e_mask = np.zeros((k + 31) // 32, np.uint32)
    for s, i in enumerate(order):
        if lights.is_point[i]:
            e_mask[s >> 5] |= np.uint32(1 << (s & 31))
    assert np.array_equal(e_mask, tmask)
    if name == "signed-zero":
        assert (np.signbit(keys) & (keys == 0)).any() and (~np.signbit(keys) & (keys == 0)).any(), "both zero keys occur"
        assert list(order) == sorted(order), "equal keys keep input order"
    if name == "ties":
        assert len(np.unique(keys)) < len(keys)
    v.close()


def _set_lights_device(v, count, **kw):
    from granite_b200 import viewer

    l = viewer.GrbhDeviceLights(count, 16, 16, 16, 16, 16, 16, 1e10, None, None)  # never dereferenced: refused first
    return viewer.lib().grbh_viewer_set_lights_device(v, C.byref(l))


def test_set_lights_device_argument_checks(built):
    """Refusals that need no CUDA call: a null viewer, a count outside 0..65536, a viewer created with shadowed lights,
    a host-only viewer; each with its message."""
    from granite_b200 import viewer

    L = viewer.lib()
    assert L.grbh_viewer_set_lights_device(None, None) < 0 and b"null" in L.grbh_last_error()
    v = viewer.Viewer(320, 192, cuda_device=-1)
    for n in (-1, viewer.MAX_DEVICE_LIGHTS + 1, 1 << 30):
        assert _set_lights_device(v._h, n) < 0
        assert b"outside 0..65536" in L.grbh_last_error()
    for n in (0, 1, viewer.MAX_DEVICE_LIGHTS):
        assert _set_lights_device(v._h, n) < 0
        assert b"host-only viewer" in L.grbh_last_error()
    v.close()
    s = viewer.Viewer(320, 192, cuda_device=-1, light_shadows=True)
    assert _set_lights_device(s._h, 4) < 0
    assert b"clustered_lights_shadows" in L.grbh_last_error()
    s.close()
    # the host path keeps working on the same viewer after a refusal
    v = viewer.Viewer(320, 192, cuda_device=-1)
    assert _set_lights_device(v._h, 4) < 0
    from granite_b200 import synth

    v.set_camera(*cases.default_camera(320, 192))
    v.set_lights(synth.make_lights(16))
    assert v.light_prep()[0] == 16
    v.close()
