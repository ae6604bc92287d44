"""A device light list whose length lives on the device, without a GPU: the live/dead decision of the cull step
(lp::live_count and lp::cull_key of granite_b200/csrc/grb_light_prep.cuh, compiled for the CPU) against today's keys, and
the argument checks of grbh_viewer_set_light_count_device and grb_light_prep[_shadowed]_counted that refuse before any
CUDA call."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import device_lights_cases as cases
from tests import test_device_lights_cpu as base

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built():
    from granite_b200 import build

    return build.build_all()


def _compile(tmp_path_factory, src):
    out = str(tmp_path_factory.mktemp("emu") / (os.path.splitext(src)[0] + ".so"))
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    cmd = ["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-x", "c++", f"-I{cuda}/include",
           os.path.join(ROOT, "tests", "cpp", src), "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(out)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return _compile(tmp_path_factory, "emulate_light_prep.cpp")


@pytest.fixture(scope="module")
def emu_count(tmp_path_factory):
    lib = _compile(tmp_path_factory, "emulate_light_prep_count.cpp")
    lib.emu_cull_keys.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    return lib


CAPACITY = 300


@pytest.mark.parametrize("live", [-3, 0, 1, 37, CAPACITY, CAPACITY + 10])
def test_dead_entries_get_the_culled_key_and_live_ones_keep_todays(built, oracle, emu, emu_count, live):
    """live = min(max(count, 0), capacity); entry i < live gets the key the cull kernel gives today (culled bit from the
    visibility, then the radix code of dot(position, front)), entry i >= live exactly 1 << 32 even when it holds NaNs."""
    from granite_b200 import viewer

    w, h, proj, view_m, lights, _ = cases.case(oracle, f"{CAPACITY}-0.25")
    lights.position[::5, 2] += 200.0  # every fifth light behind the eye: culled
    v = viewer.Viewer(w, h, cuda_device=-1)
    v.set_camera(proj, view_m)
    view = base.prep_view(oracle, v)
    v.close()
    vis, _, radix, _, _, _ = base.emulate(emu, lights, view)
    today = radix.astype(np.uint64) | ((~vis).astype(np.uint64) << np.uint64(32))
    assert vis.any() and (~vis).any(), "the case has both visible and culled lights"

    k = min(max(live, 0), CAPACITY)
    arrs = [np.ascontiguousarray(a, t).copy() for a, t in ((lights.color, np.float32), (lights.position, np.float32), (lights.is_point, np.uint8),
                                                           (lights.rot, np.float32), (lights.inner_cone, np.float32),
                                                           (lights.outer_cone, np.float32))]
    for a in arrs:
        a[k:] = 0xFF if a.dtype == np.uint8 else np.float32(np.nan)  # dead entries: garbage the kernel must not read
    ll = base.GrbLightList(CAPACITY, *[base._p(a) for a in arrs], 1e10)
    keys = np.zeros(CAPACITY, np.uint64)
    got_live = emu_count.emu_cull_keys(C.byref(ll), C.byref(view), live, base._p(keys))
    assert got_live == k
    assert keys[:k].tolist() == today[:k].tolist()
    assert keys[k:].tolist() == [1 << 32] * (CAPACITY - k)
    # the stable sort puts the visible live lights first, in today's order for the first k lights
    order = np.argsort(keys, kind="stable")
    visible_live = int((keys >> np.uint64(32) == 0).sum())
    assert visible_live == int(vis[:k].sum())
    assert order[:visible_live].tolist() == np.argsort(today[:k], kind="stable")[:visible_live].tolist()


def test_set_light_count_device_argument_checks(built):
    """Refusals a host-only viewer reaches, each with its message: a null viewer, a host-only viewer (with a null, an
    aligned and a misaligned count); the host path keeps working after them."""
    from granite_b200 import synth, viewer

    L = viewer.lib()
    buf = (C.c_int32 * 2)()
    assert L.grbh_viewer_set_light_count_device(None, None) < 0
    assert b"grbh_viewer_set_light_count_device: null viewer" in L.grbh_last_error()
    for shadows in (False, True):
        v = viewer.Viewer(320, 192, cuda_device=-1, light_shadows=shadows)
        for p in (None, C.addressof(buf), C.addressof(buf) + 2):
            assert L.grbh_viewer_set_light_count_device(v._h, p) < 0
            assert b"grbh_viewer_set_light_count_device: host-only viewer" in L.grbh_last_error()
        v.set_camera(*cases.default_camera(320, 192))
        v.set_lights(synth.make_lights(16))
        assert v.light_prep()[0] == 16
        v.close()


def _prep_args():
    """Arguments grb_light_prep would accept up to its first CUDA call (never dereferenced on the host)."""
    dummy = C.c_void_p(64)
    ll = base.GrbLightList(4, dummy, dummy, dummy, dummy, dummy, dummy, 1e10)
    view = base.GrbLightPrepView()
    return ll, view, dummy


def test_counted_prep_refuses_before_any_cuda_call(built):
    """grb_light_prep_counted and grb_light_prep_shadowed_counted refuse a null input count (and the shadowed form a
    null shadow list), and both a count that is not 4-byte aligned, with GRB_ERR_INVALID_ARGUMENT and a message."""
    from granite_b200 import capi

    L = capi.lib()
    ll, view, d = _prep_args()
    sh = (C.c_void_p * 2)(64, 64)  # a GrbLightShadowList: transforms, maps
    counted = L.grb_light_prep_counted
    counted.argtypes = [C.c_void_p] * 9 + [C.c_uint64, C.c_void_p]
    shadowed = L.grb_light_prep_shadowed_counted
    shadowed.argtypes = [C.c_void_p] * 12 + [C.c_uint64, C.c_void_p]

    assert counted(C.byref(ll), None, C.byref(view), d, d, d, d, d, d, 1 << 30, None) == -1
    assert b"grb_light_prep_counted: a null input count" in L.grb_last_error_string()
    assert shadowed(C.byref(ll), None, sh, C.byref(view), d, d, d, d, d, d, d, d, 1 << 30, None) == -1
    assert b"grb_light_prep_shadowed_counted: a null input count or shadow table" in L.grb_last_error_string()
    assert shadowed(C.byref(ll), d, None, C.byref(view), d, d, d, d, d, d, d, d, 1 << 30, None) == -1
    assert b"grb_light_prep_shadowed_counted: a null input count or shadow table" in L.grb_last_error_string()
    odd = C.c_void_p(66)
    assert counted(C.byref(ll), odd, C.byref(view), d, d, d, d, d, d, 1 << 30, None) == -1
    assert b"grb_light_prep_counted: the input count is not 4-byte aligned" in L.grb_last_error_string()
    assert shadowed(C.byref(ll), odd, sh, C.byref(view), d, d, d, d, d, d, d, d, 1 << 30, None) == -1
    assert b"grb_light_prep_shadowed_counted: the input count is not 4-byte aligned" in L.grb_last_error_string()
