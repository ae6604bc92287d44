"""Shadowed device lights without a GPU: the shadow part of the device prep's pack kernel (lp::pack_shadow of
granite_b200/csrc/grb_light_prep.cuh, compiled for the CPU through tests/cpp/cuda_host_emul.h) against the host prep's
shadow tables, and the argument checks of grbh_viewer_set_lights_device_shadowed that refuse before any CUDA call."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from granite_b200 import synth
from tests import device_lights_cases as cases
from tests.test_device_lights_cpu import emulate, prep_view

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# odd slot counts: the transform table then starts 8 bytes past a 16-byte boundary
ODD_CASES = ["odd-1", "odd-37", "odd-4095"]


@pytest.fixture(scope="module")
def built():
    from granite_b200 import build

    return build.build_all()


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emu") / "libemu_light_prep_shadows.so")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    srcs = [os.path.join(ROOT, "tests", "cpp", f) for f in ("emulate_light_prep.cpp", "emulate_light_prep_shadows.cpp")]
    cmd = ["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-x", "c++", f"-I{cuda}/include", *srcs, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(out)


class GrbLightShadowList(C.Structure):
    _fields_ = [("transforms", C.c_void_p), ("maps", C.c_void_p)]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def shadow_case(oracle, name):
    """(w, h, proj, view, lights) of a named case: the device-light cases, or an odd light count."""
    if name in ODD_CASES:
        n = int(name.split("-")[1])
        w, h = 1920, 1080
        lights = synth.make_lights(n, spot_fraction=0.4)
        lights.position[::5, 2] += 200.0  # every fifth light behind the eye: culled, so count < slots
        return w, h, *cases.default_camera(w, h), cases.shuffled(lights)
    w, h, proj, view, lights, _ = cases.case(oracle, name)
    return w, h, proj, view, lights


def fake_maps(n):
    """Distinct fake map pointers by input light (never dereferenced), every sixth light without a map."""
    maps = np.uint64(0x7F0000000000) + np.arange(n, dtype=np.uint64) * np.uint64(0x1000)
    maps[5::6] = 0
    return maps


def packed_size(n):
    """Bytes of "cluster-transforms" before the shadow tables (host/clusterer.cpp packed_size): records, model rows,
    the type mask, the Z ranges."""
    return 48 * n + 48 * n + 4 * 128 + 8 * max(n, 1)


@pytest.mark.parametrize("name", cases.HOST_PREP_CASES + cases.TIE_CASES + cases.LIMIT_CASES + ODD_CASES)
def test_pack_shadow_gives_the_host_prep_tables(built, oracle, emu, name):
    """Slot s holds the transform bytes and map pointer of input light order[s], exactly the host prep's tables; slots
    past the kept count hold a zero matrix and a null map; the maps of lights culled or dropped past 4096 never appear;
    the two tables fill [packed_size(slots), + 72 x slots) of the buffer and no byte around them."""
    from granite_b200 import viewer
    from tests import common

    w, h, proj, view_m, lights = shadow_case(oracle, name)
    n = len(lights.color)
    v = viewer.Viewer(w, h, cuda_device=-1, light_shadows=True)
    v.set_camera(proj, view_m)
    v.set_lights(lights)
    maps_in = fake_maps(n)
    v.set_light_shadow_maps([int(m) for m in maps_in])
    k = v.light_prep()[0]
    want_t, want_m = v.light_shadow_prep()
    assert len(want_t) == k

    # the caller's transforms, in input order: the reference's shadow cameras of every light, culled ones included
    cam = common.oracle_camera_from_viewer(oracle, v)
    transforms = np.ascontiguousarray(oracle.shadow_transforms(oracle.prepare_lights(cam, lights, cull=False)), np.float32)
    assert transforms.shape == (n, 16)

    vis, _, radix, _, _, _ = emulate(emu, lights, prep_view(oracle, v))
    sort_key = radix.astype(np.uint64) | ((~vis).astype(np.uint64) << np.uint64(32))
    order = np.ascontiguousarray(np.argsort(sort_key, kind="stable")[: min(int(vis.sum()), 4096)], np.uint32)
    assert len(order) == k
    # the oracle's transforms are the host prep's, put back in input order
    assert transforms[order].tobytes() == want_t.tobytes()

    slots = min(n, 4096)
    base = packed_size(slots)
    # the input transforms 4 bytes past an 8-byte boundary: read one float at a time
    t_in = np.zeros(16 * n + 1, np.float32)[1:]
    t_in[:] = transforms.reshape(-1)
    assert t_in.ctypes.data % 8 == 4 or n == 0
    buf = np.full(base + 72 * slots + 64, 0xA5, np.uint8)
    sh = GrbLightShadowList(t_in.ctypes.data if n else None, maps_in.ctypes.data if n else None)
    emu.emu_pack_shadows(C.byref(sh), _p(order), len(order), slots, C.c_void_p(buf.ctypes.data + base),
                         C.c_void_p(buf.ctypes.data + base + 64 * slots))
    assert (buf[:base] == 0xA5).all() and (buf[base + 72 * slots:] == 0xA5).all(), "a byte outside the shadow tables was written"
    got_t = buf[base:base + 64 * slots].view(np.float32).reshape(slots, 16)
    got_m = buf[base + 64 * slots:base + 72 * slots].view(np.uint64)
    assert got_t[:k].tobytes() == want_t.tobytes()
    assert np.array_equal(got_m[:k], want_m)
    assert np.array_equal(got_m[:k], maps_in[order])
    assert not got_t[k:].view(np.uint32).any() and not got_m[k:].any()
    dropped = np.setdiff1d(np.arange(n), order)
    assert not np.isin(got_m[got_m != 0], maps_in[dropped][maps_in[dropped] != 0]).any()
    if name == "6000-visible":
        assert k == 4096 and len(dropped) >= 6000 - 4096
    if name in ODD_CASES:
        assert slots % 2 == 1 and base % 16 == 8 and k < slots
    v.close()


def _set_shadowed(v, count, transforms=16, maps=16, shadows=True):
    from granite_b200 import viewer

    l = viewer.GrbhDeviceLights(count, 16, 16, 16, 16, 16, 16, 1e10, None, None)  # never dereferenced: refused first
    sh = viewer.GrbhDeviceLightShadows(transforms, maps, None, None)
    return viewer.lib().grbh_viewer_set_lights_device_shadowed(v, C.byref(l), C.byref(sh) if shadows else None)


def test_set_lights_device_shadowed_argument_checks(built):
    """Refusals that need no CUDA call, each with its message: a null argument, a count outside 0..65536, a viewer
    created without clustered_lights_shadows, null tables with lights to shadow, a host-only viewer.  The unshadowed
    entry still refuses a shadowed viewer."""
    from granite_b200 import viewer

    L = viewer.lib()
    assert L.grbh_viewer_set_lights_device_shadowed(None, None, None) < 0 and b"null viewer" in L.grbh_last_error()
    s = viewer.Viewer(320, 192, cuda_device=-1, light_shadows=True)
    assert _set_shadowed(s._h, 4, shadows=False) < 0 and b"null viewer, light list or shadow list" in L.grbh_last_error()
    for n in (-1, viewer.MAX_DEVICE_LIGHTS + 1, 1 << 30):
        assert _set_shadowed(s._h, n) < 0
        assert b"outside 0..65536" in L.grbh_last_error()
    for t, m in ((None, 16), (16, None), (None, None)):
        assert _set_shadowed(s._h, 3, t, m) < 0
        assert b"null shadow transforms or shadow maps table" in L.grbh_last_error()
    for n, t in ((0, None), (1, 16), (viewer.MAX_DEVICE_LIGHTS, 16)):
        assert _set_shadowed(s._h, n, t, t) < 0
        assert b"host-only viewer" in L.grbh_last_error()
    l = viewer.GrbhDeviceLights(4, 16, 16, 16, 16, 16, 16, 1e10, None, None)
    assert L.grbh_viewer_set_lights_device(s._h, C.byref(l)) < 0
    assert b"clustered_lights_shadows" in L.grbh_last_error() and b"grbh_viewer_set_lights_device_shadowed" in L.grbh_last_error()
    s.close()
    v = viewer.Viewer(320, 192, cuda_device=-1)
    assert _set_shadowed(v._h, 4) < 0
    assert b"created without clustered_lights_shadows" in L.grbh_last_error()
    v.close()
    # the host path keeps working on the same viewer after a refusal, shadow tables included
    s = viewer.Viewer(320, 192, cuda_device=-1, light_shadows=True)
    assert _set_shadowed(s._h, 4) < 0
    s.set_camera(*cases.default_camera(320, 192))
    s.set_lights(synth.make_lights(16))
    s.set_light_shadow_maps([0x1000 * (i + 1) for i in range(16)])
    t, m = s.light_shadow_prep()
    assert len(t) == 16 and sorted(m.tolist()) == [0x1000 * (i + 1) for i in range(16)]
    s.close()

