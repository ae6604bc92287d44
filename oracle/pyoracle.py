"""ctypes binding of the CPU oracle -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py (cpu_baseline / --impl reference) may
import this module.  The product package granite_b200 must never import it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from types import SimpleNamespace

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "liboracle.so")
_REF_PATH = os.path.join(_HERE, "_ref", "libgranite_refmath.so")


_REF_KERNEL_PATHS = [os.path.join(_HERE, "_ref", f"libgranite_ref_k{k}.so") for k in (1, 2, 3, 4, 5)]
# post-processing shaders K7-K13 (ref_post_shim.cpp); ids as in oracle/Makefile POST_IDS
_REF_POST_IDS = (7, 8, 18, 9, 10, 11, 12, 22, 13, 23, 33, 43, 14, 150, 151, 152, 153, 160, 161, 162, 163, 170, 171, 172, 173, 24, 25, 26, 27)
_REF_POST_PATHS = {k: os.path.join(_HERE, "_ref", f"libgranite_ref_p{k}.so") for k in _REF_POST_IDS}
# deferred-lighting fragment shaders K5 (clustering.frag) and K6 (directional.frag), ref_light_shim.cpp
_REF_LIGHT_PATHS = {k: os.path.join(_HERE, "_ref", f"libgranite_ref_l{k}.so") for k in (5, 6, 7, 8, 9)}


def build(ref: bool = True) -> None:
    """Compile liboracle.so (always) and oracle/_ref (only where /root/reference exists):
    the reference's math/ (`make ref`) and its clusterer compute shaders run on the CPU through its
    vendored glslang + spirv-cross (`make ref-shaders`, ~1 min the first time)."""
    subprocess.run(["make", "-s", "-C", _HERE], check=True)
    if ref and os.path.isdir("/root/reference/math"):
        subprocess.run(["make", "-s", "-C", _HERE, "ref"], check=True)
    if ref and os.path.isdir("/root/reference/third_party/spirv-cross") and os.path.isdir("/root/reference/third_party/glslang"):
        shim = os.path.join(_HERE, "ref_shader_shim.cpp")
        stale = any(not os.path.exists(p) or os.path.getmtime(p) < os.path.getmtime(shim) for p in _REF_KERNEL_PATHS)
        pshim = os.path.join(_HERE, "ref_post_shim.cpp")
        stale = stale or any(not os.path.exists(p) or os.path.getmtime(p) < os.path.getmtime(pshim) for p in _REF_POST_PATHS.values())
        lshim = os.path.join(_HERE, "ref_light_shim.cpp")
        stale = stale or any(not os.path.exists(p) or os.path.getmtime(p) < os.path.getmtime(lshim) for p in _REF_LIGHT_PATHS.values())
        if stale:
            r = subprocess.run(["make", "-s", "-j8", "-C", _HERE, "ref-shaders"], capture_output=True, text=True)
            if r.returncode != 0:  # checker infrastructure: report, never break the product build
                print("oracle: `make ref-shaders` failed (the reference-shader pin is unavailable):\n" + r.stdout[-2000:] + r.stderr[-2000:])


class Light(C.Structure):
    _fields_ = [("color", C.c_float * 3), ("spot_scale_bias", C.c_uint16 * 2),
                ("position", C.c_float * 3), ("offset_radius", C.c_uint16 * 2),
                ("direction", C.c_float * 3), ("inv_radius", C.c_float)]


LIGHT_DTYPE = np.dtype([("color", "<f4", 3), ("spot_scale_bias", "<u2", 2), ("position", "<f4", 3),
                        ("offset_radius", "<u2", 2), ("direction", "<f4", 3), ("inv_radius", "<f4")])
assert LIGHT_DTYPE.itemsize == 48 and C.sizeof(Light) == 48


class ClusterParams(C.Structure):
    _fields_ = [("transform", C.c_float * 16), ("clip_scale", C.c_float * 4),
                ("camera_base", C.c_float * 3), ("camera_front", C.c_float * 3),
                ("xy_scale", C.c_float * 2), ("resolution_xy", C.c_int32 * 2),
                ("inv_resolution_xy", C.c_float * 2), ("num_lights", C.c_int32),
                ("num_lights_32", C.c_int32), ("z_max_index", C.c_int32), ("z_scale", C.c_float)]


class Camera(C.Structure):
    _fields_ = [("projection", C.c_float * 16), ("view", C.c_float * 16),
                ("view_projection", C.c_float * 16), ("inv_projection", C.c_float * 16),
                ("inv_view", C.c_float * 16), ("inv_view_projection", C.c_float * 16),
                ("camera_position", C.c_float * 3), ("camera_front", C.c_float * 3),
                ("z_near", C.c_float), ("z_far", C.c_float)]


class GBuffer(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("albedo", C.c_void_p), ("normal", C.c_void_p),
                ("pbr", C.c_void_p), ("depth", C.c_void_p), ("emissive", C.c_void_p),
                ("dir_color", C.c_float * 3), ("dir_direction", C.c_float * 3)]


_lib = None
_ref = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build(ref=False)
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_float_to_half.restype = C.c_uint16
        _lib.orc_float_to_half.argtypes = [C.c_float]
        _lib.orc_pack_r11g11b10.restype = C.c_uint32
        _lib.orc_pack_r11g11b10.argtypes = [C.c_float] * 3
        _lib.orc_f32_to_f16.restype = C.c_uint16
        _lib.orc_f32_to_f16.argtypes = [C.c_float]
        _lib.orc_f16_to_f32.restype = C.c_float
        _lib.orc_f16_to_f32.argtypes = [C.c_uint16]
        _lib.orc_linear_to_srgb8.restype = C.c_uint32
        _lib.orc_linear_to_srgb8.argtypes = [C.c_float]
        _lib.orc_srgb8_to_linear.restype = C.c_float
        _lib.orc_srgb8_to_linear.argtypes = [C.c_uint32]
    return _lib


def ref():
    """The reference's own math/ compiled into oracle/_ref (None when it was not built)."""
    global _ref
    if _ref is None and os.path.exists(_REF_PATH):
        _ref = C.CDLL(_REF_PATH)
        _ref.ref_float_to_half.restype = C.c_uint16
        _ref.ref_float_to_half.argtypes = [C.c_float]
        _ref.ref_infinite_far_plane.restype = C.c_float
    return _ref


_ref_kernels = None


def ref_kernels():
    """{1..4: CDLL} of the reference's clusterer compute shaders compiled for the CPU
    (oracle/_ref/libgranite_ref_k*.so, see ref_shader_shim.cpp), or None when they were not built."""
    global _ref_kernels
    if _ref_kernels is None and all(os.path.exists(p) for p in _REF_KERNEL_PATHS):
        _ref_kernels = {k: C.CDLL(p) for k, p in zip((1, 2, 3, 4, 5), _REF_KERNEL_PATHS)}
    return _ref_kernels


_ref_post = None


def ref_post_kernels():
    """{id: CDLL} of the reference's post-processing shaders (K7-K13) compiled for the CPU
    (oracle/_ref/libgranite_ref_p*.so, see ref_post_shim.cpp), or None when they were not built."""
    global _ref_post
    if _ref_post is None and all(os.path.exists(p) for p in _REF_POST_PATHS.values()):
        lib()  # liboracle.so supplies the storage-format helpers the shim links against
        _ref_post = {k: C.CDLL(p) for k, p in _REF_POST_PATHS.items()}
    return _ref_post


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f(x):
    return C.c_float(float(x))


def _c(a, dtype):
    if a is None:
        return None
    return np.ascontiguousarray(a, dtype=dtype)


# ---------------- host math ----------------
def perspective(fovy, aspect, near, far):
    out = np.zeros(16, np.float32)
    lib().orc_perspective(_f(fovy), _f(aspect), _f(near), _f(far), _p(out))
    return out.reshape(4, 4)


def mat4_inverse(m):
    m = _c(m, np.float32)
    out = np.zeros(16, np.float32)
    lib().orc_mat4_inverse(_p(m), _p(out))
    return out.reshape(4, 4)


def mat4_mul(a, b):
    a = _c(a, np.float32); b = _c(b, np.float32)
    out = np.zeros(16, np.float32)
    lib().orc_mat4_mul(_p(a), _p(b), _p(out))
    return out.reshape(4, 4)


def camera_setup(projection, view) -> Camera:
    cam = Camera()
    pr = _c(projection, np.float32); vw = _c(view, np.float32)
    lib().orc_camera_setup(_p(pr), _p(vw), C.byref(cam))
    return cam


# ---------------- light prep ----------------
def visible_lights(cam: Camera, lights, cutoff=1e10):
    """renderer/scene.cpp:333-358: boolean mask of the lights whose world AABB passes the camera's
    visibility frustum (the list the clusterer then sorts and truncates)."""
    L = lib()
    L.orc_light_visible.restype = C.c_int
    planes = np.zeros(24, np.float32)
    ivp = np.array(list(cam.inv_view_projection), np.float32)
    L.orc_frustum_planes(_p(ivp), _p(planes))
    keep = np.zeros(len(lights.color), bool)
    for i in range(len(lights.color)):
        col = _c(lights.color[i], np.float32); pos = lights.position[i]
        if lights.is_point[i]:
            rows = np.array([[1, 0, 0, pos[0]], [0, 1, 0, pos[1]], [0, 0, 1, pos[2]]], np.float32)
        else:
            r = np.asarray(lights.rot[i], np.float32).reshape(-1)  # column-major 3x3, as the host API takes it
            rows = np.array([[r[0], r[3], r[6], pos[0]], [r[1], r[4], r[7], pos[1]], [r[2], r[5], r[8], pos[2]]], np.float32)
        rows = np.ascontiguousarray(rows)
        keep[i] = bool(L.orc_light_visible(_p(planes), int(bool(lights.is_point[i])), _p(col), _f(cutoff), _f(lights.outer_cone[i]), _p(rows)))
    return keep


def prepare_lights(cam: Camera, lights, res=(128, 64, 4096), cutoff=1e10, cull=True):
    """Host prep: frustum cull (scene.cpp:333-358), then records (sorted order as given), model rows,
    type mask, cluster params, z ranges."""
    if cull and len(lights.color):
        keep = visible_lights(cam, lights, cutoff)
        if not keep.all():
            lights = type(lights)(lights.color[keep], lights.position[keep], lights.is_point[keep], lights.rot[keep],
                                  lights.inner_cone[keep], lights.outer_cone[keep])
    n = len(lights.color)
    n32 = (n + 31) // 32
    recs = np.zeros(max(n, 1), LIGHT_DTYPE)
    model = np.zeros((max(n, 1), 12), np.float32)
    type_mask = np.zeros(max(n32, 1), np.uint32)
    L = lib()
    for i in range(n):
        col = _c(lights.color[i], np.float32); pos = _c(lights.position[i], np.float32)
        rec = Light()
        if lights.is_point[i]:
            L.orc_point_light_info(_p(col), _p(pos), _f(cutoff), C.byref(rec))
            type_mask[i >> 5] |= np.uint32(1 << (i & 31))
            model[i, 0:3] = pos
            model[i, 3] = np.float32(1.0) / np.float32(rec.inv_radius)  # clusterer.cpp:647-650
        else:
            rot = _c(lights.rot[i], np.float32)
            rows = np.zeros(12, np.float32)
            L.orc_spot_light_info(_p(col), _p(pos), _p(rot), _f(lights.inner_cone[i]), _f(lights.outer_cone[i]),
                                  _f(cutoff), C.byref(rec), _p(rows))
            model[i] = rows
        recs[i:i + 1] = np.frombuffer(bytes(rec), LIGHT_DTYPE)
    params = ClusterParams()
    L.orc_cluster_params(C.byref(cam), n, res[0], res[1], res[2], C.byref(params))
    z_ranges = np.zeros((max(n, 1), 2), np.uint32)
    L.orc_light_z_ranges(C.byref(cam), _p(recs), _p(model), _p(type_mask), n, res[2], _p(z_ranges))
    return SimpleNamespace(n=n, n32=n32, records=recs, model=model, type_mask=type_mask, params=params,
                           z_ranges=z_ranges, res=res, outer_cone=np.asarray(lights.outer_cone, np.float32).copy())


def spot_xy_range(outer_cone):
    """SpotLight::set_spot_parameters (lights.cpp:82-86): tan of the outer half angle from its cosine, in fp32."""
    oc = np.float32(outer_cone)
    return np.float32(np.sqrt(np.float32(np.float32(1.0) - oc * oc)) / oc)


def shadow_transforms(prep):
    """ClustererBindlessTransforms::shadow of every light of prep (clusterer.cpp:467-474, 518-521): (n, 16) f32."""
    L = lib()
    out = np.zeros((max(prep.n, 1), 16), np.float32)
    for i in range(prep.n):
        rec = Light.from_buffer_copy(prep.records[i:i + 1].tobytes())
        m = np.zeros(16, np.float32)
        if (int(prep.type_mask[i >> 5]) >> (i & 31)) & 1:
            L.orc_point_shadow_transform(C.byref(rec), _p(m))
        else:
            L.orc_spot_shadow_transform(C.byref(rec), _f(spot_xy_range(prep.outer_cone[i])), _p(m))
        out[i] = m
    return out[:prep.n] if prep.n else out[:0]


class Shadows(C.Structure):
    _fields_ = [("transforms", C.c_void_p), ("maps", C.c_void_p), ("resolution", C.c_int), ("pcf_wide", C.c_int)]


def deferred_lighting_shadowed(scene, cam: Camera, prep, clus, transforms, maps, resolution, rows=None, pcf_wide=False):
    """The lighting pass with POSITIONAL_LIGHTS_SHADOW.  maps: one uint16 array per light (res x res for a spot light,
    6 x res x res for a point light) or None (no shadow)."""
    H, W = scene.depth.shape
    g = GBuffer()
    g.width, g.height = W, H
    keep = [_c(scene.albedo, np.uint32), _c(scene.normal, np.uint32), _c(scene.pbr, np.uint16),
            _c(scene.depth, np.float32), _c(scene.emissive, np.uint32)]
    g.albedo, g.normal, g.pbr, g.depth, g.emissive = [k.ctypes.data for k in keep]
    g.dir_color = (C.c_float * 3)(*scene.dir_color)
    g.dir_direction = (C.c_float * 3)(*scene.dir_direction)
    hdr = np.zeros((H, W), np.uint32)
    y0, y1 = rows if rows else (0, H)
    t = _c(transforms, np.float32)
    held = [None if m is None else _c(m, np.uint16) for m in maps]
    table = (C.c_void_p * max(len(held), 1))(*[None if m is None else m.ctypes.data for m in held])
    sh = Shadows(t.ctypes.data, C.cast(table, C.c_void_p), int(resolution), int(pcf_wide))
    lib().orc_deferred_lighting_shadowed(C.byref(g), C.byref(cam), C.byref(prep.params), _p(prep.records), _p(prep.type_mask),
                                         _p(clus.bitmask), _p(clus.range), C.byref(sh), _p(hdr), y0, y1)
    return hdr


def cluster_build(cam: Camera, prep):
    """K1..K4. Returns transformed_spots, cull_setup, bitmask, cluster_range."""
    L = lib()
    n, n32 = prep.n, prep.n32
    rx, ry, rz = prep.res
    spots = np.zeros((max(n, 1), 24), np.float32)
    L.orc_spot_transform(C.byref(cam), _p(prep.model), n, _p(spots))
    cull = np.zeros((max(n, 1), 128), np.float32)
    L.orc_cull_setup(C.byref(cam), C.byref(prep.params), _p(prep.records), _p(prep.type_mask), _p(spots), _p(cull))
    bitmask = np.zeros((ry, rx, max(n32, 1)), np.uint32)
    if n:
        L.orc_binning(C.byref(prep.params), _p(prep.type_mask), _p(cull), _p(bitmask))
    crange = np.zeros((rz, 2), np.uint32)
    L.orc_z_range(_p(prep.z_ranges), max(n, 1), rz, _p(crange))
    return SimpleNamespace(spots=spots, cull=cull, bitmask=bitmask, range=crange)


def _farr(x, dtype=np.float32):
    return np.ascontiguousarray(np.array(list(x), dtype))


def ref_spot_transform(cam: Camera, prep):
    """K1 through the reference's own shader (clusterer_bindless_spot_transform.comp)."""
    n = prep.n
    out = np.zeros((max(n, 1), 24), np.float32)
    vp, cp, cf = _farr(cam.view_projection), _farr(cam.camera_position), _farr(cam.camera_front)
    ref_kernels()[1].refk1_spot_transform(_p(vp), _p(cp), _p(cf), _f(cam.z_near), _f(cam.z_far), _p(prep.model), n, _p(out))
    return out


def ref_cull_setup(cam: Camera, prep, spots):
    """K2 through the reference's own shader (clusterer_bindless_setup.comp)."""
    n, pr = prep.n, prep.params
    out = np.zeros((max(n, 1), 128), np.float32)
    keep = [_farr(cam.view), _farr(pr.transform), _farr(pr.clip_scale), _farr(pr.camera_base), _farr(pr.camera_front), _farr(pr.xy_scale),
            _farr(pr.resolution_xy, np.int32), _farr(pr.inv_resolution_xy)]
    spots = _c(spots, np.float32)
    ref_kernels()[2].refk2_cull_setup(*[_p(k) for k in keep], pr.num_lights_32, pr.z_max_index, _f(pr.z_scale), _p(prep.records),
                                      _p(prep.type_mask), _p(spots), n, _p(out))
    return out


def ref_binning(prep, cull, window=None):
    """K3 through the reference's own shader.  The reference runs the SUBGROUPS=1 variant on NVIDIA
    (clusterer.cpp:1519-1561): a coarse test of each 8x4-tile block AND the per-tile test, both with
    the shader's test_point_light / test_spot_light.  Only the SUBGROUPS=0 variant (per-tile test
    alone) can execute without subgroup hardware, so the coarse pass is that same executable run on
    the 16x16 grid of 8x4-tile blocks (resolution 128x64 makes `2 * tile * inv_resolution` exact in
    both forms), and the two masks are ANDed.  window = (tx0, tx1, ty0, ty1) in tiles, multiples of
    (8, 4); tiles outside it are returned as zeros.  Returns (composite, fine_only)."""
    pr = prep.params
    n, n32 = prep.n, pr.num_lights_32
    rx, ry = int(pr.resolution_xy[0]), int(pr.resolution_xy[1])
    tx0, tx1, ty0, ty1 = window if window else (0, rx, 0, ry)
    assert tx0 % 8 == 0 and tx1 % 8 == 0 and ty0 % 4 == 0 and ty1 % 4 == 0
    cull = _c(cull, np.float32)
    k3 = ref_kernels()[3].refk3_binning
    clip, res, inv = _farr(pr.clip_scale), _farr(pr.resolution_xy, np.int32), _farr(pr.inv_resolution_xy)
    fine = np.zeros((ry, rx, max(n32, 1)), np.uint32)
    k3(_p(clip), _p(res), _p(inv), n32, _p(prep.type_mask), _p(cull), n, tx0, tx1, ty0, ty1, _p(fine))
    res_c = np.array([rx // 8, ry // 4], np.int32)
    inv_c = np.array([np.float32(8.0) * np.float32(pr.inv_resolution_xy[0]), np.float32(4.0) * np.float32(pr.inv_resolution_xy[1])], np.float32)
    coarse = np.zeros((ry // 4, rx // 8, max(n32, 1)), np.uint32)
    k3(_p(clip), _p(res_c), _p(inv_c), n32, _p(prep.type_mask), _p(cull), n, tx0 // 8, tx1 // 8, ty0 // 4, ty1 // 4, _p(coarse))
    return fine & np.repeat(np.repeat(coarse, 4, 0), 8, 1), fine


def ref_z_range(prep):
    """K4 through the reference's own shader (clusterer_bindless_z_range.comp, the naive form)."""
    rz = prep.res[2]
    out = np.zeros((rz, 2), np.uint32)
    ref_kernels()[4].refk4_z_range(_p(prep.z_ranges), max(prep.n, 1), rz, _p(out))
    return out


def deferred_lighting(scene, cam: Camera, prep, clus, rows=None, want_indices=False):
    H, W = scene.depth.shape
    g = GBuffer()
    g.width, g.height = W, H
    keep = [_c(scene.albedo, np.uint32), _c(scene.normal, np.uint32), _c(scene.pbr, np.uint16),
            _c(scene.depth, np.float32), _c(scene.emissive, np.uint32)]
    g.albedo, g.normal, g.pbr, g.depth, g.emissive = [k.ctypes.data for k in keep]
    g.dir_color = (C.c_float * 3)(*scene.dir_color)
    g.dir_direction = (C.c_float * 3)(*scene.dir_direction)
    hdr = np.zeros((H, W), np.uint32)
    tile = np.zeros((H, W), np.int32) if want_indices else None
    zidx = np.zeros((H, W), np.int32) if want_indices else None
    cnt = np.zeros((H, W), np.int32) if want_indices else None
    y0, y1 = rows if rows else (0, H)
    lib().orc_deferred_lighting(C.byref(g), C.byref(cam), C.byref(prep.params), _p(prep.records),
                                _p(prep.type_mask), _p(clus.bitmask), _p(clus.range), _p(hdr),
                                _p(tile), _p(zidx), _p(cnt), y0, y1)
    if want_indices:
        return hdr, tile, zidx, cnt
    return hdr


def deferred_lighting_fp16(scene, cam: Camera, prep, clus, emissive16, rows=None, shadows=None):
    """The lighting pass into an R16G16B16A16_SFLOAT HDR-main ("renderTargetFp16").  emissive16: (H, W, 4) uint16.
    shadows = (transforms, maps, resolution) or None.  Returns (H, W, 4) uint16."""
    H, W = scene.depth.shape
    g = GBuffer()
    g.width, g.height = W, H
    keep = [_c(scene.albedo, np.uint32), _c(scene.normal, np.uint32), _c(scene.pbr, np.uint16),
            _c(scene.depth, np.float32), _c(emissive16, np.uint16)]
    g.albedo, g.normal, g.pbr, g.depth, g.emissive = [k.ctypes.data for k in keep]
    g.dir_color = (C.c_float * 3)(*scene.dir_color)
    g.dir_direction = (C.c_float * 3)(*scene.dir_direction)
    hdr = np.zeros((H, W, 4), np.uint16)
    y0, y1 = rows if rows else (0, H)
    sh = None
    if shadows is not None:
        t = _c(shadows[0], np.float32)
        held = [None if m is None else _c(m, np.uint16) for m in shadows[1]]
        table = (C.c_void_p * max(len(held), 1))(*[None if m is None else m.ctypes.data for m in held])
        sh = C.byref(Shadows(t.ctypes.data, C.cast(table, C.c_void_p), int(shadows[2]), int(shadows[3]) if len(shadows) > 3 else 0))
    lib().orc_deferred_lighting_fp16(C.byref(g), C.byref(cam), C.byref(prep.params), _p(prep.records), _p(prep.type_mask),
                                     _p(clus.bitmask), _p(clus.range), sh, _p(hdr), y0, y1)
    return hdr


_ref_light = None


def ref_light_kernels():
    """{5, 6: CDLL} of the reference's clustering.frag / directional.frag compiled for the CPU, or None."""
    global _ref_light
    if _ref_light is None and all(os.path.exists(p) for p in _REF_LIGHT_PATHS.values()):
        lib()
        _ref_light = {k: C.CDLL(p) for k, p in _REF_LIGHT_PATHS.items()}
    return _ref_light


def ref_deferred_lighting(scene, cam: Camera, prep, clus, rows=None, shadows=None, emissive16=None):
    """renderer.cpp:1004-1156 with the reference's own fragment shaders: the two draws' colours
    (fp32), then the two additive blends into B10G11R11 with DESIGN.md section 2's store rule:
    q(q(emissive + directional) + clustered).  Returns (hdr, directional_rgb, clustered_rgb).
    shadows = (transforms (n, 16) f32, maps [uint16 array | None per light], resolution): clustering.frag compiled with
    POSITIONAL_LIGHTS_SHADOW (ref_light_shim.cpp KERNEL=7)."""
    H, W = scene.depth.shape
    k = ref_light_kernels()
    y0, y1 = rows if rows else (0, H)
    alb, nrm, pbr, dep = _c(scene.albedo, np.uint32), _c(scene.normal, np.uint32), _c(scene.pbr, np.uint16), _c(scene.depth, np.float32)
    ivp = _farr(list(cam.inv_view_projection))
    cpos, cfront = _farr(list(cam.camera_position)), _farr(list(cam.camera_front))
    d_rgb = np.zeros((H, W, 3), np.float32)
    c_rgb = np.zeros((H, W, 3), np.float32)
    k[6].refk6_directional(W, H, _p(alb), _p(nrm), _p(pbr), _p(dep), _p(ivp), _p(cpos), _p(cfront), _p(_farr(list(scene.dir_color))),
                           _p(_farr(list(scene.dir_direction))), y0, y1, _p(d_rgb))
    P = prep.params
    if shadows is not None:
        t = _c(shadows[0], np.float32)
        held = [None if m is None else _c(m, np.uint16) for m in shadows[1]]
        table = (C.c_void_p * max(len(held), 1))(*[None if m is None else m.ctypes.data for m in held])
        if len(shadows) > 3 and shadows[3]:  # SHADOW_MAP_PCF_KERNEL_WIDE
            clustering = lambda *a: k[8].refk8_clustering_shadowed_pcf_wide(_p(t), table, int(shadows[2]), *a)  # noqa: E731
        else:
            clustering = lambda *a: k[7].refk7_clustering_shadowed(_p(t), table, int(shadows[2]), *a)  # noqa: E731
    else:
        clustering = k[5].refk5_clustering
    clustering(W, H, _p(alb), _p(nrm), _p(pbr), _p(dep), _p(ivp), _p(cpos), _p(_farr(list(P.camera_base))), _p(_farr(list(P.camera_front))),
                          _p(_farr(list(P.xy_scale))), _p(np.array(list(P.resolution_xy), np.int32)), int(P.num_lights), int(P.num_lights_32),
                          int(P.z_max_index), _f(P.z_scale), _p(prep.records), _p(_c(prep.type_mask, np.uint32)), _p(_c(clus.bitmask, np.uint32)),
                          _p(_c(clus.range, np.uint32)), y0, y1, _p(c_rgb))
    L = lib()
    L.orc_blend_add_r11g11b10.restype = None
    L.orc_blend_add_rgba16f.restype = None
    lit = dep != 0.0
    lit[:y0] = False
    lit[y1:] = False
    if emissive16 is not None:  # R16G16B16A16_SFLOAT HDR-main: each blend rounds to fp16
        hdr = _c(emissive16, np.uint16).copy()
        for rgb in (d_rgb, c_rgb):
            L.orc_blend_add_rgba16f(_p(hdr), _p(np.ascontiguousarray(rgb)), _p(np.ascontiguousarray(lit, dtype=np.uint8)), H * W)
        return hdr, d_rgb, c_rgb
    hdr = _c(scene.emissive, np.uint32).copy()
    for rgb in (d_rgb, c_rgb):
        L.orc_blend_add_r11g11b10(_p(hdr), _p(np.ascontiguousarray(rgb)), _p(np.ascontiguousarray(lit, dtype=np.uint8)), hdr.size)
    return hdr, d_rgb, c_rgb


# ---------------- HDR chain ----------------
def bloom_threshold(hdr, lum3, out_wh):
    h_in, w_in = hdr.shape[:2]
    w, h = out_wh
    out = np.zeros((h, w, 4), np.uint16)
    l3 = None if lum3 is None else _c(lum3, np.float32)
    if hdr.ndim == 3:  # R16G16B16A16_SFLOAT HDR image ("renderTargetFp16")
        lib().orc_bloom_threshold_fp16(_p(_c(hdr, np.uint16)), w_in, h_in, _p(l3), _p(out), w, h)
    else:
        lib().orc_bloom_threshold(_p(_c(hdr, np.uint32)), w_in, h_in, _p(l3), _p(out), w, h)
    return out


def bloom_downsample(src, out_wh, history=None, lerp=0.0):
    h_in, w_in = src.shape[:2]
    w, h = out_wh
    out = np.zeros((h, w, 4), np.uint16)
    hist = None if history is None else _c(history, np.uint16)
    lib().orc_bloom_downsample(_p(_c(src, np.uint16)), w_in, h_in, _p(hist), _f(lerp), _p(out), w, h)
    return out


def bloom_upsample(src, out_wh):
    h_in, w_in = src.shape[:2]
    w, h = out_wh
    out = np.zeros((h, w, 4), np.uint16)
    lib().orc_bloom_upsample(_p(_c(src, np.uint16)), w_in, h_in, _p(out), w, h)
    return out


def luminance(d3, lum3, lerp, lo=-3.0, hi=2.0, want_grid=False):
    h, w = d3.shape[:2]
    l3 = _c(lum3, np.float32).copy()
    grid = np.zeros((h // 2, w // 2), np.float32) if want_grid else None
    lib().orc_luminance(_p(_c(d3, np.uint16)), w, h, _f(lerp), _f(lo), _f(hi), _p(l3), _p(grid))
    return (l3, grid) if want_grid else l3


def tonemap(hdr, bloom, lum3, exposure=1.0, rows=None, target_srgb=True):
    """target_srgb: an R8G8B8A8_SRGB attachment (the swapchain) or, when False, the UNORM store of the linear value."""
    h, w = hdr.shape[:2]
    bh, bw = bloom.shape[:2]
    out = np.zeros((h, w), np.uint32)
    l3 = None if lum3 is None else _c(lum3, np.float32)
    y0, y1 = rows if rows else (0, h)
    if hdr.ndim == 3:
        lib().orc_tonemap_fp16(_p(_c(hdr, np.uint16)), w, h, _p(_c(bloom, np.uint16)), bw, bh, _p(l3), _f(exposure), int(target_srgb), _p(out), y0, y1)
    else:
        lib().orc_tonemap(_p(_c(hdr, np.uint32)), w, h, _p(_c(bloom, np.uint16)), bw, bh, _p(l3), _f(exposure), int(target_srgb), _p(out), y0, y1)
    return out


def fxaa(img, target_srgb=True, rows=None):
    h, w = img.shape
    out = np.zeros((h, w), np.uint32)
    y0, y1 = rows if rows else (0, h)
    lib().orc_fxaa(_p(_c(img, np.uint32)), w, h, int(target_srgb), _p(out), y0, y1)
    return out


def taa_resolve(hdr, depth, mv, history, reproj, quality=2, rows=None):
    h, w = hdr.shape[:2]
    out_c = np.zeros((h, w), np.uint32)
    out_h = np.zeros((h, w, 4), np.uint16)
    hist = None if history is None else _c(history, np.uint16)
    y0, y1 = rows if rows else (0, h)
    fn, dt = (lib().orc_taa_resolve_fp16, np.uint16) if hdr.ndim == 3 else (lib().orc_taa_resolve, np.uint32)
    fn(_p(_c(hdr, dt)), _p(_c(depth, np.float32)), _p(_c(mv, np.uint16)), _p(hist), w, h,
       _p(_c(reproj, np.float32)), int(quality), _p(out_c), _p(out_h), y0, y1)
    return out_c, out_h


# ---------------- the reference's own post shaders on the CPU (oracle/_ref) ----------------
def _hdr_arg(k, hdr):
    """The shim's HDR sampler reads B10G11R11 (2-D uint32 array) or, for a (H, W, 4) uint16 array, RGBA16F."""
    k.refk_set_hdr_fp16(1 if hdr.ndim == 3 else 0)
    return _c(hdr, np.uint16 if hdr.ndim == 3 else np.uint32)


def ref_bloom_threshold(hdr, lum3, out_wh):
    h_in, w_in = hdr.shape[:2]
    w, h = out_wh
    out = np.zeros((h, w, 4), np.uint16)
    k = ref_post_kernels()[7]
    a = _hdr_arg(k, hdr)
    k.refk7_bloom_threshold(_p(a), w_in, h_in, _p(_c(lum3, np.float32)), _p(out), w, h)
    k.refk_set_hdr_fp16(0)
    return out


def ref_bloom_downsample(src, out_wh, history=None, lerp=0.0):
    h_in, w_in = src.shape[:2]
    w, h = out_wh
    out = np.zeros((h, w, 4), np.uint16)
    k = ref_post_kernels()
    if history is None:
        k[8].refk8_bloom_downsample(_p(_c(src, np.uint16)), w_in, h_in, None, _f(0.0), _p(out), w, h)
    else:
        k[18].refk8_bloom_downsample_feedback(_p(_c(src, np.uint16)), w_in, h_in, _p(_c(history, np.uint16)), _f(lerp), _p(out), w, h)
    return out


def ref_bloom_upsample(src, out_wh):
    h_in, w_in = src.shape[:2]
    w, h = out_wh
    out = np.zeros((h, w, 4), np.uint16)
    ref_post_kernels()[9].refk9_bloom_upsample(_p(_c(src, np.uint16)), w_in, h_in, _p(out), w, h)
    return out


def ref_luminance(d3, lum3, lerp, lo=-3.0, hi=2.0):
    h, w = d3.shape[:2]
    l3 = _c(lum3, np.float32).copy()
    ref_post_kernels()[10].refk10_luminance(_p(_c(d3, np.uint16)), w, h, _f(lerp), _f(lo), _f(hi), _p(l3))
    return l3


def ref_tonemap(hdr, bloom, lum3, exposure=1.0, rows=None):
    h, w = hdr.shape[:2]
    bh, bw = bloom.shape[:2]
    out = np.zeros((h, w), np.uint32)
    y0, y1 = rows if rows else (0, h)
    k = ref_post_kernels()[11]
    a = _hdr_arg(k, hdr)
    k.refk11_tonemap(_p(a), w, h, _p(_c(bloom, np.uint16)), bw, bh, _p(_c(lum3, np.float32)), _f(exposure), _p(out), y0, y1)
    k.refk_set_hdr_fp16(0)
    return out


def ref_fxaa(img, target_srgb=True, rows=None):
    h, w = img.shape
    out = np.zeros((h, w), np.uint32)
    y0, y1 = rows if rows else (0, h)
    k = ref_post_kernels()
    (k[22].refk12_fxaa_srgb if target_srgb else k[12].refk12_fxaa_unorm)(_p(_c(img, np.uint32)), w, h, _p(out), y0, y1)
    return out


def ref_taa_resolve(hdr, depth, mv, history, reproj, quality=2, rows=None):
    h, w = hdr.shape[:2]
    out_c = np.zeros((h, w), np.uint32)
    out_h = np.zeros((h, w, 4), np.uint16)
    y0, y1 = rows if rows else (0, h)
    k = ref_post_kernels()
    if history is None:
        kk, fn = k[43], k[43].refk13_taa_nohistory
    else:
        kk = {0: k[23], 1: k[33], 2: k[13]}[int(quality)]
        fn = {0: k[23].refk13_taa_q0, 1: k[33].refk13_taa_q1, 2: k[13].refk13_taa_q2}[int(quality)]
    hdr = _hdr_arg(kk, hdr)
    fn(_p(hdr), _p(_c(depth, np.float32)), _p(_c(mv, np.uint16)), None if history is None else _p(_c(history, np.uint16)), w, h,
       _p(_c(reproj, np.float32)), _p(out_c), _p(out_h), y0, y1)
    kk.refk_set_hdr_fp16(0)
    return out_c, out_h


# BT.2020 primaries + D65, the HDR10 swapchain metadata the tests use
BT2020_PRIMARIES = (0.708, 0.292, 0.170, 0.797, 0.131, 0.046, 0.3127, 0.3290)


def rec709_to_display_primaries(primaries8=BT2020_PRIMARIES):
    """hdr.cpp:580-593 as a column-major mat4 (upper 3x3 filled), ready for pq10_encode."""
    out = np.zeros(9, np.float32)
    lib().orc_rec709_to_display_primaries(_p(_farr(primaries8)), _p(out))
    m = np.zeros((4, 4), np.float32)
    m[:3, :3] = out.reshape(3, 3)  # rows of `m` are COLUMNS (column-major storage)
    m[3, 3] = 1.0
    return m.reshape(-1)


def ref_rec709_to_display_primaries(primaries8=BT2020_PRIMARIES):
    """The same matrix from the reference's own fp32 chain (oracle/ref_shim.cpp), as a column-major mat4."""
    out = np.zeros(9, np.float32)
    ref().ref_rec709_to_display_primaries(_p(_farr(primaries8)), _p(out))
    m = np.zeros((4, 4), np.float32)
    m[:3, :3] = out.reshape(3, 3)
    m[3, 3] = 1.0
    return m.reshape(-1)


def pq10_encode(hdr, ui, primary16, hdr_pre=500.0, ui_pre=400.0, max_light=1000.0, rows=None):
    h, w = hdr.shape
    out = np.zeros((h, w), np.uint32)
    y0, y1 = rows if rows else (0, h)
    lib().orc_pq10_encode(_p(_c(hdr, np.uint32)), _p(_c(ui, np.uint32)), w, h, _p(_c(primary16, np.float32)), _f(hdr_pre), _f(ui_pre), _f(max_light),
                          _p(out), y0, y1)
    return out


def ref_pq10_encode(hdr, ui, primary16, hdr_pre=500.0, ui_pre=400.0, max_light=1000.0, rows=None):
    h, w = hdr.shape
    out = np.zeros((h, w), np.uint32)
    y0, y1 = rows if rows else (0, h)
    ref_post_kernels()[14].refk14_pq10_encode(_p(_c(hdr, np.uint32)), _p(_c(ui, np.uint32)), w, h, _p(_c(primary16, np.float32)), _f(hdr_pre), _f(ui_pre),
                                              _f(max_light), _p(out), y0, y1)
    return out


# ------------------------------------------------------------------------------------------- SMAA
SMAA_MAX_SEARCH_STEPS = (4, 8, 16, 32)   # SMAA.hlsl:304-324, presets Low / Medium / High / Ultra (SMAA_QUALITY 0..3)
SMAA_LUT_DIR = "/root/reference/assets/textures/smaa"


def load_gtx(path):
    """Granite's memory-mapped texture container (vulkan/texture/memory_mapped_texture.cpp:29-46): 64-byte header
    (magic, type, VkFormat, width, height, depth, layers, levels, flags, payload size), then the texels."""
    raw = open(path, "rb").read()
    assert raw[:15] == b"GRANITE TEXFMT1"
    hdr = np.frombuffer(raw[16:48], np.uint32)
    fmt, w, h = int(hdr[1]), int(hdr[2]), int(hdr[3])
    ch = {9: 1, 16: 2}[fmt]  # VK_FORMAT_R8_UNORM, VK_FORMAT_R8G8_UNORM
    return np.frombuffer(raw[64:64 + w * h * ch], np.uint8).reshape(h, w, ch).copy()


def smaa_luts():
    """(area 560x160x2, search 16x64x1) from the reference's assets."""
    return load_gtx(os.path.join(SMAA_LUT_DIR, "area.gtx")), load_gtx(os.path.join(SMAA_LUT_DIR, "search.gtx"))


def smaa_edge(color_unorm, quality, rows=None):
    h, w = color_unorm.shape
    out = np.zeros((h, w, 2), np.uint8)
    y0, y1 = rows if rows else (0, h)
    lib().orc_smaa_edge_detection(_p(_c(color_unorm, np.uint32)), w, h, int(quality), _p(out), y0, y1)
    return out


def smaa_weights(edges, area, search, quality, rows=None):
    h, w = edges.shape[:2]
    out = np.zeros((h, w), np.uint32)
    y0, y1 = rows if rows else (0, h)
    lib().orc_smaa_blend_weights(_p(_c(edges, np.uint8)), w, h, _p(_c(area, np.uint8)), _p(_c(search, np.uint8)), int(quality), _p(out), y0, y1)
    return out


def smaa_blend(color_unorm, weights, rows=None):
    h, w = color_unorm.shape
    out = np.zeros((h, w), np.uint32)
    y0, y1 = rows if rows else (0, h)
    lib().orc_smaa_neighborhood_blend(_p(_c(color_unorm, np.uint32)), _p(_c(weights, np.uint32)), w, h, _p(out), y0, y1)
    return out


def ref_smaa_edge(color_unorm, quality, rows=None):
    h, w = color_unorm.shape
    out = np.zeros((h, w, 2), np.uint8)
    y0, y1 = rows if rows else (0, h)
    ref_post_kernels()[150 + quality].refk_smaa_edge(_p(_c(color_unorm, np.uint32)), w, h, _p(out), y0, y1)
    return out


def ref_smaa_weights(edges, area, search, quality, rows=None):
    h, w = edges.shape[:2]
    out = np.zeros((h, w), np.uint32)
    y0, y1 = rows if rows else (0, h)
    ref_post_kernels()[160 + quality].refk_smaa_weights(_p(_c(edges, np.uint8)), w, h, _p(_c(area, np.uint8)), _p(_c(search, np.uint8)),
                                                        SMAA_MAX_SEARCH_STEPS[quality], _p(out), y0, y1)
    return out


def ref_smaa_blend(color_unorm, weights, quality, rows=None):
    h, w = color_unorm.shape
    out = np.zeros((h, w), np.uint32)
    y0, y1 = rows if rows else (0, h)
    ref_post_kernels()[170 + quality].refk_smaa_blend(_p(_c(color_unorm, np.uint32)), _p(_c(weights, np.uint32)), w, h, _p(out), y0, y1)
    return out


def pyramid_sizes(w, h):
    """ceil(parent * scale), renderer/render_graph.cpp:3160-3171; scales 1/2 .. 1/32 of the HDR input."""
    import math
    return [(int(math.ceil(w * s)), int(math.ceil(h * s))) for s in (0.5, 0.25, 0.125, 0.0625, 0.03125)]


def hdr_chain(hdr, lum3, d3_history, frame_time=1.0 / 60.0, exposure=1.0, dynamic_exposure=True):
    """One frame of setup_hdr_postprocess_compute (renderer/post/hdr.cpp:354-379) + tonemap.  hdr: (H, W) uint32 B10G11R11 or
    (H, W, 4) uint16 RGBA16F."""
    h, w = hdr.shape[:2]
    sz = pyramid_sizes(w, h)
    lerp_d3 = np.float32(1.0 - 0.001 ** frame_time)   # hdr.cpp:182 (double math, then float)
    lerp_lum = np.float32(1.0 - 0.5 ** frame_time)    # hdr.cpp:93
    lum_in = _c(lum3, np.float32) if dynamic_exposure else None
    t = bloom_threshold(hdr, lum_in, sz[0])
    d0 = bloom_downsample(t, sz[1])
    d1 = bloom_downsample(d0, sz[2])
    d2 = bloom_downsample(d1, sz[3])
    d3 = bloom_downsample(d2, sz[4], d3_history, lerp_d3)
    lum_out = luminance(d3, lum3, lerp_lum) if dynamic_exposure else None
    u2 = bloom_upsample(d3, sz[3])
    u1 = bloom_upsample(u2, sz[2])
    u0 = bloom_upsample(u1, sz[1])
    ldr = tonemap(hdr, u0, lum_out, exposure)
    return SimpleNamespace(t=t, d0=d0, d1=d1, d2=d2, d3=d3, u2=u2, u1=u1, u0=u0, lum=lum_out, ldr=ldr)


# ---------------- FSR 1 (renderer/post/aa.cpp:34-174) ----------------
def fsr_easu_constants(w_in, h_in, w_out, h_out):
    con = np.zeros(16, np.float32)
    lib().orc_fsr_easu_constants(int(w_in), int(h_in), int(w_out), int(h_out), _p(con))
    return con


def fsr_rcas_constants(sharpness_stops=0.5):
    con = np.zeros(4, np.float32)
    lib().orc_fsr_rcas_constants(_f(sharpness_stops), _p(con))
    return con


def fsr_upscale(img, out_wh, target_srgb=False, rows=None):
    """upscale.frag: img (h, w) uint32 RGBA8 read as UNORM -> (h_out, w_out) uint32."""
    h, w = img.shape
    wo, ho = out_wh
    out = np.zeros((ho, wo), np.uint32)
    y0, y1 = rows if rows else (0, ho)
    lib().orc_fsr_easu(_p(_c(img, np.uint32)), w, h, _p(fsr_easu_constants(w, h, wo, ho)), _p(out), wo, ho, int(target_srgb), y0, y1)
    return out


def fsr_sharpen(img, sharpness_stops=0.5, srgb=True, rows=None):
    """sharpen.frag: srgb = the target is an sRGB attachment (input read through an sRGB view)."""
    h, w = img.shape
    out = np.zeros((h, w), np.uint32)
    y0, y1 = rows if rows else (0, h)
    lib().orc_fsr_rcas(_p(_c(img, np.uint32)), w, h, _p(fsr_rcas_constants(sharpness_stops)), _p(out), int(srgb), y0, y1)
    return out


def ref_fsr_upscale(img, out_wh, target_srgb=False, rows=None):
    """The reference's upscale.frag on the CPU (oracle/_ref/libgranite_ref_p24 / p25)."""
    k = ref_post_kernels()
    h, w = img.shape
    wo, ho = out_wh
    out = np.zeros((ho, wo), np.uint32)
    y0, y1 = rows if rows else (0, ho)
    fn = k[25].refk25_fsr_upscale_srgb if target_srgb else k[24].refk24_fsr_upscale_unorm
    fn(_p(_c(img, np.uint32)), w, h, _p(fsr_easu_constants(w, h, wo, ho)), _p(out), wo, ho, y0, y1)
    return out


def ref_fsr_sharpen(img, sharpness_stops=0.5, srgb=True, rows=None):
    """The reference's sharpen.frag on the CPU (oracle/_ref/libgranite_ref_p26)."""
    k = ref_post_kernels()
    h, w = img.shape
    out = np.zeros((h, w), np.uint32)
    y0, y1 = rows if rows else (0, h)
    k[26].refk26_fsr_sharpen(_p(_c(img, np.uint32)), w, h, _p(fsr_rcas_constants(sharpness_stops)), int(srgb), _p(out), y0, y1)
    return out


# ---------------- volumetric-decal binning (clusterer.cpp:1348-1461) ----------------
def decal_mvps(cam: Camera, world_rows):
    """world_rows: (n, 12) f32 mat_affine rows -> (n, 16) f32 view_projection * world."""
    w = _c(world_rows, np.float32).reshape(-1, 12)
    out = np.zeros((len(w), 16), np.float32)
    vp = _farr(list(cam.view_projection))
    for i in range(len(w)):
        lib().orc_decal_mvp(_p(vp), _p(w[i]), _p(out[i]))
    return out


def decal_z_ranges(cam: Camera, world_rows):
    w = _c(world_rows, np.float32).reshape(-1, 12)
    out = np.zeros((len(w), 2), np.float32)
    for i in range(len(w)):
        lib().orc_decal_z_range(C.byref(cam), _p(w[i]), _p(out[i]))
    return out


def decal_binning(res_xy, mvps):
    rx, ry = res_xy
    m = _c(mvps, np.float32).reshape(-1, 16)
    n = len(m)
    inv = np.array([1.0 / rx, 1.0 / ry], np.float32)
    out = np.zeros((ry, rx, max((n + 31) // 32, 1)), np.uint32)
    lib().orc_decal_binning(rx, ry, _p(inv), n, _p(m), _p(out))
    return out


def ref_decal_binning(res_xy, mvps):
    """The reference's clusterer_bindless_binning_decal.comp (SUBGROUPS=0) on the CPU."""
    rx, ry = res_xy
    m = _c(mvps, np.float32).reshape(-1, 16)
    n = len(m)
    out = np.zeros((ry, rx, max((n + 31) // 32, 1)), np.uint32)
    ref_kernels()[5].refk5_decal_binning(_p(np.array([rx, ry], np.int32)), _p(np.array([1.0 / rx, 1.0 / ry], np.float32)), n, _p(m), _p(out))
    return out


# ---------------- volumetric fog, accumulation pass (volumetric_fog.cpp:236-254) ----------------
def fog_accumulate(light):
    """light: (d, h, w, 4) uint16 RGBA16F froxel grid (rgb in-scattered light, a optical depth) -> fog, same shape."""
    d, h, w = light.shape[:3]
    out = np.zeros((d, h, w, 4), np.uint16)
    lib().orc_fog_accumulate(_p(_c(light, np.uint16)), w, h, d, _p(out))
    return out


def ref_fog_accumulate(light):
    """The reference's fog_accumulate.comp on the CPU (oracle/_ref/libgranite_ref_p27)."""
    d, h, w = light.shape[:3]
    out = np.zeros((d, h, w, 4), np.uint16)
    ref_post_kernels()[27].refk27_fog_accumulate(_p(_c(light, np.uint16)), w, h, d, _p(out))
    return out


# ---------------- volumetric fog, light-density pass (volumetric_fog.cpp:115-228), base variant ----------------
class FogParams(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("depth", C.c_int), ("dither_offset", C.c_int),
                ("slice_z_log2_scale", C.c_float), ("density_mod", C.c_float), ("in_scatter_strength", C.c_float)]


def fog_params(w, h, d, z_range=80.0, density=0.5, in_scatter=1.0, dither_offset=0):
    """slice_z_log2_scale = 1 / log2(1 + z_range), in fp32 (volumetric_fog.cpp:87-91)."""
    s = np.float32(1.0) / np.float32(np.log2(np.float32(1.0) + np.float32(z_range)))
    return FogParams(int(w), int(h), int(d), int(dither_offset), float(s), float(density), float(in_scatter))


def fog_slice_extents(fp: FogParams):
    out = np.zeros(fp.depth, np.float32)
    lib().orc_fog_slice_extents(fp.depth, _f(fp.slice_z_log2_scale), _p(out))
    return out


def fog_light_density(fp: FogParams, cam: Camera, prep, clus, dir_color, dir_direction, dither_lut):
    """dither_lut: (layers, 128, 128) uint32 RGBA8.  Returns (d, h, w, 4) uint16 RGBA16F."""
    out = np.zeros((fp.depth, fp.height, fp.width, 4), np.uint16)
    ext = fog_slice_extents(fp)
    lib().orc_fog_light_density(C.byref(fp), C.byref(cam), C.byref(prep.params), _p(prep.records), _p(prep.type_mask), _p(_c(clus.bitmask, np.uint32)),
                                _p(_c(clus.range, np.uint32)), _p(_farr(list(dir_color))), _p(_farr(list(dir_direction))), _p(ext),
                                _p(_c(dither_lut, np.uint32)), _p(out))
    return out


def ref_fog_light_density(fp: FogParams, cam: Camera, prep, clus, dir_color, dir_direction, dither_lut):
    """The reference's fog_light_density.comp (base variant) on the CPU (oracle/_ref/libgranite_ref_l9)."""
    out = np.zeros((fp.depth, fp.height, fp.width, 4), np.uint16)
    ext = fog_slice_extents(fp)
    P = prep.params
    ref_light_kernels()[9].refk9_fog_light_density(
        fp.width, fp.height, fp.depth, fp.dither_offset, _f(fp.slice_z_log2_scale), _f(fp.density_mod), _f(fp.in_scatter_strength),
        _p(_farr(list(cam.inv_view_projection))), _p(_farr(list(cam.projection))), _p(_farr(list(cam.inv_projection))),
        _p(_farr(list(cam.camera_position))), _p(_farr(list(cam.camera_front))), _p(_farr(list(dir_color))), _p(_farr(list(dir_direction))),
        _p(_farr(list(P.transform))), _p(_farr(list(P.camera_base))), _p(_farr(list(P.camera_front))), _p(_farr(list(P.xy_scale))),
        _p(np.array(list(P.resolution_xy), np.int32)), int(P.num_lights), int(P.num_lights_32), int(P.z_max_index), _f(P.z_scale),
        _p(prep.records), _p(_c(prep.type_mask, np.uint32)), _p(_c(clus.bitmask, np.uint32)), _p(_c(clus.range, np.uint32)), _p(ext),
        _p(_c(dither_lut, np.uint32)), _p(out))
    return out
