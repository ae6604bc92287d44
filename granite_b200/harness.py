"""numpy-in / numpy-out helpers over the C ABI, one per entry point, for the parity tests.

Each helper uploads its inputs with torch (device memory only), calls the extern "C" function
on the current stream and downloads the result.  No arithmetic happens in Python.
"""
from __future__ import annotations

import ctypes as C
from types import SimpleNamespace

import numpy as np
import torch

from . import capi


def _dev(a: np.ndarray) -> torch.Tensor:
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint32:
        return torch.from_numpy(a.view(np.int32)).cuda()
    if a.dtype == np.uint16:
        return torch.from_numpy(a.view(np.int16)).cuda()
    return torch.from_numpy(a).cuda()


def _host(t: torch.Tensor, dtype) -> np.ndarray:
    return t.cpu().numpy().view(dtype)


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def camera_struct(cam) -> capi.GrbCamera:
    """cam: any object with view, view_projection, inv_view_projection (16 floats), camera_position,
    camera_front (3 floats), z_near, z_far."""
    c = capi.GrbCamera()
    c.view = (C.c_float * 16)(*list(cam.view))
    c.view_projection = (C.c_float * 16)(*list(cam.view_projection))
    c.inv_view_projection = (C.c_float * 16)(*list(cam.inv_view_projection))
    c.camera_position = (C.c_float * 3)(*list(cam.camera_position))
    c.camera_front = (C.c_float * 3)(*list(cam.camera_front))
    c.z_near = cam.z_near
    c.z_far = cam.z_far
    return c


def params_struct(p) -> capi.GrbClusterParameters:
    q = capi.GrbClusterParameters()
    for name, _ in capi.GrbClusterParameters._fields_:
        v = getattr(p, name)
        if hasattr(v, "__len__"):
            getattr(q, name)[:] = list(v)
        else:
            setattr(q, name, v)
    return q


class ClusterDevice:
    """Device-side light cluster buffers (what the render graph would own)."""

    def __init__(self, records, model, type_mask, z_ranges, params, res):
        n = params.num_lights
        n32 = params.num_lights_32
        rx, ry, rz = res
        self.res = res
        self.params = params_struct(params)
        self.records = _dev(np.frombuffer(np.ascontiguousarray(records).tobytes(), np.uint8))
        self.model = _dev(np.ascontiguousarray(model, np.float32))
        self.type_mask = _dev(np.ascontiguousarray(type_mask, np.uint32))
        self.z_ranges = _dev(np.ascontiguousarray(z_ranges, np.uint32))
        # graph buffers are zero-initialised at creation (renderer/render_graph.cpp:2587)
        self.spots = torch.zeros((max(n, 1), 24), dtype=torch.float32, device="cuda")
        self.cull = torch.zeros((max(n, 1), 128), dtype=torch.float32, device="cuda")
        self.bitmask = torch.zeros((ry, rx, max(n32, 1)), dtype=torch.int32, device="cuda")
        self.range = torch.zeros((rz, 2), dtype=torch.int32, device="cuda")
        b = capi.GrbClusterBuffers()
        b.lights = self.records.data_ptr()
        b.model = self.model.data_ptr()
        b.type_mask = self.type_mask.data_ptr()
        b.z_ranges = self.z_ranges.data_ptr()
        b.transformed_spots = self.spots.data_ptr()
        b.cull_setup = self.cull.data_ptr()
        b.bitmask = self.bitmask.data_ptr()
        b.cluster_range = self.range.data_ptr()
        b.resolution_z = rz
        self.buffers = b

    def build(self, cam: capi.GrbCamera):
        capi.check(capi.lib().grb_cluster_build(C.byref(cam), C.byref(self.params), C.byref(self.buffers), capi.stream_ptr()),
                   "grb_cluster_build")

    def download(self):
        return SimpleNamespace(spots=_host(self.spots, np.float32), cull=_host(self.cull, np.float32),
                               bitmask=_host(self.bitmask, np.uint32), range=_host(self.range, np.uint32))


class GBufferDevice:
    def __init__(self, scene):
        self.h, self.w = scene.depth.shape
        self.albedo = _dev(scene.albedo)
        self.normal = _dev(scene.normal)
        self.pbr = _dev(scene.pbr)
        self.depth = _dev(scene.depth)
        self.emissive = _dev(scene.emissive)
        g = capi.GrbGBuffer()
        g.albedo = capi.image(self.albedo, capi.FORMAT_R8G8B8A8_SRGB)
        g.normal = capi.image(self.normal, capi.FORMAT_A2B10G10R10_UNORM)
        g.pbr = capi.image(self.pbr, capi.FORMAT_R8G8_UNORM)
        g.depth = capi.image(self.depth, capi.FORMAT_D32_SFLOAT)
        g.directional_color = (C.c_float * 3)(*scene.dir_color)
        g.directional_direction = (C.c_float * 3)(*scene.dir_direction)
        self.struct = g


def _hdr_img(t):
    """HDR-main / emissive: an (H, W) int32 tensor is B10G11R11_UFLOAT, an (H, W, 4) int16 tensor R16G16B16A16_SFLOAT ("renderTargetFp16")."""
    return capi.image(t, capi.FORMAT_R16G16B16A16_SFLOAT if t.dim() == 3 else capi.FORMAT_B10G11R11_UFLOAT)


def lighting_schedule(height: int) -> torch.Tensor:
    """Zero-initialised schedule buffer for grb_deferred_lighting_scheduled (kept across frames)."""
    return torch.zeros(int(capi.lib().grb_lighting_schedule_bytes(height)) // 4, dtype=torch.int32, device="cuda")


def deferred_lighting(gb: GBufferDevice, cam: capi.GrbCamera, cluster: ClusterDevice, hdr: torch.Tensor, rows=None, schedule=None):
    """hdr: int32 (H, W) tensor (or int16 (H, W, 4): RGBA16F) holding the emissive / HDR-main attachment; updated in place."""
    img = _hdr_img(hdr)
    if schedule is not None:
        capi.check(capi.lib().grb_deferred_lighting_scheduled(C.byref(gb.struct), C.byref(cam), C.byref(cluster.params), C.byref(cluster.buffers),
                                                              C.byref(img), capi.rows(rows), _ptr(schedule), capi.stream_ptr()),
                   "grb_deferred_lighting_scheduled")
        return
    capi.check(capi.lib().grb_deferred_lighting(C.byref(gb.struct), C.byref(cam), C.byref(cluster.params), C.byref(cluster.buffers),
                                                C.byref(img), capi.rows(rows), capi.stream_ptr()), "grb_deferred_lighting")


def deferred_lighting_blocks(gb: GBufferDevice, cam: capi.GrbCamera, cluster: ClusterDevice, hdr: torch.Tensor, rows=None):
    """grb_deferred_lighting_blocks: the pass as a grid of short-lived CTAs (the non-persistent pairs kernel)."""
    img = _hdr_img(hdr)
    capi.check(capi.lib().grb_deferred_lighting_blocks(C.byref(gb.struct), C.byref(cam), C.byref(cluster.params), C.byref(cluster.buffers),
                                                       C.byref(img), capi.rows(rows), capi.stream_ptr()), "grb_deferred_lighting_blocks")


def deferred_lighting_shadowed(gb: GBufferDevice, cam: capi.GrbCamera, cluster: ClusterDevice, transforms: torch.Tensor, map_table: torch.Tensor,
                              resolution: int, hdr: torch.Tensor, rows=None, pcf_wide=False):
    """Lighting with shadowed positional lights.  transforms: float32 (n, 16) device tensor (cluster order); map_table: int64 (n,)
    device tensor of device pointers to each light's D16 map (0 = no shadow)."""
    img = _hdr_img(hdr)
    sh = capi.GrbLightShadows(_ptr(transforms), _ptr(map_table), int(resolution), int(pcf_wide))
    capi.check(capi.lib().grb_deferred_lighting_shadowed(C.byref(gb.struct), C.byref(cam), C.byref(cluster.params), C.byref(cluster.buffers),
                                                         C.byref(sh), C.byref(img), capi.rows(rows), capi.stream_ptr()), "grb_deferred_lighting_shadowed")


def deferred_lighting_stripes(gb: GBufferDevice, cam: capi.GrbCamera, cluster: ClusterDevice, hdr: torch.Tensor, stripes, schedule=None, shadows=None):
    """grb_deferred_lighting_stripes over the stripe set stripes = (first, rows, period).  shadows: None, or
    (transforms, map_table, resolution) as for deferred_lighting_shadowed."""
    img = _hdr_img(hdr)
    sh = None
    if shadows is not None:
        transforms, map_table, resolution = shadows
        sh = C.byref(capi.GrbLightShadows(_ptr(transforms), _ptr(map_table), int(resolution), 0))
    capi.check(capi.lib().grb_deferred_lighting_stripes(C.byref(gb.struct), C.byref(cam), C.byref(cluster.params), C.byref(cluster.buffers), sh,
                                                        C.byref(img), capi.GrbStripes(*stripes), None if schedule is None else _ptr(schedule),
                                                        capi.stream_ptr()),
               "grb_deferred_lighting_stripes")


def hdr_rows_to_peers(hdr_t, slots, flag_arrays, peer_rows, flag_index, epoch, counter_t, stripes, width=None):
    """grb_hdr_rows_to_peers with every rank's HDR slot and flag array as tensors on this device: hdr_t and slots[q]
    (H, P) int32 (B10G11R11) or (H, P, 4) int16 (RGBA16F), the image the first `width` texels of each row (all P by
    default); peer_rows[q] = rank q's lighting rows (y0, y1)."""
    img = _hdr_img(hdr_t)
    if width is not None:
        img.width = int(width)
    n = len(slots)
    images = (C.c_void_p * n)(*[t.data_ptr() for t in slots])
    flags = (C.c_void_p * n)(*[t.data_ptr() for t in flag_arrays])
    rows = (capi.GrbRows * n)(*[capi.GrbRows(int(a), int(b)) for a, b in peer_rows])
    capi.check(capi.lib().grb_hdr_rows_to_peers(C.byref(img), images, flags, rows, n, int(flag_index), int(epoch), _ptr(counter_t),
                                                capi.GrbStripes(*stripes), capi.stream_ptr()),
               "grb_hdr_rows_to_peers")


def _img16(t):
    return capi.image(t, capi.FORMAT_R16G16B16A16_SFLOAT)


def new_rgba16f(w, h):
    return torch.zeros((h, w, 4), dtype=torch.int16, device="cuda")


def bloom_threshold(hdr_t, lum_t, out_t, rows=None):
    hi = _hdr_img(hdr_t)
    oi = _img16(out_t)
    capi.check(capi.lib().grb_bloom_threshold(C.byref(hi), _ptr(lum_t), C.byref(oi), capi.rows(rows), capi.stream_ptr()), "grb_bloom_threshold")


def bloom_threshold_downsample(hdr_t, lum_t, d0_t, threshold_t=None, rows=None):
    """Fused K7 + first K8 (TMA tiles); raises GrbError when the shape is not eligible."""
    hi = _hdr_img(hdr_t)
    oi = _img16(d0_t)
    ti = C.byref(_img16(threshold_t)) if threshold_t is not None else None
    capi.check(capi.lib().grb_bloom_threshold_downsample(C.byref(hi), _ptr(lum_t), ti, C.byref(oi), capi.rows(rows), capi.stream_ptr()),
               "grb_bloom_threshold_downsample")


def bloom_downsample(in_t, out_t, history_t=None, lerp=0.0, rows=None):
    ii, oi = _img16(in_t), _img16(out_t)
    hi = C.byref(_img16(history_t)) if history_t is not None else None
    capi.check(capi.lib().grb_bloom_downsample(C.byref(ii), hi, C.c_float(lerp), C.byref(oi), capi.rows(rows), capi.stream_ptr()),
               "grb_bloom_downsample")


def bloom_upsample(in_t, out_t, rows=None):
    ii, oi = _img16(in_t), _img16(out_t)
    capi.check(capi.lib().grb_bloom_upsample(C.byref(ii), C.byref(oi), capi.rows(rows), capi.stream_ptr()), "grb_bloom_upsample")


def bloom_upsample_exact(in_t, out_t, rows=None):
    """The shader's arithmetic at every size (no tile kernel): the u0 a frame computes when the fused tail does not run."""
    ii, oi = _img16(in_t), _img16(out_t)
    capi.check(capi.lib().grb_bloom_upsample_exact(C.byref(ii), C.byref(oi), capi.rows(rows), capi.stream_ptr()), "grb_bloom_upsample_exact")


def bloom_tail(d0_t, d1_t, d2_t, d3_t, history_t, lerp_d3, lum_t, lerp_lum, u2_t, u1_t, lo=-3.0, hi=2.0, u0_t=None, u0_rows=None, max_ctas=0):
    """d1, d2, d3 (+feedback), luminance, u2, u1 in one cooperative launch; with u0_t also (rows of) u0."""
    im = [_img16(t) for t in (d0_t, d1_t, d2_t, d3_t, u2_t, u1_t)]
    hi_ = C.byref(_img16(history_t)) if history_t is not None else None
    if u0_t is not None or max_ctas:
        opt = capi.GrbBloomTailOptions()
        u0i = _img16(u0_t) if u0_t is not None else None
        opt.u0 = C.cast(C.pointer(u0i), C.c_void_p) if u0i is not None else None
        opt.u0_rows = capi.rows(u0_rows)
        opt.max_ctas = int(max_ctas)
        capi.check(capi.lib().grb_bloom_tail_ex(C.byref(im[0]), C.byref(im[1]), C.byref(im[2]), C.byref(im[3]), hi_, C.c_float(lerp_d3), _ptr(lum_t),
                                                C.c_float(lerp_lum), C.c_float(lo), C.c_float(hi), C.byref(im[4]), C.byref(im[5]), C.byref(opt),
                                                capi.stream_ptr()), "grb_bloom_tail_ex")
        return
    capi.check(capi.lib().grb_bloom_tail(C.byref(im[0]), C.byref(im[1]), C.byref(im[2]), C.byref(im[3]), hi_, C.c_float(lerp_d3), _ptr(lum_t),
                                         C.c_float(lerp_lum), C.c_float(lo), C.c_float(hi), C.byref(im[4]), C.byref(im[5]), capi.stream_ptr()),
               "grb_bloom_tail")


def luminance(d3_t, lum_t, lerp, lo=-3.0, hi=2.0):
    di = _img16(d3_t)
    capi.check(capi.lib().grb_luminance(C.byref(di), _ptr(lum_t), C.c_float(lerp), C.c_float(lo), C.c_float(hi), capi.stream_ptr()), "grb_luminance")


def luminance_grid(d3_t, grid_t, rows=None):
    di = _img16(d3_t)
    capi.check(capi.lib().grb_luminance_grid(C.byref(di), _ptr(grid_t), capi.rows(rows), capi.stream_ptr()), "grb_luminance_grid")


def luminance_finalize(grid_t, size_x, size_y, lum_t, lerp, lo=-3.0, hi=2.0):
    capi.check(capi.lib().grb_luminance_finalize(_ptr(grid_t), size_x, size_y, _ptr(lum_t), C.c_float(lerp), C.c_float(lo), C.c_float(hi),
                                                 capi.stream_ptr()), "grb_luminance_finalize")


def tonemap(hdr_t, bloom_t, lum_t, out_t, exposure=1.0, srgb=True, rows=None):
    hi = _hdr_img(hdr_t)
    bi = _img16(bloom_t)
    oi = capi.image(out_t, capi.FORMAT_R8G8B8A8_SRGB if srgb else capi.FORMAT_R8G8B8A8_UNORM)
    capi.check(capi.lib().grb_tonemap(C.byref(hi), C.byref(bi), _ptr(lum_t), C.c_float(exposure), C.byref(oi), capi.rows(rows), capi.stream_ptr()),
               "grb_tonemap")


def fxaa(in_t, out_t, target_srgb=True, rows=None):
    fmt = capi.FORMAT_R8G8B8A8_SRGB if target_srgb else capi.FORMAT_R8G8B8A8_UNORM
    ii, oi = capi.image(in_t, fmt), capi.image(out_t, fmt)
    capi.check(capi.lib().grb_fxaa(C.byref(ii), C.byref(oi), capi.rows(rows), capi.stream_ptr()), "grb_fxaa")


def pq10_encode(hdr_t, ui_t, primary16, hdr_pre, ui_pre, max_light, out_t, rows=None):
    hi = _hdr_img(hdr_t)
    ui = capi.image(ui_t, capi.FORMAT_R8G8B8A8_UNORM)
    oi = capi.image(out_t, capi.FORMAT_A2B10G10R10_UNORM)
    m = (C.c_float * 16)(*np.asarray(primary16, np.float32).reshape(-1).tolist())
    capi.check(capi.lib().grb_pq10_encode(C.byref(hi), C.byref(ui), m, float(hdr_pre), float(ui_pre), float(max_light), C.byref(oi), capi.rows(rows),
                                          capi.stream_ptr()), "grb_pq10_encode")


def smaa_edge_detection(color_t, quality, edges_t, rows=None):
    """color_t: (H, W) int32 RGBA8 (read as UNORM); edges_t: (H, W, 2) uint8."""
    ci, ei = capi.image(color_t, capi.FORMAT_R8G8B8A8_UNORM), capi.image(edges_t, capi.FORMAT_R8G8_UNORM)
    capi.check(capi.lib().grb_smaa_edge_detection(C.byref(ci), int(quality), C.byref(ei), capi.rows(rows), capi.stream_ptr()), "grb_smaa_edge_detection")


def smaa_edge_detection_to_peers(color_t, quality, edge_images, flag_arrays, windows, flag_index, epoch, counter_t, rows=None):
    """grb_smaa_edge_detection_to_peers with every rank's edge image and flag array as a tensor on this device:
    edge_images[q]: (H, W, 2) uint8, flag_arrays[q]: int32 tensor, windows[q]: (y0, y1); counter_t: one zeroed int32."""
    n = len(edge_images)
    ci, li = capi.image(color_t, capi.FORMAT_R8G8B8A8_UNORM), capi.image(edge_images[0], capi.FORMAT_R8G8_UNORM)
    images = (C.c_void_p * n)(*[t.data_ptr() for t in edge_images])
    flags = (C.c_void_p * n)(*[t.data_ptr() for t in flag_arrays])
    wins = (capi.GrbRows * n)(*[capi.GrbRows(int(a), int(b)) for a, b in windows])
    capi.check(capi.lib().grb_smaa_edge_detection_to_peers(C.byref(ci), int(quality), C.byref(li), images, flags, wins, n, int(flag_index), int(epoch),
                                                           _ptr(counter_t), capi.rows(rows), capi.stream_ptr()), "grb_smaa_edge_detection_to_peers")


def smaa_blend_weights(edges_t, area_t, search_t, quality, weights_t, rows=None):
    """area_t: (560, 160, 2) uint8, search_t: (16, 64) or (16, 64, 1) uint8, weights_t: (H, W) int32."""
    ei, ai = capi.image(edges_t, capi.FORMAT_R8G8_UNORM), capi.image(area_t, capi.FORMAT_R8G8_UNORM)
    si, wi = capi.image(search_t, capi.FORMAT_R8_UNORM), capi.image(weights_t, capi.FORMAT_R8G8B8A8_UNORM)
    capi.check(capi.lib().grb_smaa_blend_weights(C.byref(ei), C.byref(ai), C.byref(si), int(quality), C.byref(wi), capi.rows(rows), capi.stream_ptr()),
               "grb_smaa_blend_weights")


def smaa_neighborhood_blend(color_t, weights_t, out_t, target_srgb=True, rows=None):
    ci, wi = capi.image(color_t, capi.FORMAT_R8G8B8A8_UNORM), capi.image(weights_t, capi.FORMAT_R8G8B8A8_UNORM)
    oi = capi.image(out_t, capi.FORMAT_R8G8B8A8_SRGB if target_srgb else capi.FORMAT_R8G8B8A8_UNORM)
    capi.check(capi.lib().grb_smaa_neighborhood_blend(C.byref(ci), C.byref(wi), C.byref(oi), capi.rows(rows), capi.stream_ptr()), "grb_smaa_neighborhood_blend")


def fsr_upscale(color_t, out_t, target_srgb=False, rows=None):
    """color_t: (h_in, w_in) int32 RGBA8; out_t: (h_out, w_out) int32 RGBA8 (UNORM when a sharpen pass follows)."""
    ci = capi.image(color_t, capi.FORMAT_R8G8B8A8_UNORM)
    oi = capi.image(out_t, capi.FORMAT_R8G8B8A8_SRGB if target_srgb else capi.FORMAT_R8G8B8A8_UNORM)
    capi.check(capi.lib().grb_fsr_upscale(C.byref(ci), C.byref(oi), capi.rows(rows), capi.stream_ptr()), "grb_fsr_upscale")


def fsr_sharpen(color_t, out_t, sharpness_stops=0.5, srgb=True, rows=None):
    fmt = capi.FORMAT_R8G8B8A8_SRGB if srgb else capi.FORMAT_R8G8B8A8_UNORM
    ci, oi = capi.image(color_t, capi.FORMAT_R8G8B8A8_UNORM), capi.image(out_t, fmt)
    capi.check(capi.lib().grb_fsr_sharpen(C.byref(ci), C.byref(oi), C.c_float(sharpness_stops), capi.rows(rows), capi.stream_ptr()), "grb_fsr_sharpen")


def taa_resolve(hdr_t, depth_t, mv_t, history_t, reproj, quality, out_color_t, out_history_t, rows=None):
    hi = _hdr_img(hdr_t)
    oc = capi.image(out_color_t, capi.FORMAT_B10G11R11_UFLOAT)
    oh = _img16(out_history_t)
    di = C.byref(capi.image(depth_t, capi.FORMAT_D32_SFLOAT)) if depth_t is not None else None
    mi = C.byref(capi.image(mv_t, capi.FORMAT_R16G16_SFLOAT)) if mv_t is not None else None
    hs = C.byref(_img16(history_t)) if history_t is not None else None
    rp = None
    if reproj is not None:
        rp = (C.c_float * 16)(*np.asarray(reproj, np.float32).reshape(-1).tolist())
    capi.check(capi.lib().grb_taa_resolve(C.byref(hi), di, mi, hs, rp, int(quality), C.byref(oc), C.byref(oh), capi.rows(rows), capi.stream_ptr()),
               "grb_taa_resolve")


def taa_resolve_to_peers(hdr_t, depth_t, mv_t, history_t, reproj, quality, out_color_t, history_images, flag_arrays, flag_index, epoch, counter_t,
                         rows=None, own=None):
    """grb_taa_resolve_to_peers with every rank's history image and flag array as a tensor on this device:
    history_images[r]: (H, W, 4) uint16, flag_arrays[r]: int32 tensor; counter_t: one zeroed int32."""
    n = len(history_images)
    hi = _hdr_img(hdr_t)
    oc = capi.image(out_color_t, capi.FORMAT_B10G11R11_UFLOAT)
    layout = _img16(history_images[0])
    di = C.byref(capi.image(depth_t, capi.FORMAT_D32_SFLOAT)) if depth_t is not None else None
    mi = C.byref(capi.image(mv_t, capi.FORMAT_R16G16_SFLOAT)) if mv_t is not None else None
    hs = C.byref(_img16(history_t)) if history_t is not None else None
    rp = (C.c_float * 16)(*np.asarray(reproj, np.float32).reshape(-1).tolist()) if reproj is not None else None
    images = (C.c_void_p * n)(*[t.data_ptr() for t in history_images])
    flags = (C.c_void_p * n)(*[t.data_ptr() for t in flag_arrays])
    capi.check(capi.lib().grb_taa_resolve_to_peers(C.byref(hi), di, mi, hs, rp, int(quality), C.byref(oc), C.byref(layout), images, flags, n, int(flag_index),
                                                   int(epoch), _ptr(counter_t), capi.rows(rows), capi.rows(own), capi.stream_ptr()),
               "grb_taa_resolve_to_peers")


def peer_publish(flag_arrays, flag_index, epoch, counter_t):
    """grb_peer_publish with every rank's flag array as tensors on this device: flag_arrays[r] an int32 tensor;
    counter_t: one zeroed int32."""
    flags = (C.c_void_p * len(flag_arrays))(*[t.data_ptr() for t in flag_arrays])
    capi.check(capi.lib().grb_peer_publish(flags, len(flag_arrays), int(flag_index), int(epoch), _ptr(counter_t), capi.stream_ptr()),
               "grb_peer_publish")


def present_rows_to_peer(src_t, dst_t, flag_arrays, flag_index, epoch, counter_t, own, fmt=capi.FORMAT_R8G8B8A8_SRGB, width=None):
    """grb_present_rows_to_peer with the presenting rank's slot and every rank's flag array as tensors on this device:
    src_t / dst_t: (H, P) int32 (one 4-byte texel each; the image is the first `width` texels of each row, all P by
    default), flag_arrays[r]: int32 tensor; counter_t: one zeroed int32."""
    si = capi.image(src_t, fmt)
    if width is not None:
        si.width = int(width)
    flags = (C.c_void_p * len(flag_arrays))(*[t.data_ptr() for t in flag_arrays])
    capi.check(capi.lib().grb_present_rows_to_peer(C.byref(si), dst_t.data_ptr(), flags, len(flag_arrays), int(flag_index), int(epoch),
                                                   _ptr(counter_t), capi.rows(own), capi.stream_ptr()),
               "grb_present_rows_to_peer")


def gbuffer_planes(**planes) -> capi.GrbGBufferPlanes:
    """A GrbGBufferPlanes from keyword planes (capi.GBUFFER_PLANES names) given as (tensor, format): CUDA tensors laid
    out (H, W[, C]) whose rows may be strided, the pitch being the row stride.  Planes not given are absent."""
    g = capi.GrbGBufferPlanes()
    for name, (t, fmt) in planes.items():
        g.plane[capi.GBUFFER_PLANES.index(name)] = capi.pitched_image(t, fmt)
    return g


def gbuffer_copy_rows(src, dst, ranges):
    """grb_gbuffer_copy_rows of the (y0, y1) `ranges` from the GrbGBufferPlanes src into dst on the current stream."""
    rs = (capi.GrbRows * max(len(ranges), 1))(*[capi.GrbRows(int(a), int(b)) for a, b in ranges])
    capi.check(capi.lib().grb_gbuffer_copy_rows(C.byref(src), C.byref(dst), rs, len(ranges), capi.stream_ptr()), "grb_gbuffer_copy_rows")


def gbuffer_slot_layout(layout, base=None):
    """grb_gbuffer_slot_layout: (the planes of a slot at device address `base`, the slot's bytes)."""
    out, size = capi.GrbGBufferPlanes(), C.c_uint64()
    capi.check(capi.lib().grb_gbuffer_slot_layout(C.byref(layout), None if base is None else C.c_void_p(base), C.byref(out), C.byref(size)),
               "grb_gbuffer_slot_layout")
    return out, size.value


def gbuffer_rows_to_peers(src, slots, flag_arrays, rows_per_rank, flag_index, epoch, counter_t):
    """grb_gbuffer_rows_to_peers with every rank's slot and flag array as tensors on this device: slots[q] a uint8
    tensor of the slot's bytes, rows_per_rank[q] rank q's (y0, y1) list."""
    n = len(flag_arrays)
    flat = [r for lst in rows_per_rank for r in lst]
    rs = (capi.GrbRows * max(len(flat), 1))(*[capi.GrbRows(int(a), int(b)) for a, b in flat])
    counts = (C.c_int32 * n)(*[len(lst) for lst in rows_per_rank])
    images = (C.c_void_p * n)(*[t.data_ptr() for t in slots])
    flags = (C.c_void_p * n)(*[t.data_ptr() for t in flag_arrays])
    capi.check(capi.lib().grb_gbuffer_rows_to_peers(C.byref(src), images, flags, rs, counts, n, int(flag_index), int(epoch), _ptr(counter_t),
                                                    capi.stream_ptr()),
               "grb_gbuffer_rows_to_peers")


def light_list(color, position, is_point, rotation, inner_cone, outer_cone, cutoff=1e10, count=None) -> capi.GrbLightList:
    """A GrbLightList over CUDA tensors in synth.Lights' shapes (Viewer.set_lights_device's); count (default: the
    tensors' length) is the list's capacity."""
    n = int(color.shape[0]) if count is None else int(count)
    return capi.GrbLightList(n, *[t.data_ptr() for t in (color, position, is_point, rotation, inner_cone, outer_cone)], float(cutoff))


def light_slot_layout(base=None):
    """grb_light_slot_layout: (the GrbLightList of a slot at device address `base`, its count word's address, the
    slot's bytes); base None queries the size (null pointers)."""
    out, count, size = capi.GrbLightList(), C.c_void_p(), C.c_uint64()
    capi.check(capi.lib().grb_light_slot_layout(None if base is None else C.c_void_p(base), C.byref(out), C.byref(count), C.byref(size)),
               "grb_light_slot_layout")
    return out, count.value, size.value


def light_list_to_peers(lights, input_count_t, slots, flag_arrays, flag_index, epoch, counter_t):
    """grb_light_list_to_peers with every rank's slot and flag array as tensors on this device: lights a GrbLightList,
    input_count_t a one-element int32 tensor or None, slots[r] a uint8 tensor of the slot's bytes."""
    n = len(flag_arrays)
    images = (C.c_void_p * n)(*[t.data_ptr() for t in slots])
    flags = (C.c_void_p * n)(*[t.data_ptr() for t in flag_arrays])
    capi.check(capi.lib().grb_light_list_to_peers(C.byref(lights), _ptr(input_count_t), images, flags, n, int(flag_index), int(epoch), _ptr(counter_t),
                                                  capi.stream_ptr()),
               "grb_light_list_to_peers")


def light_prep_shadow_ids(lights, input_count_t, transforms_t, map_ids_t, table_t, view, records_t, model_t, type_mask_t, z_ranges_t,
                          shadow_transforms_t, shadow_maps_t, count_t, scratch_t):
    """grb_light_prep_shadow_ids on the current stream: lights a GrbLightList, view a GrbLightPrepView, every other
    argument a CUDA tensor (input_count_t None: every entry live); table_t an int64 tensor of map pointers whose length
    is the table's size; the outputs as grb_light_prep_shadowed takes them."""
    ids = capi.GrbLightShadowIdList(_ptr(transforms_t), _ptr(map_ids_t))
    capi.check(capi.lib().grb_light_prep_shadow_ids(C.byref(lights), _ptr(input_count_t), C.byref(ids), _ptr(table_t), int(table_t.numel()), C.byref(view),
                                                    _ptr(records_t), _ptr(model_t), _ptr(type_mask_t), _ptr(z_ranges_t), _ptr(shadow_transforms_t),
                                                    _ptr(shadow_maps_t), _ptr(count_t), _ptr(scratch_t), scratch_t.numel() * scratch_t.element_size(),
                                                    capi.stream_ptr()),
               "grb_light_prep_shadow_ids")


def light_shadow_slot_layout(base=None):
    """grb_light_shadow_slot_layout: (the transforms' address, the map ids' address, the whole shadowed slot's bytes) of a
    slot at device address `base`; base None queries the size (null addresses)."""
    t, m, size = C.c_void_p(), C.c_void_p(), C.c_uint64()
    capi.check(capi.lib().grb_light_shadow_slot_layout(None if base is None else C.c_void_p(base), C.byref(t), C.byref(m), C.byref(size)),
               "grb_light_shadow_slot_layout")
    return t.value, m.value, size.value


def light_list_shadowed_to_peers(lights, transforms_t, map_ids_t, input_count_t, slots, flag_arrays, flag_index, epoch, counter_t):
    """grb_light_list_shadowed_to_peers with every rank's slot and flag array as tensors on this device: lights a
    GrbLightList, transforms_t / map_ids_t its shadow transforms and map ids, slots[r] a uint8 tensor of the shadowed
    slot's bytes."""
    n = len(flag_arrays)
    ids = capi.GrbLightShadowIdList(_ptr(transforms_t), _ptr(map_ids_t))
    images = (C.c_void_p * n)(*[t.data_ptr() for t in slots])
    flags = (C.c_void_p * n)(*[t.data_ptr() for t in flag_arrays])
    capi.check(capi.lib().grb_light_list_shadowed_to_peers(C.byref(lights), C.byref(ids), _ptr(input_count_t), images, flags, n, int(flag_index), int(epoch),
                                                           _ptr(counter_t), capi.stream_ptr()),
               "grb_light_list_shadowed_to_peers")


def to_dev(a):
    return _dev(a)


def to_host(t, dtype):
    return _host(t, dtype)
