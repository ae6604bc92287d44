"""Light-clusterer geometry cases beyond the default view, and a float64 coverage check of a built cluster (test
infrastructure).

The default view (common.build_lights_case / synth.make_scene) looks down -Z from (0, 0, 8) with an infinite far plane
at lights 2-150 m ahead, so most branches of the clusterer's set-up never run there.  build(oracle, name) returns
(scene, cam, lights, prep) for one named case, shaped like common.build_case: a random G-buffer whose reverse-Z depth
holds sky pixels and pixels right at the near plane, a camera, the lights in the host clusterer's order and the
oracle's host prep.  Each case names the branches it exists for (CASES) and build() asserts from the oracle's K1 / K2
outputs that it reaches every one of them (branches()).

coverage() is the check independent of the clusterer: every (pixel, light) pair whose falloff is nonzero, found by
brute force in float64, must be in the pixel's cluster list (the light's bit set in the pixel's tile, its index within
the pixel's Z slice's range)."""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np

from granite_b200 import synth
from tests import lighting_ref64 as R

NEAR = 1.0 / 16.0

# name -> the branches of grb_cluster.cu / oracle_cluster.c the case must reach (see branches())
CASES = {
    "turned": ("points", "spots", "cull+1", "cull-1", "w-clip"),
    "around-eye": ("ellipse-off", "infinite-extent", "on-axis", "behind-eye"),
    "spots-at-eye": ("cull-1", "w1", "w2", "w3", "w4", "w5", "w6", "over-8-triangles"),
    "finite-far": ("cull0", "z-single", "z-dual"),
    "tall": ("scale-clamp", "outer-0.98", "sub-tile"),
}


# ------------------------------------------------------------------------------------------------ cameras
def perspective(fovy, aspect, near, far=None):
    """host/math.cpp perspective() in float32, column-major m[c, r]: reverse-Z, Y flipped, infinite far when far is
    None."""
    f = np.float32
    t = f(math.tan(f(fovy) / f(2.0)))
    m = np.zeros((4, 4), np.float32)
    m[0, 0] = f(1.0) / (f(aspect) * t)
    m[1, 1] = -(f(1.0) / t)
    m[2, 3] = f(-1.0)
    if far is None:
        m[3, 2] = f(near)
    else:
        n, fa = f(near), f(far)
        m[2, 2] = f(-1.0) - fa / (n - fa)
        m[3, 2] = -(fa * n) / (n - fa)
    return m


def turned_view(eye, yaw, pitch, roll):
    """View matrix (column-major m[c, r]) of a camera at `eye` turned by yaw (about +Y), pitch (about +X), roll
    (about the view axis), in that order; it looks down its local -Z."""
    cy, sy, cp, sp, cr, sr = (math.cos(yaw), math.sin(yaw), math.cos(pitch), math.sin(pitch), math.cos(roll), math.sin(roll))
    ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    rx = np.array([[1, 0, 0], [0, cp, -sp], [0, sp, cp]])
    rz = np.array([[cr, -sr, 0], [sr, cr, 0], [0, 0, 1]])
    c2w = ry @ rx @ rz
    m = np.eye(4)
    m[:3, :3] = c2w.T
    m[:3, 3] = -c2w.T @ np.asarray(eye, np.float64)
    return np.ascontiguousarray(m.T.astype(np.float32)) + np.float32(0.0)


def _frame(view):
    """(eye, right, up, front) in float64 from a view matrix."""
    m = view.astype(np.float64).T  # row-major
    rot = m[:3, :3]
    eye = -rot.T @ m[:3, 3]
    return eye, rot[0], rot[1], -rot[2]


def ndc_depth(projection, z):
    """Reverse-Z NDC depth of view depth z (> 0) through `projection`."""
    p = projection.astype(np.float64)
    return (p[2, 2] * -z + p[3, 2]) / z


# ------------------------------------------------------------------------------------------------ scene
def random_scene(rng, w, h, projection, view, z_max, sky=0.08, at_near=0.02):
    """Random G-buffer words and a random reverse-Z depth buffer: view depths log-uniform in [near, z_max], `sky` of the
    pixels 0 (sky) and `at_near` of them exactly 1 (the near plane)."""
    near = NEAR if projection[2, 2] == 0 else float(projection[3, 2] / (projection[2, 2] + 1.0))
    z = np.exp(rng.uniform(np.log(near), np.log(z_max), (h, w)))
    depth = ndc_depth(projection, z).astype(np.float32)
    u = rng.random((h, w))
    depth[u < sky] = 0.0
    depth[(u >= sky) & (u < sky + at_near)] = 1.0
    n = rng.normal(size=(h, w, 3))
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    n10 = np.clip(np.rint((n * 0.5 + 0.5) * 1023.0), 0, 1023).astype(np.uint32)
    normal = (n10[..., 0] | (n10[..., 1] << np.uint32(10)) | (n10[..., 2] << np.uint32(20)) | np.uint32(3 << 30)).astype(np.uint32)
    alb = rng.integers(13, 243, size=(h, w, 3), dtype=np.uint32)
    albedo = (alb[..., 0] | (alb[..., 1] << np.uint32(8)) | (alb[..., 2] << np.uint32(16)) | np.uint32(0xFF000000)).astype(np.uint32)
    pbr = ((rng.random((h, w)) < 0.2) * 255 | (rng.integers(26, 256, size=(h, w)) << 8)).astype(np.uint16)
    emis = np.zeros((h, w, 3), np.float32)
    hot = rng.random((h, w)) < 0.002
    emis[hot] = rng.uniform(0.0, 20.0, size=(int(hot.sum()), 3)).astype(np.float32)
    return synth.Scene(w, h, projection, view, albedo, normal, pbr, depth, synth.pack_r11g11b10(emis))


# ------------------------------------------------------------------------------------------------ lights
class _Lights:
    """Accumulates lights; spots are given by the direction they point along."""

    def __init__(self):
        self.pos, self.col, self.pt, self.fwd, self.inner, self.outer = [], [], [], [], [], []

    def add(self, pos, radius, point, fwd=(0.0, 0.0, -1.0), outer=0.8, inner=None):
        fwd = np.asarray(fwd, np.float64)
        self.pos.append(np.asarray(pos, np.float64))
        self.col.append(np.full(3, 0.1 * radius * radius))  # falloff radius sqrt(max colour / 0.1) (lights.cpp recompute_range)
        self.pt.append(bool(point))
        self.fwd.append(fwd / np.linalg.norm(fwd))
        self.outer.append(outer)
        self.inner.append(min(outer + 0.05, 0.999) if inner is None else inner)

    def build(self, front):
        """synth.Lights in the host clusterer's order: ascending view depth of the centre, dot(position, front) in
        float32 (clusterer.cpp refresh_bindless_prepare).  Each light moves 1e-4 m per rank along the view axis so that
        no two keys are within rounding of each other."""
        pos = np.asarray(self.pos)
        order = np.argsort(pos @ front, kind="stable")
        pos = pos[order] + np.arange(len(order))[:, None] * 1e-4 * front
        n = len(order)
        rot = np.zeros((n, 3, 3), np.float32)
        for k, i in enumerate(order):
            f = self.fwd[i]
            up = np.array([0.0, 0.0, 1.0]) if abs(f[1]) > 0.9 else np.array([0.0, 1.0, 0.0])
            r = np.cross(f, up)
            r /= np.linalg.norm(r)
            rot[k, 0], rot[k, 1], rot[k, 2] = r, np.cross(r, f), -f  # columns: right, up, -forward
        pick = lambda a, dt=np.float32: np.asarray(a)[order].astype(dt)  # noqa: E731
        return synth.Lights(pick(self.col), pos.astype(np.float32), pick(self.pt, bool), rot, pick(self.inner), pick(self.outer))


def _unit(rng, n):
    v = rng.normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _ball(rng, n, centre, radius):
    return centre + _unit(rng, n) * radius * rng.random((n, 1)) ** (1.0 / 3.0)


def _mixed(L, rng, n, centre, radius, spots=0.35, r_lo=2.0, r_hi=20.0):
    for p in _ball(rng, n, centre, radius):
        L.add(p, rng.uniform(r_lo, r_hi), rng.random() >= spots, _unit(rng, 1)[0], outer=rng.uniform(0.5, 0.95))


def _case_geometry(name):
    """(width, height, projection, view, z_max of the scene, lights builder)."""
    rng = np.random.default_rng(sum(map(ord, name)) * 7919)
    L = _Lights()
    if name == "turned":
        w, h = 320, 180
        proj = perspective(math.radians(70.0), w / h, NEAR)
        view = turned_view((13.5, 4.25, -7.75), 0.65, -0.35, 0.25)
        eye, right, up, front = _frame(view)
        _mixed(L, rng, 260, eye + 30.0 * front, 60.0)
        z_max = 600.0
    elif name == "around-eye":
        w, h = 256, 192
        proj = perspective(math.radians(60.0), w / h, NEAR)
        view = turned_view((-3.0, 1.5, 6.0), 0.3, 0.1, 0.0)
        eye, right, up, front = _frame(view)
        for p in _ball(rng, 12, eye, 1.5):  # spheres holding the eye
            L.add(p, rng.uniform(2.5, 6.0), True)
        for k in range(40):  # behind the eye and beside the frustum
            side = (right if k % 2 else -right) * rng.uniform(3.0, 25.0) + up * rng.uniform(-8.0, 8.0)
            L.add(eye - front * rng.uniform(0.5, 20.0) + side, rng.uniform(3.0, 20.0), k % 3 != 0, _unit(rng, 1)[0])
        L.add(eye + 12.0 * front, 4.0, True)  # on the view axis
        _mixed(L, rng, 150, eye + 25.0 * front, 30.0)
        z_max = 400.0
    elif name == "spots-at-eye":
        w, h = 320, 180
        proj = perspective(math.radians(75.0), w / h, NEAR)
        view = turned_view((2.0, 1.0, 3.0), -0.4, 0.2, -0.3)
        eye, right, up, front = _frame(view)
        for p in _ball(rng, 60, eye, 8.0):  # aimed at the eye, reaching it
            d = np.linalg.norm(p - eye)
            L.add(p, d * rng.uniform(1.2, 3.0), False, eye - p + _unit(rng, 1)[0] * 0.3 * d, outer=rng.uniform(0.5, 0.9))
        for _ in range(60):  # straddling the camera plane
            p = eye + front * rng.uniform(-2.0, 2.0) + right * rng.uniform(-6.0, 6.0) + up * rng.uniform(-6.0, 6.0)
            L.add(p, rng.uniform(3.0, 20.0), False, _unit(rng, 1)[0], outer=rng.uniform(0.4, 0.9))
        for _ in range(60):  # behind the eye, pointing through it
            p = eye - front * rng.uniform(0.3, 5.0) + _unit(rng, 1)[0] * 0.5
            L.add(p, np.linalg.norm(p - eye) * rng.uniform(1.5, 6.0), False, front + _unit(rng, 1)[0] * 0.4, outer=rng.uniform(0.4, 0.9))
        _mixed(L, rng, 40, eye + 10.0 * front, 15.0, spots=0.0)
        z_max = 300.0
    elif name == "finite-far":
        w, h = 320, 180
        far = 120.0
        proj = perspective(math.radians(60.0), w / h, 0.1, far)
        view = turned_view((-5.0, 2.0, 10.0), 0.2, -0.15, 0.05)
        eye, right, up, front = _frame(view)
        for _ in range(50):  # from the near plane to beyond the far plane
            p = eye + front * rng.uniform(-1.0, 0.05) + right * rng.uniform(-3.0, 3.0) + up * rng.uniform(-2.0, 2.0)
            L.add(p, rng.uniform(150.0, 250.0), False, front + _unit(rng, 1)[0] * 0.2, outer=rng.uniform(0.85, 0.97))
        for _ in range(60):  # in front, reaching past the far plane
            p = eye + front * rng.uniform(20.0, 110.0) + right * rng.uniform(-30.0, 30.0) + up * rng.uniform(-15.0, 15.0)
            L.add(p, rng.uniform(30.0, 100.0), False, front + _unit(rng, 1)[0] * 0.5, outer=rng.uniform(0.6, 0.95))
        for _ in range(40):  # beyond the far plane, pointing back
            p = eye + front * rng.uniform(125.0, 180.0) + right * rng.uniform(-40.0, 40.0) + up * rng.uniform(-20.0, 20.0)
            L.add(p, rng.uniform(20.0, 90.0), False, -front + _unit(rng, 1)[0] * 0.5, outer=rng.uniform(0.6, 0.95))
        _mixed(L, rng, 100, eye + 60.0 * front, 50.0)
        z_max = far * 0.999
    elif name == "tall":
        w, h = 180, 320
        proj = perspective(math.radians(100.0), w / h, NEAR)
        view = turned_view((0.0, 3.0, 0.0), 1.1, -0.5, 0.1)
        eye, right, up, front = _frame(view)
        for k in range(80):  # narrow cones, half of them with inner - outer under 0.001
            outer = rng.uniform(0.9, 0.98)
            inner = outer + (rng.uniform(0.0, 0.0009) if k % 2 else rng.uniform(0.002, 0.02))
            L.add(_ball(rng, 1, eye + 20.0 * front, 20.0)[0], rng.uniform(5.0, 40.0), False, _unit(rng, 1)[0], outer=outer, inner=inner)
        for _ in range(80):  # radius under one tile
            p = eye + front * rng.uniform(30.0, 150.0) + right * rng.uniform(-20.0, 20.0) + up * rng.uniform(-60.0, 60.0)
            L.add(p, rng.uniform(0.2, 0.45), rng.random() < 0.7, _unit(rng, 1)[0])
        _mixed(L, rng, 90, eye + 25.0 * front, 30.0)
        z_max = 500.0
    else:
        raise KeyError(name)
    return w, h, proj, view, front, z_max, L


# ------------------------------------------------------------------------------------------------ branches
_HULL = ((0, 1, 2), (0, 2, 3), (0, 3, 4), (0, 4, 1), (2, 1, 3), (4, 3, 1))  # the six hull triangles K2 sets up
_MIN_W = np.float32(1.0 / 1024.0)


def is_point(prep):
    i = np.arange(prep.n)
    return ((prep.type_mask[i >> 5] >> (i & 31).astype(np.uint32)) & 1).astype(bool)


def branches(cam, prep, clus, lights=None, scene=None):
    """How often the clusterer's set-up branches are reached, from the oracle's K1 / K2 outputs (and numpy on the hull's
    clip coordinates): {branch: count}."""
    n, pt = prep.n, is_point(prep)
    spots = clus.spots[:n].reshape(n, 6, 4)
    cull = clus.cull[:n]
    sp = ~pt
    sign, count = spots[:, 5, 0], cull[:, 3].view(np.uint32)
    out = {"points": int(pt.sum()), "spots": int(sp.sum()),
           "cull0": int((sp & (sign == 0)).sum()), "cull-1": int((sp & (sign < 0)).sum()), "cull+1": int((sp & (sign > 0)).sum()),
           "over-8-triangles": int((sp & (sign != 0) & (count > 8)).sum())}
    assert (count[sp & (sign == 0)] == 0xFFFFFFFF).all(), "cull sign 0 stores the 'always passes' count"
    # K2's w clip code per hull triangle (clip_w_and_emit) and, for triangles in front of w = 1/1024, the z clip code
    # of the projected triangle (clip_z_and_emit)
    wc, zc = np.zeros(8, np.int64), np.zeros(8, np.int64)
    for i in np.nonzero(sp & (sign != 0))[0]:
        c = spots[i, :5]
        for t in _HULL:
            w = c[list(t), 3]
            code = int((w[0] < _MIN_W) + 2 * (w[1] < _MIN_W) + 4 * (w[2] < _MIN_W))
            wc[code] += 1
            if code == 0:
                z = c[list(t), 2] / w
                zc[int((z[0] < 0) + 2 * (z[1] < 0) + 4 * (z[2] < 0))] += 1
    for k in range(1, 7):
        out[f"w{k}"] = int(wc[k])
    out["w-clip"] = int(wc[1:7].sum())
    out["z-single"], out["z-dual"] = int(zc[[3, 5, 6]].sum()), int(zc[[1, 2, 4]].sum())
    # point lights: data[3].x is the ellipse flag, data[1] project_sphere_flat's extents, data[2] the rotation that
    # the xy_length < 1e-5 branch leaves at exactly (1, +0, +0, 1)
    out["ellipse-off"] = int((pt & (cull[:, 12] == 0.0)).sum())
    out["infinite-extent"] = int((pt & np.isinf(cull[:, 4:8]).any(1)).sum())
    ident = np.array([1.0, 0.0, 0.0, 1.0], np.float32).view(np.uint32)
    out["on-axis"] = int((pt & (cull[:, 8:12].view(np.uint32) == ident).all(1)).sum())
    # view-space position of the light centres (float64)
    eye = np.asarray(list(cam.camera_position), np.float64)
    front = np.asarray(list(cam.camera_front), np.float64)
    lpos = prep.records["position"][:n].astype(np.float64)
    zc_ = (lpos - eye) @ front
    out["behind-eye"] = int((zc_ < 0).sum())
    # spot_scale = 1 / max(0.001, inner - outer): the clamp leaves exactly fp16(1000)
    scale = prep.records["spot_scale_bias"][:n, 0].view(np.float16).astype(np.float64)
    out["scale-clamp"] = int((sp & (scale == np.float64(np.float16(1000.0)))).sum())
    out["outer-0.98"] = int((sp & (prep.outer_cone[:n] >= 0.975)).sum())
    # radius under one tile's width at the light's view depth
    tile_w = 2.0 * np.maximum(zc_, 1e-6) / (float(cam.projection[0]) * float(prep.params.resolution_xy[0]))
    out["sub-tile"] = int(((1.0 / prep.records["inv_radius"][:n].astype(np.float64)) < tile_w).sum())
    return out


def build(oracle, name, res=synth.CLUSTER_RES, check=True):
    """(scene, cam, lights, prep) of the named case.  check: assert that the oracle's clusterer reaches every branch the
    case names."""
    w, h, proj, view, front, z_max, L = _case_geometry(name)
    rng = np.random.default_rng(sum(map(ord, name)) * 104729)
    scene = random_scene(rng, w, h, proj, view, z_max)
    cam = oracle.camera_setup(proj, view)
    lights = L.build(np.asarray(list(cam.camera_front), np.float32).astype(np.float64))
    prep = oracle.prepare_lights(cam, lights, res=res)
    if check:
        got = branches(cam, prep, oracle.cluster_build(cam, prep))
        missing = [b for b in CASES[name] if got[b] == 0]
        assert not missing, f"case {name} does not reach {missing}: {got}"
    return scene, cam, lights, prep


def count_case(oracle, n, res=synth.CLUSTER_RES):
    """The turned case's camera and G-buffer with exactly n mixed lights (no frustum culling: grb_cluster_build and the
    oracle take up to 4097 lights through the raw ABI): (scene, cam, prep)."""
    w, h, proj, view, front, z_max, _ = _case_geometry("turned")
    rng = np.random.default_rng(n + 17)
    eye = _frame(view)[0]
    L = _Lights()
    _mixed(L, rng, n, eye + 30.0 * front, 60.0)
    cam = oracle.camera_setup(proj, view)
    lights = L.build(np.asarray(list(cam.camera_front), np.float32).astype(np.float64)) if n else synth.make_lights(0)
    scene = random_scene(np.random.default_rng(5), w, h, proj, view, z_max)
    return scene, cam, oracle.prepare_lights(cam, lights, res=res, cull=False)


# ------------------------------------------------------------------------------------------------ coverage
def grid_depth(prep, cam):
    """View depth the Z slices end at: res_z * get_z_slice_extent (clusterer.cpp:700-703)."""
    rz = prep.res[2]
    return rz * float(min(np.float32(0.5), np.float32(cam.z_far) / np.float32(rz)))


def brute_pairs(scene, cam, prep, ys=None, xs=None):
    """Every (pixel, light) pair of lit pixels (ys, xs) (default: every lit pixel, row-major) whose falloff is nonzero,
    in float64: |P - L| < r, and for spots also cos * scale + bias > 0 with scale and bias the record's fp16 words, as
    the shader reads them.  Returns (pix, light, borderline): pix indexes (ys, xs), pairs in ascending (pix, light)
    order; borderline marks pairs within float32 rounding of the boundary (|d / r - 1| < 1e-5 or a cone value under
    1e-6)."""
    from scipy.spatial import cKDTree

    if ys is None:
        ys, xs = np.nonzero(scene.depth != 0)
    P = R.positions(scene.depth, cam.inv_view_projection, ys, xs, np.float64)
    n = prep.n
    if n == 0 or len(ys) == 0:
        e = np.zeros(0, np.int64)
        return e, e, np.zeros(0, bool)
    tree = cKDTree(P)
    recs = prep.records[:n]
    lpos = recs["position"].astype(np.float64)
    r = 1.0 / recs["inv_radius"].astype(np.float64)
    pt = is_point(prep)
    sb = recs["spot_scale_bias"].view(np.float16).astype(np.float64)
    ldir = recs["direction"].astype(np.float64)
    pix, light, border = [], [], []
    for i, cand in enumerate(tree.query_ball_point(lpos, r * (1.0 + 1e-9))):
        if not cand:
            continue
        cand = np.asarray(cand, np.int64)
        d = np.linalg.norm(P[cand] - lpos[i], axis=1)
        keep = d < r[i]
        edge = np.abs(d / r[i] - 1.0) < 1e-5
        if not pt[i]:
            with np.errstate(invalid="ignore", divide="ignore"):
                cos = ((P[cand] - lpos[i]) @ ldir[i]) / d  # dot(-L, direction), L = normalize(light - P)
            cone = np.where(d > 0, cos * sb[i, 0] + sb[i, 1], 1.0)
            keep &= cone > 0
            edge |= np.abs(cone) < 1e-6
        pix.append(cand[keep])
        light.append(np.full(int(keep.sum()), i, np.int64))
        border.append(edge[keep])
    pix, light, border = np.concatenate(pix), np.concatenate(light), np.concatenate(border)
    order = np.lexsort((light, pix))
    return pix[order], light[order], border[order]


def covered(prep, bitmask, crange, tile, zi, ys, xs, pix, light):
    """Boolean per pair: the light is in its pixel's cluster list (bit set in the tile's mask, index within the slice's
    range)."""
    n32 = max(int(prep.params.num_lights_32), 1)
    t = tile[ys[pix], xs[pix]].astype(np.int64)
    z = zi[ys[pix], xs[pix]].astype(np.int64)
    words = bitmask.reshape(-1, n32)[t, light >> 5]
    bit = ((words >> (light & 31).astype(np.uint32)) & 1).astype(bool)
    rng = crange.astype(np.int64)
    return bit & (rng[z, 0] <= light) & (light <= rng[z, 1])


def coverage(scene, cam, prep, bitmask, crange, tile, zi, max_depth=None):
    """The float64 coverage check of a built cluster.  Pixels whose view depth reaches max_depth (default the Z grid's
    end, grid_depth) are left out: see test_cluster_cases_cpu.py::test_pixels_beyond_the_z_grid_lose_lights_beyond_it.
    Returns SimpleNamespace(pairs, missed (pairs not covered, away from the boundary), borderline_missed,
    borderline, pix, light, ys, xs)."""
    if max_depth is None:
        max_depth = grid_depth(prep, cam)
    ys, xs = np.nonzero(scene.depth != 0)
    P = R.positions(scene.depth, cam.inv_view_projection, ys, xs, np.float64)
    vz = (P - np.asarray(list(cam.camera_position), np.float64)) @ np.asarray(list(cam.camera_front), np.float64)
    inside = vz < max_depth
    ys, xs = ys[inside], xs[inside]
    pix, light, border = brute_pairs(scene, cam, prep, ys, xs)
    ok = covered(prep, bitmask, crange, tile, zi, ys, xs, pix, light)
    return SimpleNamespace(pairs=len(pix), missed=int((~ok & ~border).sum()), borderline_missed=int((~ok & border).sum()),
                           borderline=int(border.sum()), pix=pix, light=light, ok=ok, ys=ys, xs=xs)


def assert_cluster_equal(got, ref, prep):
    """K1..K4 outputs of two cluster builds bit for bit (NaNs canonicalised): spot hulls, point-light set-up words,
    each spot's triangle count and the triangles it stores, the bitmask and the Z-slice ranges; bits at or above
    num_lights zero."""
    def canon(a):
        """fp32 bit patterns with every NaN mapped to one pattern (x86 and NVIDIA differ in the default NaN they
        generate; any NaN compares the same way in the shaders)."""
        a = np.ascontiguousarray(a, np.float32)
        return np.where(np.isnan(a), np.uint32(0x7FC00000), a.view(np.uint32))

    n, pt = prep.n, is_point(prep)
    assert np.array_equal(canon(got.spots[:n][~pt]), canon(ref.spots[:n][~pt])), "K1 spot hulls"
    assert np.array_equal(canon(got.cull[:n][pt][:, :16]), canon(ref.cull[:n][pt][:, :16])), "K2 point lights"
    for i in np.nonzero(~pt)[0]:
        cnt = int(ref.cull[i].view(np.uint32)[3])
        assert int(got.cull[i].view(np.uint32)[3]) == cnt, f"K2 spot {i}: triangle count"
        used = 16 * cnt if cnt <= 8 else 0
        a, b = canon(got.cull[i][:used]).copy(), canon(ref.cull[i][:used]).copy()
        if used:
            a[3] = b[3] = 0
        assert np.array_equal(a, b), f"K2 spot {i}"
    assert np.array_equal(got.bitmask, ref.bitmask), f"K3 bitmask: {int((got.bitmask != ref.bitmask).sum())} words differ"
    assert np.array_equal(got.range, ref.range), f"K4 ranges: {int((got.range != ref.range).any(1).sum())} slices differ"
    if n % 32:
        assert not (got.bitmask[..., (n - 1) >> 5] >> np.uint32(n % 32)).any(), "bits at or above num_lights"


def assert_covers(cov, what=""):
    assert cov.pairs > 1000, f"{what}: only {cov.pairs} lit pairs: the case does not test coverage"
    assert cov.missed == 0, f"{what}: {cov.missed} of {cov.pairs} (pixel, light) pairs with a nonzero falloff are not in the pixel's cluster"
    # within float32 rounding of the falloff boundary either answer is right; there must be few such pairs
    assert cov.borderline_missed <= max(4, cov.pairs // 100000), f"{what}: {cov.borderline_missed} borderline pairs missed"


def lighting_pairs(scene, cam, prep):
    """The brute-force pairs of every lit pixel (row-major), as lighting_ref64.reference takes them."""
    pix, light, _ = brute_pairs(scene, cam, prep)
    return pix, light


def debug_cluster_indices(cam, prep, depth_np):
    """grb_debug_cluster_indices: each pixel's (tile, Z slice) as the lighting pass computes them, (H, W) int32 each."""
    import ctypes as C

    import torch

    from granite_b200 import capi, harness

    h, w = depth_np.shape
    depth = harness.to_dev(depth_np)
    out_t = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    out_z = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    img = capi.image(depth, capi.FORMAT_D32_SFLOAT)
    gcam = harness.camera_struct(cam)
    params = harness.params_struct(prep.params)
    capi.check(capi.lib().grb_debug_cluster_indices(C.byref(img), C.byref(gcam), C.byref(params), C.c_void_p(out_t.data_ptr()),
                                                    C.c_void_p(out_z.data_ptr()), capi.rows(), capi.stream_ptr()))
    return out_t.cpu().numpy(), out_z.cpu().numpy()
