"""The deferred lighting pass (orc_deferred_lighting, oracle/oracle_lighting.c) restated in numpy float64, and the
bar every lighting kernel form is held to against it (test infrastructure).

What is restated: the G-buffer decode through the same sRGB table, draw 1 (directional.frag: the directional light
and the 5 % ambient), the B10G11R11 store of draw 1, draw 2 (clustering.frag: point and spot falloff, the cone term,
the Cook-Torrance BRDF with the half vector formed as normalize(V + L)) and the final store.  What is not restated:
each pixel's cluster (tile, Z slice), the cluster bitmask and the Z-slice light ranges.  They are integers with their
own bit-exact tests, so they are taken from the oracle.

The bar.  A B10G11R11 store truncates a float to its code (6 / 6 / 5 mantissa bits).  For each lit pixel and channel
let v64 be the float64 value of the sum a store quantises, and s a per-pixel slack:

    s = REL * (|destination| + sum over terms |term|) + GAP * sum over terms |t64 - t32|

where t32 is the same term evaluated in float32 with the reference's own formulation.  The first part covers the
rounding of a well-conditioned fp32 evaluation (fast reciprocal square roots, FMA, sums over a few hundred lights,
all near 1e-7 relative per operation).  The second part is where the formulation itself is ill-conditioned: a term
that fp32 cannot evaluate better than the reference does gets the reference's own fp32 error, times GAP.  A kernel
whose formulation is worse-conditioned than the reference's (the half vector from |V+L|^2 = 2 + 2 V.L near
L = -V, for example) misses it.

The stored code must lie between code(v64 - s) and code(v64 + s).  Draw 1 is stored before draw 2 adds to it, so
where the float64 draw-1 value lies within its slack of a code boundary, the final value computed from either
neighbouring draw-1 code is accepted.  Sky pixels (depth 0) keep the destination's bits.

Against "at most one code from the fp32 oracle" this is about twice as tight away from code boundaries (one code
either way becomes zero codes), and it does not take the oracle's own rounding as the truth where the oracle is
ill-conditioned.  tests/test_lighting_ref64_cpu.py pins it: the fp32 oracle meets this bar."""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np

PI = float(np.float32(3.1415628))  # assets/shaders/lights/pbr.h:5 (sic), as the oracle and the kernels use it
REL = 2e-5
GAP = 4.0
MBITS = (6, 6, 5)  # R, G, B mantissa bits of B10G11R11


# ----------------------------------------------------------------------------------------------- B10G11R11 codes
def ufloat_code(v, mbits):
    """Code of the store of v (float64, any sign): truncation to a 5-bit-exponent unsigned float, as f32_to_ufloat."""
    v = np.asarray(v, np.float64)
    pos = np.where(v > 0, v, 1.0)
    mant, exp = np.frexp(pos)  # pos = mant 2^exp, mant in [0.5, 1)
    e = exp.astype(np.int64) - 1
    normal = ((e + 15) << mbits) + np.floor((pos / np.ldexp(1.0, e) - 1.0) * (1 << mbits)).astype(np.int64)
    denorm = np.floor(pos * 2.0 ** (14 + mbits)).astype(np.int64)
    code = np.where(e >= -14, normal, denorm)
    code = np.minimum(code, (30 << mbits) | ((1 << mbits) - 1))
    return np.where(v > 0, code, 0)


def ufloat_value(code, mbits):
    code = np.asarray(code, np.int64)
    e, m = code >> mbits, code & ((1 << mbits) - 1)
    return np.where(e == 0, m * 2.0 ** (-14 - mbits), np.ldexp(1.0 + m / (1 << mbits), (e - 15).astype(np.int64)))


def codes(packed):
    """(..., 3) int64 channel codes of packed B10G11R11 words."""
    p = np.asarray(packed).astype(np.uint32).astype(np.int64)
    return np.stack([p & 0x7FF, (p >> 11) & 0x7FF, p >> 22], -1)


def decode(packed):
    c = codes(packed)
    return np.stack([ufloat_value(c[..., k], MBITS[k]) for k in range(3)], -1)


def pack(rgb):
    """Store of float values (..., 3): truncating, as pack_r11g11b10."""
    c = [ufloat_code(rgb[..., k], MBITS[k]) for k in range(3)]
    return (c[0] | (c[1] << 11) | (c[2] << 22)).astype(np.uint32)


# ----------------------------------------------------------------------------------------------- inputs
def srgb_table(oracle):
    """The 256-entry sRGB8 -> linear table (float32) the oracle and the kernels decode albedo through."""
    L = oracle.lib()
    return np.array([L.orc_srgb8_to_linear(i) for i in range(256)], np.float32)


def light_pairs(prep, clus, tile, zi, ys, xs):
    """(pixel, light) pairs of draw 2: for lit pixel k = (ys[k], xs[k]) every light of its (tile, Z slice) mask,
    cut to the slice's light range (cluster_mask_range), in ascending light order.  Returns (pix, light) int64."""
    n = prep.n
    if n == 0 or len(ys) == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    n32 = int(prep.params.num_lights_32)
    rng = clus.range.astype(np.int64)
    t, z = tile[ys, xs].astype(np.int64), zi[ys, xs].astype(np.int64)
    key = t * rng.shape[0] + z
    ukeys, inv = np.unique(key, return_inverse=True)
    rows = clus.bitmask.reshape(-1, n32)
    utiles, tinv = np.unique(ukeys // rng.shape[0], return_inverse=True)
    bits = np.unpackbits(np.ascontiguousarray(rows[utiles]).view(np.uint8), axis=1, bitorder="little").astype(bool)
    lists = []
    for k, uk in enumerate(ukeys):
        rx, ry = rng[uk % rng.shape[0]]
        hi = min(ry + 1, 32 * n32, n)
        lists.append(np.nonzero(bits[tinv[k], rx:hi])[0] + rx if rx < hi else np.zeros(0, np.int64))
    counts = np.array([len(a) for a in lists], np.int64)
    flat = np.concatenate(lists).astype(np.int64)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    per_pix = counts[inv]
    pix = np.repeat(np.arange(len(ys)), per_pix)
    first = np.concatenate([[0], np.cumsum(per_pix)[:-1]])
    light = flat[np.repeat(starts[inv], per_pix) + np.arange(len(pix)) - np.repeat(first, per_pix)]
    return pix, light


def positions(depth, ivp, ys, xs, dt):
    """World position of pixels (ys, xs): invVP * (ndc.xy, depth, 1) at the pixel centre, divided by w."""
    H, W = depth.shape
    m = np.asarray(list(ivp), np.float32).astype(dt).reshape(4, 4)  # column-major: m[column, row]
    nx = (xs.astype(dt) + dt(0.5)) * dt(2.0) / dt(W) - dt(1.0)
    ny = (ys.astype(dt) + dt(0.5)) * dt(2.0) / dt(H) - dt(1.0)
    d = depth[ys, xs].astype(dt)
    c = [m[0, r] * nx + m[1, r] * ny + m[3, r] + d * m[2, r] for r in range(4)]
    return np.stack([c[0] / c[3], c[1] / c[3], c[2] / c[3]], -1)


def _dot(a, b):
    return a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1] + a[..., 2] * b[..., 2]


def _normalize(a):
    return a / np.sqrt(_dot(a, a))[..., None]


def brdf(form, N, V, L, base, metallic, rough_in, dt):
    """NoL * (F G D + (1 - F) base (1 - metallic) / PI) per channel, (..., 3).  form selects how the half-vector
    terms are evaluated: "ref" the oracle's normalize(V + L); "h" the explicit h = V + L of the persistent kernel
    (NoL = N.h - N.V, HoV = |h| / 2); "vol" the |V + L|^2 = 2 + 2 V.L algebra the pairs kernel used before it formed
    h (NoH = (N.L + N.V) / |h|, HoV = (1 + V.L) / |h|)."""
    one = dt(1.0)
    r = rough_in * dt(0.75) + dt(0.25)
    m = r * r
    m2 = m * m
    NoVr = _dot(N, V)
    NoV = np.clip(NoVr, dt(0.001), one)
    if form == "ref":
        H = _normalize(V + L)
        NoL = np.clip(_dot(N, L), dt(0.001), one)
        f = one - np.clip(_dot(H, V), dt(0.001), one)
        NoH = np.clip(_dot(N, H), dt(0.0001), one)
    elif form == "h":
        h = V + L
        hh = _dot(h, h)
        inv_h = one / np.sqrt(hh)
        Nh = _dot(N, h)
        NoL = np.clip(Nh - NoVr, dt(0.001), one)
        NoH = np.clip(Nh * inv_h, dt(0.0001), one)
        f = np.minimum(one - hh * inv_h * dt(0.5), dt(0.999))
    elif form == "vol":
        VoL, NoLr = _dot(V, L), _dot(N, L)
        inv_h = one / np.sqrt(VoL * dt(2.0) + dt(2.0))
        NoL = np.clip(NoLr, dt(0.001), one)
        NoH = np.clip((NoLr + NoVr) * inv_h, dt(0.0001), one)
        f = one - np.maximum(VoL * inv_h + inv_h, dt(0.001))
    else:
        raise ValueError(form)
    f5 = f * f * f * f * f
    d = (NoH * m2 - NoH) * NoH + one
    D = m2 / (dt(PI) * d * d)
    k = (r + one) * (r + one) * dt(0.125)
    G = dt(0.25) / np.maximum((NoV * (one - k) + k) * (NoL * (one - k) + k), dt(0.001))
    F0 = dt(0.04) * (one - metallic)[..., None] + base * metallic[..., None]
    F = F0 * (one - f5)[..., None] + f5[..., None]
    spec = F * (G * D)[..., None]
    diff = (one - F) * dt(1.0 / PI) * base * (one - metallic)[..., None]
    return NoL[..., None] * (spec + diff)


def _light_color(recs, type_mask, light, P, dt):
    """point.h compute_point_color / spot.h compute_spot_color: (colour x falloff / dist^2 (..., 3), L (..., 3))."""
    one = dt(1.0)
    lpos = recs["position"][light].astype(dt)
    inv_r = recs["inv_radius"][light].astype(dt)
    col = recs["color"][light].astype(dt)
    full = lpos - P
    dist2 = _dot(full, full)
    L = full / np.sqrt(dist2)[..., None]
    dist = np.maximum(dt(0.1), np.sqrt(dist2))
    e0 = dt(np.float32(0.9))  # smoothstep(0.9, 1.0, .): the shader's constants are fp32
    t = np.clip((dist * inv_r - e0) / (one - e0), dt(0.0), one)
    fall = one - t * t * (dt(3.0) - dt(2.0) * t)
    is_point = ((type_mask[light >> 5].astype(np.int64) >> (light & 31)) & 1) == 1
    sb = recs["spot_scale_bias"][light].view(np.float16).astype(dt)
    cone = np.clip(_dot(-L, recs["direction"][light].astype(dt)) * sb[:, 0] + sb[:, 1], dt(0.0), one)
    fall = np.where(is_point, fall, fall * cone * cone)
    return col * (fall / (dist * dist))[..., None], L


def evaluate(scene, cam, prep, pairs, ys, xs, srgb, form, dt):
    """Draw 1 (value before its store, (P, 3)) and draw 2's per-pair terms ((Q, 3)) for lit pixels (ys, xs)."""
    a8 = scene.albedo[ys, xs].astype(np.int64)
    base = np.stack([srgb[a8 & 255], srgb[(a8 >> 8) & 255], srgb[(a8 >> 16) & 255]], -1).astype(dt)
    n10 = scene.normal[ys, xs].astype(np.int64)
    N = np.stack([(n10 >> s) & 1023 for s in (0, 10, 20)], -1).astype(dt) / dt(1023.0) * dt(2.0) - dt(1.0)
    mr = scene.pbr[ys, xs].astype(np.int64)
    metallic, rough = (mr & 255).astype(dt) / dt(255.0), (mr >> 8).astype(dt) / dt(255.0)
    P = positions(scene.depth, cam.inv_view_projection, ys, xs, dt)
    V = _normalize(np.asarray(list(cam.camera_position), np.float32).astype(dt) - P)
    dir_dir = np.broadcast_to(np.asarray(scene.dir_direction, np.float32).astype(dt), P.shape)
    dir_col = np.asarray(scene.dir_color, np.float32).astype(dt)
    draw1 = dir_col * brdf(form, N, V, dir_dir, base, metallic, rough, dt) + base * dt(0.05)
    pix, light = pairs
    color, L = _light_color(prep.records, prep.type_mask, light, P[pix], dt)
    terms = color * brdf(form, N[pix], V[pix], L, base[pix], metallic[pix], rough[pix], dt)
    return draw1, terms


def _per_pixel_sum(pix, v, n):
    return np.stack([np.bincount(pix, weights=v[:, k].astype(np.float64), minlength=n) for k in range(3)], -1)


# ----------------------------------------------------------------------------------------------- reference + bar
def reference(oracle, scene, cam, prep, clus, indices=None, emissive=None, pairs=None):
    """Float64 values and slacks of every lit pixel.  indices = (tile, zi) from oracle.deferred_lighting(...,
    want_indices=True) (computed here when None); emissive: the destination's initial words (scene.emissive).
    pairs: draw 2's (pixel, light) pairs over the lit pixels in row-major order, in place of the cluster's (clus and
    indices are then not read); tests/cluster_cases.py brute_pairs gives the pairs whose falloff is nonzero."""
    emissive = scene.emissive if emissive is None else emissive
    lit = scene.depth != 0
    ys, xs = np.nonzero(lit)
    tile = zi = None
    if pairs is None:
        if indices is None:
            _, tile, zi, _ = oracle.deferred_lighting(scene, cam, prep, clus, want_indices=True)
        else:
            tile, zi = indices
        pairs = light_pairs(prep, clus, tile, zi, ys, xs)
    srgb = srgb_table(oracle)
    d64, t64 = evaluate(scene, cam, prep, pairs, ys, xs, srgb, "ref", np.float64)
    d32, t32 = evaluate(scene, cam, prep, pairs, ys, xs, srgb, "ref", np.float32)
    e = decode(emissive[ys, xs])
    s1 = REL * (e + np.abs(d64)) + GAP * np.abs(d64 - d32.astype(np.float64))
    P = len(ys)
    l64 = _per_pixel_sum(pairs[0], t64, P)
    mag = _per_pixel_sum(pairs[0], np.abs(t64), P)
    gap = _per_pixel_sum(pairs[0], np.abs(t64 - t32.astype(np.float64)), P)
    return SimpleNamespace(lit=lit, ys=ys, xs=xs, pairs=pairs, emissive=emissive, e=e, d1=d64, s1=s1, l64=l64, mag=mag, gap=gap,
                           tile=tile, zi=zi, srgb=srgb)


def _code_bounds(dst, v, s):
    """(lo, hi) codes of the store of dst + (v -+ s), where dst is a stored value and v >= 0 a sum of terms that are
    all >= 0: an fp32 sum of such terms onto dst never falls below dst."""
    lo = np.stack([ufloat_code(np.maximum(dst[..., k] + v[..., k] - s[..., k], dst[..., k]), MBITS[k]) for k in range(3)], -1)
    hi = np.stack([ufloat_code(dst[..., k] + v[..., k] + s[..., k], MBITS[k]) for k in range(3)], -1)
    return lo, hi


def allowed_codes(ref):
    """(lo, hi) final codes per lit pixel and channel, (P, 3) each."""
    q_lo, q_hi = _code_bounds(ref.e, ref.d1, ref.s1)
    base_lo = np.stack([ufloat_value(q_lo[:, k], MBITS[k]) for k in range(3)], -1)
    base_hi = np.stack([ufloat_value(q_hi[:, k], MBITS[k]) for k in range(3)], -1)
    s2 = REL * (base_hi + ref.mag) + GAP * ref.gap
    lo, _ = _code_bounds(base_lo, ref.l64, s2)
    _, hi = _code_bounds(base_hi, ref.l64, s2)
    return lo, hi


def bar_misses(got, ref):
    """Boolean (P, 3): lit pixel channels of `got` ((H, W) packed words) outside the bar."""
    c = codes(got[ref.ys, ref.xs])
    lo, hi = allowed_codes(ref)
    return (c < lo) | (c > hi)


def assert_meets_bar(got, ref, what=""):
    """Every lit channel within the float64 bar, and every sky pixel the destination's bits."""
    sky = ~ref.lit
    assert np.array_equal(got[sky], ref.emissive[sky]), f"{what}: sky pixels must keep the destination's value"
    bad = bar_misses(got, ref)
    if bad.any():
        c = codes(got[ref.ys, ref.xs])
        lo, hi = allowed_codes(ref)
        k = np.argwhere(bad)[:5]
        detail = ", ".join(f"({int(ref.xs[i])},{int(ref.ys[i])})[{j}] code {int(c[i, j])} not in [{int(lo[i, j])}, {int(hi[i, j])}]" for i, j in k)
        raise AssertionError(f"{what}: {int(bad.sum())} channels outside the float64 bar, e.g. {detail}")


def emulate(oracle, scene, cam, prep, ref, form, dt=np.float32):
    """The frame a kernel evaluating the BRDF with `form` in `dt` would store (draw 1, its store, draw 2, the store),
    with the reference's pairs; sky pixels keep the destination.  For checking on the CPU that a case discriminates
    between formulations."""
    d, t = evaluate(scene, cam, prep, ref.pairs, ref.ys, ref.xs, ref.srgb, form, dt)
    e = decode(ref.emissive[ref.ys, ref.xs]).astype(dt)
    q1 = pack((e + d).astype(np.float64))
    acc = _per_pixel_sum(ref.pairs[0], t, len(ref.ys)).astype(dt)
    out = ref.emissive.copy()
    out[ref.ys, ref.xs] = pack((decode(q1).astype(dt) + acc).astype(np.float64))
    return out



# ----------------------------------------------------------------------------------------------- cases
def grazing_case(oracle, w=640, h=360, patches=12, theta=(0.01, 0.03), distance=4.0, color=300.0):
    """A specular peak seen at a grazing angle: `patches` 2x2-pixel patches of the lit ground get roughness input 0
    and normals along h = V + L, and each gets one bright point light `distance` metres behind it along the view ray
    of its first pixel, turned by an angle in `theta` away from -V.  Returns (scene, cam, lights, prep, patch mask,
    per-pixel angle between L and -V)."""
    from granite_b200 import synth

    scene = synth.make_scene(w, h)
    cam = oracle.camera_setup(scene.projection, scene.view)
    eye = np.asarray(list(cam.camera_position), np.float64)
    rng = np.random.default_rng(0x6A2E)
    lit = scene.depth != 0
    mask = np.zeros((h, w), bool)
    angle = np.full((h, w), np.nan)
    pos, cols = [], []
    cands = [(y, x) for y in range(h // 2 + 8, h - 8, 6) for x in range(16, w - 16, 12) if lit[y:y + 2, x:x + 2].all()]
    for k in rng.choice(len(cands), patches, replace=False):
        y, x = cands[k]
        ys, xs = np.mgrid[y:y + 2, x:x + 2]
        P = positions(scene.depth, cam.inv_view_projection, ys.ravel(), xs.ravel(), np.float64)
        fwd = P[0] - eye
        fwd /= np.linalg.norm(fwd)
        side = np.cross(fwd, (0.0, 1.0, 0.0))
        side /= np.linalg.norm(side)
        t = rng.uniform(*theta)
        q = (P[0] + distance * (np.cos(t) * fwd + np.sin(t) * side)).astype(np.float32)
        V = eye - P
        V /= np.linalg.norm(V, axis=1, keepdims=True)
        L = q.astype(np.float64) - P
        L /= np.linalg.norm(L, axis=1, keepdims=True)
        Nv = V + L
        Nv /= np.linalg.norm(Nv, axis=1, keepdims=True)
        n10 = np.clip(np.rint((Nv * 0.5 + 0.5) * 1023.0), 0, 1023).astype(np.uint32)
        scene.normal[ys.ravel(), xs.ravel()] = n10[:, 0] | (n10[:, 1] << 10) | (n10[:, 2] << 20) | np.uint32(3 << 30)
        scene.pbr[ys.ravel(), xs.ravel()] = 0  # metallic 0, roughness input 0
        mask[y:y + 2, x:x + 2] = True
        angle[ys.ravel(), xs.ravel()] = np.arccos(np.clip(np.sum(L * (P - eye) / np.linalg.norm(P - eye, axis=1, keepdims=True), 1), -1.0, 1.0))
        pos.append(q)
        cols.append(np.full(3, color, np.float32))
    pos = np.asarray(pos, np.float32)
    order = np.argsort(-pos[:, 2], kind="stable")  # front to back, as the clusterer expects
    n = len(pos)
    lights = synth.Lights(np.asarray(cols, np.float32)[order], pos[order], np.ones(n, bool), np.zeros((n, 3, 3), np.float32),
                          np.full(n, 0.9, np.float32), np.full(n, 0.8, np.float32))
    prep = oracle.prepare_lights(cam, lights, res=synth.CLUSTER_RES, cull=False)
    return scene, cam, lights, prep, mask, angle


def dense_case(oracle, w=256, h=144, n=320, seed=0xDE5E):
    """Point lights crowded into a 2 m box on the ground 10 m in front of the camera (colours 0.5..2, radii of a few
    metres): the pixel blocks around it keep far more lights than one list batch holds."""
    from granite_b200 import synth

    scene = synth.make_scene(w, h)
    cam = oracle.camera_setup(scene.projection, scene.view)
    rng = np.random.default_rng(seed)
    pos = np.stack([rng.uniform(-1.0, 1.0, n), rng.uniform(-1.8, 0.2, n), rng.uniform(-3.0, -1.0, n)], -1).astype(np.float32)
    pos = pos[np.argsort(-pos[:, 2], kind="stable")]
    lights = synth.Lights(rng.uniform(0.5, 2.0, (n, 3)).astype(np.float32), pos, np.ones(n, bool), np.zeros((n, 3, 3), np.float32),
                          np.full(n, 0.9, np.float32), np.full(n, 0.8, np.float32))
    return scene, cam, lights, oracle.prepare_lights(cam, lights, res=synth.CLUSTER_RES)


def block_batches(scene, cam, prep, clus, zi, list_cap=160):
    """The persistent kernel's light lists, recomputed: for every 16x4 pixel block, the candidates of the bitmask
    rows of the cluster tiles under it, cut to the hull of its lit pixels' Z-slice ranges, that pass the sphere-box
    test against the box of its lit pixels; compacted a 32-light word at a time into batches that close once they
    hold more than list_cap - 32 entries.  Returns {(bx, by): [batch lengths]} for blocks with candidates."""
    H, W = scene.depth.shape
    pr = prep.params
    n32 = int(pr.num_lights_32)
    f = np.float32
    inv_x, inv_y = f(1.0) / f(W), f(1.0) / f(H)
    tx_of = lambda x: min(max(int((f(x) + f(0.5)) * inv_x * f(pr.xy_scale[0])), 0), int(pr.resolution_xy[0]) - 1)  # noqa: E731
    ty_of = lambda y: min(max(int((f(y) + f(0.5)) * inv_y * f(pr.xy_scale[1])), 0), int(pr.resolution_xy[1]) - 1)  # noqa: E731
    rows = clus.bitmask.reshape(-1, n32)
    lpos = prep.records["position"].astype(np.float64)
    inv_r = prep.records["inv_radius"].astype(np.float64)
    out = {}
    for by in range(0, H, 4):
        for bx in range(0, W, 16):
            ys, xs = np.nonzero(scene.depth[by:by + 4, bx:bx + 16] != 0)
            if len(ys) == 0:
                continue
            ys, xs = ys + by, xs + bx
            rng = clus.range[zi[ys, xs]].astype(np.int64)
            lo, hi = int(rng[:, 0].min()), int(rng[:, 1].max())
            if lo > hi:
                continue
            words = np.zeros(n32, np.uint64)
            for ty in range(ty_of(by), ty_of(min(by + 3, H - 1)) + 1):
                for tx in range(tx_of(bx), tx_of(min(bx + 15, W - 1)) + 1):
                    words |= rows[ty * int(pr.resolution_xy[0]) + tx].astype(np.uint64)
            idx = np.nonzero(np.unpackbits(words.astype("<u4").view(np.uint8), bitorder="little"))[0]
            idx = idx[(idx >= lo) & (idx <= hi)]
            P = positions(scene.depth, cam.inv_view_projection, ys, xs, np.float64)
            d = np.maximum(np.maximum(P.min(0) - lpos[idx], lpos[idx] - P.max(0)), 0.0)
            idx = idx[(d * d).sum(1) * inv_r[idx] ** 2 < 1.0005]
            if len(idx) == 0:
                continue
            batches, count = [], 0
            for word_count in np.bincount(idx >> 5, minlength=n32):
                if not word_count:
                    continue
                count += int(word_count)
                if count > list_cap - 32:
                    batches.append(count)
                    count = 0
            if count:
                batches.append(count)
            out[(bx // 16, by // 4)] = batches
    return out
