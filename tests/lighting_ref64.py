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
ill-conditioned.  tests/test_lighting_ref64_cpu.py pins it: the fp32 oracle meets this bar.

RGBA16F destinations (fmt=RGBA16F): the store rounds to nearest even with fp16 subnormals, 65520 and above to +inf;
draw 1 and the final sum are each stored; alpha keeps the destination's bits.  Non-negative fp16 bit patterns are
ordered like the values, so the same two-stage code bounds apply; a draw 1 stored as +inf stays +inf.

Shadowed lights (shadows=(transforms, maps, res[, pcf_wide])): each pair's shadow factor is restated in float64 (the
2 x 2 comparison sample, the 6 x 6 wide PCF, the cube sample with its edge and corner handling; the cube's edge
neighbours are taken from the oracle).  A comparison ref >= texel / 65535 is ambiguous where the two sides are closer
than fp32 can tell apart, and so is a cube major-axis tie; both outcomes are admitted.  Every filter is a
non-negative combination of comparisons, so the interval comes from two evaluations (ambiguous comparisons all 0,
then all 1).  A pair contributes its term times the interval's midpoint, and half the interval's width times the
term's magnitude goes into the slack.

The receiver's position.  t32 uses the reference's own fp32 position, which can by chance be far more accurate than a
kernel's (another association of the same sums): at 1920 x 1080 a light 0.68 m from a receiver 27 m away, almost in
the surface's plane (N.L = 0.005), moves its term by 8e-4 relative for 3 ulps of the position, ten times GAP |t64 -
t32| there.  So the slack also holds each value's change over a bound of the fp32 position error (position_error),
which covers a shadow footprint that moves by res times that error as well."""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np

PI = float(np.float32(3.1415628))  # assets/shaders/lights/pbr.h:5 (sic), as the oracle and the kernels use it
REL = 2e-5
GAP = 4.0
MBITS = (6, 6, 5)  # R, G, B mantissa bits of B10G11R11
B10G11R11, RGBA16F = "b10g11r11", "rgba16f"


# ----------------------------------------------------------------------------------------------- stored codes
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


def half_code(v):
    """Code of the RGBA16F store of v >= 0 (float64): round to nearest even, fp16 subnormals, >= 65520 -> +inf.  The
    bit patterns of non-negative fp16 values (+inf included) are ordered like the values."""
    with np.errstate(over="ignore"):
        return np.maximum(np.asarray(v, np.float64), 0.0).astype(np.float16).view(np.uint16).astype(np.int64)


def half_value(code):
    return np.asarray(code).astype(np.uint16).view(np.float16).astype(np.float64)


def channel_code(v, k, fmt):
    return ufloat_code(v, MBITS[k]) if fmt == B10G11R11 else half_code(v)


def channel_value(code, k, fmt):
    return ufloat_value(code, MBITS[k]) if fmt == B10G11R11 else half_value(code)


def codes(packed, fmt=None):
    """(..., 3) int64 channel codes: of packed B10G11R11 words ((H, W) uint32), or the RGB of RGBA16F texels ((H, W, 4)
    uint16).  fmt None takes the format from the array."""
    p = np.asarray(packed)
    if (fmt or (RGBA16F if p.dtype == np.uint16 else B10G11R11)) == RGBA16F:
        return p[..., :3].astype(np.int64)
    p = p.astype(np.uint32).astype(np.int64)
    return np.stack([p & 0x7FF, (p >> 11) & 0x7FF, p >> 22], -1)


def decode(packed, fmt=None):
    c = codes(packed, fmt)
    fmt = fmt or (RGBA16F if np.asarray(packed).dtype == np.uint16 else B10G11R11)
    return np.stack([channel_value(c[..., k], k, fmt) for k in range(3)], -1)


def pack(rgb):
    """Store of float values (..., 3): truncating, as pack_r11g11b10."""
    c = [ufloat_code(rgb[..., k], MBITS[k]) for k in range(3)]
    return (c[0] | (c[1] << 11) | (c[2] << 22)).astype(np.uint32)


def store_f16(rgb, alpha, rounding="rne"):
    """RGBA16F texels (..., 4) uint16 of float values rgb (..., 3), alpha the bits kept.  rounding "rne" is the store;
    "trunc" rounds toward zero (for showing that a case tells the two apart)."""
    rgb = np.asarray(rgb)
    if rounding == "rne":
        c = half_code(rgb)
    else:
        c = half_code(rgb)
        over = half_value(c) > np.where(rgb > 0, rgb, 0.0)  # rounded up: step back one code (+inf included)
        c = np.where(over & (c > 0), c - 1, c)
    return np.concatenate([c, np.asarray(alpha)[..., None].astype(np.int64)], -1).astype(np.uint16)


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


def position_error(depth, ivp, ys, xs):
    """(P, 3) float64 bound of the error of an fp32 reconstruction of the world positions of pixels (ys, xs), whatever
    the association or FMA contraction of its sums: each clip component is a sum of four products (and the ndc
    coordinates carry one rounding of about 1), so its error is below 6 u times the sum of the magnitudes; the
    division by w adds |P| times w's relative error and one rounding (u = 2^-24)."""
    H, W = depth.shape
    m = np.asarray(list(ivp), np.float32).astype(np.float64).reshape(4, 4)
    nx = (xs + 0.5) * 2.0 / W - 1.0
    ny = (ys + 0.5) * 2.0 / H - 1.0
    d = depth[ys, xs].astype(np.float64)
    u = 2.0 ** -24
    mag = [np.abs(m[0, r] * nx) + np.abs(m[1, r] * ny) + abs(m[3, r]) + np.abs(d * m[2, r]) + abs(m[0, r]) + abs(m[1, r]) for r in range(4)]
    c = [m[0, r] * nx + m[1, r] * ny + m[3, r] + d * m[2, r] for r in range(4)]
    P = np.stack([c[0] / c[3], c[1] / c[3], c[2] / c[3]], -1)
    err = np.stack([6 * u * mag[r] for r in range(3)], -1)
    return (err + np.abs(P) * (6 * u * mag[3])[:, None]) / np.abs(c[3])[:, None] + 2 * u * np.abs(P)


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


def evaluate(scene, cam, prep, pairs, ys, xs, srgb, form, dt, P=None):
    """Draw 1 (value before its store, (P, 3)) and draw 2's per-pair terms ((Q, 3)) for lit pixels (ys, xs); P: their
    world positions in place of positions(...)."""
    a8 = scene.albedo[ys, xs].astype(np.int64)
    base = np.stack([srgb[a8 & 255], srgb[(a8 >> 8) & 255], srgb[(a8 >> 16) & 255]], -1).astype(dt)
    n10 = scene.normal[ys, xs].astype(np.int64)
    N = np.stack([(n10 >> s) & 1023 for s in (0, 10, 20)], -1).astype(dt) / dt(1023.0) * dt(2.0) - dt(1.0)
    mr = scene.pbr[ys, xs].astype(np.int64)
    metallic, rough = (mr & 255).astype(dt) / dt(255.0), (mr >> 8).astype(dt) / dt(255.0)
    P = positions(scene.depth, cam.inv_view_projection, ys, xs, dt) if P is None else np.asarray(P).astype(dt)
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


# ----------------------------------------------------------------------------------------------- shadow factor
class ShadowStats(SimpleNamespace):
    """What one shadow evaluation reached, counted over the pairs it sampled: pairs (shadowed pairs sampled),
    ambiguous (pairs with an ambiguous comparison), edge (cube pairs whose 2 x 2 footprint steps over a face edge),
    corner (cube pairs that take the three-texel corner average), tie (cube pairs with more than one candidate face),
    outside (spot pairs whose footprint leaves the map and is clamped to its edge), ref_hi / ref_lo (pairs whose
    reference depth clamps to 1 / to 0)."""

    def __init__(self):
        super().__init__(pairs=0, ambiguous=0, edge=0, corner=0, tie=0, outside=0, ref_hi=0, ref_lo=0)


_CUBE_TABLES = {}


def cube_texels(oracle, res):
    """(6, res + 2, res + 2) int64: the texel of face f that samples (i, j), i and j in -1 .. res (index i + 1, j + 1),
    across the cube's edges; -1 at the four corners.  Taken from orc_shadow_cube_texel, whose mapping
    test_shadow_source_cpu.py pins to the geometric neighbours."""
    if res not in _CUBE_TABLES:
        import ctypes as C

        fn = oracle.lib().orc_shadow_cube_texel
        fn.restype = C.c_int
        t = np.full((6, res + 2, res + 2), -1, np.int64)
        out = C.c_size_t()
        for f in range(6):
            for i in range(-1, res + 1):
                for j in range(-1, res + 1):
                    if fn(res, f, i, j, C.byref(out)):
                        t[f, i + 1, j + 1] = out.value
        _CUBE_TABLES[res] = t
    return _CUBE_TABLES[res]


def _ulp32(x):
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float32)).astype(np.float64)


class _Compare:
    """Comparison results ref >= texel / 65535 of one evaluation, per (pair, texel).  exact: the reference's own
    outcome in dt (emulations).  Otherwise a comparison is ambiguous where |ref64 - d| is within
    GAP |ref64 - ref32| + the fp32 rounding of ref and of d, and takes `mode` (0 or 1); the rest take the float64
    outcome."""

    def __init__(self, texels, ref64, ref32, mode=None, ref=None, dt=np.float64):
        self.d64 = texels.astype(np.float64) / 65535.0
        self.d32 = (texels.astype(np.float32) / np.float32(65535.0)).astype(np.float64)
        self.ref64, self.mode, self.ref, self.dt = ref64, mode, ref, dt
        inner = (ref64 > 0.0) & (ref64 < 1.0)
        self.w = GAP * np.abs(ref64 - ref32) + np.where(inner, _ulp32(ref64), 0.0)
        self.ambiguous = np.zeros(len(ref64), bool)

    def __call__(self, q, tex):
        if self.mode is None:
            d = self.d32 if self.dt == np.float32 else self.d64
            return (self.ref[q] >= d[tex].astype(self.dt)).astype(self.dt)
        r = self.ref64[q]
        amb = np.abs(r - self.d64[tex]) < self.w[q] + np.abs(self.d32[tex] - self.d64[tex])
        np.logical_or.at(self.ambiguous, q, amb)
        return np.where(amb, self.dt(self.mode), (r >= self.d64[tex]).astype(self.dt)).astype(self.dt)


def _bilin(s, t, res, dt, half=True):
    """oracle_math.h bilin_setup: (x0, y0) and the fractions of (s res - 0.5, t res - 0.5); half=False drops the
    half-texel offset (for showing that a case tells the two apart)."""
    o = dt(0.5) if half else dt(0.0)
    fx, fy = s * dt(res) - o, t * dt(res) - o
    flx, fly = np.floor(fx), np.floor(fy)
    a, b = fx - flx, fy - fly
    x0 = np.nan_to_num(np.clip(flx, -2, res + 1)).astype(np.int64)
    y0 = np.nan_to_num(np.clip(fly, -2, res + 1)).astype(np.int64)
    return x0, y0, a, b


def _mix(c00, c10, c01, c11, a, b):
    one = np.ones_like(a)
    ia, ib = one - a, one - b
    return (c00 * ia + c10 * a) * ib + (c01 * ia + c11 * a) * b


def _spot_factor(cmp, q, base, res, clip, dt, wide, variant, stats):
    """textureProjLod(sampler2DShadow, clip, 0) with the 2 x 2 filter, or the 6 x 6 kernel of pcf.h (wide)."""
    s, t = clip[:, 0] / clip[:, 3], clip[:, 1] / clip[:, 3]
    at = lambda x, y: cmp(q, base + np.clip(y, 0, res - 1) * res + np.clip(x, 0, res - 1))  # noqa: E731
    if not wide:
        x0, y0, a, b = _bilin(s, t, res, dt, variant != "no-half-texel")
        if stats is not None:
            stats.outside += int(((x0 < 0) | (y0 < 0) | (x0 + 1 > res - 1) | (y0 + 1 > res - 1)).sum())
        return _mix(at(x0, y0), at(x0 + 1, y0), at(x0, y0 + 1), at(x0 + 1, y0 + 1), a, b)
    ix, iy = s * dt(res) - dt(1.5), t * dt(res) - dt(1.5)
    flx, fly = np.floor(ix), np.floor(iy)
    fx, fy = ix - flx, iy - fly
    x0 = np.nan_to_num(np.clip(flx, -8, res + 8)).astype(np.int64) - 1
    y0 = np.nan_to_num(np.clip(fly, -8, res + 8)).astype(np.int64) - 1
    if variant == "origin-clamp":  # the window's origin clamped to >= -2 before the texels clamp to the edge
        x0, y0 = np.clip(x0, -2, res + 1), np.clip(y0, -2, res + 1)
    if stats is not None:
        stats.outside += int(((x0 < 0) | (y0 < 0) | (x0 + 5 > res - 1) | (y0 + 5 > res - 1)).sum())
    weight = lambda p: np.exp2(p * p * dt(-0.375)) * (dt(1.0) - p * p / dt(9.0))  # noqa: E731
    H = [weight(fx + dt(2 - k)) for k in range(6)]
    V = [weight(fy + dt(2 - k)) for k in range(6)]
    num = sum(at(x0 + c, y0 + r) * (H[c] * V[r]) for r in range(6) for c in range(6))
    if variant == "wide-unnormalised":
        return num
    return num / (sum(H) * sum(V))


def _cube_factor(cmp, q, base, res, d, axis, dt, table, variant, stats):
    """texture(samplerCubeShadow, vec4(d, ref)) on the face of major axis `axis` (per pair), with the footprint
    stepped across the cube's edges and the missing corner texel replaced by the mean of the other three."""
    rows = np.arange(len(q))
    comp = d[rows, axis]
    neg = comp < 0
    face = 2 * axis + neg
    dx, dy, dz = d[:, 0], d[:, 1], d[:, 2]
    sc = np.select([axis == 2, axis == 1], [np.where(neg, -dx, dx), dx], np.where(neg, dz, -dz))
    tc = np.select([axis == 2, axis == 1], [-dy, np.where(neg, -dz, dz)], -dy)
    ma = np.abs(comp)
    s, t = dt(0.5) * (sc / ma) + dt(0.5), dt(0.5) * (tc / ma) + dt(0.5)
    x0, y0, a, b = _bilin(s, t, res, dt)
    c, have, stepped = [], [], np.zeros(len(q), bool)
    for k in range(4):
        i, j = np.clip(x0 + (k & 1), -1, res), np.clip(y0 + (k >> 1), -1, res)
        stepped |= ((i < 0) | (i >= res)) != ((j < 0) | (j >= res))
        if variant == "edge-clamp":
            tex = (face * res + np.clip(j, 0, res - 1)) * res + np.clip(i, 0, res - 1)
        else:
            tex = table[face, i + 1, j + 1]
        have.append(tex >= 0)
        c.append(np.where(tex >= 0, cmp(q, base + np.maximum(tex, 0)), dt(0.0)))
    n = sum(h.astype(np.int64) for h in have)
    if stats is not None:
        stats.edge += int(stepped.sum())
        stats.corner += int((n == 3).sum())
    fill = np.zeros_like(c[0]) if variant == "corner-zero" else (c[0] + c[1] + c[2] + c[3]) / dt(3.0)
    c = [np.where(h, ck, np.where(n == 3, fill, dt(0.0))) for ck, h in zip(c, have)]
    return _mix(c[0], c[1], c[2], c[3], a, b)


def shadow_factors(oracle, prep, shadows, light, P64, P32, variant=None, dt=None, stats=None, live=None, float32=True):
    """Shadow factor of each (pair, light) with P64 / P32 the pairs' world positions in float64 / float32.
    shadows = (transforms, maps, res[, pcf_wide]).  Returns (lo64, hi64, lo32, hi32): the factor's interval evaluated
    in float64 and in float32, ambiguous comparisons (and both faces of a cube major-axis tie) admitting both outcomes.
    With dt set (an emulation): (factor, None, None, None), the comparisons and the face taken in dt as they fall,
    `variant` one of the deliberate errors the CPU tests show the bar rejects.  live: the pairs whose unshadowed term
    is nonzero (the kernels sample only those); the others keep factor 1.  float32=False skips the float32 evaluation
    (lo32 and hi32 are then 1)."""
    transforms, maps, res = shadows[:3]
    wide = bool(shadows[3]) if len(shadows) > 3 else False
    nq = len(light)
    out = [np.ones(nq), np.ones(nq), np.ones(nq), np.ones(nq)]
    sizes = np.array([0 if m is None else np.asarray(m).size for m in maps], np.int64)
    texels = np.concatenate([np.asarray(m, np.uint16).ravel() for m in maps if m is not None] or [np.zeros(1, np.uint16)])
    base_of = np.concatenate([[0], np.cumsum(sizes)[:-1]]) if len(sizes) else np.zeros(0, np.int64)
    has = np.zeros(nq, bool) if not len(sizes) else sizes[light] > 0
    if live is not None:
        has &= live
    is_point = ((prep.type_mask[light >> 5].astype(np.int64) >> (light & 31)) & 1) == 1
    m32 = np.asarray(transforms, np.float32)
    table = cube_texels(oracle, res) if (has & is_point).any() else None
    for point in (False, True):
        sel = np.nonzero(has & (is_point == point))[0]
        if len(sel) == 0:
            continue
        base = base_of[light[sel]]
        m = m32[light[sel]]
        lpos = prep.records["position"][light[sel]]
        vals = {}
        for t in (np.float64, np.float32):
            P, mt = (P64 if t == np.float64 else P32)[sel].astype(t), m.astype(t)
            if point:
                full = P - lpos.astype(t)
                mz = np.abs(full).max(1)
                ref = (mt[:, 2] - mt[:, 0] * mz) / (mt[:, 3] - mt[:, 1] * mz)
                vals[t] = (full, ref)
            else:
                clip = np.stack([(mt[:, r] * P[:, 0] + mt[:, 4 + r] * P[:, 1]) + (mt[:, 8 + r] * P[:, 2] + mt[:, 12 + r]) for r in range(4)], -1)
                vals[t] = (clip, clip[:, 2] / clip[:, 3])
        raw64 = vals[np.float64][1]
        ref64 = np.nan_to_num(np.clip(raw64, 0.0, 1.0))
        ref32 = np.nan_to_num(np.clip(vals[np.float32][1], 0.0, 1.0)).astype(np.float64)
        if stats is not None:
            stats.pairs += len(sel)
            stats.ref_hi += int((raw64 > 1.0).sum())
            stats.ref_lo += int((raw64 < 0.0).sum())
        q = np.arange(len(sel))

        def sample(cmp, t, idx, axis=None, st=None):
            """The factor of pairs sel[idx] in t (on the cube face of major axis `axis`)."""
            geo = vals[t][0][idx]
            if point:
                return _cube_factor(cmp, idx, base[idx], res, geo, axis, t, table, variant, st)
            return _spot_factor(cmp, idx, base[idx], res, geo, t, wide, variant, st)

        def major_axis(a):
            return np.where((a[:, 2] >= a[:, 0]) & (a[:, 2] >= a[:, 1]), 2, np.where(a[:, 1] >= a[:, 0], 1, 0))

        if dt is not None:
            ref_t = np.clip(np.nan_to_num(vals[dt][1]), dt(0.0), dt(1.0)).astype(dt)
            cmp = _Compare(texels, ref64, ref32, ref=ref_t, dt=dt)
            out[0][sel] = sample(cmp, dt, q, major_axis(np.abs(vals[dt][0])) if point else None)
            continue
        if point:
            # a face is a candidate where its axis is within fp32's reach of the largest component
            a64 = np.abs(vals[np.float64][0])
            tol = GAP * np.abs(a64 - np.abs(vals[np.float32][0]).astype(np.float64)) + _ulp32(a64)
            major = major_axis(a64)
            cand = a64 + tol + tol[q, major][:, None] >= a64[q, major][:, None]
            cand[q, major] = True
            if stats is not None:
                stats.tie += int((cand.sum(1) > 1).sum())
                sample(_Compare(texels, ref64, ref32, 0), np.float64, q, major, stats)
        for k, (t, mode) in enumerate([(np.float64, 0), (np.float64, 1), (np.float32, 0), (np.float32, 1)][:4 if float32 else 2]):
            cmp = _Compare(texels, ref64, ref32, mode, dt=t)
            if point:
                val = np.full(len(sel), np.nan)
                for axis in range(3):
                    idx = np.nonzero(cand[:, axis])[0]
                    if len(idx):
                        f = sample(cmp, t, idx, np.full(len(idx), axis))
                        val[idx] = np.where(np.isnan(val[idx]), f, np.minimum(val[idx], f) if mode == 0 else np.maximum(val[idx], f))
            else:
                val = sample(cmp, t, q, st=stats if k == 0 else None)
            out[k][sel] = val
            if stats is not None and k == 0:
                stats.ambiguous += int(cmp.ambiguous.sum())
    return tuple(out)


# ----------------------------------------------------------------------------------------------- reference + bar
def reference(oracle, scene, cam, prep, clus, indices=None, emissive=None, pairs=None, fmt=B10G11R11, shadows=None, stats=None,
              rows=None):
    """Float64 values and slacks of every lit pixel.  indices = (tile, zi) from oracle.deferred_lighting(...,
    want_indices=True) (computed here when None); emissive: the destination's initial texels (scene.emissive), of
    format fmt (B10G11R11 words (H, W) or RGBA16F texels (H, W, 4)).  pairs: draw 2's (pixel, light) pairs over the
    lit pixels in row-major order, in place of the cluster's (clus and indices are then not read);
    tests/cluster_cases.py brute_pairs gives the pairs whose falloff is nonzero.  shadows = (transforms, maps, res[,
    pcf_wide]) as for oracle.deferred_lighting_shadowed: each pair's term is scaled by the midpoint of its shadow
    factor's interval, and half the interval's width times the term's magnitude goes into the slack.  stats: a
    ShadowStats to count what the shadow evaluation reached.  rows = (y0, y1): only the pixels of those rows (the bar
    then checks nothing else)."""
    emissive = scene.emissive if emissive is None else emissive
    lit = scene.depth != 0
    region = np.zeros(lit.shape, bool)
    region[slice(*rows) if rows else slice(None)] = True
    lit &= region
    ys, xs = np.nonzero(lit)
    tile = zi = None
    if pairs is None:
        if indices is None:
            _, tile, zi, _ = oracle.deferred_lighting(scene, cam, prep, clus, want_indices=True)
        else:
            tile, zi = indices
        pairs = light_pairs(prep, clus, tile, zi, ys, xs)
    srgb = srgb_table(oracle)
    Pp64 = positions(scene.depth, cam.inv_view_projection, ys, xs, np.float64)
    Pp32 = positions(scene.depth, cam.inv_view_projection, ys, xs, np.float32)
    d64, u64 = evaluate(scene, cam, prep, pairs, ys, xs, srgb, "ref", np.float64, Pp64)
    d32, t32 = evaluate(scene, cam, prep, pairs, ys, xs, srgb, "ref", np.float32, Pp32)
    P = len(ys)
    shw = np.zeros((P, 3))
    t64 = u64
    live = (u64 != 0).any(1) | (t32 != 0).any(1)
    factor = lambda Pk: shadow_factors(oracle, prep, shadows, pairs[1], Pk[pairs[0]], Pp32[pairs[0]], live=live, float32=False)[:2]  # noqa: E731
    if shadows is not None and len(pairs[0]):
        lo64, hi64, lo32, hi32 = shadow_factors(oracle, prep, shadows, pairs[1], Pp64[pairs[0]], Pp32[pairs[0]], stats=stats, live=live)
        shw = _per_pixel_sum(pairs[0], np.abs(u64) * ((hi64 - lo64) / 2.0)[:, None], P)
        t64 = u64 * ((lo64 + hi64) / 2.0)[:, None]
        t32 = t32 * ((lo32.astype(np.float32) + hi32.astype(np.float32)) / np.float32(2.0))[:, None]
    # the receiver's position: a kernel's fp32 reconstruction is off by up to `h` per coordinate, and a term can be
    # ill-conditioned in it (a light almost in the surface's plane: N.L near 0 moves with L's direction; a shadow
    # footprint moves by res times the position's error).  Each draw-1 value and term moves by at most the sum over
    # the coordinates of its larger change with that coordinate moved by -h and +h.
    h = position_error(scene.depth, cam.inv_view_projection, ys, xs)
    pos1, pos2 = np.zeros_like(d64), np.zeros_like(t64)
    for k in range(3):
        m1, m2 = np.zeros_like(d64), np.zeros_like(t64)
        for sign in (-1.0, 1.0):
            Pk = Pp64.copy()
            Pk[:, k] += sign * h[:, k]
            dk, tk = evaluate(scene, cam, prep, pairs, ys, xs, srgb, "ref", np.float64, Pk)
            if shadows is not None and len(pairs[0]):
                lo, hi = factor(Pk)
                tk = tk * ((lo + hi) / 2.0)[:, None]
            m1, m2 = np.maximum(m1, np.abs(dk - d64)), np.maximum(m2, np.abs(tk - t64))
        pos1, pos2 = pos1 + m1, pos2 + m2
    e = decode(emissive[ys, xs], fmt)
    s1 = REL * (e + np.abs(d64)) + GAP * np.abs(d64 - d32.astype(np.float64)) + pos1
    l64 = _per_pixel_sum(pairs[0], t64, P)
    mag = _per_pixel_sum(pairs[0], np.abs(t64), P)
    gap = _per_pixel_sum(pairs[0], np.abs(t64 - t32.astype(np.float64)), P)
    pos = _per_pixel_sum(pairs[0], pos2, P)
    return SimpleNamespace(lit=lit, region=region, ys=ys, xs=xs, pairs=pairs, emissive=emissive, e=e, d1=d64, s1=s1, l64=l64, mag=mag,
                           gap=gap, shw=shw, pos=pos, tile=tile, zi=zi, srgb=srgb, fmt=fmt, shadows=shadows)


def _code_bounds(dst, v, s, fmt):
    """(lo, hi) codes of the store of dst + (v -+ s), where dst is a stored value and v >= 0 a sum of terms that are
    all >= 0: an fp32 sum of such terms onto dst never falls below dst.  An infinite dst (an RGBA16F draw 1 stored
    as +inf) stays +inf whatever is added to it."""
    with np.errstate(invalid="ignore"):
        lo = np.stack([channel_code(np.maximum(dst[..., k] + v[..., k] - s[..., k], dst[..., k]), k, fmt) for k in range(3)], -1)
        hi = np.stack([channel_code(dst[..., k] + v[..., k] + s[..., k], k, fmt) for k in range(3)], -1)
    inf = np.isinf(dst)
    if inf.any():
        lo = np.where(inf, half_code(np.inf), lo)
        hi = np.where(inf, half_code(np.inf), hi)
    return lo, hi


def allowed_codes(ref):
    """(lo, hi) final codes per lit pixel and channel, (P, 3) each."""
    fmt = ref.fmt
    q_lo, q_hi = _code_bounds(ref.e, ref.d1, ref.s1, fmt)
    base_lo = np.stack([channel_value(q_lo[:, k], k, fmt) for k in range(3)], -1)
    base_hi = np.stack([channel_value(q_hi[:, k], k, fmt) for k in range(3)], -1)
    s2 = REL * (np.where(np.isinf(base_hi), base_lo, base_hi) + ref.mag) + GAP * ref.gap + ref.shw + ref.pos
    lo, _ = _code_bounds(base_lo, ref.l64, s2, fmt)
    _, hi = _code_bounds(base_hi, ref.l64, s2, fmt)
    return lo, hi


def bar_misses(got, ref):
    """Boolean (P, 3): lit pixel channels of `got` ((H, W) packed words, or (H, W, 4) RGBA16F texels) outside the bar."""
    c = codes(got[ref.ys, ref.xs], ref.fmt)
    lo, hi = allowed_codes(ref)
    return (c < lo) | (c > hi)


def assert_meets_bar(got, ref, what=""):
    """Every lit channel of the reference's rows within the float64 bar, and every sky pixel there the destination's
    bits; RGBA16F: every lit pixel
    keeps the destination's alpha bits.  Returns the share of lit channels equal to the float64 value's own store."""
    sky = ref.region & ~ref.lit
    assert got.shape == ref.emissive.shape, f"{what}: {got.shape} is not the destination's shape {ref.emissive.shape}"
    assert np.array_equal(got[sky], ref.emissive[sky]), f"{what}: sky pixels must keep the destination's value"
    if ref.fmt == RGBA16F:
        assert np.array_equal(got[ref.ys, ref.xs, 3], ref.emissive[ref.ys, ref.xs, 3]), f"{what}: alpha must keep the destination's bits"
    bad = bar_misses(got, ref)
    c = codes(got[ref.ys, ref.xs], ref.fmt)
    lo, hi = allowed_codes(ref)
    if bad.any():
        k = np.argwhere(bad)[:5]
        detail = ", ".join(f"({int(ref.xs[i])},{int(ref.ys[i])})[{j}] code {int(c[i, j])} not in [{int(lo[i, j])}, {int(hi[i, j])}]" for i, j in k)
        raise AssertionError(f"{what}: {int(bad.sum())} channels outside the float64 bar, e.g. {detail}")
    return float((lo == hi).mean()) if c.size else 1.0


def emulate(oracle, scene, cam, prep, ref, form, dt=np.float32, store="rne", shadow_variant=None):
    """The frame a kernel evaluating the BRDF with `form` in `dt` would store (draw 1, its store, draw 2, the store),
    with the reference's pairs, destination format and shadows; sky pixels keep the destination.  For checking on the
    CPU that a case discriminates between formulations.  RGBA16F stores: store "rne" (the format's rounding), "trunc"
    (toward zero) or "single" (draw 1 not stored: one rounding of the whole sum).  shadow_variant: a deliberate error
    of the samplers (shadow_factors)."""
    d, t = evaluate(scene, cam, prep, ref.pairs, ref.ys, ref.xs, ref.srgb, form, dt)
    if ref.shadows is not None and len(ref.pairs[0]):
        P64 = positions(scene.depth, cam.inv_view_projection, ref.ys, ref.xs, np.float64)[ref.pairs[0]]
        P32 = positions(scene.depth, cam.inv_view_projection, ref.ys, ref.xs, np.float32)[ref.pairs[0]]
        f = shadow_factors(oracle, prep, ref.shadows, ref.pairs[1], P64, P32, shadow_variant, dt, live=(t != 0).any(1))[0]
        t = t * f.astype(dt)[:, None]
    e = decode(ref.emissive[ref.ys, ref.xs], ref.fmt).astype(dt)
    acc = _per_pixel_sum(ref.pairs[0], t, len(ref.ys)).astype(dt)
    out = ref.emissive.copy()
    if ref.fmt == B10G11R11:
        q1 = pack((e + d).astype(np.float64))
        out[ref.ys, ref.xs] = pack((decode(q1).astype(dt) + acc).astype(np.float64))
        return out
    alpha = ref.emissive[ref.ys, ref.xs, 3]
    with np.errstate(over="ignore", invalid="ignore"):
        if store == "single":
            out[ref.ys, ref.xs] = store_f16(((e + d) + acc).astype(np.float64), alpha)
            return out
        q1 = store_f16((e + d).astype(np.float64), alpha, store)
        out[ref.ys, ref.xs] = store_f16((decode(q1, RGBA16F).astype(dt) + acc).astype(np.float64), alpha, store)
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


def _spot_rot(direction):
    """Node rotation (columns right, up, -forward) of a spot light pointing along `direction`, as synth.make_lights."""
    f = np.asarray(direction, np.float64) / np.linalg.norm(direction)
    up = np.array([0.0, 0.0, 1.0]) if abs(f[1]) > 0.9 else np.array([0.0, 1.0, 0.0])
    r = np.cross(f, up)
    r /= np.linalg.norm(r)
    return np.stack([r, np.cross(r, f), -f]).astype(np.float32)


def shadow_edge_case(oracle, res, w=256, h=144, seed=0xC0BE):
    """Shadowed lights placed for the samplers' edges, with synthetic maps of resolution res (common.make_shadow_maps,
    every light mapped).  Point lights 0.4 .. 1.2 m above the ground at positions chosen so that the direction from the
    light to one receiver has two or three equal components (a cube edge or corner direction: a major-axis tie); the
    receivers around it see the light near that edge or corner.  Point and spot lights 1.5 cm above the ground, closer
    than their shadow near plane (0.5 % of the radius) to the receivers below them: reference depths above 1.  Spot
    lights pointing down, whose footprints at the rim of the cone reach past the map's edge.  Returns (scene, cam,
    lights, prep, clus, transforms, maps)."""
    from granite_b200 import synth
    from tests import common

    scene = synth.make_scene(w, h)
    cam = oracle.camera_setup(scene.projection, scene.view)
    rng = np.random.default_rng(seed)
    ground = [(y, x) for y in range(h // 2 + 6, h - 4, 5) for x in range(8, w - 8, 7)
              if scene.depth[y, x] != 0 and abs(scene.world_pos[y, x, 1] + 2.0) < 1e-6]
    pick = rng.choice(len(ground), 40, replace=False)
    pos, is_point, rot = [], [], []
    for n, k in enumerate(pick):
        y, x = ground[k]
        P = positions(scene.depth, cam.inv_view_projection, np.array([y]), np.array([x]), np.float64)[0]
        hgt = rng.uniform(0.4, 1.2)
        sx, sz = rng.choice([-1.0, 1.0], 2)
        if n < 24:  # P - light = hgt (sx, -1, sz): a corner direction; or hgt (sx, -1, 0.3 sz): an edge direction
            d = hgt * np.array([sx, -1.0, sz if n % 2 == 0 else 0.3 * sz])
            pos.append(P - d)
            is_point.append(True)
            rot.append(np.eye(3, dtype=np.float32))
        elif n < 30:
            pos.append(P + np.array([0.0, 0.015, 0.0]))
            is_point.append(n % 2 == 0)
            rot.append(_spot_rot((0.0, -1.0, 0.0)))
        else:
            pos.append(P + np.array([rng.uniform(-0.5, 0.5), hgt, rng.uniform(-0.5, 0.5)]))
            is_point.append(False)
            rot.append(_spot_rot((rng.uniform(-0.3, 0.3), -1.0, rng.uniform(-0.3, 0.3))))
    pos = np.asarray(pos, np.float32)
    order = np.argsort(-pos[:, 2], kind="stable")  # front to back, as the clusterer expects
    n = len(pos)
    col = rng.uniform(1.0, 3.0, (n, 3)).astype(np.float32)
    lights = synth.Lights(col[order], pos[order], np.asarray(is_point)[order], np.asarray(rot, np.float32)[order],
                          np.full(n, 0.9, np.float32), np.full(n, 0.7, np.float32))
    prep = oracle.prepare_lights(cam, lights, res=synth.CLUSTER_RES, cull=False)
    clus = oracle.cluster_build(cam, prep)
    transforms = oracle.shadow_transforms(prep)
    maps = common.make_shadow_maps(prep, res, skip_every=0)
    return scene, cam, lights, prep, clus, transforms, maps


def fp16_overflow_case(oracle, w=256, h=144, n=300):
    """RGBA16F stores that reach +inf: the emissive's red is 65504 (the largest fp16 value, half a code below the
    +inf threshold 65520 by 16) and its green 65472 (one code below); a bright directional light (draw 1 adds more
    than 16 where it faces the light) and bright point lights (draw 2 adds more than 16 near them).  Returns (scene,
    cam, prep, clus, emissive16)."""
    from tests import common

    scene, cam, lights, _ = common.build_case(oracle, w, h, 0)
    from granite_b200 import synth

    lights = synth.make_lights(n, aspect=w / h)
    lights.color *= np.float32(40.0)
    scene.dir_color = (60.0, 30.0, 1.0)
    prep = oracle.prepare_lights(cam, lights, res=synth.CLUSTER_RES)
    em = common.random_hdr_f16(np.random.default_rng(0xF16), w, h, scale=0.02, hot=0.0)
    em[..., 0] = np.float16(65504.0).view(np.uint16)
    em[..., 1] = np.float16(65472.0).view(np.uint16)
    return scene, cam, prep, oracle.cluster_build(cam, prep), em


def fp16_subnormal_case(oracle, w=256, h=144, n=300):
    """RGBA16F stores that stay fp16 subnormal (below 2^-14): directional colour 0; black metallic surfaces (albedo
    sRGB code 0, metallic 1), so that the ambient and the diffuse term are 0 and each light adds only its Fresnel
    reflection; point lights of colour 0.05 .. 0.2 (radii of about a metre) that reach the ground from 0.5 .. 3 m; and
    an emissive of random subnormals.  Returns (scene, cam, prep, clus, emissive16)."""
    from granite_b200 import synth

    scene = synth.make_scene(w, h)
    cam = oracle.camera_setup(scene.projection, scene.view)
    rng = np.random.default_rng(0x5B)
    scene.albedo[:] = 0xFF000000
    scene.pbr = (scene.pbr & np.uint16(0xFF00)) | np.uint16(255)
    scene.dir_color = (0.0, 0.0, 0.0)
    lights = synth.make_lights(n, aspect=w / h)
    lights.color = rng.uniform(0.05, 0.2, lights.color.shape).astype(np.float32)
    prep = oracle.prepare_lights(cam, lights, res=synth.CLUSTER_RES, cull=False)
    em = np.zeros((h, w, 4), np.uint16)
    em[..., :3] = rng.integers(0, 64, (h, w, 3))  # subnormal codes (value code * 2^-24)
    em[..., 3] = np.float16(1.0).view(np.uint16)
    return scene, cam, prep, oracle.cluster_build(cam, prep), em
