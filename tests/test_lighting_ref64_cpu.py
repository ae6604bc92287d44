"""The float64 lighting reference (tests/lighting_ref64.py) pinned on the CPU: the fp32 oracle meets its bar, in both
destination formats and with shadowed lights; its stores match the B10G11R11 and RGBA16F stores; each deliberate error
of a store or a shadow sampler misses the bar on the case named for it; and the cases of the GPU lighting tests reach
what they claim."""
import numpy as np
import pytest

from granite_b200 import synth
from tests import common
from tests import lighting_ref64 as R
from tests.kernel_forms_worker import LIGHTING_CASE
from tests.test_oracle_ref_light_shadows import shadow_case


def test_codes_are_the_store():
    rng = np.random.default_rng(11)
    v = np.concatenate([rng.uniform(0.0, 1.0, 4000) ** 6 * 70000.0, rng.uniform(0.0, 1e-4, 1000), [0.0, 2.0 ** -14, 65024.0, 1e9]])
    rgb = np.stack([v, v[::-1], np.roll(v, 7)], -1).astype(np.float32)
    want = synth.pack_r11g11b10(rgb)
    assert np.array_equal(R.pack(rgb.astype(np.float64)), want)
    assert np.array_equal(R.pack(R.decode(want)), want), "decoded codes store to themselves"


@pytest.mark.parametrize("case", ["C1-256x256-16pt", "small-300-25pct-spots", "dense-256x144"])
def test_oracle_meets_the_float64_bar(oracle, case):
    if case == "dense-256x144":
        scene, cam, _, prep = R.dense_case(oracle)
    else:
        w, h, n, spots = {"C1-256x256-16pt": (256, 256, 16, 0.0), "small-300-25pct-spots": (640, 360, 300, 0.25)}[case]
        scene, cam, _, prep = common.build_case(oracle, w, h, n, spots)
    clus = oracle.cluster_build(cam, prep)
    got, tile, zi, _ = oracle.deferred_lighting(scene, cam, prep, clus, want_indices=True)
    ref = R.reference(oracle, scene, cam, prep, clus, (tile, zi))
    R.assert_meets_bar(got, ref, f"oracle {case}")
    lo, hi = R.allowed_codes(ref)
    assert (hi > lo).mean() < 0.01, "away from code boundaries the bar admits one code"


def test_grazing_case_discriminates(oracle):
    """The half vector from |V+L|^2 = 2 + 2 V.L, evaluated in fp32, misses the bar at most of the grazing pixels;
    the explicit h = V + L of the persistent kernel meets it everywhere."""
    scene, cam, _, prep, mask, angle = R.grazing_case(oracle)
    assert mask.sum() >= 40 and 0.005 < np.nanmin(angle) and np.nanmax(angle) < 0.035
    clus = oracle.cluster_build(cam, prep)
    got, tile, zi, _ = oracle.deferred_lighting(scene, cam, prep, clus, want_indices=True)
    ref = R.reference(oracle, scene, cam, prep, clus, (tile, zi))
    R.assert_meets_bar(got, ref, "oracle, grazing")
    R.assert_meets_bar(R.emulate(oracle, scene, cam, prep, ref, "h"), ref, "explicit h, fp32")
    patch = mask[ref.ys, ref.xs]
    miss = R.bar_misses(R.emulate(oracle, scene, cam, prep, ref, "vol"), ref).any(1)
    assert miss[patch].mean() > 0.3, f"2 + 2 V.L misses only {int(miss[patch].sum())} of {int(patch.sum())} grazing pixels"


def test_dense_case_reaches_batching(oracle):
    """Some 16x4 blocks of the dense case keep more than one list batch (160 entries) of lights after the box test,
    and some of those batches have an odd length (padded with the dummy record)."""
    scene, cam, _, prep = R.dense_case(oracle)
    clus = oracle.cluster_build(cam, prep)
    _, _, zi, _ = oracle.deferred_lighting(scene, cam, prep, clus, want_indices=True)
    batches = R.block_batches(scene, cam, prep, clus, zi)
    several = [b for b in batches.values() if len(b) > 1]
    assert len(several) >= 10 and max(sum(b) for b in several) > 160
    assert any(x % 2 for b in several for x in b)


def test_half_codes_are_the_store():
    """half_code of float64 values is the RGBA16F store (RNE, subnormals, >= 65520 -> +inf) of their fp32 values."""
    rng = np.random.default_rng(12)
    v = np.concatenate([rng.uniform(0.0, 1.0, 4000) ** 8 * 70000.0, rng.uniform(0.0, 2.0 ** -13, 2000),
                        [0.0, 2.0 ** -25, 3 * 2.0 ** -25, 2.0 ** -14, 65504.0, 65519.996, 65520.0, 1e9]]).astype(np.float32)
    with np.errstate(over="ignore"):
        want = v.astype(np.float16).view(np.uint16).astype(np.int64)
    assert np.array_equal(R.half_code(v.astype(np.float64)), want)
    assert R.half_code(65519.996) == 0x7BFF and R.half_code(65520.0) == 0x7C00 and R.half_code(3 * 2.0 ** -25) == 2
    assert np.array_equal(R.half_code(R.half_value(want)), want), "decoded codes store to themselves"
    t = R.store_f16(np.stack([v, v, v], -1).astype(np.float64), np.zeros(len(v)), "trunc")[:, 0].astype(np.int64)
    assert (R.half_value(t) <= v).all() and ((t == want) | (t == want - 1)).all()


def _fp16_case(oracle, name):
    if name == "dense-256x144":
        scene, cam, _, prep = R.dense_case(oracle)
    elif name == "grazing-640x360":
        scene, cam, _, prep, _, _ = R.grazing_case(oracle)
    else:
        w, h, n, spots = {"small-640x360": LIGHTING_CASE, "C1-256x256": (256, 256, 16, 0.0)}[name]
        scene, cam, _, prep = common.build_case(oracle, w, h, n, spots)
    h, w = scene.depth.shape
    em = common.random_hdr_f16(np.random.default_rng(w + prep.n), w, h, scale=0.02, hot=0.001)
    return scene, cam, prep, oracle.cluster_build(cam, prep), em


def _wide_share(ref):
    lo, hi = R.allowed_codes(ref)
    return float((hi > lo).mean())


@pytest.mark.parametrize("case", ["small-640x360", "C1-256x256", "dense-256x144", "grazing-640x360"])
def test_oracle_fp16_meets_the_float64_bar(oracle, case):
    """The oracle's RGBA16F frames meet the bar, which admits more than one code on under 10 % of the lit channels
    (6 - 9 % on these cases: an fp16 code is 8x finer than a B10G11R11 one).  A truncating store and a single store of
    the whole sum (no rounding of draw 1) both miss it."""
    scene, cam, prep, clus, em = _fp16_case(oracle, case)
    ref = R.reference(oracle, scene, cam, prep, clus, emissive=em, fmt=R.RGBA16F)
    R.assert_meets_bar(oracle.deferred_lighting_fp16(scene, cam, prep, clus, em), ref, f"oracle fp16 {case}")
    share = _wide_share(ref)
    print(f"{case}: the bar admits more than one code on {share:.4f} of the lit channels")
    assert share < 0.10
    R.assert_meets_bar(R.emulate(oracle, scene, cam, prep, ref, "ref"), ref, "fp32 emulation with the RNE store")
    for store in ("trunc", "single"):
        assert R.bar_misses(R.emulate(oracle, scene, cam, prep, ref, "ref", store=store), ref).any(), f"{store} store meets the bar"


def test_fp16_overflow_case_reaches_inf(oracle):
    """The overflow case stores +inf from draw 1 on some pixels and only from draw 2 on others; the oracle meets the
    bar there, and the truncating store (65504 instead of +inf) misses it."""
    scene, cam, prep, clus, em = R.fp16_overflow_case(oracle)
    ref = R.reference(oracle, scene, cam, prep, clus, emissive=em, fmt=R.RGBA16F)
    got = oracle.deferred_lighting_fp16(scene, cam, prep, clus, em)
    R.assert_meets_bar(got, ref, "oracle fp16 overflow")
    inf = R.half_code(np.inf)
    q_lo, _ = R._code_bounds(ref.e, ref.d1, ref.s1, R.RGBA16F)
    lo, hi = R.allowed_codes(ref)
    draw1 = (q_lo == inf).any(1)
    draw2 = (lo == inf).any(1) & ~draw1
    print(f"draw 1 stores +inf on {int(draw1.sum())} pixels, draw 2 on {int(draw2.sum())} more; finite: {int((hi < inf).all(1).sum())}")
    assert draw1.sum() >= 3 and draw2.sum() >= 50 and (hi < inf).all(1).sum() > 0.9 * len(ref.ys)
    assert R.bar_misses(R.emulate(oracle, scene, cam, prep, ref, "ref", store="trunc"), ref).any()


def test_fp16_subnormal_case_stays_subnormal(oracle):
    """The dim case's stores are fp16 subnormals (nonzero codes below 0x400) on over 95 % of the lit channels (98 %
    measured: the brightest Fresnel peaks leave the subnormal range); the oracle meets
    the bar there, and the truncating store misses it."""
    scene, cam, prep, clus, em = R.fp16_subnormal_case(oracle)
    ref = R.reference(oracle, scene, cam, prep, clus, emissive=em, fmt=R.RGBA16F)
    got = oracle.deferred_lighting_fp16(scene, cam, prep, clus, em)
    R.assert_meets_bar(got, ref, "oracle fp16 subnormal")
    c = R.codes(got[ref.ys, ref.xs])
    assert ((c > 0) & (c < 0x400)).mean() > 0.95
    assert len(ref.pairs[0]) > 200 and (ref.l64 > 0).any(), "the dim lights must reach the receivers"
    assert R.bar_misses(R.emulate(oracle, scene, cam, prep, ref, "ref", store="trunc"), ref).any()


SHADOW_CASES = {"narrow-160x96-res32": ((160, 96, 300, 0.25, 32), False), "wide-320x180-res64": ((320, 180, 300, 0.6, 64), True),
                "spot-edge-narrow-res8": ((320, 180, 300, 1.0, 8), False), "spot-edge-wide-res8": ((320, 180, 300, 1.0, 8), True),
                "cube-res3": (3, False), "cube-res48": (48, False)}
# the deliberate sampler error each case must reject
SHADOW_VARIANTS = {"narrow-160x96-res32": ["no-half-texel"], "wide-320x180-res64": ["wide-unnormalised"],
                   "spot-edge-narrow-res8": ["no-half-texel"], "spot-edge-wide-res8": ["origin-clamp", "wide-unnormalised"],
                   "cube-res3": ["corner-zero", "edge-clamp"], "cube-res48": ["corner-zero", "edge-clamp"]}


def shadowed_case(oracle, name):
    """(scene, cam, prep, clus, shadows) of a named shadow case: shadow_case's narrow and wide PCF cases; the spot-edge
    cases, spot lights only with 8 x 8 maps of independent texels (no two neighbours alike, so a footprint that
    reaches past the map's edge and is clamped wrongly reads other depths); or R.shadow_edge_case at a cube
    resolution."""
    args, wide = SHADOW_CASES[name]
    if name.startswith("cube"):
        scene, cam, _, prep, clus, transforms, maps = R.shadow_edge_case(oracle, args)
        return scene, cam, prep, clus, (transforms, maps, args, False)
    scene, cam, prep, clus, transforms, maps = shadow_case(oracle, *args)
    if name.startswith("spot-edge"):
        maps = common.make_shadow_maps(prep, args[-1], block=1)
    return scene, cam, prep, clus, (transforms, maps, args[-1], wide)


@pytest.mark.parametrize("fmt", [R.B10G11R11, R.RGBA16F])
@pytest.mark.parametrize("case", list(SHADOW_CASES))
def test_oracle_shadowed_meets_the_float64_bar(oracle, case, fmt):
    """The oracle's shadowed frames meet the bar with the float64 shadow factor, which admits more than one code on
    under 1 % (B10G11R11) / 10 % (RGBA16F) of the lit channels; each case's deliberate sampler error misses it."""
    scene, cam, prep, clus, shadows = shadowed_case(oracle, case)
    st = R.ShadowStats()
    if fmt == R.RGBA16F:
        h, w = scene.depth.shape
        em = common.random_hdr_f16(np.random.default_rng(w + prep.n), w, h, scale=0.02, hot=0.001)
        got = oracle.deferred_lighting_fp16(scene, cam, prep, clus, em, shadows=shadows)
    else:
        em = scene.emissive
        got = oracle.deferred_lighting_shadowed(scene, cam, prep, clus, *shadows[:3], pcf_wide=shadows[3])
    ref = R.reference(oracle, scene, cam, prep, clus, emissive=em, fmt=fmt, shadows=shadows, stats=st)
    R.assert_meets_bar(got, ref, f"oracle shadowed {case} {fmt}")
    share = _wide_share(ref)
    print(f"{case} {fmt}: the bar admits more than one code on {share:.4f} of the lit channels; "
          f"{st.ambiguous} of {st.pairs} shadowed pairs have an ambiguous comparison")
    assert share < (0.01 if fmt == R.B10G11R11 else 0.10)
    assert st.pairs > 500
    for v in SHADOW_VARIANTS[case]:
        assert R.bar_misses(R.emulate(oracle, scene, cam, prep, ref, "ref", shadow_variant=v), ref).any(), f"{v} meets the bar"
    R.assert_meets_bar(R.emulate(oracle, scene, cam, prep, ref, "ref"), ref, "fp32 emulation of the samplers")


@pytest.mark.parametrize("res", [3, 48])
def test_shadow_edge_case_reaches_its_paths(oracle, res):
    """From the geometry, counted over the pairs the kernels sample (nonzero unshadowed term): cube footprints that
    step over a face edge, three-texel corners, major-axis ties, and reference depths above 1 (clamped); the spot-edge
    cases reach footprints (2 x 2 and 6 x 6) past the map's edge.  A reference depth below 0 lies beyond the light's radius, where the
    falloff is 0 and nothing is sampled."""
    scene, cam, prep, clus, shadows = shadowed_case(oracle, f"cube-res{res}")
    st = R.ShadowStats()
    R.reference(oracle, scene, cam, prep, clus, shadows=shadows, stats=st)
    print(f"cube res {res}: {st}")
    assert st.edge >= (10000 if res == 3 else 1000) and st.corner >= (1000 if res == 3 else 10) and st.tie >= 100 and st.ref_hi >= 3
    for case in ("spot-edge-narrow-res8", "spot-edge-wide-res8"):
        scene, cam, prep, clus, shadows = shadowed_case(oracle, case)
        st = R.ShadowStats()
        R.reference(oracle, scene, cam, prep, clus, shadows=shadows, stats=st)
        print(f"{case}: {st}")
        assert st.outside >= (300 if "wide" in case else 100) and st.ref_lo == 0
