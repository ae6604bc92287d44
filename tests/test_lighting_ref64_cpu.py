"""The float64 lighting reference (tests/lighting_ref64.py) pinned on the CPU: the fp32 oracle meets its bar, its
store matches the B10G11R11 store, and the grazing and dense cases of the GPU lighting tests reach what they claim."""
import numpy as np
import pytest

from granite_b200 import synth
from tests import common
from tests import lighting_ref64 as R


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
