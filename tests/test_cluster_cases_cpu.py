"""The clusterer's geometry cases (tests/cluster_cases.py) on the CPU oracle: each case reaches the branches it exists
for, the oracle's cluster covers every (pixel, light) pair whose falloff is nonzero by the float64 brute-force count,
the oracle's frame meets the float64 lighting bar with those brute-force pairs in place of the cluster's, and the
coverage check fails on a cluster that lacks one needed bit or one slice of a range."""
import math

import numpy as np
import pytest

from granite_b200 import synth
from tests import cluster_cases as CC
from tests import lighting_ref64 as R

_CACHE = {}


def _case(oracle, name):
    """(scene, cam, prep, oracle cluster, tile, zi), computed once per case."""
    if name not in _CACHE:
        scene, cam, _, prep = CC.build(oracle, name)
        clus = oracle.cluster_build(cam, prep)
        _, tile, zi, _ = oracle.deferred_lighting(scene, cam, prep, clus, want_indices=True)
        _CACHE[name] = (scene, cam, prep, clus, tile, zi)
    return _CACHE[name]


@pytest.mark.parametrize("name", list(CC.CASES))
def test_case_reaches_its_branches(oracle, name):
    scene, cam, prep, clus, tile, zi = _case(oracle, name)
    got = CC.branches(cam, prep, clus)
    assert all(got[b] > 0 for b in CC.CASES[name]), got
    # every case keeps sky pixels and pixels right at the near plane, and sees lights of both kinds
    assert (scene.depth == 0).any() and (scene.depth == 1.0).any()
    assert got["points"] > 0 and got["spots"] > 0


@pytest.mark.parametrize("name", list(CC.CASES))
def test_oracle_cluster_covers_every_lit_pair(oracle, name):
    scene, cam, prep, clus, tile, zi = _case(oracle, name)
    cov = CC.coverage(scene, cam, prep, clus.bitmask, clus.range, tile, zi)
    print(f"{name}: {cov.pairs} pairs, {cov.borderline} borderline, {cov.borderline_missed} borderline missed")
    CC.assert_covers(cov, name)


@pytest.mark.parametrize("name", ["turned", "spots-at-eye"])
def test_oracle_frame_meets_the_bar_with_brute_force_pairs(oracle, name):
    scene, cam, prep, clus, tile, zi = _case(oracle, name)
    frame = oracle.deferred_lighting(scene, cam, prep, clus)
    ref = R.reference(oracle, scene, cam, prep, None, pairs=CC.lighting_pairs(scene, cam, prep))
    R.assert_meets_bar(frame, ref, name)


def test_coverage_check_has_teeth(oracle):
    """One needed bit cleared, or one slice's range shortened by one light: the check reports a missed pair."""
    scene, cam, prep, clus, tile, zi = _case(oracle, "turned")
    cov = CC.coverage(scene, cam, prep, clus.bitmask, clus.range, tile, zi)
    assert cov.missed == 0
    solid = np.nonzero(cov.ok)[0]
    # a bit: the light of one covered pair, cleared in that pixel's tile
    k = solid[len(solid) // 2]
    y, x, light = cov.ys[cov.pix[k]], cov.xs[cov.pix[k]], cov.light[k]
    bitmask = clus.bitmask.copy()
    bitmask.reshape(-1, prep.n32)[tile[y, x], light >> 5] &= ~np.uint32(1 << (light & 31))
    assert CC.coverage(scene, cam, prep, bitmask, clus.range, tile, zi).missed >= 1
    # a range: a slice whose last light reaches one of its pixels, ended one light earlier
    z = zi[cov.ys[cov.pix[solid]], cov.xs[cov.pix[solid]]]
    last = cov.light[solid] == clus.range[z, 1].astype(np.int64)
    assert last.any()
    crange = clus.range.copy()
    crange[z[np.nonzero(last)[0][0]], 1] -= 1
    assert CC.coverage(scene, cam, prep, clus.bitmask, crange, tile, zi).missed >= 1


def test_pixels_beyond_the_z_grid_lose_lights_beyond_it(oracle):
    """The Z slices end at res_z * extent (2048 m at the default grid).  compute_uint_range (clusterer.cpp:1265-1275)
    clamps only the high end of a light's slice range, so a light entirely beyond the last slice gets an inverted range
    (lo > res_z - 1, hi = res_z - 1) that no slice contains; pixels beyond the grid clamp into the last slice and lose
    that light.  This is the reference's behaviour, and the shaders' bit-exactness with it keeps it: the coverage
    check leaves those pixels out (coverage's max_depth).  Here they are kept, and exactly those pairs are missed."""
    w, h = 64, 32
    proj = synth.perspective_inf(math.radians(0.5), w / h, CC.NEAR)  # 17 m across at 2 km: the lights reach most pixels
    view = synth.look_at_view((0.0, 0.0, 8.0), (0.0, 0.0, 0.0))
    rng = np.random.default_rng(3)
    scene = CC.random_scene(rng, w, h, proj, view, 10.0)
    z = rng.uniform(1990.0, 2130.0, (h, w))
    scene.depth[:] = np.where(scene.depth == 0, 0.0, CC.ndc_depth(proj, z)).astype(np.float32)
    cam = oracle.camera_setup(proj, view)
    L = CC._Lights()
    for depth in (2010.0, 2040.0, 2090.0, 2110.0):  # straddling the grid's end, and entirely beyond it
        L.add((0.0, 0.0, 8.0 - depth), 40.0 if depth < 2080.0 else 25.0, True)
    prep = oracle.prepare_lights(cam, L.build(np.array([0.0, 0.0, -1.0])))
    assert prep.n == 4 and CC.grid_depth(prep, cam) == 2048.0
    beyond = prep.z_ranges[:, 0] > prep.res[2] - 1
    assert beyond.tolist() == [False, False, True, True] and (prep.z_ranges[beyond, 1] == prep.res[2] - 1).all()
    clus = oracle.cluster_build(cam, prep)
    _, tile, zi, _ = oracle.deferred_lighting(scene, cam, prep, clus, want_indices=True)
    assert CC.coverage(scene, cam, prep, clus.bitmask, clus.range, tile, zi).missed == 0
    cov = CC.coverage(scene, cam, prep, clus.bitmask, clus.range, tile, zi, max_depth=np.inf)
    P = R.positions(scene.depth, cam.inv_view_projection, cov.ys[cov.pix], cov.xs[cov.pix], np.float64)
    pix_beyond = 8.0 - P[:, 2] >= 2048.0
    want_missed = pix_beyond & beyond[cov.light]
    assert want_missed.sum() > 100
    assert np.array_equal(~cov.ok, want_missed)
