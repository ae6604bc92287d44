"""The light clusterer (grb_cluster.cu) at the launch shapes the default view never reaches, and the cluster it builds
checked for coverage in float64, independently of the oracle.

Bit for bit with the oracle: light counts whose 32-light words end partly filled and whose word count leaves every
remainder of the binning's four warps per CTA, and counts past K4's 2048-range staging round; tile grids with odd
block counts and Z resolutions below and off multiples of 32; grb_cluster_z_range on synthetic range lists with
sentinel, inverted and edge ranges; grb_cluster_binning_rows on ragged and inverted tile-row ranges.

Coverage (tests/cluster_cases.py): on every geometry case, every (pixel, light) pair whose falloff is nonzero by a
float64 brute-force count is in the GPU cluster's list for the pixel, with the pixel's tile and slice taken from
grb_debug_cluster_indices.  End to end, the persistent lighting pass on the GPU's own cluster meets the float64 bar
with the brute-force pairs in place of any cluster's."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import cluster_cases as CC
from tests import lighting_ref64 as R

pytestmark = pytest.mark.gpu

SENTINEL = 0x5EA5EA5E


def _device(cam, prep):
    from granite_b200 import harness

    dev = harness.ClusterDevice(prep.records, prep.model, prep.type_mask, prep.z_ranges, prep.params, prep.res)
    gcam = harness.camera_struct(cam)
    dev.build(gcam)
    torch.cuda.synchronize()
    return dev, gcam


@pytest.mark.parametrize("n", [0, 1, 31, 33, 65, 97, 2049, 4097])
def test_light_counts(cuda, oracle, n):
    """n % 32 != 0 leaves a partly filled last word (its bits at or above num_lights must be 0); num_lights_32 % 4 =
    1, 2, 3, 0 for 1, 33, 65, 97 lights; 2049 and 4097 lights end K4's staging in a partial round.  Zero lights: the
    one (~0u, 0) range entry, and every slice empty."""
    _, cam, prep = CC.count_case(oracle, n)
    assert prep.n == n
    ref = oracle.cluster_build(cam, prep)
    dev, _ = _device(cam, prep)
    got = dev.download()
    CC.assert_cluster_equal(got, ref, prep)
    if n == 0:
        assert prep.z_ranges.tolist() == [[0xFFFFFFFF, 0]]
        assert (got.range[:, 0] == 0xFFFFFFFF).all() and (got.range[:, 1] == 0).all()
    else:
        assert got.bitmask.any() and (got.range[:, 0] != 0xFFFFFFFF).any()


@pytest.mark.parametrize("res", [(8, 4, 1), (16, 8, 33), (136, 68, 100), (128, 64, 4096)], ids=lambda r: "x".join(map(str, r)))
@pytest.mark.parametrize("name", ["turned", "finite-far"])
def test_grids(cuda, oracle, name, res):
    """Tile grids of one block, of odd block counts (17 x 17 blocks of 8 x 4 tiles), and Z resolutions of 1, 33 and
    100 slices: K1-K4 and each pixel's (tile, slice) bit for bit."""
    scene, cam, _, prep = CC.build(oracle, name, res=res, check=False)
    ref = oracle.cluster_build(cam, prep)
    dev, _ = _device(cam, prep)
    CC.assert_cluster_equal(dev.download(), ref, prep)
    _, tile, zi, _ = oracle.deferred_lighting(scene, cam, prep, ref, want_indices=True)
    got_t, got_z = CC.debug_cluster_indices(cam, prep, scene.depth)
    assert np.array_equal(got_t, tile) and np.array_equal(got_z, zi)


def _synthetic_ranges(rng, num, res_z):
    """Light slice ranges as the host makes them, and the forms around them: random spans, sentinels (culled lights),
    inverted ranges (lo > hi), the inverted form of a light beyond the last slice (lo > res_z - 1, hi = res_z - 1),
    ranges touching slices 0 and res_z - 1, and a band of slices no range touches."""
    lo = rng.integers(0, res_z, num)
    hi = np.minimum(lo + rng.integers(0, max(res_z // 8, 1) + 1, num), res_z - 1)
    z = np.stack([lo, hi], -1).astype(np.int64)
    kind = rng.integers(0, 10, num)
    z[kind == 0] = (0xFFFFFFFF, 0)
    inv = kind == 1
    z[inv] = np.stack([z[inv, 1] + 1 + rng.integers(0, 5, int(inv.sum())), z[inv, 0]], -1)
    beyond = kind == 2
    z[beyond] = np.stack([res_z + rng.integers(0, 50, int(beyond.sum())), np.full(int(beyond.sum()), res_z - 1)], -1)
    z[kind == 3, 0] = 0
    z[kind == 4, 1] = res_z - 1
    if res_z >= 8:  # slices [res_z // 3, res_z // 3 + 3) touched by nothing
        gap0, gap1 = res_z // 3, res_z // 3 + 3
        normal = (z[:, 0] <= z[:, 1]) & (z[:, 0] < gap1) & (z[:, 1] >= gap0)
        z[normal & (z[:, 0] >= gap0), 0] = gap1
        z[normal & (z[:, 0] < gap0), 1] = gap0 - 1
        z[normal & (z[:, 0] > z[:, 1])] = (0xFFFFFFFF, 0)
    if res_z >= 96:  # K4's third 32-slice segment, [64, 96), touched by one range and only at its last slice
        normal = (z[:, 0] <= z[:, 1]) & (z[:, 0] < 96) & (z[:, 1] >= 64)
        z[normal & (z[:, 0] >= 64), 0] = 96
        z[normal & (z[:, 0] < 64), 1] = 63
        z[normal & (z[:, 0] > z[:, 1])] = (0xFFFFFFFF, 0)
        z[num // 2] = (95, 95)
    return np.ascontiguousarray(np.clip(z, 0, 0xFFFFFFFF).astype(np.uint32))


@pytest.mark.parametrize("res_z", [1, 31, 33, 4096])
@pytest.mark.parametrize("num", [1, 2047, 2048, 2049, 6000])
def test_z_range_on_synthetic_ranges(cuda, oracle, num, res_z):
    """grb_cluster_z_range bit for bit with the oracle's per-slice scan; nothing past slice res_z - 1 is written."""
    from granite_b200 import capi, harness

    rng = np.random.default_rng(num * 7 + res_z)
    z = _synthetic_ranges(rng, num, res_z)
    ref = np.zeros((res_z, 2), np.uint32)
    oracle.lib().orc_z_range(z.ctypes.data_as(C.c_void_p), num, res_z, ref.ctypes.data_as(C.c_void_p))
    z_t = harness.to_dev(z)
    out = torch.full((res_z + 40, 2), SENTINEL, dtype=torch.int32, device="cuda")
    b = capi.GrbClusterBuffers()
    b.z_ranges, b.cluster_range, b.resolution_z = z_t.data_ptr(), out.data_ptr(), res_z
    capi.check(capi.lib().grb_cluster_z_range(C.byref(b), num, capi.stream_ptr()), "grb_cluster_z_range")
    got = harness.to_host(out, np.uint32)
    assert np.array_equal(got[:res_z], ref)
    assert (got[res_z:] == SENTINEL).all()
    if res_z >= 8 and num > 1:
        assert (ref[res_z // 3:res_z // 3 + 3, 0] == 0xFFFFFFFF).all() and (ref[:, 0] != 0xFFFFFFFF).any()
    if res_z >= 96:
        assert (ref[64:95, 0] == 0xFFFFFFFF).all() and ref[95].tolist() == [num // 2, num // 2]


@pytest.mark.parametrize("res", [(128, 64, 4096), (136, 68, 100)], ids=lambda r: "x".join(map(str, r)))
def test_binning_rows(cuda, oracle, res):
    """grb_cluster_binning_rows on ragged tile-row ranges: the block rows [4 floor(y0 / 4), 4 ceil(min(y1, res_y) / 4))
    equal the whole build's, every other row keeps its fill; an inverted range means every row, a range starting at
    res_y none."""
    from granite_b200 import capi, harness

    _, cam, _, prep = CC.build(oracle, "turned", res=res, check=False)
    dev, _ = _device(cam, prep)
    full = dev.download().bitmask
    ry = res[1]
    for y0, y1 in ((5, 9), (ry - 1, ry), (3, ry + 7), (ry, ry + 4), (9, 5)):
        bm = torch.full_like(dev.bitmask, SENTINEL)
        b = capi.GrbClusterBuffers.from_buffer_copy(dev.buffers)
        b.bitmask = bm.data_ptr()
        capi.check(capi.lib().grb_cluster_binning_rows(C.byref(dev.params), C.byref(b), y0, y1, capi.stream_ptr()), "grb_cluster_binning_rows")
        got = harness.to_host(bm, np.uint32)
        r0, r1 = (0, ry) if y1 <= y0 else (4 * (y0 // 4), 4 * -(-min(y1, ry) // 4))
        assert np.array_equal(got[r0:r1], full[r0:r1]), (y0, y1)
        assert (got[:r0] == SENTINEL).all() and (got[r1:] == SENTINEL).all(), (y0, y1)


_CASES = {}


def _gpu_case(oracle, name):
    """(scene, cam, prep, device cluster, gcam, GPU tile, GPU slice), built once per case."""
    if name not in _CASES:
        scene, cam, _, prep = CC.build(oracle, name)
        dev, gcam = _device(cam, prep)
        tile, zi = CC.debug_cluster_indices(cam, prep, scene.depth)
        _CASES[name] = (scene, cam, prep, dev, gcam, tile, zi)
    return _CASES[name]


@pytest.mark.parametrize("name", list(CC.CASES))
def test_gpu_cluster_covers_every_lit_pair(cuda, oracle, name):
    scene, cam, prep, dev, gcam, tile, zi = _gpu_case(oracle, name)
    got = dev.download()
    cov = CC.coverage(scene, cam, prep, got.bitmask, got.range, tile, zi)
    print(f"{name}: {cov.pairs} pairs, {cov.borderline} borderline, {cov.borderline_missed} borderline missed")
    CC.assert_covers(cov, name)


@pytest.mark.parametrize("name", ["turned", "spots-at-eye"])
def test_lighting_on_the_gpu_cluster_meets_the_brute_force_bar(cuda, oracle, name):
    """The persistent lighting pass on the GPU's cluster: a dropped light, a wrong (tile, slice) or an off Z range
    changes stored codes against the float64 frame of the brute-force pairs."""
    from granite_b200 import harness

    scene, cam, prep, dev, gcam, tile, zi = _gpu_case(oracle, name)
    gb = harness.GBufferDevice(scene)
    hdr = gb.emissive.clone()
    harness.deferred_lighting(gb, gcam, dev, hdr)
    ref = R.reference(oracle, scene, cam, prep, None, pairs=CC.lighting_pairs(scene, cam, prep))
    R.assert_meets_bar(harness.to_host(hdr, np.uint32), ref, name)
