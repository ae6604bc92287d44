"""Row-sharded frames on CPU: world_size-2 (and emulated 4/8) runs of the multi-GPU protocol with
`gloo` collectives and the oracle standing in for the kernels.  What is under test is the HOST
logic the GPUs rely on: the band partition, the per-stage row plan (granite_b200/host/shard_plan.cpp,
through its C entry point), the all-gather of 1/4-res bloom bands and the zero-padded all-reduce
that assembles the luminance grid exactly.  A plan with a halo one row too small would leak
never-computed (zero) rows into a band and break the bit-equality asserted here."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import common

W, H, N_LIGHTS = 512, 384, 64  # 6 bands of 64 rows


def _reference_frame(oracle, scene, cam, prep):
    clus = oracle.cluster_build(cam, prep)
    hdr = oracle.deferred_lighting(scene, cam, prep, clus)
    lum0 = np.array([0.2, 2 ** 0.2, 2 ** -0.2], np.float32)
    f = oracle.hdr_chain(hdr, lum0, None)
    ldr_fxaa = oracle.fxaa(f.ldr, True)
    return clus, hdr, lum0, f, ldr_fxaa


def _sharded_rank(rank, world, bands, fxaa, gather_fn, reduce_fn):
    """One rank's frame.  Everything outside the planned rows is left ZERO on purpose."""
    from granite_b200 import synth, viewer
    from oracle import pyoracle as oracle
    from tests import common

    scene, cam, lights, prep = common.build_case(oracle, W, H, N_LIGHTS, 0.25)
    plan = viewer.shard_plan(W, H, bands, rank, fxaa)
    clus = oracle.cluster_build(cam, prep)  # replicated on every rank
    hdr = oracle.deferred_lighting(scene, cam, prep, clus, rows=plan["lighting"])
    lo, hi = plan["lighting"]
    hdr[:lo] = 0
    hdr[hi:] = 0
    lum0 = np.array([0.2, 2 ** 0.2, 2 ** -0.2], np.float32)
    sz = oracle.pyramid_sizes(W, H)

    def keep(img, rows):
        out = np.zeros_like(img)
        out[rows[0]:rows[1]] = img[rows[0]:rows[1]]
        return out

    t = keep(oracle.bloom_threshold(hdr, lum0, sz[0]), plan["threshold"])
    d0 = keep(oracle.bloom_downsample(t, sz[1]), plan["downsample0"])
    d0 = gather_fn(d0, [viewer.shard_plan(W, H, bands, r, fxaa)["downsample0"] for r in range(world)])
    d1 = oracle.bloom_downsample(d0, sz[2])
    d2 = oracle.bloom_downsample(d1, sz[3])
    d3 = oracle.bloom_downsample(d2, sz[4])
    _, grid = oracle.luminance(d3, lum0, 0.0115, want_grid=True)
    g = keep(grid, plan["lum_grid"])
    g = reduce_fn(g)
    # the assembled grid IS the full grid; the finalisation is then the single-device reduction
    assert np.array_equal(g.view(np.uint32), grid.view(np.uint32))
    lum = oracle.luminance(d3, lum0, float(np.float32(1.0 - 0.5 ** (1 / 60))))
    u2 = oracle.bloom_upsample(d3, sz[3])
    u1 = oracle.bloom_upsample(u2, sz[2])
    u0 = keep(oracle.bloom_upsample(u1, sz[1]), plan["upsample0"])
    ldr = keep(oracle.tonemap(hdr, u0, lum, 1.0, rows=plan["tonemap"]), plan["tonemap"])
    out = oracle.fxaa(ldr, True, rows=plan["fxaa"]) if fxaa else ldr
    return plan, out


def _worker(rank, world, port, fxaa, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from granite_b200 import viewer

        bands = viewer.band_partition(H, world)

        def gather(img, rows_per_rank):
            t = torch.from_numpy(np.ascontiguousarray(img).view(np.uint8).copy())  # gloo has no 16-bit integer types
            for r, (a, b) in enumerate(rows_per_rank):  # one broadcast per band, like the NCCL group
                part = t[a:b].contiguous()
                dist.broadcast(part, r)
                t[a:b] = part
            return t.numpy().view(np.uint16).reshape(img.shape)

        def reduce(grid):
            t = torch.from_numpy(grid.copy())
            dist.all_reduce(t, op=dist.ReduceOp.SUM)
            return t.numpy()

        plan, out = _sharded_rank(rank, world, bands, fxaa, gather, reduce)
        q.put((rank, plan["own"], out[plan["own"][0]:plan["own"][1]].copy()))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("fxaa", [False, True])
def test_two_rank_gloo_frame_equals_single_rank(oracle, fxaa):
    from tests import common

    scene, cam, lights, prep = common.build_case(oracle, W, H, N_LIGHTS, 0.25)
    clus, hdr, lum0, f, ldr_fxaa = _reference_frame(oracle, scene, cam, prep)
    expect = ldr_fxaa if fxaa else f.ldr
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = common.free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, fxaa, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    covered = 0
    for rank, (a, b), rows in sorted(got):
        assert np.array_equal(rows, expect[a:b]), f"rank {rank} rows [{a},{b}) differ from the unsharded frame"
        covered += b - a
    assert covered == H


def _bands_for(world, weighted):
    from granite_b200 import synth, viewer

    if weighted == "thin":
        # what the feedback balancer produces around light-dense rows: bands of one or two 8-row units
        cuts = [0, H // 2 - 24, H // 2 - 16, H // 2 - 8, H // 2 + 8, H // 2 + 16, H][: world] + [H]
        cuts = sorted(set(c - c % 8 for c in cuts[:-1])) + [H]
        return list(zip(cuts[:-1], cuts[1:]))
    if not weighted:
        return viewer.band_partition(H, world)
    # cost-balanced bands in 8-row units, as bench.py builds them for N > 1
    scene = synth.make_scene(W, H)
    lights = synth.make_lights(N_LIGHTS, spot_fraction=0.25, aspect=W / H)
    cost = viewer.estimate_band_cost(scene.projection, scene.view, lights.position, lights.color, W, H, depth=scene.depth, align=8)
    return viewer.band_partition_weighted(H, world, cost, align=8)


@pytest.mark.parametrize("world,weighted", [(3, False), (6, False), (4, True), (8, True), (6, "thin")])
def test_emulated_many_ranks(oracle, world, weighted):
    """Same protocol with the collectives emulated in-process (every band count the frame allows)."""
    from granite_b200 import viewer
    from tests import common

    scene, cam, lights, prep = common.build_case(oracle, W, H, N_LIGHTS, 0.25)
    _, _, _, f, _ = _reference_frame(oracle, scene, cam, prep)
    bands = _bands_for(world, weighted)
    assert len(bands) == world
    assert bands[0][0] == 0 and bands[-1][1] == H and all(a[1] == b[0] and a[1] % 8 == 0 for a, b in zip(bands, bands[1:]))
    # three passes emulate the two exchange steps: (0) collect every rank's d0 band, (1) with the
    # gathered d0, collect every rank's luminance-grid rows, (2) the real frame
    contributions = {}

    def hooks(rank, stage):
        def gather(img, rows_per_rank):
            if stage == 0:
                contributions[("d0", rank)] = img
                return img
            full = np.zeros_like(img)
            for r, (a, b) in enumerate(rows_per_rank):
                full[a:b] = contributions[("d0", r)][a:b]
            return full

        def reduce(grid):
            if stage <= 1:
                contributions[("grid", rank)] = grid
                return grid
            return sum(contributions[("grid", r)] for r in range(world))
        return gather, reduce

    for stage in (0, 1):
        for r in range(world):
            g, rd = hooks(r, stage)
            try:
                _sharded_rank(r, world, bands, False, g, rd)
            except AssertionError:
                pass  # the grid is not assembled yet in the collection passes
    for r in range(world):
        g, rd = hooks(r, 2)
        plan, out = _sharded_rank(r, world, bands, False, g, rd)
        a, b = plan["own"]
        assert np.array_equal(out[a:b], f.ldr[a:b]), f"rank {r}"


def test_plan_invariants():
    from granite_b200 import viewer

    for h, world in [(2160, 2), (2160, 4), (2160, 8), (1080, 8), (384, 6)]:
        bands = viewer.band_partition(h, world)
        hq = -(-h // 4)
        plans = [viewer.shard_plan(3840, h, bands, r, True) for r in range(world)]
        # d0 bands and luminance-grid rows tile their images exactly
        assert plans[0]["downsample0"][0] == 0 and plans[-1]["downsample0"][1] == hq
        assert all(a["downsample0"][1] == b["downsample0"][0] for a, b in zip(plans, plans[1:]))
        assert all(a["lum_grid"][1] == b["lum_grid"][0] for a, b in zip(plans, plans[1:]))
        for p in plans:
            assert p["lighting"][0] <= p["tonemap"][0] <= p["own"][0] and p["own"][1] <= p["tonemap"][1] <= p["lighting"][1]
            assert p["lighting"][1] - p["lighting"][0] <= (p["own"][1] - p["own"][0]) + 24  # halo stays small
