"""torchrun worker for tests/test_zq_gpu_present_sharded.py: renders row-sharded frames presented from one rank (the
bands pushed to it inside the C++ graph, by peer stores or NCCL as GRB_SHARD_EXCHANGE says) and, on rank 0, unsharded;
every frame the presenting rank reads must equal the unsharded one bit for bit, with rows {0, height}, and every other
rank must still read its band.

The presenting rank reads with read_output_async + wait_outputs(1), which keeps one readback in flight, into pinned
buffers; one run also sleeps on the host before every read, so the other ranks run ahead until the credit holds them.
The camera moves every frame, so a slot that is stale or torn shows up as a wrong frame.  Tonemap-only frames without
bloom have no d0 exchange that couples the ranks, so only the credit holds the producers back there; that config is
first checked sharded without presenting (its bands gathered with an all-reduce)."""
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FRAMES = 6
# (band layout, presenting rank: 0 or -1 = the last rank, sleep before each read)
RUNS = (("equal", 0, False), ("equal", -1, True), ("narrow", 0, False), ("narrow", -1, False))
CONFIGS = ("no AA", "FXAA", "SMAA Ultra", "TAA High + FXAA", "FSR 0.67 + RCAS", "HDR10 + TAA", "tonemap-only")


def config_args(name):
    from granite_b200 import viewer

    return {"no AA": dict(post_aa=viewer.AA_NONE), "FXAA": dict(post_aa=viewer.AA_FXAA), "SMAA Ultra": dict(post_aa=viewer.AA_SMAA_ULTRA),
            "TAA High + FXAA": dict(post_aa=viewer.AA_TAA_HIGH_PLUS_FXAA), "FSR 0.67 + RCAS": dict(resolution_scale=0.67, resolution_scale_sharpen=True),
            "HDR10 + TAA": dict(post_aa=viewer.AA_TAA_HIGH, hdr10_output=True), "tonemap-only": dict(hdr_bloom=False)}[name]


def motion_vectors(w, h):
    rng = np.random.default_rng(5)
    mv = np.zeros((h, w, 2), np.float16)
    moving = rng.random((h, w)) < 0.15
    n = int(moving.sum())
    mv[moving] = np.stack([rng.uniform(-4.0, 4.0, n) / w, rng.uniform(-0.5, 0.5, n)], -1).astype(np.float16)
    return mv


def main():
    w, h, n_lights = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    gpus = torch.cuda.device_count()
    if world > gpus:
        # ranks share a device: each names a host of its own so that NCCL accepts them (see multi_gpu_worker.py)
        os.environ["NCCL_HOSTID"] = f"granite-test-rank-{rank}"
        os.environ.setdefault("NCCL_SOCKET_IFNAME", "lo")
        os.environ.setdefault("NCCL_IB_DISABLE", "1")
    local = local % gpus
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from granite_b200 import synth, viewer

    luts = np.load(os.path.join(ROOT, "tests", "golden", "refsmaa_160x96.npz"))
    scene = synth.make_scene(w, h)
    lights = synth.make_lights(n_lights, spot_fraction=0.25, aspect=w / h)
    keep = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, scene.emissive)]
    keep.append(np.ascontiguousarray(motion_vectors(w, h)).view(np.uint32).reshape(h, w))
    gb = viewer.Viewer.host_gbuffer(*keep)
    views = [synth.look_at_view((0.15 * i, 0.1 * i, 8.0 - 0.2 * i), (0.0, 0.0, 0.0)) for i in range(FRAMES)]
    # Narrow bands are 16 rows: the FXAA tile kernel's result depends on a pixel's position in its 16-row tile, so a
    # band that starts off a multiple of 16 is not bit-exact without FSR (a known limitation of sharded FXAA), and at
    # FSR 0.67 8-row bands would leave rank 0 without render rows.
    layouts = {"equal": viewer.band_partition(h, world),
               "narrow": [(16 * r, 16 * (r + 1)) for r in range(world - 1)] + [(16 * (world - 1), h)]}

    def make(cfg, bands, present_rank=-1):
        v = viewer.Viewer(w, h, cuda_device=local, **config_args(cfg))
        v.set_directional(scene.dir_color, scene.dir_direction)
        v.set_lights(lights)
        v.set_smaa_lookup_textures(luts["area"], luts["search"])
        if bands:
            uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
            if rank == 0:
                uid.copy_(torch.frombuffer(bytearray(viewer.nccl_unique_id()), dtype=torch.uint8))
            dist.broadcast(uid, 0)
            v.init_collectives(uid.cpu().numpy().tobytes(), rank, world)
            v.set_row_shards(bands, rank)
            v.set_present_rank(present_rank)
        v.set_camera(scene.projection, views[0])
        v.bake()
        return v

    ok = True
    for cfg in CONFIGS:
        reference = []
        if rank == 0:
            v1 = make(cfg, None)
            for i in range(FRAMES):
                v1.set_camera(scene.projection, views[i])
                v1.render_frame(gb if i == 0 else None)
                ref = np.zeros((h, w), np.uint32)
                v1.read_output(ref)
                reference.append(ref)
            v1.close()

        if cfg == "tonemap-only":
            # sharded without presenting first: the bands alone must assemble the unsharded frame
            for name, bands in layouts.items():
                vs = make(cfg, bands)
                for i in range(FRAMES):
                    vs.set_camera(scene.projection, views[i])
                    vs.render_frame(gb if i == 0 else None)
                    out = np.zeros((h, w), np.uint32)
                    ok &= vs.read_output(out) == tuple(bands[rank])
                    full = torch.from_numpy(out.view(np.int32)).cuda()
                    dist.all_reduce(full, op=dist.ReduceOp.SUM)  # bands are disjoint, zeros elsewhere
                    if rank == 0:
                        same = np.array_equal(full.cpu().numpy().view(np.uint32), reference[i])
                        print(f"{cfg} {name} frame {i}: tonemap-only sharded == single GPU: {same}", flush=True)
                        ok &= same
                vs.close()

        for name, p, sleep in RUNS:
            bands = layouts[name]
            present = p % world
            vs = make(cfg, bands, present)
            frames = torch.zeros((FRAMES, h, w), dtype=torch.int32).pin_memory()
            rows = []
            for i in range(FRAMES):
                vs.set_camera(scene.projection, views[i])
                vs.render_frame(gb if i == 0 else None)
                if rank == present:
                    if sleep:
                        time.sleep(0.02)
                    rows.append(vs.read_output_async(frames[i]))
                    vs.wait_outputs(1)
                else:
                    out = np.zeros((h, w), np.uint32)
                    ok &= vs.read_output(out) == tuple(bands[rank])
            vs.wait_outputs(0)
            ok &= all(r == (0, h) for r in rows)
            # every rank's pushes and flag stores have landed before any rank frees its channel
            vs.sync()
            dist.barrier()
            vs.close()
            gathered = frames.cuda()
            dist.broadcast(gathered, present)
            if rank == 0:
                got = gathered.cpu().numpy().view(np.uint32)
                for i in range(FRAMES):
                    same = np.array_equal(got[i], reference[i])
                    print(f"{cfg} {name} P={present}{' sleep' if sleep else ''} frame {i}: presented == single GPU: {same}", flush=True)
                    ok &= same
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.destroy_process_group()
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()
