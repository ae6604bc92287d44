"""torchrun worker for tests/test_zs_gpu_taa_sharded.py: renders frames with TAA row-sharded over all ranks (the
history rows exchanged inside the C++ graph, by peer stores or NCCL as GRB_SHARD_EXCHANGE says) and, on rank 0,
unsharded; every assembled sharded frame must equal the unsharded one bit for bit.  TAA Low, TAA High, TAA High + FXAA
and TAA High with HDR10 output; two band layouts (equal bands, and narrow 64-row bands at the top); 6 frames each, so
both slots of the exchange are reused.  The camera moves every frame, and 15 % of the pixels carry a motion vector of
up to half the image height: rank 0 checks on the host that every rank's motion vectors reach other ranks' bands."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FRAMES = 6


def motion_vectors(w, h):
    rng = np.random.default_rng(11)
    mv = np.zeros((h, w, 2), np.float16)
    moving = rng.random((h, w)) < 0.15
    n = int(moving.sum())
    mv[moving] = np.stack([rng.uniform(-4.0, 4.0, n) / w, rng.uniform(-0.5, 0.5, n)], -1).astype(np.float16)
    return mv


def reaches_other_bands(mv, bands):
    """For every band: moving pixels whose history read (at v - mv) lands in another band."""
    h = mv.shape[0]
    mvy = mv[..., 1].astype(np.float32)
    src = np.arange(h)[:, None] + 0.5 - mvy * h
    return [int(((src[y0:y1] < y0) | (src[y0:y1] >= y1))[mvy[y0:y1] != 0].sum()) for y0, y1 in bands]


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

    scene = synth.make_scene(w, h)
    lights = synth.make_lights(n_lights, spot_fraction=0.25, aspect=w / h)
    mv = motion_vectors(w, h)
    keep = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, scene.emissive)]
    keep.append(np.ascontiguousarray(mv).view(np.uint32).reshape(h, w))
    gb = viewer.Viewer.host_gbuffer(*keep)
    views = [synth.look_at_view((0.15 * i, 0.1 * i, 8.0 - 0.2 * i), (0.0, 0.0, 0.0)) for i in range(FRAMES)]
    layouts = {"equal": viewer.band_partition(h, world),
               "narrow": [(64 * r, 64 * (r + 1)) for r in range(world - 1)] + [(64 * (world - 1), h)]}
    configs = {"TAA Low": dict(post_aa=viewer.AA_TAA_LOW), "TAA High": dict(post_aa=viewer.AA_TAA_HIGH),
               "TAA High + FXAA": dict(post_aa=viewer.AA_TAA_HIGH_PLUS_FXAA), "TAA High HDR10": dict(post_aa=viewer.AA_TAA_HIGH, hdr10_output=True)}

    ok = True
    if rank == 0:
        for name, bands in layouts.items():
            reach = reaches_other_bands(mv, bands)
            print(f"{name}: motion vectors reach other bands from every rank: {all(n > 0 for n in reach)} {reach}", flush=True)
            ok &= all(n > 0 for n in reach)

    def make(cfg, bands):
        v = viewer.Viewer(w, h, cuda_device=local, **cfg)
        v.set_directional(scene.dir_color, scene.dir_direction)
        v.set_lights(lights)
        if bands:
            uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
            if rank == 0:
                uid.copy_(torch.frombuffer(bytearray(viewer.nccl_unique_id()), dtype=torch.uint8))
            dist.broadcast(uid, 0)
            v.init_collectives(uid.cpu().numpy().tobytes(), rank, world)
            v.set_row_shards(bands, rank)
        v.set_camera(scene.projection, views[0])
        v.bake()
        return v

    for cfg_name, cfg in configs.items():
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
        for name, bands in layouts.items():
            vs = make(cfg, bands)
            for i in range(FRAMES):
                vs.set_camera(scene.projection, views[i])
                vs.render_frame(gb if i == 0 else None)
                out = np.zeros((h, w), np.uint32)
                y0, y1 = vs.read_output(out)
                ok &= (y0, y1) == tuple(bands[rank])
                full = torch.from_numpy(out.view(np.int32)).cuda()
                dist.all_reduce(full, op=dist.ReduceOp.SUM)  # bands are disjoint, zeros elsewhere
                if rank == 0:
                    same = np.array_equal(full.cpu().numpy().view(np.uint32), reference[i])
                    print(f"{cfg_name} {name} frame {i}: sharded over {world} ranks == single GPU: {same}", flush=True)
                    ok &= same
            vs.close()
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.destroy_process_group()
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()
