"""torchrun worker for tests/test_zt_gpu_smaa_sharded.py: renders frames with SMAA row-sharded over all ranks (the
edge rows exchanged inside the C++ graph, by peer stores or NCCL as GRB_SHARD_EXCHANGE says) and, on rank 0, unsharded;
every assembled sharded frame must equal the unsharded one bit for bit.  Two band layouts (equal bands, and narrow
64-row bands at the top so that an edge window spans two ranks), presets Low and Ultra, 4 frames each (both slots of
the exchange are reused).  Rank 0 also checks that the unsharded weights are non-zero near every band border, so that
the frame really depends on the exchanged rows."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FRAMES = 4


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
    gb = viewer.Viewer.host_gbuffer(*keep)
    layouts = {"equal": viewer.band_partition(h, world),
               "narrow": [(64 * r, 64 * (r + 1)) for r in range(world - 1)] + [(64 * (world - 1), h)]}

    def make(aa, bands):
        v = viewer.Viewer(w, h, post_aa=aa, cuda_device=local)
        v.set_camera(scene.projection, scene.view)
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
        v.bake()
        return v

    ok = True
    for quality, aa in ((0, viewer.AA_SMAA_LOW), (3, viewer.AA_SMAA_ULTRA)):
        reference = []
        if rank == 0:
            v1 = make(aa, None)
            for i in range(FRAMES):
                v1.render_frame(gb if i == 0 else None)
                ref = np.zeros((h, w), np.uint32)
                v1.read_output(ref)
                reference.append(ref)
            weights = v1.download_image("smaa-weights")
            v1.close()
        for name, bands in layouts.items():
            vs = make(aa, bands)
            for i in range(FRAMES):
                vs.render_frame(gb if i == 0 else None)
                out = np.zeros((h, w), np.uint32)
                y0, y1 = vs.read_output(out)
                ok &= (y0, y1) == tuple(bands[rank])
                full = torch.from_numpy(out.view(np.int32)).cuda()
                dist.all_reduce(full, op=dist.ReduceOp.SUM)  # bands are disjoint, zeros elsewhere
                if rank == 0:
                    same = np.array_equal(full.cpu().numpy().view(np.uint32), reference[i])
                    print(f"preset {quality} {name} frame {i}: sharded over {world} ranks == single GPU: {same}", flush=True)
                    ok &= same
            vs.close()
            if rank == 0:
                reach = 2 * (4 << quality)
                near = [bool(weights[max(b - reach, 0):b + reach].any()) for _, b in bands[:-1]]
                print(f"preset {quality} {name}: weights near every border: {all(near)}", flush=True)
                ok &= all(near)
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.destroy_process_group()
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()
