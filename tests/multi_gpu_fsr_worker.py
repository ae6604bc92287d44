"""torchrun worker for tests/test_zr_gpu_fsr_sharded.py: renders frames with FSR 1 upscaling row-sharded over all ranks
(the bands are display rows; every pass before FSR runs on the render rows of grbh_shard_plan_fsr, and the bloom d0,
SMAA edge and TAA history rows are exchanged inside the C++ graph by peer stores or NCCL as GRB_SHARD_EXCHANGE says)
and, on rank 0, unsharded; every assembled sharded frame must equal the unsharded one bit for bit, and every rank
must read back exactly its display band.  Scales 0.67 and 0.5, RCAS on and off, no AA, FXAA, SMAA Ultra / Low, TAA
High + FXAA and TAA Low; two band layouts (equal bands, and narrow 64-row bands at the top); 4 frames each with a
moving camera."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FRAMES = 4


def motion_vectors(w, h):
    rng = np.random.default_rng(11)
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
    layouts = {"equal": viewer.band_partition(h, world),
               "narrow": [(64 * r, 64 * (r + 1)) for r in range(world - 1)] + [(64 * (world - 1), h)]}
    views = [synth.look_at_view((0.15 * i, 0.1 * i, 8.0 - 0.2 * i), (0.0, 0.0, 0.0)) for i in range(FRAMES)]
    configs = {"0.67 RCAS none": (0.67, True, viewer.AA_NONE), "0.67 RCAS FXAA": (0.67, True, viewer.AA_FXAA),
               "0.67 SMAA Ultra": (0.67, False, viewer.AA_SMAA_ULTRA), "0.5 RCAS SMAA Low": (0.5, True, viewer.AA_SMAA_LOW),
               "0.67 RCAS TAA High + FXAA": (0.67, True, viewer.AA_TAA_HIGH_PLUS_FXAA), "0.5 TAA Low": (0.5, False, viewer.AA_TAA_LOW)}

    inputs = {}

    def gbuffer(scale):
        """The G-buffer at the render size of `scale` (the viewer's own rule)."""
        if scale not in inputs:
            probe = viewer.Viewer(w, h, cuda_device=-1, resolution_scale=scale)
            rw, rh = probe.render_size()
            probe.close()
            scene = synth.make_scene(rw, rh)
            keep = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, scene.emissive)]
            keep.append(np.ascontiguousarray(motion_vectors(rw, rh)).view(np.uint32).reshape(rh, rw))
            lights = synth.make_lights(n_lights, spot_fraction=0.25, aspect=rw / rh)
            inputs[scale] = (scene, lights, keep, viewer.Viewer.host_gbuffer(*keep))
        return inputs[scale]

    def make(scale, rcas, aa, bands):
        scene, lights, _, _ = gbuffer(scale)
        v = viewer.Viewer(w, h, post_aa=aa, cuda_device=local, resolution_scale=scale, resolution_scale_sharpen=rcas)
        v.set_directional(scene.dir_color, scene.dir_direction)
        v.set_lights(lights)
        if viewer.AA_SMAA_LOW <= aa <= viewer.AA_SMAA_ULTRA:
            v.set_smaa_lookup_textures(luts["area"], luts["search"])
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

    ok = True
    for cfg_name, (scale, rcas, aa) in configs.items():
        scene, _, _, gb = gbuffer(scale)
        reference = []
        if rank == 0:
            v1 = make(scale, rcas, aa, None)
            for i in range(FRAMES):
                v1.set_camera(scene.projection, views[i])
                v1.render_frame(gb if i == 0 else None)
                ref = np.zeros((h, w), np.uint32)
                v1.read_output(ref)
                reference.append(ref)
            v1.close()
        for name, bands in layouts.items():
            vs = make(scale, rcas, aa, bands)
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
