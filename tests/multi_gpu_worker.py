"""torchrun worker for tests/test_multi_gpu.py: renders the same frames row-sharded over all ranks
(NCCL exchange steps inside the C++ graph) and, on rank 0, unsharded; the assembled sharded image
must equal the unsharded one bit for bit.

Row-sharded frames and the unsharded reference frame are lit by the same (persistent) form of the lighting kernel:
a light that cannot reach a pixel adds exactly 0 to it, so the result does not depend on which 16x4 pixel blocks a
rank happens to own."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    w, h, n_lights, fxaa = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    gpus = torch.cuda.device_count()
    if world > gpus:
        # More ranks than GPUs: ranks share a device.  NCCL refuses two ranks of one host on one device (it compares
        # host hash and bus id), so each rank names a host of its own and NCCL connects them through its socket
        # transport on the loopback interface.  The frame's own exchange -- the downsample kernel's stores into the
        # IPC-mapped images of every rank, the epoch flags the pyramid tail waits on -- runs unchanged.
        os.environ["NCCL_HOSTID"] = f"granite-test-rank-{rank}"
        os.environ.setdefault("NCCL_SOCKET_IFNAME", "lo")
        os.environ.setdefault("NCCL_IB_DISABLE", "1")
    local = local % gpus
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from granite_b200 import synth, viewer

    scene = synth.make_scene(w, h)
    lights = synth.make_lights(n_lights, spot_fraction=0.25, aspect=w / h)
    aa = viewer.AA_FXAA if fxaa else viewer.AA_NONE
    keep = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, scene.emissive)]
    gb = viewer.Viewer.host_gbuffer(*keep)

    def make(sharded):
        v = viewer.Viewer(w, h, post_aa=aa, cuda_device=local)
        v.set_camera(scene.projection, scene.view)
        v.set_directional(scene.dir_color, scene.dir_direction)
        v.set_lights(lights)
        if sharded:
            uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
            if rank == 0:
                uid.copy_(torch.frombuffer(bytearray(viewer.nccl_unique_id()), dtype=torch.uint8))
            dist.broadcast(uid, 0)
            v.init_collectives(uid.cpu().numpy().tobytes(), rank, world)
            v.set_row_shards(viewer.band_partition(h, world), rank)
        v.bake()
        return v

    vs = make(True)
    frames = []
    for i in range(3):
        vs.render_frame(gb if i == 0 else None)
        out = np.zeros((h, w), np.uint32)
        y0, y1 = vs.read_output(out)
        full = torch.from_numpy(out.view(np.int32)).cuda()
        dist.all_reduce(full, op=dist.ReduceOp.SUM)  # bands are disjoint, zeros elsewhere
        frames.append(full.cpu().numpy().view(np.uint32))
    lum_sharded = vs.download_buffer("average-luminance", np.float32, 3).copy()
    vs.close()
    ok = True
    if rank == 0:
        v1 = make(False)
        for i in range(3):
            v1.render_frame(gb if i == 0 else None)
            ref = np.zeros((h, w), np.uint32)
            v1.read_output(ref)
            same = np.array_equal(ref, frames[i])
            print(f"frame {i}: sharded over {world} ranks == single GPU: {same}", flush=True)
            ok &= same
        lum1 = v1.download_buffer("average-luminance", np.float32, 3)
        same = np.array_equal(lum1.view(np.uint32), lum_sharded.view(np.uint32))
        print(f"average luminance identical: {same}", flush=True)
        ok &= same
        v1.close()
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.broadcast(flag, 0)
    dist.destroy_process_group()
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()
