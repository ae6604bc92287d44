"""torchrun worker for tests/test_zfg_gpu_light_source_rank_sharded.py: row-sharded frames whose device light list and
live count come from one rank (Viewer.set_light_source_rank).  The source rank binds its list with a device count, which
the same torch ops rewrite every frame while the entries past it are NaN; every other rank binds a receiving list of
the same capacity.  Between two frames every rank rebinds at a smaller capacity, and before the last frame the bands
move.  Each assembled frame must equal, bit for bit, rank 0's unsharded host-light frame of the first `live` lights,
and every rank's light prep must equal the source rank's."""
import hashlib
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import synth, viewer  # noqa: E402
from tests import device_lights_cases as cases  # noqa: E402
from tests import sharded  # noqa: E402

# (capacity bound, count written on the device) per frame: a drop from 6000 to 10, a clamp past the capacity, a
# rebinding at capacity 1024 (frame 3) and a clamp to it
SCHEDULE = ((8192, 6000), (8192, 10), (8192, 9000), (1024, 500), (1024, 2000))
FRAMES = len(SCHEDULE)
MOVE_AT = 4  # the bands move before this frame
# (configuration, lighting stripe rows, light source rank (-1: the last), the G-buffer fed from the same rank)
RUNS = (("no AA", 0, 0, False), ("no AA", 8, -1, False), ("TAA High + FXAA", 0, -1, True), ("TAA High + FXAA", 8, 0, False))


def first(lights, k):
    return synth.Lights(lights.color[:k], lights.position[:k], lights.is_point[:k], lights.rot[:k], lights.inner_cone[:k], lights.outer_cone[:k])


def live(i):
    capacity, count = SCHEDULE[i]
    return min(max(count, 0), capacity)


def to_torch(a):
    return torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else (a.view(np.int16) if a.dtype == np.uint16 else a)).cuda()


def main():
    w, h = int(sys.argv[1]), int(sys.argv[2])
    rank, world, _ = sharded.init_ranks()
    views = [synth.look_at_view((0.15 * i, 0.1 * i, 8.0 - 0.2 * i), (0.0, 0.0, 0.0)) for i in range(FRAMES)]
    equal = viewer.band_partition(h, world, align=16)
    moved = [(0, 32)] + [(32 + (h - 32) * r // (world - 1) // 16 * 16, 32 + (h - 32) * (r + 1) // (world - 1) // 16 * 16) for r in range(world - 1)]
    moved[-1] = (moved[-1][0], h)
    capacity = SCHEDULE[0][0]
    ok = True
    references = {}
    for cfg, stripes, source, gbuffer_fed in RUNS:
        source = source % world
        args = sharded.config_args(cfg)
        scene, lights, arrays, gb = sharded.inputs(w, h, capacity, mv=sharded.motion_vectors(w, h, 3))
        if cfg not in references:
            references[cfg] = []
            if rank == 0:
                v = viewer.Viewer(w, h, cuda_device=torch.cuda.current_device(), **args)
                v.set_directional(scene.dir_color, scene.dir_direction)
                v.set_camera(scene.projection, views[0])
                v.bake()
                for i in range(FRAMES):
                    v.set_lights(first(lights, live(i)))
                    v.set_camera(scene.projection, views[i])
                    v.render_frame(gb if i == 0 else None)
                    out = np.zeros((h, w), np.uint32)
                    v.read_output(out)
                    references[cfg].append(out)
                v.close()

        v = viewer.Viewer(w, h, cuda_device=torch.cuda.current_device(), **args)
        v.set_directional(scene.dir_color, scene.dir_direction)
        uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
        if rank == 0:
            uid.copy_(torch.frombuffer(bytearray(viewer.nccl_unique_id()), dtype=torch.uint8))
        dist.broadcast(uid, 0)
        v.init_collectives(uid.cpu().numpy().tobytes(), rank, world)
        v.set_row_shards(equal, rank)
        v.set_lighting_stripes(stripes)
        v.set_light_source_rank(source)
        if gbuffer_fed:
            v.set_gbuffer_source_rank(source)
            planes = [to_torch(a) for a in arrays] if rank == source else None  # alive while frames read them
            dev_gb = v.device_gbuffer(*planes[:5], mv=planes[5]) if rank == source else None
        d = cases.to_device(lights) if rank == source else None
        clean = {k: t.clone() for k, t in d.items()} if d else None
        count = torch.zeros(1, dtype=torch.int32, device="cuda")
        ready, consumed = torch.cuda.Event(), torch.cuda.Event()
        v.set_camera(scene.projection, views[0])
        v.bake()
        bound = None
        for i in range(FRAMES):
            cap, raw = SCHEDULE[i]
            if cap != bound:
                # every rank rebinds between the same two frames: the source its list, the others a receiving list
                if rank == source:
                    v.set_lights_device(**{k: t[:cap] for k, t in d.items()}, ready=ready, consumed=consumed, count=count)
                else:
                    v.set_lights_device_from_source(cap)
                bound = cap
            if i == MOVE_AT:
                v.move_row_shards(moved)
            if rank == source:
                torch.cuda.current_stream().wait_event(consumed)
                count.fill_(raw)
                for name in ("position", "color"):
                    d[name].copy_(clean[name])
                    d[name][live(i):] = float("nan")
                ready.record()
            v.set_camera(scene.projection, views[i])
            if gbuffer_fed:
                v.render_frame_device(dev_gb)
            else:
                v.render_frame(gb if i in (0, MOVE_AT) else None)
            out = np.zeros((h, w), np.uint32)
            rows = v.read_output(out)
            ok &= rows == tuple((moved if i >= MOVE_AT else equal)[rank])
            full = sharded.assemble(out)
            n, recs, model, mask, zr = v.light_prep(capacity=4096)
            digest = hashlib.sha256(b"".join(np.ascontiguousarray(a).tobytes() for a in (recs, model, mask, zr)) + n.to_bytes(4, "little")).hexdigest()
            digests = [None] * world
            dist.all_gather_object(digests, digest)
            if rank == 0:
                label = f"{cfg} stripes={stripes} source={source}{' G-buffer from the source' if gbuffer_fed else ''} live={live(i)}"
                same = np.array_equal(full, references[cfg][i])
                print(f"{label} frame {i}: device lights from one rank sharded == host lights single GPU: {same}", flush=True)
                preps = all(x == digests[source] for x in digests)
                print(f"{label} frame {i}: light prep on every rank == the source rank's: {preps}", flush=True)
                ok &= same and preps
        sharded.close_sharded(v)
    sharded.finish(ok)


if __name__ == "__main__":
    main()
