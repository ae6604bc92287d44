"""torchrun worker for tests/test_zfi_gpu_light_shadow_ids_sharded.py: row-sharded frames whose shadowed device light list
comes from one rank by map id (Viewer.set_light_shadow_map_table, set_light_source_rank, set_lights_device(
shadow_map_ids=)).  Every rank builds its own map pool from the same seed, so the ranks' tables hold different pointers
to the same texels, in the same permuted order; some ids are out of range.  The source rank binds its list, transforms
and ids with a device count, which the same torch ops rewrite every frame while the entries past it are poisoned; every
other rank binds a receiving list of the same capacity.  Between two frames every rank rebinds at a smaller capacity,
and before the last frame the bands move.  Each assembled frame must equal, bit for bit, rank 0's unsharded host-light
shadowed frame of the first `live` lights given table[id]; every rank's light prep and shadow transforms must equal the
source rank's, and every rank's map pointers must be its own table's pointers to the same maps."""
import hashlib
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import synth, viewer  # noqa: E402
from oracle import pyoracle  # noqa: E402
from tests import device_lights_cases as cases  # noqa: E402
from tests import sharded  # noqa: E402
from tests.device_shadow_cases import MapPool, transforms_in_input_order  # noqa: E402
from tests.multi_gpu_light_source_worker import first, to_torch  # noqa: E402

# (capacity bound, count written on the device) per frame: a drop, a clamp past the capacity, a rebinding at capacity
# 256 (frame 3) and a clamp to it
SCHEDULE = ((600, 500), (600, 10), (600, 900), (256, 200), (256, 400))
FRAMES = len(SCHEDULE)
MOVE_AT = 4  # the bands move before this frame
# (configuration, lighting stripe rows, light source rank (-1: the last), the G-buffer fed from the same rank)
RUNS = (("no AA", 0, 0, False), ("no AA", 8, -1, False), ("TAA High + FXAA", 0, -1, True), ("TAA High + FXAA", 8, 0, False))
RES = 16


def live(i):
    capacity, count = SCHEDULE[i]
    return min(max(count, 0), capacity)


def ids_and_table(pool):
    """(table, ids, table[id] per light, 0 out of range): this rank's map pointers in an order every rank draws the same,
    a few null entries, and ids out of range (-1, the table size, INT32_MIN, INT32_MAX)."""
    pointers = pool.pointers()
    n = len(pointers)
    rng = np.random.default_rng(31)
    size = n + 9
    slot = rng.permutation(size)[:n]
    table = np.zeros(size, np.int64)
    table[slot] = pointers
    ids = slot.astype(np.int32)
    ids[::17] = size
    ids[4::23] = -1
    ids[6] = -(1 << 31)
    ids[9] = (1 << 31) - 1
    valid = (ids >= 0) & (ids < size)
    return table, ids, np.where(valid, table[np.clip(ids, 0, size - 1)], 0).astype(np.int64)


def map_indices(maps, pool):
    """Map pointers of this rank as offsets into its own pool (-1: no map): the same on every rank for the same maps."""
    m = np.asarray(maps, np.int64)
    return np.where(m == 0, -1, (m - pool.pool.data_ptr()) // 2)


def digest(*arrays):
    return hashlib.sha256(b"".join(np.ascontiguousarray(a).tobytes() for a in arrays)).hexdigest()


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
        args = dict(sharded.config_args(cfg), light_shadows=True, shadow_resolution=RES)
        scene, lights, arrays, gb = sharded.inputs(w, h, capacity, mv=sharded.motion_vectors(w, h, 3))
        pool = MapPool(lights, RES)  # this rank's own maps: the same texels on every rank, other pointers
        table, ids, eff = ids_and_table(pool)
        if cfg not in references:
            references[cfg] = []
            if rank == 0:
                v = viewer.Viewer(w, h, cuda_device=torch.cuda.current_device(), **args)
                v.set_directional(scene.dir_color, scene.dir_direction)
                v.set_camera(scene.projection, views[0])
                v.bake()
                for i in range(FRAMES):
                    v.set_lights(first(lights, live(i)))
                    v.set_light_shadow_maps(eff[:live(i)].tolist())
                    v.set_camera(scene.projection, views[i])
                    v.render_frame(gb if i == 0 else None)
                    out = np.zeros((h, w), np.uint32)
                    v.read_output(out)
                    t, m = v.light_shadow_prep()
                    references[cfg].append((out, digest(t), digest(map_indices(m, pool))))
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
        v.set_light_shadow_map_table(table.tolist())
        v.set_light_source_rank(source)
        if gbuffer_fed:
            v.set_gbuffer_source_rank(source)
            planes = [to_torch(a) for a in arrays] if rank == source else None  # alive while frames read them
            dev_gb = v.device_gbuffer(*planes[:5], mv=planes[5]) if rank == source else None
        d = cases.to_device(lights) if rank == source else None
        if d:
            d["shadow_transforms"] = torch.from_numpy(transforms_in_input_order(pyoracle, v, lights)).cuda()
            d["shadow_map_ids"] = torch.from_numpy(ids).cuda()
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
                for name in ("position", "color", "shadow_transforms"):
                    d[name].copy_(clean[name])
                    d[name][live(i):] = float("nan")
                d["shadow_map_ids"].copy_(clean["shadow_map_ids"])
                d["shadow_map_ids"][live(i):] = 0  # an id that resolves: a read of a dead entry would show
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
            t, m = v.light_shadow_prep()
            mine = map_indices(m, pool)
            # this rank's pointers are its own table's: inside its pool, or null
            m = m.astype(np.int64)
            own = bool(np.isin(m[m != 0], table[table != 0]).all())
            local = (digest(recs, model, mask, zr, np.int32(n)), digest(t), digest(mine), own)
            gathered = [None] * world
            dist.all_gather_object(gathered, local)
            if rank == 0:
                label = f"{cfg} stripes={stripes} source={source}{' G-buffer from the source' if gbuffer_fed else ''} live={live(i)}"
                want, want_t, want_m = references[cfg][i]
                same = np.array_equal(full, want)
                print(f"{label} frame {i}: shadowed device lights by map id from one rank sharded == host lights single GPU: {same}", flush=True)
                preps = all(g[0] == gathered[source][0] and g[1] == gathered[source][1] == want_t for g in gathered)
                print(f"{label} frame {i}: light prep and shadow transforms on every rank == the source rank's: {preps}", flush=True)
                maps = all(g[2] == want_m and g[3] for g in gathered)
                print(f"{label} frame {i}: every rank's maps are its own table's pointers to the same maps: {maps}", flush=True)
                ok &= same and preps and maps
        sharded.close_sharded(v)
    sharded.finish(ok)


if __name__ == "__main__":
    main()
