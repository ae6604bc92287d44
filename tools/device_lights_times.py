#!/usr/bin/env python3
"""Frames/s of BASELINE config c3 (3840x2160, bloom + tonemap) fed from device G-buffers, with the positional lights
moved every frame by a small torch op on the device, by where the light prep runs:
- "host lights": the moved positions are copied to the host and handed over with set_lights every frame, so the
  clusterer culls, sorts and packs them on the CPU and uploads the result;
- "device lights": set_lights_device binds the tensors once; every frame's clustering pass culls, sorts and packs them
  on the GPU.

    python tools/device_lights_times.py [--frames 100] [--shadows [--map-ids] | --live-count]
    torchrun --nproc-per-node=<GPUs> tools/device_lights_times.py [--frames 100] [--shadows [--map-ids] | [--shadows] --live-count [--source-rank]]

--shadows: viewers created with clustered_lights_shadows, every light shadowed by one of 64 static synthetic cube maps
(64 x 64 texels a face).  Host lights get the map pointers with set_lights every frame and the clusterer computes the
shadow transforms; device lights bind the transforms (the reference's, computed once: a point light's depends only on
its range) and the pointers with the lights, and the clustering pass moves them into cluster order.

--shadows --map-ids: a third mode, "device lights by map id": the same lights and transforms bound with map ids into a
table of the 64 maps (set_light_shadow_map_table, set_lights_device(shadow_map_ids=)), so the clustering pass resolves
each kept light's id through the table.  Its "clustering-bindless" time against the pointer form's is what the id
costs.

--live-count: a particle-style list whose length is known only on the device.  16384 particle lights, each alive for a
lifetime of its own in a cycle of its own, so that about half are alive and the set changes every frame.  Every frame a
torch op compacts the alive particles into a light list and writes its length, with a cumsum scatter and no host sync.
Three ways to hand that list over are timed in the same run:
- "device count": the list and its count are bound once (set_lights_device(..., count=)); the clustering pass reads
  the count on the device;
- "count read back": the count is read to the host and the list rebound with that length every frame;
- "parked": no compaction: the whole capacity is bound and dead particles are parked behind the camera, where the
  frustum cull drops them.
The torch ops run on the caller's stream and the viewer waits on them through the lights' ready / consumed events.

--live-count --source-rank (under torchrun): the same particle workload on row-sharded frames, with three hand-overs of
the list from the rank that simulates it:
- "every rank updates": every rank runs the particle update and the compaction on its own copy and binds its own list
  and count (what a caller does without a source rank);
- "caller broadcast": rank 0 updates and compacts; every frame the caller broadcasts the capacity-sized list and the
  count from rank 0 (torch.distributed.broadcast on its stream, between the lights' ready / consumed events), and every
  rank binds its copy once;
- "viewer push": rank 0 updates, compacts and binds once; every other rank binds a receiving list once
  (set_light_source_rank(0), set_lights_device_from_source), and rank 0's clustering pass pushes the live entries and
  the count to the other ranks.
With --shadows every particle is shadowed by one of the 64 static cube maps, named by map id: every rank sets its own
table of its own copy of the maps, and the transforms and ids follow the compaction, the broadcast and the push.

Two light lists: 4096 input lights (all in view), and 16384 input lights of which 4096 are kept.  Under torchrun, one
rank per GPU, row-sharded frames with every rank binding its own copy of the lights; the sharded rate is that of the
slowest rank.

Each viewer renders 4 untimed frames, then --frames timed frames (CUDA events on the viewer's stream), and reports the
host time spent recording them (the frame calls and the light hand-over, per frame).  The "clustering-bindless" pass
time comes from a second run of the same frames with the viewer's timestamps on.  The card's name and power limit come
from a read-only nvidia-smi query in the same run and are printed beside every number.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import synth, viewer  # noqa: E402
from tests import device_lights_cases as cases  # noqa: E402
from tests import sharded  # noqa: E402
from tools.device_gbuffer_times import FILL, H, W, device_gbuffers  # noqa: E402


def light_list(n):
    """n lights: the first 4096 in view (synth.make_lights), the rest behind the eye, so at most 4096 are kept."""
    kept = synth.make_lights(min(n, 4096), spot_fraction=0.0, aspect=W / H)
    if n <= 4096:
        return kept
    extra = synth.make_lights(n - 4096, spot_fraction=0.0, aspect=W / H)
    extra.position[:, 2] += 400.0
    return synth.Lights(*[np.concatenate([a, b]) for a, b in zip((kept.color, kept.position, kept.is_point, kept.rot, kept.inner_cone, kept.outer_cone),
                                                                   (extra.color, extra.position, extra.is_point, extra.rot, extra.inner_cone,
                                                                    extra.outer_cone))])


SHADOW_RES = 64
SHADOW_MAPS = 64


def shadow_inputs(scene, lights):
    """(maps tensor, (N,) int64 pointers, (N, 16) float32 transforms in input order) for the --shadows runs.  The
    transforms are the host clusterer's, put back in input order through distinct stand-in pointers."""
    n = len(lights.color)
    rng = np.random.default_rng(7)
    maps = torch.from_numpy(rng.integers(0, 3000, (SHADOW_MAPS, 6, SHADOW_RES, SHADOW_RES)).astype(np.int16)).cuda()
    pointers = maps.data_ptr() + 2 * 6 * SHADOW_RES * SHADOW_RES * (np.arange(n, dtype=np.int64) % SHADOW_MAPS)
    host = viewer.Viewer(W, H, cuda_device=-1, light_shadows=True, shadow_resolution=SHADOW_RES)
    host.set_camera(scene.projection, scene.view)
    transforms = np.zeros((n, 16), np.float32)
    # in chunks the host prep keeps whole (4096 lights): a light it culls keeps a zero matrix, which no frame packs
    for at in range(0, n, 4096):
        k = min(4096, n - at)
        host.set_lights(synth.Lights(*[a[at:at + k] for a in (lights.color, lights.position, lights.is_point, lights.rot, lights.inner_cone,
                                                              lights.outer_cone)]))
        host.set_light_shadow_maps(list(range(1, k + 1)))
        t, m = host.light_shadow_prep()
        transforms[at + m.astype(np.int64) - 1] = t
    host.close()
    return maps, pointers, transforms


PARTICLES = 16384


def particles():
    """(lights, per-particle cycle, per-particle lifetime): 16384 particle lights in view, alive at frame f when
    (f + offset) % cycle < lifetime, which holds for about half of them in every frame."""
    lights = synth.make_lights(PARTICLES, spot_fraction=0.0, aspect=W / H)
    rng = np.random.default_rng(11)
    cycle = rng.integers(8, 64, PARTICLES)
    lifetime = np.maximum(1, (cycle * rng.uniform(0.3, 0.7, PARTICLES)).astype(np.int64))
    offset = rng.integers(0, 64, PARTICLES)
    return lights, cycle, lifetime, offset


def live_count_stepper(mode, lights, cycle, lifetime, offset, rank=0, shadows=None):
    """step(v, i) for one --live-count mode: the particle update, the compaction (or the parking) and the frame.  The
    --source-rank modes: "every rank updates" is "device count" on every rank; under "caller broadcast" and "viewer
    push" only rank 0 updates.  shadows: (transforms, map ids, table) of shadowed particles by map id, or None."""
    n = PARTICLES
    src = cases.to_device(lights)
    if shadows is not None:
        src["shadow_transforms"] = torch.from_numpy(shadows[0]).cuda()
        src["shadow_map_ids"] = torch.from_numpy(shadows[1]).cuda()
    cycle_t, lifetime_t, offset_t = (torch.from_numpy(a).cuda() for a in (cycle, lifetime, offset))
    # the compacted list, one row more than the capacity: dead particles are scattered into the last row
    out = {k: torch.empty((n + 1, *t.shape[1:]), dtype=t.dtype, device="cuda") for k, t in src.items()}
    bound = {k: t[:n] for k, t in out.items()}
    parked = {k: t.clone() for k, t in src.items()}
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    ready, consumed = torch.cuda.Event(), torch.cuda.Event()
    state = {"viewer": None}

    receiver = mode in ("caller broadcast", "viewer push") and rank != 0

    def step(v, i):
        if state["viewer"] is not v:
            state["viewer"] = v
            state["gbs"] = [v.device_gbuffer(*g) for g in state["dev"]]
            if shadows is not None and mode != "viewer push":  # source_rank_viewer sets it before the source rank
                v.set_light_shadow_map_table(shadows[2])
            if mode == "viewer push" and receiver:
                v.set_lights_device_from_source(n)
            elif mode in ("device count", "every rank updates", "caller broadcast", "viewer push"):
                v.set_lights_device(**bound, ready=ready, consumed=consumed, count=count)
            elif mode == "parked":
                v.set_lights_device(**parked, ready=ready, consumed=consumed)
        else:
            torch.cuda.current_stream().wait_event(consumed)
        if mode == "viewer push" and receiver:
            v.render_frame_device(state["gbs"][i % 2])
            return
        if receiver:
            # the caller's broadcast of the capacity: the live length is only on the device
            for t in (*bound.values(), count):
                torch.distributed.broadcast(t, 0)
            ready.record()
            v.render_frame_device(state["gbs"][i % 2])
            return
        alive = (i + offset_t) % cycle_t < lifetime_t
        if mode == "parked":
            for k in parked:
                parked[k].copy_(src[k])
            parked["position"][:, 2].masked_fill_(~alive, 1000.0)  # behind the eye: culled
        else:
            csum = torch.cumsum(alive, 0, dtype=torch.int32)
            dest = torch.where(alive, csum.long() - 1, n)
            for k in out:
                out[k].index_copy_(0, dest, src[k])
            count.copy_(csum[-1:])
        if mode == "caller broadcast":
            for t in (*bound.values(), count):
                torch.distributed.broadcast(t, 0)
        ready.record()
        if mode == "count read back":
            k = int(count.item())
            v.set_lights_device(**{name: t[:k] for name, t in out.items()}, ready=ready, consumed=consumed)
        v.render_frame_device(state["gbs"][i % 2])

    return step, state


def source_rank_viewer(scene, bands, table=None, **config):
    """sharded.make_viewer's row-sharded viewer with light source rank 0, which must be set before bake (collective); a
    shadowed viewer sets its map table first."""
    v = viewer.Viewer(W, H, cuda_device=torch.cuda.current_device(), **config)
    v.set_directional(scene.dir_color, scene.dir_direction)
    rank = torch.distributed.get_rank()
    uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
    if rank == 0:
        uid.copy_(torch.frombuffer(bytearray(viewer.nccl_unique_id()), dtype=torch.uint8))
    torch.distributed.broadcast(uid, 0)
    v.init_collectives(uid.cpu().numpy().tobytes(), rank, torch.distributed.get_world_size())
    v.set_row_shards(bands, rank)
    if table is not None:
        v.set_light_shadow_map_table(table)
    v.set_light_source_rank(0)
    v.set_camera(scene.projection, scene.view)
    v.bake()
    return v


def live_count_runs(args, scene, dev, bands, card, distributed, rank, world):
    lights, cycle, lifetime, offset = particles()
    shadows, shadow_cfg = None, {}
    if args.shadows:
        maps, _, transforms = shadow_inputs(scene, lights)
        shadows = (transforms, (np.arange(PARTICLES) % SHADOW_MAPS).astype(np.int32), map_table(maps))
        shadow_cfg = dict(light_shadows=True, shadow_resolution=SHADOW_RES)
    closer = sharded.close_sharded if distributed else (lambda v: v.close())
    runs = []
    modes = ("every rank updates", "caller broadcast", "viewer push") if args.source_rank else ("device count", "count read back", "parked")
    for mode in modes:
        times = []
        for timestamps in (False, True):
            step, state = live_count_stepper(mode, lights, cycle, lifetime, offset, rank, shadows)
            state["dev"] = dev
            stream = torch.cuda.Stream()
            if mode == "viewer push":
                v = source_rank_viewer(scene, bands, shadows[2] if shadows else None, stream=stream.cuda_stream, timestamps=timestamps, **shadow_cfg)
            else:
                v = sharded.make_viewer(W, H, scene, synth.make_lights(0), scene.view, bands=bands, stream=stream.cuda_stream, timestamps=timestamps,
                                        **shadow_cfg)
            times.append(timed(v, stream, args.frames, step))
            if timestamps:
                t, c = v.collect_timings().get("clustering-bindless", (0.0, 0))
            else:
                kept = v.light_prep()[0]
            closer(v)
        ms, host_ms = times[0]
        run = {"capacity": PARTICLES, "kept_lights_last_frame": kept, "mode": mode, "ms": ms, "host_ms_per_frame": round(host_ms, 4),
               "clustering_pass_ms": round(t / max(c, 1), 4), "gpu": card}
        if distributed:
            gathered = [None] * world
            torch.distributed.all_gather_object(gathered, dict(run, rank=rank))
            run = {"capacity": PARTICLES, "mode": mode, "frames_per_s": round(args.frames / (max(g["ms"] for g in gathered) * 1e-3), 2),
                   "ranks": gathered}
        else:
            run["frames_per_s"] = round(args.frames / (ms * 1e-3), 2)
        runs.append(run)
    return runs


def map_table(maps):
    """The map pointers of the 64 cube maps of `maps`, in order: the table whose id k names map k."""
    return [maps[k].data_ptr() for k in range(SHADOW_MAPS)]


def timed(v, stream, frames, step):
    """(ms of `frames` frames of step(v, i) after FILL untimed ones, host ms per frame spent in the step calls)."""
    for i in range(FILL):
        step(v, i)
    v.sync()
    if torch.distributed.is_initialized():
        torch.distributed.barrier()
    a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a0.record(stream)
    t0 = time.perf_counter()
    for i in range(frames):
        step(v, FILL + i)
    host_ms = (time.perf_counter() - t0) * 1e3 / frames
    v.join_streams()
    a1.record(stream)
    torch.cuda.synchronize()
    return a0.elapsed_time(a1), host_ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--shadows", action="store_true", help="shadowed lights with static synthetic maps")
    ap.add_argument("--live-count", action="store_true", help="a compacted particle list whose length is known only on the device")
    ap.add_argument("--source-rank", action="store_true", help="with --live-count under torchrun: hand the list over from rank 0")
    ap.add_argument("--map-ids", action="store_true", help="with --shadows: also bind the shadowed lights by map id")
    args = ap.parse_args()
    if args.shadows and args.live_count and not args.source_rank:
        ap.error("--shadows with --live-count is the --source-rank workload (shadows by map id)")
    if args.map_ids and not args.shadows:
        ap.error("--map-ids is a form of --shadows")
    distributed = "RANK" in os.environ
    if args.source_rank and not (args.live_count and distributed):
        ap.error("--source-rank times the --live-count workload on row-sharded frames: run it with --live-count under torchrun")
    if distributed:
        rank, world, local = sharded.init_ranks(allow_shared=False)
    else:
        rank, world, local = 0, 1, 0
        torch.cuda.set_device(0)
    card = sharded.card(local)
    scene = synth.make_scene(W, H)
    dev = device_gbuffers(W, H)
    bands = viewer.band_partition(H, world) if world > 1 else None
    result = {"workload": "c3: 3840x2160, bloom + tonemap, device G-buffer every frame, lights moved on the device every frame" +
                          (f", every light shadowed ({SHADOW_RES}^2 cube maps, static)" if args.shadows else ""),
              "frames_timed": args.frames, "fill_frames": FILL, "ranks": world, "gpu": card, "runs": []}
    if args.live_count:
        result["workload"] = (f"c3: 3840x2160, bloom + tonemap, device G-buffer every frame, {PARTICLES} particle lights of which about half "
                              "are alive, compacted on the device every frame" + (", handed over from rank 0" if args.source_rank else "") +
                              (f", every light shadowed by map id ({SHADOW_RES}^2 cube maps, static)" if args.shadows else ""))
        result["runs"] = live_count_runs(args, scene, dev, bands, card, distributed, rank, world)
        if rank == 0:
            print(json.dumps(result), flush=True)
        if distributed:
            torch.distributed.destroy_process_group()
        return
    shadow_cfg = dict(light_shadows=True, shadow_resolution=SHADOW_RES) if args.shadows else {}

    for n in (4096, 16384):
        lights = light_list(n)
        if args.shadows:
            maps, pointers, transforms = shadow_inputs(scene, lights)
            shadow_args = dict(shadow_transforms=torch.from_numpy(transforms).cuda(), shadow_maps=torch.from_numpy(pointers).cuda())
            id_args = dict(shadow_transforms=shadow_args["shadow_transforms"],
                           shadow_map_ids=torch.from_numpy((np.arange(n) % SHADOW_MAPS).astype(np.int32)).cuda())
        modes = ("host lights", "device lights") + (("device lights by map id",) if args.map_ids else ())
        for mode in modes:
            def make(extra):
                v = sharded.make_viewer(W, H, scene, lights, scene.view, bands=bands, **shadow_cfg, **extra)
                if args.shadows:
                    v.set_light_shadow_maps(pointers.tolist())
                return v

            def stepper():
                state = {"viewer": None}
                d = cases.to_device(lights)
                phase = 0.01 * torch.sin(torch.arange(n, device="cuda", dtype=torch.float32))[:, None]

                def step(v, i):
                    if state["viewer"] is not v:
                        state["viewer"] = v
                        state["gbs"] = [v.device_gbuffer(*g) for g in dev]
                        if mode == "device lights":
                            v.set_lights_device(**d, **(shadow_args if args.shadows else {}))
                        elif mode == "device lights by map id":
                            v.set_light_shadow_map_table(map_table(maps))
                            v.set_lights_device(**d, **id_args)
                    d["position"].add_(phase)  # the lights' own per-frame update, on the device
                    if mode == "host lights":
                        v.set_lights(synth.Lights(lights.color, d["position"].cpu().numpy(), lights.is_point, lights.rot, lights.inner_cone,
                                                  lights.outer_cone))
                        if args.shadows:
                            v.set_light_shadow_maps(pointers.tolist())
                    v.render_frame_device(state["gbs"][i % 2])
                return step

            closer = sharded.close_sharded if distributed else (lambda v: v.close())
            stream = torch.cuda.Stream()
            v = make(dict(stream=stream.cuda_stream))
            ms, host_ms = timed(v, stream, args.frames, stepper())
            kept = v.light_prep()[0]
            closer(v)
            stream = torch.cuda.Stream()
            v = make(dict(stream=stream.cuda_stream, timestamps=True))
            timed(v, stream, args.frames, stepper())
            t, c = v.collect_timings().get("clustering-bindless", (0.0, 0))
            closer(v)
            run = {"input_lights": n, "kept_lights": kept, "mode": mode, "ms": ms, "host_ms_per_frame": round(host_ms, 4),
                   "clustering_pass_ms": round(t / max(c, 1), 4), "gpu": card}
            if distributed:
                gathered = [None] * world
                torch.distributed.all_gather_object(gathered, dict(run, rank=rank))
                run = {"input_lights": n, "mode": mode, "frames_per_s": round(args.frames / (max(g["ms"] for g in gathered) * 1e-3), 2),
                       "ranks": gathered}
            else:
                run["frames_per_s"] = round(args.frames / (ms * 1e-3), 2)
            result["runs"].append(run)
    if rank == 0:
        print(json.dumps(result), flush=True)
    if distributed:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
