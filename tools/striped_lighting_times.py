#!/usr/bin/env python3
"""Lighting in stripes against band schedules on a row-sharded renderer whose camera moves every frame: BASELINE
config c3 by default (3840x2160, 4096 lights, bloom + tonemap).  Schedules: equal bands; bands cut once from the row
cost measured after the first frame; measure + move every 16 frames (measure_row_cost -> band_partition_measured ->
move_row_shards); and equal bands lit in stripes of 16, 32 and 64 rows (set_lighting_stripes).

    torchrun --nproc-per-node=<GPUs> tools/striped_lighting_times.py [--frames 200] [--warmup 8]

Each schedule renders --warmup frames to fill the pipeline, then times a window of --frames frames: per rank the mean
`lighting` and `lighting-exchange` pass times (the viewer's timestamp events), and frames/s of the slowest rank over
the window (CUDA events on the rank's stream around every frame, measure and move of the window).  A frame after a
move brings the host G-buffer; the others find it resident.  One rank per GPU: timings from ranks that share a GPU are
not scaling numbers, so the tool refuses to run that way.  The card's name and power limit come from a read-only
nvidia-smi query in the same run.
"""
import argparse
import json
import math
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import synth, viewer  # noqa: E402
from tests import sharded  # noqa: E402

EVERY = 16  # frames between two measure + move steps of the live schedule
SCHEDULES = ("equal", "measured once", "measure + move every 16", "stripes 16", "stripes 32", "stripes 64")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--lights", type=int, default=4096)
    args = ap.parse_args()
    rank, world, local = sharded.init_ranks(allow_shared=False)
    w, h = args.width, args.height
    total = args.warmup + args.frames
    scene, lights, keep, gb = sharded.inputs(w, h, args.lights, spot_fraction=0.0)
    # the camera circles the origin: the light-dense rows move from frame to frame
    views = [synth.look_at_view((1.5 * math.sin(0.05 * i), 0.6 * math.cos(0.03 * i), 8.0 + 0.5 * math.sin(0.02 * i)), (0.0, 0.0, 0.0))
             for i in range(total)]
    equal = viewer.band_partition(h, world)
    stream = torch.cuda.Stream()

    def run(schedule):
        v = sharded.make_viewer(w, h, scene, lights, views[0], equal, timestamps=True, stream=stream.cuda_stream)
        if schedule.startswith("stripes"):
            v.set_lighting_stripes(int(schedule.split()[1]))
            v.bake()
        a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for i in range(total):
            if i == args.warmup:
                v.join_streams()
                torch.cuda.synchronize()
                v.collect_timings()
                dist.barrier()
                a0.record(stream)
            move = i > 0 and ((schedule == "measured once" and i == 1) or (schedule == "measure + move every 16" and i % EVERY == 1))
            if move:
                cost = v.measure_row_cost()
                v.move_row_shards([tuple(int(y) for y in b) for b in viewer.band_partition_measured(h, w, world, cost, align=8)])
            v.set_camera(scene.projection, views[i])
            v.render_frame(gb if i == 0 or move else None)
        v.join_streams()
        a1.record(stream)
        torch.cuda.synchronize()
        t = v.collect_timings()
        sharded.close_sharded(v)
        mean = lambda name: round(t[name][0] / max(t[name][1], 1), 4) if name in t else None
        mine = {"rank": rank, "lighting_ms": mean("lighting"), "lighting_exchange_ms": mean("lighting-exchange"), "window_ms": round(a0.elapsed_time(a1), 2)}
        every = [None] * world
        dist.all_gather_object(every, mine)
        slowest = max(r["window_ms"] for r in every)
        return {"schedule": schedule, "frames_per_s": round(args.frames / (slowest * 1e-3), 2), "ranks": every}

    result = {"workload": f"{w}x{h}, {args.lights} lights, bloom + tonemap, camera moving every frame", "ranks": world, "frames": args.frames,
              "warmup": args.warmup, "gpu": sharded.card(local), "schedules": [run(s) for s in SCHEDULES]}
    if rank == 0:
        print(json.dumps(result), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
