#!/usr/bin/env python3
"""A row-sharded renderer whose camera moves every frame, under three band schedules: equal bands, fixed; bands cut
once from the row cost measured after the first frame; and measure + move every 16 frames (the live loop:
measure_row_cost -> band_partition_measured -> move_row_shards, no re-bake).  BASELINE config c3 by default (3840x2160,
4096 lights, bloom + tonemap).

    torchrun --nproc-per-node=<GPUs> tools/live_bands_times.py [--frames 200]

Per schedule: each rank's mean lighting-pass time (the viewer's timestamp events), frames/s of the slowest rank over
the whole loop (CUDA events on the rank's stream around every frame, measure and move of the loop), and the host time
of one measure call and of one move plus the frame that follows it, against one re-bake (set_row_shards + bake) plus
its first frame.  A frame after a move or a re-bake brings the host G-buffer; the others find it resident.

One rank per GPU: timings from ranks that share a GPU are not scaling numbers; --shared-ok runs anyway (for a check of
the tool itself; tests/sharded.py's init_ranks says how ranks share a GPU) and marks the result "one_rank_per_gpu": false.  The card's name and power limit come from a read-only
nvidia-smi query in the same run.
"""
import argparse
import json
import math
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import synth, viewer  # noqa: E402
from tests import sharded  # noqa: E402

EVERY = 16  # frames between two measure + move steps of the live schedule


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--lights", type=int, default=4096)
    ap.add_argument("--shared-ok", action="store_true", help="allow more ranks than GPUs (not a scaling number)")
    args = ap.parse_args()
    rank, world, local = sharded.init_ranks(allow_shared=args.shared_ok, refusal_hint=" (--shared-ok to run anyway)")
    w, h, frames = args.width, args.height, args.frames
    scene, lights, keep, gb = sharded.inputs(w, h, args.lights, spot_fraction=0.0)
    # the camera circles the origin: the light-dense rows move from frame to frame
    views = [synth.look_at_view((1.5 * math.sin(0.05 * i), 0.6 * math.cos(0.03 * i), 8.0 + 0.5 * math.sin(0.02 * i)), (0.0, 0.0, 0.0))
             for i in range(frames)]
    equal = viewer.band_partition(h, world)
    stream = torch.cuda.Stream()

    def make(bands):
        return sharded.make_viewer(w, h, scene, lights, views[0], bands, timestamps=True, stream=stream.cuda_stream)

    def measured_bands(v):
        return [tuple(int(y) for y in b) for b in viewer.band_partition_measured(h, w, world, v.measure_row_cost(), align=8)]

    def run(schedule):
        v = make(equal)
        bands = equal
        v.set_camera(scene.projection, views[0])
        v.render_frame(gb)
        v.sync()
        v.collect_timings()
        dist.barrier()
        measure_s, move_s = [], []
        a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a0.record(stream)
        for i in range(1, frames):
            moved = False
            if (schedule == "measured once" and i == 1) or (schedule == "measure + move every 16" and i % EVERY == 1):
                t0 = time.perf_counter()
                new = measured_bands(v)
                measure_s.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                v.move_row_shards(new)
                v.set_camera(scene.projection, views[i])
                v.render_frame(gb)
                v.sync()
                move_s.append(time.perf_counter() - t0)
                bands, moved = new, True
            if not moved:
                v.set_camera(scene.projection, views[i])
                v.render_frame(None)
        v.join_streams()
        a1.record(stream)
        torch.cuda.synchronize()
        ms = a0.elapsed_time(a1)
        lighting = v.collect_timings().get("lighting", (0.0, 0))
        sharded.close_sharded(v)
        mine = {"rank": rank, "band": bands[rank], "lighting_ms": round(lighting[0] / max(lighting[1], 1), 4), "loop_ms": round(ms, 2),
                "measure_host_ms": round(1e3 * float(np.median(measure_s)), 3) if measure_s else None,
                "move_and_frame_host_ms": round(1e3 * float(np.median(move_s)), 3) if move_s else None}
        every = [None] * world
        dist.all_gather_object(every, mine)
        slowest = max(r["loop_ms"] for r in every)
        return {"schedule": schedule, "moves": len(move_s), "frames_per_s": round((frames - 1) / (slowest * 1e-3), 2), "ranks": every}

    def rebake():
        # the alternative to a move: set the new layout, re-bake (histories and attachments restart), render its first frame
        v = make(equal)
        v.set_camera(scene.projection, views[0])
        v.render_frame(gb)
        v.sync()
        new = measured_bands(v)
        dist.barrier()
        t0 = time.perf_counter()
        v.set_row_shards(new, rank)
        v.bake()
        v.set_camera(scene.projection, views[1])
        v.render_frame(gb)
        v.sync()
        s = time.perf_counter() - t0
        sharded.close_sharded(v)
        every = [None] * world
        dist.all_gather_object(every, round(1e3 * s, 3))
        return every

    result = {"workload": f"{w}x{h}, {args.lights} lights, bloom + tonemap, camera moving every frame", "ranks": world, "frames": frames,
              "one_rank_per_gpu": world <= torch.cuda.device_count(), "gpu": sharded.card(local), "schedules": []}
    for schedule in ("equal, fixed", "measured once", "measure + move every 16"):
        result["schedules"].append(run(schedule))
    result["rebake_and_frame_host_ms"] = rebake()
    if rank == 0:
        print(json.dumps(result), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
