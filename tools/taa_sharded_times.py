#!/usr/bin/env python3
"""Frames/s and per-pass GPU times of BASELINE config c5 (3840x2160, 4096 lights, TAA High + FXAA with history),
row-sharded over every rank and, on rank 0, unsharded.

    torchrun --nproc-per-node=<GPUs> tools/taa_sharded_times.py [--frames 50]

One rank per GPU: timings from ranks that share a GPU are not scaling numbers.  Each viewer renders 4 untimed frames
that fill the pipeline, then --frames timed frames with the G-buffer resident (CUDA events on the rank's stream; the
sharded rate is that of the slowest rank).  Per-pass times are the viewer's timestamp events, averaged over the
timed frames.  The card's name and power limit come from a read-only nvidia-smi query in the same run.
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import viewer  # noqa: E402
from tests import sharded  # noqa: E402

FILL = 4


def run(scene, lights, gb, frames, bands):
    w, h = scene.width, scene.height
    stream = torch.cuda.Stream()
    v = sharded.make_viewer(w, h, scene, lights, scene.view, bands, post_aa=viewer.AA_TAA_HIGH_PLUS_FXAA, timestamps=True,
                            stream=stream.cuda_stream)
    v.render_frame(gb)
    for _ in range(FILL - 1):
        v.render_frame(None)
    v.sync()
    v.collect_timings()
    if bands:
        dist.barrier()
    a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a0.record(stream)
    for _ in range(frames):
        v.render_frame(None)
    v.join_streams()
    a1.record(stream)
    torch.cuda.synchronize()
    ms = a0.elapsed_time(a1)
    passes = {k: round(t / max(c, 1), 4) for k, (t, c) in v.collect_timings().items()}
    if bands:
        sharded.close_sharded(v)
    else:
        v.close()
    return ms, passes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50)
    args = ap.parse_args()
    rank, world, local = sharded.init_ranks(allow_shared=False)
    w, h, n_lights = 3840, 2160, 4096
    scene, lights, keep, gb = sharded.inputs(w, h, n_lights, spot_fraction=0.0, mv=sharded.c5_motion_vectors(w, h))

    result = {"workload": "c5 3840x2160 TAA(q2) + FXAA, 4096 lights, G-buffer resident", "ranks": world, "frames_timed": args.frames,
              "fill_frames": FILL, "gpu": sharded.card(local)}
    if rank == 0:
        ms, passes = run(scene, lights, gb, args.frames, None)
        result["unsharded"] = {"frames_per_s": round(args.frames / (ms * 1e-3), 2), "pass_ms": passes}
    dist.barrier()
    bands = viewer.band_partition(h, world)
    ms, passes = run(scene, lights, gb, args.frames, bands)
    gathered = [None] * world
    dist.all_gather_object(gathered, {"rank": rank, "band": bands[rank], "ms": ms, "pass_ms": passes, "gpu": sharded.card(local)})
    if rank == 0:
        slowest = max(g["ms"] for g in gathered)
        result["sharded"] = {"frames_per_s": round(args.frames / (slowest * 1e-3), 2), "ranks": gathered}
        print(json.dumps(result), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
