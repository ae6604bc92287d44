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
import subprocess
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FILL = 4


def card(index):
    q = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() or "unknown"


def run(viewer, scene, lights, gb, local, frames, bands, rank, world):
    w, h = scene.width, scene.height
    stream = torch.cuda.Stream()
    v = viewer.Viewer(w, h, post_aa=viewer.AA_TAA_HIGH_PLUS_FXAA, cuda_device=local, timestamps=True, stream=stream.cuda_stream)
    v.set_camera(scene.projection, scene.view)
    v.set_directional(scene.dir_color, scene.dir_direction)
    v.set_lights(lights)
    if bands:
        uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
        if rank == 0:
            uid.copy_(torch.frombuffer(bytearray(viewer.nccl_unique_id()), dtype=torch.uint8))
        dist.broadcast(uid, 0)
        v.init_collectives(uid.cpu().numpy().tobytes(), rank, world)
        v.set_row_shards(bands, rank)
    v.bake()
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
    v.close()
    return ms, passes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50)
    args = ap.parse_args()
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    if world > torch.cuda.device_count():
        raise SystemExit(f"{world} ranks on {torch.cuda.device_count()} GPUs: one rank per GPU is needed for a scaling number")
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from granite_b200 import synth, viewer

    w, h, n_lights = 3840, 2160, 4096
    scene = synth.make_scene(w, h)
    lights = synth.make_lights(n_lights, aspect=w / h)
    # as bench.py's c5: zero motion vectors on 90 % of the pixels, <= 2 px on the rest
    rng = np.random.default_rng(5)
    mv = np.zeros((h, w, 2), np.float16)
    m = rng.random((h, w)) < 0.1
    mv[m] = (rng.uniform(-2, 2, size=(int(m.sum()), 2)) / np.array([w, h])).astype(np.float16)
    keep = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, scene.emissive)]
    keep.append(np.ascontiguousarray(mv).view(np.uint32).reshape(h, w))
    gb = viewer.Viewer.host_gbuffer(*keep)

    result = {"workload": "c5 3840x2160 TAA(q2) + FXAA, 4096 lights, G-buffer resident", "ranks": world, "frames_timed": args.frames,
              "fill_frames": FILL, "gpu": card(local)}
    if rank == 0:
        ms, passes = run(viewer, scene, lights, gb, local, args.frames, None, rank, world)
        result["unsharded"] = {"frames_per_s": round(args.frames / (ms * 1e-3), 2), "pass_ms": passes}
    dist.barrier()
    bands = viewer.band_partition(h, world)
    ms, passes = run(viewer, scene, lights, gb, local, args.frames, bands, rank, world)
    gathered = [None] * world
    dist.all_gather_object(gathered, {"rank": rank, "band": bands[rank], "ms": ms, "pass_ms": passes, "gpu": card(local)})
    if rank == 0:
        slowest = max(g["ms"] for g in gathered)
        result["sharded"] = {"frames_per_s": round(args.frames / (slowest * 1e-3), 2), "ranks": gathered}
        print(json.dumps(result), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
