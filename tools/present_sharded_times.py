#!/usr/bin/env python3
"""Frames/s of BASELINE configs c3 (3840x2160, 4096 lights, bloom + tonemap) and c5 (the same with TAA High + FXAA)
row-sharded over every rank, with presenting from rank 0 off and on, over both exchange paths (peer-memory stores and
NCCL), and the time of the "present" pass on every rank.

    torchrun --nproc-per-node=<GPUs> tools/present_sharded_times.py [--frames 50]

One rank per GPU: timings from ranks that share a GPU are not scaling numbers.  Each viewer renders 4 untimed frames
that fill the pipeline, then --frames timed frames with the G-buffer resident (CUDA events on the rank's stream; the
sharded rate is that of the slowest rank).  No host readback runs in the timed window, so the numbers are those of the
frames and their pushes alone.  Per-pass times are the viewer's timestamp events, averaged over the timed frames.  The
card's name and power limit come from a read-only nvidia-smi query in the same run.
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


def run(viewer, scene, lights, gb, local, frames, bands, rank, world, post_aa, present_rank):
    w, h = scene.width, scene.height
    stream = torch.cuda.Stream()
    v = viewer.Viewer(w, h, post_aa=post_aa, cuda_device=local, timestamps=True, stream=stream.cuda_stream)
    v.set_camera(scene.projection, scene.view)
    v.set_directional(scene.dir_color, scene.dir_direction)
    v.set_lights(lights)
    uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
    if rank == 0:
        uid.copy_(torch.frombuffer(bytearray(viewer.nccl_unique_id()), dtype=torch.uint8))
    dist.broadcast(uid, 0)
    v.init_collectives(uid.cpu().numpy().tobytes(), rank, world)
    v.set_row_shards(bands, rank)
    v.set_present_rank(present_rank)
    v.bake()
    v.render_frame(gb)
    for _ in range(FILL - 1):
        v.render_frame(None)
    v.sync()
    v.collect_timings()
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
    # every rank's pushes and flag stores have landed before any rank frees its channel
    v.sync()
    dist.barrier()
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
    bands = viewer.band_partition(h, world)

    result = {"workload": "3840x2160, 4096 lights, G-buffer resident, presenting rank 0", "ranks": world, "frames_timed": args.frames,
              "fill_frames": FILL, "gpu": card(local), "runs": []}
    for workload, post_aa in (("c3", viewer.AA_NONE), ("c5", viewer.AA_TAA_HIGH_PLUS_FXAA)):
        for exchange in ("peer", "nccl"):
            # read when each channel's buffers are created, so it applies to the viewers made below
            os.environ["GRB_SHARD_EXCHANGE"] = exchange
            for present_rank in (-1, 0):
                ms, passes = run(viewer, scene, lights, gb, local, args.frames, bands, rank, world, post_aa, present_rank)
                gathered = [None] * world
                dist.all_gather_object(gathered, {"rank": rank, "band": bands[rank], "ms": ms, "present_ms": passes.get("present"), "gpu": card(local)})
                slowest = max(g["ms"] for g in gathered)
                result["runs"].append({"workload": workload, "exchange": exchange, "present_rank": present_rank,
                                       "frames_per_s": round(args.frames / (slowest * 1e-3), 2), "ranks": gathered})
    if rank == 0:
        print(json.dumps(result), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
