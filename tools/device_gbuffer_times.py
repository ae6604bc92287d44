#!/usr/bin/env python3
"""Frames/s of BASELINE config c3 (3840x2160, 4096 lights, bloom + tonemap) fed from a G-buffer in device memory.

    python tools/device_gbuffer_times.py [--frames 100]
    torchrun --nproc-per-node=<GPUs> tools/device_gbuffer_times.py [--frames 100]

On one GPU (no torchrun, or one rank) three modes over one window each:
- "device": two seeded G-buffers in device memory, alternated, so every frame copies a new G-buffer
  (grbh_viewer_render_frame_device);
- "host": the host-fed end-to-end path (a pinned host G-buffer uploaded every frame, grbh_viewer_render_frame);
- "resident": the G-buffer left resident (render_frame(None)).
Under torchrun, one rank per GPU, row-sharded frames fed per rank (every rank copies its input rows from its own device
G-buffer) and from rank 0 (which pushes every rank's rows through the G-buffer channel), over both exchange paths.

Each viewer renders 4 untimed frames, then --frames timed frames (CUDA events on the viewer's stream; the sharded rate is
that of the slowest rank).  The time of the "gbuffer" pass comes from a second run of the same frames with the
viewer's timestamps on, so that the events do not slow the timed window.  The card's name and power limit come from a
read-only nvidia-smi query in the same run and are printed beside every number.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import synth, viewer  # noqa: E402
from tests import sharded  # noqa: E402

FILL = 4
W, H, LIGHTS = 3840, 2160, 4096


def device_gbuffers(w, h):
    """Two seeded G-buffers as torch tensors on this device (host_gbuffer order, no motion vectors)."""
    out = []
    for seed in (synth.GBUFFER_SEED, synth.GBUFFER_SEED + 1):
        s = synth.make_scene(w, h, seed=seed)
        out.append([torch.from_numpy(np.ascontiguousarray(a).view(np.int32) if a.dtype == np.uint32 else
                                     (np.ascontiguousarray(a).view(np.int16) if a.dtype == np.uint16 else np.ascontiguousarray(a))).cuda()
                    for a in (s.albedo, s.normal, s.pbr, s.depth, s.emissive)])
    return out


def timed(v, stream, frames, step):
    """ms of `frames` frames of step(v, i) after FILL untimed ones."""
    for i in range(FILL):
        step(v, i)
    v.sync()
    if torch.distributed.is_initialized():
        torch.distributed.barrier()
    a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a0.record(stream)
    for i in range(frames):
        step(v, FILL + i)
    v.join_streams()
    a1.record(stream)
    torch.cuda.synchronize()
    return a0.elapsed_time(a1)


def run(make, frames, step):
    """(ms of the timed window, ms of the "gbuffer" pass per frame from a second run with timestamps)."""
    stream = torch.cuda.Stream()
    v = make(dict(stream=stream.cuda_stream))
    ms = timed(v, stream, frames, step)
    sharded.close_sharded(v) if torch.distributed.is_initialized() else v.close()
    stream = torch.cuda.Stream()
    v = make(dict(stream=stream.cuda_stream, timestamps=True))
    timed(v, stream, frames, step)
    t, c = v.collect_timings().get("gbuffer", (0.0, 0))
    sharded.close_sharded(v) if torch.distributed.is_initialized() else v.close()
    return ms, round(t / max(c, 1), 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100)
    args = ap.parse_args()
    distributed = "RANK" in os.environ
    if distributed:
        rank, world, local = sharded.init_ranks(allow_shared=False)
    else:
        rank, world, local = 0, 1, 0
        torch.cuda.set_device(0)
    card = sharded.card(local)
    scene, lights, keep, host_gb = sharded.inputs(W, H, LIGHTS, spot_fraction=0.0)
    pinned = [torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else (a.view(np.int16) if a.dtype == np.uint16 else a)).pin_memory() for a in keep]
    host_pinned = viewer.Viewer.host_gbuffer(*pinned)
    dev = device_gbuffers(W, H)
    result = {"workload": "c3: 3840x2160, 4096 lights, bloom + tonemap", "frames_timed": args.frames, "fill_frames": FILL, "ranks": world, "gpu": card,
              "runs": []}

    if world == 1:
        def make(extra):
            return sharded.make_viewer(W, H, scene, lights, scene.view, **extra)

        gbs = []

        def device_step(v, i):
            if not gbs:
                gbs.extend(v.device_gbuffer(*d) for d in dev)
            v.render_frame_device(gbs[i % 2])

        modes = {"device": device_step, "host": lambda v, i: v.render_frame(host_pinned),
                 "resident": lambda v, i: v.render_frame(host_pinned if i == 0 else None)}
        for name, step in modes.items():
            gbs.clear()
            ms, gbuffer_ms = run(make, args.frames, step)
            result["runs"].append({"mode": name, "frames_per_s": round(args.frames / (ms * 1e-3), 2), "gbuffer_pass_ms": gbuffer_ms, "gpu": card})
    else:
        bands = viewer.band_partition(H, world)
        for exchange in ("peer", "nccl"):
            os.environ["GRB_SHARD_EXCHANGE"] = exchange  # read when each channel's buffers are created
            for feeding in ("per rank", "from rank 0"):
                source = None if feeding == "per rank" else 0

                def make(extra, source=source):
                    v = viewer.Viewer(W, H, cuda_device=local, **extra)
                    v.set_directional(scene.dir_color, scene.dir_direction)
                    v.set_lights(lights)
                    uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
                    if rank == 0:
                        uid.copy_(torch.frombuffer(bytearray(viewer.nccl_unique_id()), dtype=torch.uint8))
                    torch.distributed.broadcast(uid, 0)
                    v.init_collectives(uid.cpu().numpy().tobytes(), rank, world)
                    v.set_row_shards(bands, rank)
                    if source is not None:
                        v.set_gbuffer_source_rank(source)
                    v.set_camera(scene.projection, scene.view)
                    v.bake()
                    return v

                gbs = []

                def step(v, i, source=source):
                    if not gbs:
                        gbs.extend(v.device_gbuffer(*d) for d in dev)
                    v.render_frame_device(None if source is not None and rank != source else gbs[i % 2])

                ms, gbuffer_ms = run(make, args.frames, step)
                gathered = [None] * world
                torch.distributed.all_gather_object(gathered, {"rank": rank, "band": bands[rank], "ms": ms, "gbuffer_pass_ms": gbuffer_ms, "gpu": card})
                slowest = max(g["ms"] for g in gathered)
                result["runs"].append({"exchange": exchange, "feeding": feeding, "frames_per_s": round(args.frames / (slowest * 1e-3), 2),
                                       "ranks": gathered})
    if rank == 0:
        print(json.dumps(result), flush=True)
    if distributed:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
