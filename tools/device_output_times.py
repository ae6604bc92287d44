#!/usr/bin/env python3
"""Frames/s of BASELINE config c3 (3840x2160, 4096 lights, bloom + tonemap) fed from device G-buffers, by where each
frame goes: into a ring of caller-owned output images (grbh_viewer_set_output_images / grbh_viewer_acquire_output),
left in the graph-owned image, or read back to host memory.

    python tools/device_output_times.py [--frames 100]
    torchrun --nproc-per-node=<GPUs> tools/device_output_times.py [--frames 100]

Every frame copies a new G-buffer: two seeded device G-buffers alternate, as in tools/device_gbuffer_times.py.
On one GPU (no torchrun, or one rank) three modes over one window each:
- "ring": a ring of 3 output images; a consumer stream waits on each frame's `rendered` event and records the image's
  `acquired` event, as a compositor that hands the image on would;
- "graph-owned": the output left in the graph-owned image;
- "readback": read_output_async of every frame into pinned host memory (at most 2 in flight).
Under torchrun, one rank per GPU, row-sharded frames on both exchange paths: each rank's band into a ring of its own or
left in place, and presented to rank 0 with or without a ring there.  The sharded rate is that of the slowest rank.

Each viewer renders 4 untimed frames, then --frames timed frames (CUDA events on the viewer's stream).  The time of the
final pass ("tonemap" on one GPU, "present" on the presenting rank) comes from a second run of the same frames with
the viewer's timestamps on, so that the events do not slow the timed window.  The card's name and power limit come
from a read-only nvidia-smi query in the same run and are printed beside every number.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import viewer  # noqa: E402
from tests import sharded  # noqa: E402
from tools.device_gbuffer_times import FILL, H, LIGHTS, W, device_gbuffers, timed  # noqa: E402

RING = 3


class Ring:
    """A ring of output images on this device and the consumer that releases each one once its frame is rendered."""

    def __init__(self):
        self.images = [torch.zeros((H, W), dtype=torch.int32, device="cuda") for _ in range(RING)]
        self.acquired = [torch.cuda.Event() for _ in range(RING)]
        self.rendered = [torch.cuda.Event() for _ in range(RING)]
        self.consumer = torch.cuda.Stream()

    def acquire(self, v, i):
        k = i % RING
        v.acquire_output(k, acquired=self.acquired[k], rendered=self.rendered[k])
        return k

    def release(self, k):
        self.consumer.wait_event(self.rendered[k])
        self.acquired[k].record(self.consumer)


def run(make, frames, step, pass_name):
    """(ms of the timed window, ms of `pass_name` per frame from a second run with timestamps, 0 where it did not run)."""
    closer = sharded.close_sharded if torch.distributed.is_initialized() else (lambda v: v.close())
    stream = torch.cuda.Stream()
    v = make(dict(stream=stream.cuda_stream))
    ms = timed(v, stream, frames, step)
    closer(v)
    stream = torch.cuda.Stream()
    v = make(dict(stream=stream.cuda_stream, timestamps=True))
    timed(v, stream, frames, step)
    t, c = v.collect_timings().get(pass_name, (0.0, 0))
    closer(v)
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
    scene, lights, _, _ = sharded.inputs(W, H, LIGHTS, spot_fraction=0.0)
    dev = device_gbuffers(W, H)
    result = {"workload": "c3: 3840x2160, 4096 lights, bloom + tonemap, device G-buffer every frame", "frames_timed": args.frames, "fill_frames": FILL,
              "ranks": world, "gpu": card, "runs": []}

    def stepper(ring=None, readback=None, holds_ring=True):
        """step(v, i) of one mode: a new viewer gets the device G-buffers (and the ring) on its first frame."""
        state = {"viewer": None, "gbs": []}

        def step(v, i):
            if state["viewer"] is not v:
                state["viewer"] = v
                state["gbs"] = [v.device_gbuffer(*d) for d in dev]
                if ring is not None and holds_ring:
                    v.set_output_images(ring.images)
            k = ring.acquire(v, i) if ring is not None and holds_ring else None
            v.render_frame_device(state["gbs"][i % 2])
            if k is not None:
                ring.release(k)
            if readback is not None:
                v.read_output_async(readback[i % 3])
                v.wait_outputs(2)
        return step

    if world == 1:
        def make(extra):
            return sharded.make_viewer(W, H, scene, lights, scene.view, **extra)

        pinned = [torch.zeros((H, W), dtype=torch.int32, pin_memory=True) for _ in range(3)]
        modes = {"ring": stepper(ring=Ring()), "graph-owned": stepper(), "readback": stepper(readback=pinned)}
        for name, step in modes.items():
            ms, tonemap_ms = run(make, args.frames, step, "tonemap")
            result["runs"].append({"mode": name, "frames_per_s": round(args.frames / (ms * 1e-3), 2), "tonemap_pass_ms": tonemap_ms, "gpu": card})
    else:
        bands = viewer.band_partition(H, world)
        for exchange in ("peer", "nccl"):
            os.environ["GRB_SHARD_EXCHANGE"] = exchange  # read when each channel's buffers are created
            for present in (None, 0):
                for use_ring in (True, False):
                    def make(extra, present=present):
                        return sharded.make_viewer(W, H, scene, lights, scene.view, bands=bands, present_rank=present, **extra)

                    step = stepper(ring=Ring() if use_ring else None, holds_ring=present is None or rank == present)
                    ms, present_ms = run(make, args.frames, step, "present")
                    gathered = [None] * world
                    torch.distributed.all_gather_object(gathered, {"rank": rank, "band": bands[rank], "ms": ms, "present_pass_ms": present_ms, "gpu": card})
                    slowest = max(g["ms"] for g in gathered)
                    output = ("band per rank" if present is None else f"presented to rank {present}") + (" into a ring" if use_ring else ", left in place")
                    result["runs"].append({"exchange": exchange, "output": output, "frames_per_s": round(args.frames / (slowest * 1e-3), 2),
                                           "ranks": gathered})
    if rank == 0:
        print(json.dumps(result), flush=True)
    if distributed:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
