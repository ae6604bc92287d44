#!/usr/bin/env python3
"""GPU time of grb_deferred_lighting_blocks (the pairs kernel, deferred_lighting2_kernel) at BASELINE config 3:
3840x2160, 4096 point lights.

    python tools/lighting_blocks_time.py [--iters 50] [--repeats 5]

The cluster is built once; each repeat times --iters back-to-back launches on the current stream with CUDA events,
after 5 untimed ones, and prints the mean per launch.  The card's name and power limit come from a read-only
nvidia-smi query in the same run.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    from granite_b200 import capi, harness
    from oracle import pyoracle as oracle
    from tests import common, sharded

    capi.lib()
    capi.init()
    oracle.build(ref=False)
    scene, cam, _, prep = common.build_case(oracle, 3840, 2160, 4096, 0.0)
    dev = harness.ClusterDevice(prep.records, prep.model, prep.type_mask, prep.z_ranges, prep.params, prep.res)
    gcam = harness.camera_struct(cam)
    dev.build(gcam)
    gb = harness.GBufferDevice(scene)
    hdr = gb.emissive.clone()
    for _ in range(5):
        harness.deferred_lighting_blocks(gb, gcam, dev, hdr)
    ms = []
    for _ in range(args.repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            harness.deferred_lighting_blocks(gb, gcam, dev, hdr)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b) / args.iters)
    print(json.dumps({"kernel": "grb_deferred_lighting_blocks", "size": "3840x2160", "lights": prep.n, "ms_per_launch": ms,
                      "card": sharded.card(0)}))


if __name__ == "__main__":
    main()
