"""Diagnostic (debug build of the library only, -DGRB_LIGHTING_DEBUG): per-block cycles and
per-warp finish times of the persistent lighting kernel at the bench configuration."""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from granite_b200 import capi, harness, synth
from oracle import pyoracle as oracle
from tests import common

oracle.build(ref=False)
capi.lib(); capi.init()
w, h, n = 3840, 2160, 4096
scene, cam, lights, prep = common.build_case(oracle, w, h, n, 0.0)
dev = harness.ClusterDevice(prep.records, prep.model, prep.type_mask, prep.z_ranges, prep.params, prep.res)
gcam = harness.camera_struct(cam)
dev.build(gcam)
gb = harness.GBufferDevice(scene)
sched = harness.lighting_schedule(h)
sms = torch.cuda.get_device_properties(0).multi_processor_count  # one persistent CTA per SM
for it in range(4):
    hdr = gb.emissive.clone()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    harness.deferred_lighting(gb, gcam, dev, hdr, schedule=sched if it >= 1 else None)
    e1.record(); torch.cuda.synchronize()
    blocks = np.zeros((240 * 540, 2), np.uint32); warps = np.zeros((256 * 16, 2), np.uint32)
    capi.lib().grb_debug_lighting_dump(C.c_void_p(blocks.ctypes.data), C.c_void_p(warps.ctypes.data))
    items = np.zeros(256 * 16, np.uint32); last = np.zeros((256 * 16, 8, 2), np.uint32)
    capi.lib().grb_debug_lighting_dump2(C.c_void_p(items.ctypes.data), C.c_void_p(last.ctypes.data))
    wv = warps[: sms * 16]
    start = wv[:, 0].astype(np.int64); start -= start.min()
    end = start + wv[:, 1]
    cyc = blocks[:, 0].astype(np.float64).reshape(540, 240)
    print(f"iter {it} ({'scheduled' if it >= 2 else 'raster' if it == 0 else 'first scheduled (raster order)'}): kernel {e0.elapsed_time(e1) * 1e3:.0f} us; "
          f"warp start spread {start.max() / 1e3:.1f} us; warp end min/median/p90/max = {end.min() / 1e3:.0f}/{np.median(end) / 1e3:.0f}/{np.percentile(end, 90) / 1e3:.0f}/{end.max() / 1e3:.0f} us")
    per_sm = end.reshape(sms, 16).max(1)
    print("   per-SM finish min/median/max us:", per_sm.min() / 1e3, np.median(per_sm) / 1e3, per_sm.max() / 1e3)
    print(f"   block cycles: mean {cyc.mean():.0f} median {np.median(cyc):.0f} p99 {np.percentile(cyc, 99):.0f} max {cyc.max():.0f}; rows with mean > 30000: {(cyc.mean(1) > 30000).sum()}")
    top = np.argsort(-cyc.reshape(-1))[:5]
    print("   slowest blocks (by, bx, cycles, start us):", [(int(t // 240), int(t % 240), int(blocks[t, 0]), round(blocks[t, 1] / 1e3, 1)) for t in top])
    slow = np.argsort(-end)[:4]
    for wq in slow:
        k = int(items[wq]); ring = [tuple(int(v) for v in last[wq, (k - j) & 7]) for j in range(min(k, 8))]
        print(f"   straggler warp {wq} (sm {wq // 16}): end {end[wq] / 1e3:.1f} us, {k} items; last fetches (item, us): {[(a, round(b / 1e3, 1)) for a, b in ring]}")
    print("   items per warp min/median/max:", items[:sms * 16].min(), np.median(items[:sms * 16]), items[:sms * 16].max())
    late = np.argsort(-(blocks[:, 1].astype(np.int64)))[:5]
    print("   latest-started blocks (by, bx, cycles, start us):", [(int(t // 240), int(t % 240), int(blocks[t, 0]), round(blocks[t, 1] / 1e3, 1)) for t in late])
