"""torchrun worker for tests/test_zn_gpu_live_bands.py: row-sharded viewers whose band cuts move between frames
(grbh_viewer_move_row_shards, no re-bake) against the unsharded viewer on rank 0, with the exchanges inside the C++ graph
(peer-memory stores or NCCL, as GRB_SHARD_EXCHANGE says).

Every run renders FRAMES frames with a moving camera.  The cuts move after frame 2 (each cut 16 rows down) and after
frame 5 (to a layout with one 16-row band in the middle); every cut stays on a multiple of 16 rows, which sharded FXAA
needs to stay bit-exact.  Every frame, assembled from the bands (or read on the presenting rank), must equal the
unsharded frame bit for bit -- also the frames right after a move, which read the TAA history and the bloom feedback
written under the old layout.  Right after a move, render_frame(None), render_frame without motion vectors under TAA,
read_output and measure_row_cost are refused; the frame that brings the G-buffer and the resident frames after it must
be right.  Where a run measures, the sharded measure_row_cost after a frame must equal the unsharded one bit for bit on
every rank; the last run moves its cuts to band_partition_measured of that measurement, which must give every rank the
same bands."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import synth, viewer  # noqa: E402
from tests import sharded  # noqa: E402

FRAMES = 8
MOVES = (3, 6)  # frames rendered first on a new layout
# (config, presenting rank: None = off, -1 = the last rank; whether the run measures the row cost; the layouts)
RUNS = (("no AA", None, True, "fixed"), ("FXAA", None, False, "fixed"), ("SMAA Ultra", None, False, "fixed"),
        ("TAA High + FXAA", None, False, "fixed"), ("FSR 0.67 + RCAS", None, True, "fixed"), ("HDR10 + TAA", None, False, "fixed"),
        ("TAA High + FXAA", -1, False, "fixed"), ("no AA", None, True, "measured"))


def uses_taa(name):
    return "TAA" in name


def expect_refusal(fn, what):
    try:
        fn()
    except Exception as e:  # noqa: BLE001 -- the binding raises capi.GrbError
        return "grbh_viewer_move_row_shards" in str(e)
    print(f"{what} right after a move was not refused", flush=True)
    return False


def main():
    w, h, n_lights = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
    rank, world, _ = sharded.init_ranks()
    scene, lights, keep, gb = sharded.inputs(w, h, n_lights, mv=sharded.motion_vectors(w, h, 5))
    gb_no_mv = viewer.Viewer.host_gbuffer(*keep[:5])
    views = [synth.look_at_view((0.15 * i, 0.1 * i, 8.0 - 0.2 * i), (0.0, 0.0, 0.0)) for i in range(FRAMES)]
    equal = viewer.band_partition(h, world)
    assert all(y0 % 16 == 0 for y0, _ in equal) and all(y1 + 16 < h for _, y1 in equal[:-1])
    shifted = [(0 if r == 0 else y0 + 16, h if r == world - 1 else y1 + 16) for r, (y0, y1) in enumerate(equal)]
    # one 16-row band in the middle (rank 1); the others share the rest on multiples of 16
    mid = (h // 2) // 16 * 16
    narrow = [(0, mid), (mid, mid + 16)]
    rest = (h - mid - 16) // 16
    for r in range(2, world):
        y0 = narrow[-1][1]
        narrow.append((y0, h if r == world - 1 else y0 + 16 * max(rest // (world - 2), 1)))
    fixed_layouts = {0: equal, MOVES[0]: shifted, MOVES[1]: narrow}

    ok = True
    references = {}
    for cfg, present, measure, layouts in RUNS:
        if cfg not in references:
            # the unsharded frames (and row costs) on rank 0, shared with every rank
            frames, costs = [], []
            if rank == 0:
                v1 = sharded.make_viewer(w, h, scene, lights, views[0], **sharded.config_args(cfg))
                for ref, _ in sharded.frames(v1, gb, scene.projection, views):
                    frames.append(ref)
                    costs.append(v1.measure_row_cost())
                v1.close()
            shared = [costs]
            dist.broadcast_object_list(shared, 0)
            references[cfg] = (frames, shared[0])
        reference, ref_costs = references[cfg]

        p = None if present is None else present % world
        bands = equal
        vs = sharded.make_viewer(w, h, scene, lights, views[0], bands, p, **sharded.config_args(cfg))
        label = f"{cfg} {layouts}{'' if p is None else f' P={p}'}"
        for i in range(FRAMES):
            if i in MOVES:
                if layouts == "fixed":
                    bands = fixed_layouts[i]
                else:
                    cost = vs.measure_row_cost()
                    same = np.array_equal(cost, ref_costs[i - 1])
                    bands = [tuple(int(y) for y in b) for b in viewer.band_partition_measured(h, w, world, cost, align=8)]
                    every = [None] * world
                    dist.all_gather_object(every, bands)
                    agree = all(b == bands for b in every)
                    if rank == 0:
                        print(f"{label} after frame {i - 1}: measured bands identical on every rank: {agree} {bands}", flush=True)
                    ok &= agree and same
                vs.move_row_shards(bands)
                ok &= expect_refusal(lambda: vs.render_frame(None), "render_frame(None)")
                if uses_taa(cfg):
                    ok &= expect_refusal(lambda: vs.render_frame(gb_no_mv), "render_frame without motion vectors")
                ok &= expect_refusal(lambda: vs.read_output(np.zeros((h, w), np.uint32)), "read_output")
                ok &= expect_refusal(vs.measure_row_cost, "measure_row_cost")
            vs.set_camera(scene.projection, views[i])
            vs.render_frame(gb if i == 0 or i in MOVES else None)
            out = np.zeros((h, w), np.uint32)
            rows = vs.read_output(out)
            ok &= rows == ((0, h) if rank == p else tuple(bands[rank]))
            full = sharded.assemble(out, p)
            if rank == 0:
                same = np.array_equal(full, reference[i])
                print(f"{label} frame {i} bands {bands}: live bands == single GPU: {same}", flush=True)
                ok &= same
            if measure and layouts == "fixed" and i in (1, MOVES[0] + 1, MOVES[1] + 1):
                cost = vs.measure_row_cost()
                same = torch.tensor([1 if np.array_equal(cost, ref_costs[i]) else 0], device="cuda")
                dist.all_reduce(same, op=dist.ReduceOp.MIN)
                if rank == 0:
                    print(f"{label} frame {i}: sharded row cost == single GPU on every rank: {bool(same.item())}", flush=True)
                ok &= bool(same.item())
        sharded.close_sharded(vs)
    sharded.finish(ok)


if __name__ == "__main__":
    main()
