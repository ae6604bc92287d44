"""torchrun worker for tests/test_zq_gpu_present_sharded.py: renders row-sharded frames presented from one rank (the
bands pushed to it inside the C++ graph, by peer stores or NCCL as GRB_SHARD_EXCHANGE says) and, on rank 0, unsharded;
every frame the presenting rank reads must equal the unsharded one bit for bit, with rows {0, height}, and every other
rank must still read its band.

The presenting rank reads with read_output_async + wait_outputs(1), which keeps one readback in flight, into pinned
buffers; one run also sleeps on the host before every read, so the other ranks run ahead until the credit holds them.
The camera moves every frame, so a slot that is stale or torn shows up as a wrong frame.  Tonemap-only frames without
bloom have no d0 exchange that couples the ranks, so only the credit holds the producers back there; that config is
first checked sharded without presenting (its bands gathered with an all-reduce)."""
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import synth, viewer  # noqa: E402
from tests import sharded  # noqa: E402

FRAMES = 6
# (band layout, presenting rank: 0 or -1 = the last rank, sleep before each read)
RUNS = (("equal", 0, False), ("equal", -1, True), ("narrow", 0, False), ("narrow", -1, False))
CONFIGS = ("no AA", "FXAA", "SMAA Ultra", "TAA High + FXAA", "FSR 0.67 + RCAS", "HDR10 + TAA", "tonemap-only")


def main():
    w, h, n_lights = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
    rank, world, _ = sharded.init_ranks()
    scene, lights, keep, gb = sharded.inputs(w, h, n_lights, mv=sharded.motion_vectors(w, h, 5))
    views = [synth.look_at_view((0.15 * i, 0.1 * i, 8.0 - 0.2 * i), (0.0, 0.0, 0.0)) for i in range(FRAMES)]
    # Narrow bands are 16 rows: the FXAA tile kernel's result depends on a pixel's position in its 16-row tile, so a
    # band that starts off a multiple of 16 is not bit-exact without FSR (a known limitation of sharded FXAA), and at
    # FSR 0.67 8-row bands would leave rank 0 without render rows.
    layouts = {"equal": viewer.band_partition(h, world),
               "narrow": [(16 * r, 16 * (r + 1)) for r in range(world - 1)] + [(16 * (world - 1), h)]}

    ok = True
    for cfg in CONFIGS:
        reference = sharded.reference_frames(w, h, scene, lights, gb, views, **sharded.config_args(cfg))

        if cfg == "tonemap-only":
            # sharded without presenting first: the bands alone must assemble the unsharded frame
            for name, bands in layouts.items():
                vs = sharded.make_viewer(w, h, scene, lights, views[0], bands, **sharded.config_args(cfg))
                ok &= sharded.check_frames(vs, gb, scene.projection, views, bands, reference, f"{cfg} {name}",
                                           "tonemap-only sharded == single GPU")
                sharded.close_sharded(vs)

        for name, p, sleep in RUNS:
            bands = layouts[name]
            present = p % world
            vs = sharded.make_viewer(w, h, scene, lights, views[0], bands, present, **sharded.config_args(cfg))
            frames = torch.zeros((FRAMES, h, w), dtype=torch.int32).pin_memory()
            rows = []
            for i in range(FRAMES):
                vs.set_camera(scene.projection, views[i])
                vs.render_frame(gb if i == 0 else None)
                if rank == present:
                    if sleep:
                        time.sleep(0.02)
                    rows.append(vs.read_output_async(frames[i]))
                    vs.wait_outputs(1)
                else:
                    out = np.zeros((h, w), np.uint32)
                    ok &= vs.read_output(out) == tuple(bands[rank])
            vs.wait_outputs(0)
            ok &= all(r == (0, h) for r in rows)
            sharded.close_sharded(vs)
            got = sharded.assemble(frames.numpy(), present)
            if rank == 0:
                for i in range(FRAMES):
                    same = np.array_equal(got[i], reference[i])
                    print(f"{cfg} {name} P={present}{' sleep' if sleep else ''} frame {i}: presented == single GPU: {same}", flush=True)
                    ok &= same
    sharded.finish(ok)


if __name__ == "__main__":
    main()
