"""torchrun worker for tests/test_zj_gpu_lighting_stripes_sharded.py: row-sharded viewers lit in stripes
(grbh_viewer_set_lighting_stripes) against the unsharded viewer on rank 0, with the exchanges inside the C++ graph
(peer-memory stores or NCCL, as GRB_SHARD_EXCHANGE says).

Every run renders FRAMES frames with a moving camera, and the band cuts move 16 rows down after frame MOVE - 1
(grbh_viewer_move_row_shards): the stripes a rank lights do not depend on the bands, the rows it pushes and receives
do.  Every frame, assembled from the bands (or read on the presenting rank), must equal the unsharded frame bit for
bit.  After the first frame and after the first frame on the moved bands, the striped measure_row_cost must equal the
unsharded one on every rank."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import synth, viewer  # noqa: E402
from tests import sharded  # noqa: E402

FRAMES = 8
MOVE = 4  # the first frame rendered on the moved bands
STRIPES = (8, 64)
# (config, presenting rank: None = off, -1 = the last rank)
CONFIGS = (("no AA", None), ("FXAA", None), ("SMAA Ultra", None), ("TAA High + FXAA", None), ("HDR10 + TAA", None), ("tonemap-only", None),
           ("RGBA16F", None), ("TAA High + FXAA", -1))


def config_args(name):
    return dict(render_target_fp16=True) if name == "RGBA16F" else sharded.config_args(name)


def main():
    w, h, n_lights = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
    rank, world, _ = sharded.init_ranks()
    scene, lights, keep, gb = sharded.inputs(w, h, n_lights, mv=sharded.motion_vectors(w, h, 7))
    views = [synth.look_at_view((0.15 * i, 0.1 * i, 8.0 - 0.2 * i), (0.0, 0.0, 0.0)) for i in range(FRAMES)]
    equal = viewer.band_partition(h, world)
    # FXAA needs cuts on multiples of 16 rows to stay bit-exact
    assert all(y0 % 16 == 0 for y0, _ in equal) and all(y1 + 16 < h for _, y1 in equal[:-1])
    moved = [(0 if r == 0 else y0 + 16, h if r == world - 1 else y1 + 16) for r, (y0, y1) in enumerate(equal)]

    ok = True
    references = {}
    for cfg, present in CONFIGS:
        if cfg not in references:
            frames, costs = [], []
            if rank == 0:
                v1 = sharded.make_viewer(w, h, scene, lights, views[0], **config_args(cfg))
                for ref, _ in sharded.frames(v1, gb, scene.projection, views):
                    frames.append(ref)
                    costs.append(v1.measure_row_cost())
                v1.close()
            shared = [costs]
            dist.broadcast_object_list(shared, 0)
            references[cfg] = (frames, shared[0])
        reference, ref_costs = references[cfg]
        p = None if present is None else present % world
        for stripe_rows in STRIPES:
            bands = equal
            vs = sharded.make_viewer(w, h, scene, lights, views[0], bands, p, **config_args(cfg))
            vs.set_lighting_stripes(stripe_rows)
            vs.bake()
            names = vs.pass_names()
            ok &= "lighting-exchange" in names
            label = f"{cfg} stripes {stripe_rows}{'' if p is None else f' P={p}'}"
            for i in range(FRAMES):
                if i == MOVE:
                    bands = moved
                    vs.move_row_shards(bands)
                vs.set_camera(scene.projection, views[i])
                vs.render_frame(gb if i in (0, MOVE) else None)
                out = np.zeros((h, w), np.uint32)
                rows = vs.read_output(out)
                ok &= rows == ((0, h) if rank == p else tuple(bands[rank]))
                full = sharded.assemble(out, p)
                if rank == 0:
                    same = np.array_equal(full, reference[i])
                    print(f"{label} frame {i}: striped == single GPU: {same}", flush=True)
                    ok &= same
                if i in (0, MOVE):
                    cost = vs.measure_row_cost()
                    same = torch.tensor([1 if np.array_equal(cost, ref_costs[i]) else 0], device="cuda")
                    dist.all_reduce(same, op=dist.ReduceOp.MIN)
                    if rank == 0:
                        print(f"{label} frame {i}: striped row cost == single GPU on every rank: {bool(same.item())}", flush=True)
                    ok &= bool(same.item())
            sharded.close_sharded(vs)
    sharded.finish(ok)


if __name__ == "__main__":
    main()
