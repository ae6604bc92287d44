"""torchrun worker for tests/test_zt_gpu_smaa_sharded.py: renders frames with SMAA row-sharded over all ranks (the
edge rows exchanged inside the C++ graph, by peer stores or NCCL as GRB_SHARD_EXCHANGE says) and, on rank 0, unsharded;
every assembled sharded frame must equal the unsharded one bit for bit.  Two band layouts (equal bands, and narrow
64-row bands at the top so that an edge window spans two ranks), presets Low and Ultra, 4 frames each (both slots of
the exchange are reused).  Rank 0 also checks that the unsharded weights are non-zero near every band border, so that
the frame really depends on the exchanged rows."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import viewer  # noqa: E402
from tests import sharded  # noqa: E402

FRAMES = 4


def main():
    w, h, n_lights = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
    rank, world, _ = sharded.init_ranks()
    scene, lights, keep, gb = sharded.inputs(w, h, n_lights)
    views = [scene.view] * FRAMES
    layouts = {"equal": viewer.band_partition(h, world),
               "narrow": [(64 * r, 64 * (r + 1)) for r in range(world - 1)] + [(64 * (world - 1), h)]}

    ok = True
    for quality, aa in ((0, viewer.AA_SMAA_LOW), (3, viewer.AA_SMAA_ULTRA)):
        reference = []
        if rank == 0:
            v1 = sharded.make_viewer(w, h, scene, lights, scene.view, post_aa=aa)
            reference = [ref for ref, _ in sharded.frames(v1, gb, scene.projection, views)]
            weights = v1.download_image("smaa-weights")
            v1.close()
        for name, bands in layouts.items():
            vs = sharded.make_viewer(w, h, scene, lights, scene.view, bands, post_aa=aa)
            ok &= sharded.check_frames(vs, gb, scene.projection, views, bands, reference, f"preset {quality} {name}",
                                       f"sharded over {world} ranks == single GPU")
            sharded.close_sharded(vs)
            if rank == 0:
                reach = 2 * (4 << quality)
                near = [bool(weights[max(b - reach, 0):b + reach].any()) for _, b in bands[:-1]]
                print(f"preset {quality} {name}: weights near every border: {all(near)}", flush=True)
                ok &= all(near)
    sharded.finish(ok)


if __name__ == "__main__":
    main()
