"""torchrun worker for tests/test_zs_gpu_taa_sharded.py: renders frames with TAA row-sharded over all ranks (the
history rows exchanged inside the C++ graph, by peer stores or NCCL as GRB_SHARD_EXCHANGE says) and, on rank 0,
unsharded; every assembled sharded frame must equal the unsharded one bit for bit.  TAA Low, TAA High, TAA High + FXAA
and TAA High with HDR10 output; two band layouts (equal bands, and narrow 64-row bands at the top); 6 frames each, so
both slots of the exchange are reused.  The camera moves every frame, and 15 % of the pixels carry a motion vector of
up to half the image height: rank 0 checks on the host that every rank's motion vectors reach other ranks' bands."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import synth, viewer  # noqa: E402
from tests import sharded  # noqa: E402

FRAMES = 6


def reaches_other_bands(mv, bands):
    """For every band: moving pixels whose history read (at v - mv) lands in another band."""
    h = mv.shape[0]
    mvy = mv[..., 1].astype(np.float32)
    src = np.arange(h)[:, None] + 0.5 - mvy * h
    return [int(((src[y0:y1] < y0) | (src[y0:y1] >= y1))[mvy[y0:y1] != 0].sum()) for y0, y1 in bands]


def main():
    w, h, n_lights = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
    rank, world, _ = sharded.init_ranks()
    mv = sharded.motion_vectors(w, h, 11)
    scene, lights, keep, gb = sharded.inputs(w, h, n_lights, mv=mv)
    views = [synth.look_at_view((0.15 * i, 0.1 * i, 8.0 - 0.2 * i), (0.0, 0.0, 0.0)) for i in range(FRAMES)]
    layouts = {"equal": viewer.band_partition(h, world),
               "narrow": [(64 * r, 64 * (r + 1)) for r in range(world - 1)] + [(64 * (world - 1), h)]}
    configs = {"TAA Low": dict(post_aa=viewer.AA_TAA_LOW), "TAA High": dict(post_aa=viewer.AA_TAA_HIGH),
               "TAA High + FXAA": dict(post_aa=viewer.AA_TAA_HIGH_PLUS_FXAA), "TAA High HDR10": dict(post_aa=viewer.AA_TAA_HIGH, hdr10_output=True)}

    ok = True
    if rank == 0:
        for name, bands in layouts.items():
            reach = reaches_other_bands(mv, bands)
            print(f"{name}: motion vectors reach other bands from every rank: {all(n > 0 for n in reach)} {reach}", flush=True)
            ok &= all(n > 0 for n in reach)

    for cfg_name, cfg in configs.items():
        reference = sharded.reference_frames(w, h, scene, lights, gb, views, **cfg)
        for name, bands in layouts.items():
            vs = sharded.make_viewer(w, h, scene, lights, views[0], bands, **cfg)
            ok &= sharded.check_frames(vs, gb, scene.projection, views, bands, reference, f"{cfg_name} {name}",
                                       f"sharded over {world} ranks == single GPU")
            sharded.close_sharded(vs)
    sharded.finish(ok)


if __name__ == "__main__":
    main()
