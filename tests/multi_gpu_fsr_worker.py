"""torchrun worker for tests/test_zr_gpu_fsr_sharded.py: renders frames with FSR 1 upscaling row-sharded over all ranks
(the bands are display rows; every pass before FSR runs on the render rows of grbh_shard_plan_fsr, and the bloom d0,
SMAA edge and TAA history rows are exchanged inside the C++ graph by peer stores or NCCL as GRB_SHARD_EXCHANGE says)
and, on rank 0, unsharded; every assembled sharded frame must equal the unsharded one bit for bit, and every rank
must read back exactly its display band.  Scales 0.67 and 0.5, RCAS on and off, no AA, FXAA, SMAA Ultra / Low, TAA
High + FXAA and TAA Low; two band layouts (equal bands, and narrow 64-row bands at the top); 4 frames each with a
moving camera."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import synth, viewer  # noqa: E402
from tests import sharded  # noqa: E402

FRAMES = 4


def main():
    w, h, n_lights = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
    _, world, _ = sharded.init_ranks()
    layouts = {"equal": viewer.band_partition(h, world),
               "narrow": [(64 * r, 64 * (r + 1)) for r in range(world - 1)] + [(64 * (world - 1), h)]}
    views = [synth.look_at_view((0.15 * i, 0.1 * i, 8.0 - 0.2 * i), (0.0, 0.0, 0.0)) for i in range(FRAMES)]
    configs = {"0.67 RCAS none": (0.67, True, viewer.AA_NONE), "0.67 RCAS FXAA": (0.67, True, viewer.AA_FXAA),
               "0.67 SMAA Ultra": (0.67, False, viewer.AA_SMAA_ULTRA), "0.5 RCAS SMAA Low": (0.5, True, viewer.AA_SMAA_LOW),
               "0.67 RCAS TAA High + FXAA": (0.67, True, viewer.AA_TAA_HIGH_PLUS_FXAA), "0.5 TAA Low": (0.5, False, viewer.AA_TAA_LOW)}

    inputs = {}

    def gbuffer(scale):
        """The inputs at the render size of `scale` (the viewer's own rule)."""
        if scale not in inputs:
            probe = viewer.Viewer(w, h, cuda_device=-1, resolution_scale=scale)
            rw, rh = probe.render_size()
            probe.close()
            inputs[scale] = sharded.inputs(rw, rh, n_lights, mv=sharded.motion_vectors(rw, rh, 11))
        return inputs[scale]

    ok = True
    for cfg_name, (scale, rcas, aa) in configs.items():
        scene, lights, _, gb = gbuffer(scale)
        cfg = dict(post_aa=aa, resolution_scale=scale, resolution_scale_sharpen=rcas)
        reference = sharded.reference_frames(w, h, scene, lights, gb, views, **cfg)
        for name, bands in layouts.items():
            vs = sharded.make_viewer(w, h, scene, lights, views[0], bands, **cfg)
            ok &= sharded.check_frames(vs, gb, scene.projection, views, bands, reference, f"{cfg_name} {name}",
                                       f"sharded over {world} ranks == single GPU")
            sharded.close_sharded(vs)
    sharded.finish(ok)


if __name__ == "__main__":
    main()
