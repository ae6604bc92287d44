"""torchrun worker for tests/test_multi_gpu.py: renders the same frames row-sharded over all ranks
(NCCL exchange steps inside the C++ graph) and, on rank 0, unsharded; the assembled sharded image
must equal the unsharded one bit for bit.

Row-sharded frames and the unsharded reference frame are lit by the same (persistent) form of the lighting kernel:
a light that cannot reach a pixel adds exactly 0 to it, so the result does not depend on which 16x4 pixel blocks a
rank happens to own."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import viewer  # noqa: E402
from tests import sharded  # noqa: E402


def main():
    w, h, n_lights, fxaa = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
    rank, world, _ = sharded.init_ranks()
    scene, lights, keep, gb = sharded.inputs(w, h, n_lights)
    aa = viewer.AA_FXAA if fxaa else viewer.AA_NONE
    views = [scene.view] * 3

    vs = sharded.make_viewer(w, h, scene, lights, scene.view, viewer.band_partition(h, world), post_aa=aa)
    frames = [sharded.assemble(out) for out, _ in sharded.frames(vs, gb, scene.projection, views)]
    lum_sharded = vs.download_buffer("average-luminance", np.float32, 3).copy()
    sharded.close_sharded(vs)
    ok = True
    if rank == 0:
        v1 = sharded.make_viewer(w, h, scene, lights, scene.view, post_aa=aa)
        for i, (ref, _) in enumerate(sharded.frames(v1, gb, scene.projection, views)):
            same = np.array_equal(ref, frames[i])
            print(f"frame {i}: sharded over {world} ranks == single GPU: {same}", flush=True)
            ok &= same
        lum1 = v1.download_buffer("average-luminance", np.float32, 3)
        same = np.array_equal(lum1.view(np.uint32), lum_sharded.view(np.uint32))
        print(f"average luminance identical: {same}", flush=True)
        ok &= same
        v1.close()
    sharded.finish(ok)


if __name__ == "__main__":
    main()
