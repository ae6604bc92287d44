"""torchrun worker for tests/test_zfa_gpu_device_lights_sharded.py: row-sharded frames whose lights come from device
memory (grbh_viewer_set_lights_device), every rank binding its own device copy of the same lights, against the
unsharded host-light frames of rank 0, bit for bit.  The lights move every frame by the same torch op on every rank; the
reference viewer is handed the same bytes through set_lights."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import synth, viewer  # noqa: E402
from tests import device_lights_cases as cases  # noqa: E402
from tests import sharded  # noqa: E402

FRAMES = 4
CONFIGS = ("no AA", "TAA High + FXAA")
STRIPES = (0, 8)


def moved_positions(lights, frame):
    """The lights' positions at `frame`, computed on the device with a fixed op sequence (the same bytes on every rank)."""
    p = torch.from_numpy(np.ascontiguousarray(lights.position)).cuda()
    phase = torch.sin(torch.arange(len(lights.color), device="cuda", dtype=torch.float32))[:, None]
    for _ in range(frame):
        p.add_(torch.tensor([0.3, -0.05, 0.7], device="cuda") * phase)
    return p


def main():
    w, h, n_lights = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
    rank, world, _ = sharded.init_ranks()
    bands = viewer.band_partition(h, world, align=16)
    views = [synth.look_at_view((0.15 * i, 0.1 * i, 8.0 - 0.2 * i), (0.0, 0.0, 0.0)) for i in range(FRAMES)]
    ok = True
    for cfg in CONFIGS:
        args = sharded.config_args(cfg)
        scene, lights, arrays, gb = sharded.inputs(w, h, n_lights, mv=sharded.motion_vectors(w, h, 3))
        positions = [moved_positions(lights, i) for i in range(FRAMES)]
        reference = []
        if rank == 0:
            v = sharded.make_viewer(w, h, scene, lights, views[0], **args)
            for i in range(FRAMES):
                v.set_lights(synth.Lights(lights.color, positions[i].cpu().numpy(), lights.is_point, lights.rot, lights.inner_cone,
                                          lights.outer_cone))
                v.set_camera(scene.projection, views[i])
                v.render_frame(gb if i == 0 else None)
                out = np.zeros((h, w), np.uint32)
                v.read_output(out)
                reference.append(out)
            v.close()
        for stripes in STRIPES:
            v = viewer.Viewer(w, h, cuda_device=torch.cuda.current_device(), **args)
            v.set_directional(scene.dir_color, scene.dir_direction)
            uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
            if rank == 0:
                uid.copy_(torch.frombuffer(bytearray(viewer.nccl_unique_id()), dtype=torch.uint8))
            torch.distributed.broadcast(uid, 0)
            v.init_collectives(uid.cpu().numpy().tobytes(), rank, world)
            v.set_row_shards(bands, rank)
            v.set_lighting_stripes(stripes)
            d = cases.to_device(lights)
            v.set_lights_device(**d)
            v.set_camera(scene.projection, views[0])
            v.bake()
            for i in range(FRAMES):
                d["position"].copy_(positions[i])
                v.set_camera(scene.projection, views[i])
                v.render_frame(gb if i == 0 else None)
                out = np.zeros((h, w), np.uint32)
                rows = v.read_output(out)
                ok &= rows == tuple(bands[rank])
                full = sharded.assemble(out)
                if rank == 0:
                    same = np.array_equal(full, reference[i])
                    print(f"{cfg} stripes={stripes} frame {i}: device lights sharded == host lights single GPU: {same}", flush=True)
                    ok &= same
            sharded.close_sharded(v)
    sharded.finish(ok)


if __name__ == "__main__":
    main()
