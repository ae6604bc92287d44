"""torchrun worker for tests/test_zfc_gpu_device_lights_shadowed_sharded.py: row-sharded frames whose shadowed lights
come from device memory (grbh_viewer_set_lights_device_shadowed), every rank binding its own device copies of the
lights, their shadow transforms and their maps, against the unsharded host-light shadowed frames of rank 0, bit for bit.
Each frame the same torch ops on every rank move the lights and rewrite texels of the maps; the reference viewer is
handed the same bytes through set_lights and set_light_shadow_maps.  Before those, host-light shadowed frames are
checked sharded too."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import synth, viewer  # noqa: E402
from oracle import pyoracle  # noqa: E402
from tests import device_lights_cases as cases  # noqa: E402
from tests import sharded  # noqa: E402
from tests.device_shadow_cases import MapPool, transforms_in_input_order  # noqa: E402
from tests.multi_gpu_lights_worker import moved_positions  # noqa: E402

FRAMES = 4
CONFIGS = ("no AA", "TAA High + FXAA")
STRIPES = (0, 8)
RES = 16


def sharded_viewer(w, h, scene, bands, rank, world, stripes, args):
    v = viewer.Viewer(w, h, cuda_device=torch.cuda.current_device(), light_shadows=True, shadow_resolution=RES, **args)
    v.set_directional(scene.dir_color, scene.dir_direction)
    uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
    if rank == 0:
        uid.copy_(torch.frombuffer(bytearray(viewer.nccl_unique_id()), dtype=torch.uint8))
    torch.distributed.broadcast(uid, 0)
    v.init_collectives(uid.cpu().numpy().tobytes(), rank, world)
    v.set_row_shards(bands, rank)
    v.set_lighting_stripes(stripes)
    return v


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
        moved = [synth.Lights(lights.color, p.cpu().numpy(), lights.is_point, lights.rot, lights.inner_cone, lights.outer_cone) for p in positions]
        # every rank its own maps: the same seeded texels, rewritten by the same ops
        pool = MapPool(lights, RES)
        texels = []
        for i in range(FRAMES):
            if i:
                pool.rewrite(i)
            texels.append(pool.pool.clone())
        reference = []
        if rank == 0:
            v = viewer.Viewer(w, h, cuda_device=torch.cuda.current_device(), light_shadows=True, shadow_resolution=RES, **args)
            v.set_directional(scene.dir_color, scene.dir_direction)
            v.set_camera(scene.projection, views[0])
            v.bake()
            for i in range(FRAMES):
                pool.pool.copy_(texels[i])
                v.set_lights(moved[i])
                v.set_light_shadow_maps(pool.pointers().tolist())
                v.set_camera(scene.projection, views[i])
                v.render_frame(gb if i == 0 else None)
                out = np.zeros((h, w), np.uint32)
                v.read_output(out)
                reference.append(out)
            v.close()
        for stripes in STRIPES:
            for kind in ("host", "device"):
                v = sharded_viewer(w, h, scene, bands, rank, world, stripes, args)
                d = cases.to_device(lights)
                t = torch.zeros(len(lights.color), 16, device="cuda")
                if kind == "device":
                    v.set_lights_device(**d, shadow_transforms=t, shadow_maps=pool.device_pointers())
                v.set_camera(scene.projection, views[0])
                v.bake()
                for i in range(FRAMES):
                    pool.pool.copy_(texels[i])
                    if kind == "device":
                        d["position"].copy_(positions[i])
                        t.copy_(torch.from_numpy(transforms_in_input_order(pyoracle, v, moved[i])))
                    else:
                        v.set_lights(moved[i])
                        v.set_light_shadow_maps(pool.pointers().tolist())
                    v.set_camera(scene.projection, views[i])
                    v.render_frame(gb if i == 0 else None)
                    out = np.zeros((h, w), np.uint32)
                    rows = v.read_output(out)
                    ok &= rows == tuple(bands[rank])
                    full = sharded.assemble(out)
                    if rank == 0:
                        same = np.array_equal(full, reference[i])
                        print(f"{cfg} stripes={stripes} frame {i}: {kind} shadowed lights sharded == host lights single GPU: {same}", flush=True)
                        ok &= same
                sharded.close_sharded(v)
    sharded.finish(ok)


if __name__ == "__main__":
    main()
