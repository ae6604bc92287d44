"""torchrun worker for tests/test_zfe_gpu_device_light_count_sharded.py: row-sharded frames whose device light list has
its length in device memory (Viewer.set_lights_device(..., count=)).  Every rank binds its own copy of the list and of
the count, and every frame the same torch ops on every rank rewrite the count and fill the entries past it with NaNs.
Each assembled frame must equal, bit for bit, rank 0's unsharded host-light frame of the first `count` lights."""
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
from tests.multi_gpu_shadowed_lights_worker import RES, sharded_viewer  # noqa: E402

COUNTS = (450, 37, 1000, 5)  # the live count of each frame; 1000 is past the capacity and clamps to it
FRAMES = len(COUNTS)
# (configuration, lighting stripes, shadowed)
RUNS = (("no AA", 0, False), ("no AA", 8, False), ("TAA High + FXAA", 0, False), ("TAA High + FXAA", 8, False), ("no AA", 8, True))


def first(lights, k):
    return synth.Lights(lights.color[:k], lights.position[:k], lights.is_point[:k], lights.rot[:k], lights.inner_cone[:k], lights.outer_cone[:k])


def main():
    w, h, n_lights = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
    rank, world, _ = sharded.init_ranks()
    bands = viewer.band_partition(h, world, align=16)
    views = [synth.look_at_view((0.15 * i, 0.1 * i, 8.0 - 0.2 * i), (0.0, 0.0, 0.0)) for i in range(FRAMES)]
    ok = True
    for cfg, stripes, shadowed in RUNS:
        args = sharded.config_args(cfg)
        scene, lights, arrays, gb = sharded.inputs(w, h, n_lights, mv=sharded.motion_vectors(w, h, 3))
        pool = MapPool(lights, RES) if shadowed else None
        live = [min(k, n_lights) for k in COUNTS]
        reference = []
        if rank == 0:
            v = viewer.Viewer(w, h, cuda_device=torch.cuda.current_device(), light_shadows=shadowed, shadow_resolution=RES, **args)
            v.set_directional(scene.dir_color, scene.dir_direction)
            v.set_camera(scene.projection, views[0])
            v.bake()
            for i in range(FRAMES):
                v.set_lights(first(lights, live[i]))
                if shadowed:
                    v.set_light_shadow_maps(pool.pointers()[: live[i]].tolist())
                v.set_camera(scene.projection, views[i])
                v.render_frame(gb if i == 0 else None)
                out = np.zeros((h, w), np.uint32)
                v.read_output(out)
                reference.append(out)
            v.close()
        if shadowed:
            v = sharded_viewer(w, h, scene, bands, rank, world, stripes, args)
        else:
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
        clean = d["position"].clone()
        count = torch.zeros(1, dtype=torch.int32, device="cuda")
        if shadowed:
            t = torch.from_numpy(transforms_in_input_order(pyoracle, v, lights)).cuda()
            v.set_lights_device(**d, shadow_transforms=t, shadow_maps=pool.device_pointers(), count=count)
        else:
            v.set_lights_device(**d, count=count)
        v.set_camera(scene.projection, views[0])
        v.bake()
        for i in range(FRAMES):
            count.fill_(COUNTS[i])
            d["position"].copy_(clean)
            d["position"][live[i]:] = float("nan")
            v.set_camera(scene.projection, views[i])
            v.render_frame(gb if i == 0 else None)
            out = np.zeros((h, w), np.uint32)
            rows = v.read_output(out)
            ok &= rows == tuple(bands[rank])
            full = sharded.assemble(out)
            if rank == 0:
                same = np.array_equal(full, reference[i])
                label = f"{cfg} stripes={stripes}{' shadowed' if shadowed else ''} count={COUNTS[i]}"
                print(f"{label} frame {i}: counted device lights sharded == host lights single GPU: {same}", flush=True)
                ok &= same
        sharded.close_sharded(v)
    sharded.finish(ok)


if __name__ == "__main__":
    main()
