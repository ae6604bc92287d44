"""torchrun worker for tests/test_zi_gpu_gbuffer_sharded.py: row-sharded frames rendered from G-buffers in device memory
(grbh_viewer_render_frame_device), with the exchanges of the C++ graph on peer stores or NCCL as GRB_SHARD_EXCHANGE
says, against the unsharded host-fed frames of rank 0, bit for bit.

Two ways to feed a frame:
- per rank: every rank holds a whole-size device G-buffer in which only its input_rows() are valid; every other row is
  poisoned (NaN depth, 0xFF bytes), so a row read outside the rank's list shows up as a wrong frame;
- from one rank: the source rank passes the whole frame's G-buffer, every other rank None
  (grbh_viewer_set_gbuffer_source_rank), from rank 0 or from the last rank.
The G-buffer changes every frame and the camera moves; each rank overwrites its one set of tensors once the viewer's
`consumed` event of the last frame has completed.  Some runs move the bands after the third frame (move_row_shards),
light in stripes, or present from the last rank."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import synth, viewer  # noqa: E402
from tests import sharded  # noqa: E402

FRAMES = 6
CONFIGS = ("no AA", "FXAA", "SMAA Ultra", "TAA High + FXAA", "FSR 0.67 + RCAS", "HDR10 + TAA", "tonemap-only")
# (feeding: "per rank" or the source rank, -1 = the last rank; lighting stripe rows; presenting rank or None; move the
# bands after frame 2)
RUNS = (("per rank", 0, None, True), ("per rank", 8, -1, False), (0, 64, None, True), (-1, 0, -1, False), (-1, 8, None, True))


def frame_inputs(rw, rh, n_lights):
    """The scene and lights, and one seeded G-buffer per frame (host arrays in host_gbuffer order, mv included)."""
    scene = synth.make_scene(rw, rh)
    lights = synth.make_lights(n_lights, spot_fraction=0.25, aspect=rw / rh)
    gbs = []
    for i in range(FRAMES):
        s = synth.make_scene(rw, rh, seed=200 + i)
        mv = sharded.motion_vectors(rw, rh, i).view(np.uint32).reshape(rh, rw)
        gbs.append([np.ascontiguousarray(a) for a in (s.albedo, s.normal, s.pbr, s.depth, s.emissive, mv)])
    return scene, lights, gbs


def to_torch(a):
    return torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else (a.view(np.int16) if a.dtype == np.uint16 else a))


def main():
    w, h, n_lights = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
    rank, world, _ = sharded.init_ranks()
    views = [synth.look_at_view((0.15 * i, 0.1 * i, 8.0 - 0.2 * i), (0.0, 0.0, 0.0)) for i in range(FRAMES)]
    # cuts on multiples of 16 rows: sharded FXAA is bit-exact only there
    equal = viewer.band_partition(h, world, align=16)
    moved = [(0, 32)] + [(32 + (h - 32) * r // (world - 1) // 16 * 16, 32 + (h - 32) * (r + 1) // (world - 1) // 16 * 16) for r in range(world - 1)]
    moved[-1] = (moved[-1][0], h)

    ok = True
    for cfg in CONFIGS:
        args = sharded.config_args(cfg)
        probe = viewer.Viewer(w, h, cuda_device=-1, **args)
        rw, rh = probe.render_size()
        probe.close()
        scene, lights, gbs = frame_inputs(rw, rh, n_lights)
        reference = []
        if rank == 0:
            v = sharded.make_viewer(w, h, scene, lights, views[0], **args)
            for i in range(FRAMES):
                v.set_camera(scene.projection, views[i])
                v.render_frame(viewer.Viewer.host_gbuffer(*gbs[i]))
                out = np.zeros((h, w), np.uint32)
                v.read_output(out)
                reference.append(out)
            v.close()

        for feeding, stripes, present, move in RUNS:
            if stripes and args.get("resolution_scale"):
                stripes = 0  # lighting in stripes is not supported with FSR 1
            source = None if feeding == "per rank" else feeding % world
            present = None if present is None else present % world
            v = viewer.Viewer(w, h, cuda_device=torch.cuda.current_device(), **args)
            v.set_directional(scene.dir_color, scene.dir_direction)
            v.set_lights(lights)
            if args.get("post_aa", 0) == viewer.AA_SMAA_ULTRA:
                luts = np.load(sharded.SMAA_LUTS)
                v.set_smaa_lookup_textures(luts["area"], luts["search"])
            uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
            if rank == 0:
                uid.copy_(torch.frombuffer(bytearray(viewer.nccl_unique_id()), dtype=torch.uint8))
            torch.distributed.broadcast(uid, 0)
            v.init_collectives(uid.cpu().numpy().tobytes(), rank, world)
            v.set_row_shards(equal, rank)
            if present is not None:
                v.set_present_rank(present)
            if source is not None:
                v.set_gbuffer_source_rank(source)
            v.set_lighting_stripes(stripes)
            v.set_camera(scene.projection, views[0])
            v.bake()

            planes = [torch.zeros(a.shape, dtype=to_torch(a).dtype, device="cuda") for a in gbs[0]]
            gb = v.device_gbuffer(*planes)
            consumed = torch.cuda.Event()
            label = f"{cfg} feeding={'per rank' if source is None else f'from {source}'} stripes={stripes} present={present} move={move}"
            for i in range(FRAMES):
                if move and i == 3:
                    v.move_row_shards(moved)
                bands = moved if move and i >= 3 else equal
                v.set_camera(scene.projection, views[i])
                consumed.synchronize()
                if source is None:
                    keep = np.zeros(rh, bool)
                    for y0, y1 in v.input_rows():
                        keep[y0:y1] = True
                    for t, a in zip(planes, gbs[i]):
                        p = np.array(a, copy=True)
                        if p.dtype == np.float32:
                            p[~keep] = np.nan
                        else:
                            p.view(np.uint8).reshape(rh, -1)[~keep] = 0xFF
                        t.copy_(to_torch(p))
                    v.render_frame_device(gb, consumed=consumed)
                elif rank == source:
                    for t, a in zip(planes, gbs[i]):
                        t.copy_(to_torch(a))
                    v.render_frame_device(gb, consumed=consumed)
                else:
                    v.render_frame_device(None)
                out = np.zeros((h, w), np.uint32)
                rows = v.read_output(out)
                want_rows = (0, h) if present == rank else tuple(bands[rank])
                ok &= rows == want_rows
                if present is None:
                    full = sharded.assemble(out)
                else:
                    full = sharded.assemble(out, present)
                if rank == 0:
                    same = np.array_equal(full, reference[i])
                    print(f"{label} frame {i}: device-fed sharded == host-fed single GPU: {same}", flush=True)
                    ok &= same
            sharded.close_sharded(v)
    sharded.finish(ok)


if __name__ == "__main__":
    main()
