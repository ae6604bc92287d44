"""torchrun worker for tests/test_zg_gpu_output_sharded.py: row-sharded frames rendered into caller-owned output images
(grbh_viewer_set_output_images / grbh_viewer_acquire_output), with the exchanges of the C++ graph on peer stores or NCCL
as GRB_SHARD_EXCHANGE says, against the unsharded host-fed frames of rank 0, bit for bit.

Three runs per configuration:
- per-rank rings: every rank holds a ring of 2 padded whole-frame images, poisoned before each acquire; the final pass
  writes the band's rows only, so every other row and the padding must keep the poison.  The bands move after the
  third frame (move_row_shards);
- presenting to rank 0, and to the last rank (with a band move): only the presenting rank holds a ring, and the
  present pass copies the assembled frame into it; every other rank reads back its band as before."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from granite_b200 import synth, viewer  # noqa: E402
from tests import sharded  # noqa: E402
from tests.multi_gpu_gbuffer_worker import FRAMES, frame_inputs  # noqa: E402

CONFIGS = ("no AA", "FXAA", "SMAA Ultra", "TAA High + FXAA", "FSR 0.67 + RCAS", "HDR10 + TAA", "tonemap-only")
# (presenting rank or None, -1 = the last rank; move the bands after frame 2)
RUNS = ((None, True), (0, False), (-1, True))
RING = 2
POISON = 0x5A5A5A5A
PAD = 4  # texels past the width of each ring image's rows


def main():
    w, h, n_lights = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
    assert (w + PAD) % 4 == 0, "ring pitches are multiples of 16 bytes"
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

        for present, move in RUNS:
            present = None if present is None else present % world
            v = sharded.make_viewer(w, h, scene, lights, views[0], bands=equal, present_rank=present, **args)
            holds_ring = present is None or rank == present
            ring = [torch.full((h, w + PAD), POISON, dtype=torch.int32, device="cuda") for _ in range(RING)]
            if holds_ring:
                v.set_output_images([t[:, :w] for t in ring])
            acquired, rendered = torch.cuda.Event(), torch.cuda.Event()
            label = f"{cfg} present={present} move={move}"
            for i in range(FRAMES):
                if move and i == 3:
                    v.move_row_shards(moved)
                bands = moved if move and i >= 3 else equal
                v.set_camera(scene.projection, views[i])
                k = i % RING
                if holds_ring:
                    ring[k].fill_(POISON)
                    acquired.record()
                    v.acquire_output(k, acquired=acquired, rendered=rendered)
                v.render_frame(viewer.Viewer.host_gbuffer(*gbs[i]))
                out = np.zeros((h, w), np.uint32)
                rows = v.read_output(out)
                want_rows = (0, h) if present == rank else tuple(bands[rank])
                ok &= rows == want_rows
                if holds_ring:
                    rendered.synchronize()
                    img = ring[k].cpu().numpy().view(np.uint32)
                    y0, y1 = want_rows
                    inside = np.array_equal(img[y0:y1, :w], out[y0:y1])
                    outside = bool((img[:y0] == POISON).all() and (img[y1:] == POISON).all() and (img[:, w:] == POISON).all())
                    if not (inside and outside):
                        print(f"{label} frame {i} rank {rank}: ring image rows {want_rows} equal the readback: {inside}, "
                              f"every other byte still poisoned: {outside}", flush=True)
                    ok &= inside and outside
                    if present is None:
                        out = np.zeros((h, w), np.uint32)
                        out[y0:y1] = img[y0:y1, :w]  # the assembled frame comes from the ring images
                full = sharded.assemble(out) if present is None else sharded.assemble(out, present)
                if rank == 0:
                    same = np.array_equal(full, reference[i])
                    print(f"{label} frame {i}: ring output sharded == host-fed single GPU: {same}", flush=True)
                    ok &= same
            sharded.close_sharded(v)
    sharded.finish(ok)


if __name__ == "__main__":
    main()
