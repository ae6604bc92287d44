"""What the row-sharded GPU workers (tests/multi_gpu*_worker.py) and the sharded timing tools (tools/*_times.py) share:
the rank bootstrap under torchrun, the seeded inputs, the viewer factory, the unsharded reference frames, the assembly
of a whole frame from the ranks' bands, the teardown, and the card query the timing tools report.  Functions that
talk to the other ranks say so; every rank calls them, in the same order."""
import os
import subprocess
import sys

import numpy as np
import torch
import torch.distributed as dist

from granite_b200 import synth, viewer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMAA_LUTS = os.path.join(ROOT, "tests", "golden", "refsmaa_160x96.npz")


def config_args(name):
    """The Viewer keyword arguments of a named configuration."""
    return {"no AA": dict(post_aa=viewer.AA_NONE), "FXAA": dict(post_aa=viewer.AA_FXAA), "SMAA Ultra": dict(post_aa=viewer.AA_SMAA_ULTRA),
            "TAA High + FXAA": dict(post_aa=viewer.AA_TAA_HIGH_PLUS_FXAA), "FSR 0.67 + RCAS": dict(resolution_scale=0.67, resolution_scale_sharpen=True),
            "HDR10 + TAA": dict(post_aa=viewer.AA_TAA_HIGH, hdr10_output=True), "tonemap-only": dict(hdr_bloom=False)}[name]


def init_ranks(allow_shared=True, refusal_hint=""):
    """Join the NCCL process group torchrun set up and select this rank's GPU; returns (rank, world, local device).

    With more ranks than GPUs the ranks share devices (allow_shared=False refuses that: timings from ranks that share a
    GPU are not scaling numbers).  NCCL refuses two ranks of one host on one device (it compares host hash and bus
    id), so each rank names a host of its own and NCCL connects them through its socket transport on the loopback
    interface.  The frame's own exchange -- the kernels' stores into the IPC-mapped images of every rank, the epoch
    flags their consumers wait on -- runs unchanged."""
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    gpus = torch.cuda.device_count()
    if world > gpus:
        if not allow_shared:
            raise SystemExit(f"{world} ranks on {gpus} GPUs: one rank per GPU is needed for a scaling number{refusal_hint}")
        os.environ["NCCL_HOSTID"] = f"granite-rank-{rank}"
        os.environ.setdefault("NCCL_SOCKET_IFNAME", "lo")
        os.environ.setdefault("NCCL_IB_DISABLE", "1")
    local = local % gpus
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    return rank, world, local


def motion_vectors(w, h, seed):
    """The workers' motion vectors: 15 % of the pixels move by up to 4 px across and half the image height down or
    up, so that history reads cross band borders."""
    rng = np.random.default_rng(seed)
    mv = np.zeros((h, w, 2), np.float16)
    moving = rng.random((h, w)) < 0.15
    n = int(moving.sum())
    mv[moving] = np.stack([rng.uniform(-4.0, 4.0, n) / w, rng.uniform(-0.5, 0.5, n)], -1).astype(np.float16)
    return mv


def c5_motion_vectors(w, h):
    """bench.py's c5 motion vectors: zero on 90 % of the pixels, <= 2 px on the rest."""
    rng = np.random.default_rng(5)
    mv = np.zeros((h, w, 2), np.float16)
    m = rng.random((h, w)) < 0.1
    mv[m] = (rng.uniform(-2, 2, size=(int(m.sum()), 2)) / np.array([w, h])).astype(np.float16)
    return mv


def inputs(w, h, n_lights, spot_fraction=0.25, mv=None):
    """The seeded scene and lights at w x h, and the host G-buffer (with motion vectors mv, if given).  Returns
    (scene, lights, arrays, gbuffer): the G-buffer holds raw pointers into `arrays`, which must outlive it."""
    scene = synth.make_scene(w, h)
    lights = synth.make_lights(n_lights, spot_fraction=spot_fraction, aspect=w / h)
    arrays = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, scene.emissive)]
    if mv is not None:
        arrays.append(np.ascontiguousarray(mv).view(np.uint32).reshape(h, w))
    return scene, lights, arrays, viewer.Viewer.host_gbuffer(*arrays)


def make_viewer(w, h, scene, lights, view, bands=None, present_rank=None, **config):
    """A baked w x h viewer on this rank's GPU with the scene's directional light, `lights` and camera `view`, and the
    SMAA lookup textures when `config` selects SMAA.  With `bands`, row-sharded over the process group (collective:
    rank 0's NCCL unique id is broadcast), presenting from `present_rank` when given."""
    v = viewer.Viewer(w, h, cuda_device=torch.cuda.current_device(), **config)
    v.set_directional(scene.dir_color, scene.dir_direction)
    v.set_lights(lights)
    if viewer.AA_SMAA_LOW <= config.get("post_aa", viewer.AA_NONE) <= viewer.AA_SMAA_ULTRA:
        luts = np.load(SMAA_LUTS)
        v.set_smaa_lookup_textures(luts["area"], luts["search"])
    if bands:
        rank = dist.get_rank()
        uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
        if rank == 0:
            uid.copy_(torch.frombuffer(bytearray(viewer.nccl_unique_id()), dtype=torch.uint8))
        dist.broadcast(uid, 0)
        v.init_collectives(uid.cpu().numpy().tobytes(), rank, dist.get_world_size())
        v.set_row_shards(bands, rank)
        if present_rank is not None:
            v.set_present_rank(present_rank)
    v.set_camera(scene.projection, view)
    v.bake()
    return v


def frames(v, gb, projection, views):
    """Render one frame per view on v, the first bringing the host G-buffer gb; after each, yields (output, rows) of
    read_output."""
    for i, view in enumerate(views):
        v.set_camera(projection, view)
        v.render_frame(gb if i == 0 else None)
        out = np.zeros((v.height, v.width), np.uint32)
        rows = v.read_output(out)
        yield out, rows


def reference_frames(w, h, scene, lights, gb, views, **config):
    """Rank 0: the unsharded frames of `views`, rendered in order by one viewer.  Other ranks: []."""
    if dist.get_rank() != 0:
        return []
    v = make_viewer(w, h, scene, lights, views[0], **config)
    reference = [out for out, _ in frames(v, gb, scene.projection, views)]
    v.close()
    return reference


def assemble(out, present=None):
    """The whole frame(s) on every rank from each rank's read (collective).  Bands are disjoint and zero elsewhere, so a
    SUM all-reduce assembles them; a presented frame is broadcast from the presenting rank."""
    full = torch.from_numpy(np.ascontiguousarray(out).view(np.int32)).cuda()
    if present is None:
        dist.all_reduce(full, op=dist.ReduceOp.SUM)
    else:
        dist.broadcast(full, present)
    return full.cpu().numpy().view(np.uint32)


def check_frames(v, gb, projection, views, bands, reference, label, what):
    """Render `views` on the row-sharded viewer v (collective): every rank must read back its own band, and every
    assembled frame must equal rank 0's `reference` frame, which rank 0 prints as "<label> frame <i>: <what>: <bool>".
    Returns whether every check of this rank held."""
    rank = dist.get_rank()
    ok = True
    for i, (out, rows) in enumerate(frames(v, gb, projection, views)):
        ok &= rows == tuple(bands[rank])
        full = assemble(out)
        if rank == 0:
            same = np.array_equal(full, reference[i])
            print(f"{label} frame {i}: {what}: {same}", flush=True)
            ok &= same
    return ok


def close_sharded(v):
    """Close a row-sharded viewer (collective): every rank's pushes and flag stores have landed before any rank frees
    the peer channels they target."""
    v.sync()
    dist.barrier()
    v.close()


def finish(ok):
    """Exit every rank with 0 if `ok` holds on every rank, else 1 (collective)."""
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.destroy_process_group()
    sys.exit(0 if int(flag.item()) == 1 else 1)


def card(index):
    """The name and power limit of GPU `index`, from a read-only nvidia-smi query."""
    q = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() or "unknown"
