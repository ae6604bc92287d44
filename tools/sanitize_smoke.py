"""One small invocation of every CUDA entry point of the hot path, for compute-sanitizer:

    compute-sanitizer --tool memcheck  python tools/sanitize_smoke.py
    compute-sanitizer --tool racecheck python tools/sanitize_smoke.py

(no parity checks here -- tests/ does that; this exists so that the shared-memory tile kernels, the
TMA boxes, the persistent lighting kernel's queue and the cooperative tail run under the sanitizer
at sizes that finish in a minute)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from granite_b200 import capi, harness, synth, viewer
from oracle import pyoracle as oracle
from tests import common
from tests.test_oracle_ref_post_shaders import taa_inputs

oracle.build(ref=False)
capi.lib(); capi.init()
rng = np.random.default_rng(0)

# clusterer + lighting (persistent with schedule, and the block form), odd and even sizes
for (w, h, n, spots) in [(320, 192, 300, 0.25), (322, 190, 64, 0.0)]:
    scene, cam, lights, prep = common.build_case(oracle, w, h, n, spots)
    dev = harness.ClusterDevice(prep.records, prep.model, prep.type_mask, prep.z_ranges, prep.params, prep.res)
    gcam = harness.camera_struct(cam)
    dev.build(gcam)
    gb = harness.GBufferDevice(scene)
    sched = harness.lighting_schedule(h)
    for _ in range(2):
        hdr = gb.emissive.clone()
        harness.deferred_lighting(gb, gcam, dev, hdr, schedule=sched)
    hdr2 = gb.emissive.clone()
    img = capi.image(hdr2, capi.FORMAT_B10G11R11_UFLOAT)
    import ctypes as C
    capi.check(capi.lib().grb_deferred_lighting_blocks(C.byref(gb.struct), C.byref(gcam), C.byref(dev.params), C.byref(dev.buffers), C.byref(img), capi.rows((8, h - 8)),
                                                       capi.stream_ptr()), "blocks")
torch.cuda.synchronize()
print("cluster + lighting ok")

# post chain: fused head (TMA), tile kernels (large level), cooperative tail, tonemap, FXAA, TAA
w, h = 1024, 512
hdr = common.random_hdr(rng, w, h)
lum = harness.to_dev(np.array([0.3, 2.0 ** 0.3, 2.0 ** -0.3], np.float32))
sz = oracle.pyramid_sizes(w, h)
lv = {k: harness.new_rgba16f(*s) for k, s in zip(("t", "d0", "d1", "d2", "d3"), sz)}
up = {"u2": harness.new_rgba16f(*sz[3]), "u1": harness.new_rgba16f(*sz[2]), "u0": harness.new_rgba16f(*sz[1])}
hist = harness.to_dev(common.random_rgba16f(rng, *sz[4]))
harness.bloom_threshold_downsample(harness.to_dev(hdr), lum, lv["d0"], lv["t"])
harness.bloom_threshold_downsample(harness.to_dev(hdr), None, lv["d0"], None, rows=(5, 77))
harness.bloom_tail(lv["d0"], lv["d1"], lv["d2"], lv["d3"], hist, 0.1, lum, 0.01, up["u2"], up["u1"])
harness.bloom_upsample(up["u1"], up["u0"])
big_src, big_dst = harness.to_dev(common.random_rgba16f(rng, 1280, 720)), harness.new_rgba16f(640, 360)
harness.bloom_downsample(big_src, big_dst)                      # TMA down tile kernel (>= 200k texels)
harness.bloom_upsample(big_dst, harness.new_rgba16f(1280, 720), rows=(3, 711))  # TMA up tile kernel, odd first row
for k in ("t", "d0", "d1"):
    harness.bloom_downsample(lv[k], lv[{"t": "d0", "d0": "d1", "d1": "d2"}[k]])  # generic kernels
ldr = torch.zeros((h, w), dtype=torch.int32, device="cuda")
harness.tonemap(harness.to_dev(hdr), up["u0"], lum, ldr)
out = torch.zeros((h, w), dtype=torch.int32, device="cuda")
harness.fxaa(ldr, out, True)
harness.fxaa(ldr, out, False, rows=(7, h - 9))
tw, th = 333, 177
thdr, depth, mv, thist, reproj = taa_inputs(rng, tw, th)
oc = torch.zeros((th, tw), dtype=torch.int32, device="cuda"); oh = harness.new_rgba16f(tw, th)
mv_t = harness.to_dev(mv.reshape(th, tw, 2)).view(torch.int32).reshape(th, tw)
for q in (0, 1, 2):
    harness.taa_resolve(harness.to_dev(thdr), harness.to_dev(depth), mv_t, harness.to_dev(thist), reproj, q, oc, oh)
pq_out = torch.zeros((h, w), dtype=torch.int32, device="cuda")
harness.pq10_encode(harness.to_dev(hdr), ldr, oracle.rec709_to_display_primaries(), 500.0, 400.0, 1000.0, pq_out)
harness.pq10_encode(harness.to_dev(thdr), oc, oracle.rec709_to_display_primaries(), 500.0, 400.0, 1000.0, torch.zeros((th, tw), dtype=torch.int32, device="cuda"),
                    rows=(3, th - 5))  # odd width: unaligned path
torch.cuda.synchronize()
print("post chain ok")

# one whole frame through the graph (streams, events, ping-pong resources)
sw, sh = 320, 192
scene = synth.make_scene(sw, sh)
v = viewer.Viewer(sw, sh, post_aa=viewer.AA_TAA_HIGH_PLUS_FXAA)
v.set_camera(scene.projection, scene.view)
v.set_directional(scene.dir_color, scene.dir_direction)
v.set_lights(synth.make_lights(64, spot_fraction=0.25, aspect=sw / sh))
v.bake()
mvz = np.zeros((sh, sw), np.uint32)
gbh = viewer.Viewer.host_gbuffer(*[np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, scene.emissive)], mvz)
o = np.zeros((sh, sw), np.uint32)
for i in range(3):
    v.render_frame(gbh if i == 0 else None)
    v.read_output(o)
v.close()
print("graph frames ok")
