"""Shadowed lights from device memory on one GPU (grbh_viewer_set_lights_device_shadowed): the device prep's shadow
tables against the host prep's, whole frames against host-light shadowed frames bit for bit, frames lit with
transforms of the caller's choosing against the oracle and the float64 reference, the maps_ready / maps_consumed
events, the lights' ready event over the transform table, and switching between host and device lights."""
import numpy as np
import pytest

from granite_b200 import viewer as _viewer
from tests import device_lights_cases as cases
from tests.device_shadow_cases import MapPool, transforms_in_input_order

pytestmark = pytest.mark.gpu

W, H = 320, 192
RES = 16


def _viewer_with_scene(proj, view, lights=None, pool=None, w=W, h=H, res=RES, **cfg):
    """A baked shadowed viewer with the scene's G-buffer arrays (host_gbuffer order; RGBA16F emissive when the config
    says so); host lights and their maps when given."""
    from granite_b200 import synth, viewer
    from tests import common

    v = viewer.Viewer(w, h, cuda_device=0, light_shadows=True, shadow_resolution=res, **cfg)
    rw, rh = v.render_size()
    scene = synth.make_scene(rw, rh)
    v.set_directional(scene.dir_color, scene.dir_direction)
    v.set_camera(proj, view)
    if lights is not None:
        v.set_lights(lights)
        v.set_light_shadow_maps(pool.pointers().tolist())
    v.bake()
    em = common.random_hdr_f16(np.random.default_rng(3), rw, rh, scale=0.02, hot=0.001) if cfg.get("render_target_fp16") else scene.emissive
    keep = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, em)]
    return v, keep, scene


def _frame(v, keep, first):
    from granite_b200 import viewer

    v.render_frame(viewer.Viewer.host_gbuffer(*keep) if first else None)
    out = np.zeros((v.height, v.width), np.uint32)
    v.read_output(out)
    return out


def _bind(v, d, transforms, pool, **events):
    import torch

    t = transforms if isinstance(transforms, torch.Tensor) else torch.from_numpy(transforms).cuda()
    m = pool.device_pointers()
    v.set_lights_device(**d, shadow_transforms=t, shadow_maps=m, **events)
    return t, m


@pytest.mark.parametrize("name", cases.HOST_PREP_CASES + cases.TIE_CASES + cases.LIMIT_CASES + ["odd-37"])
def test_device_shadow_prep_equals_host_prep(cuda, oracle, name):
    """The caller's transforms (the oracle's, input order) equal the host prep's put back in input order; the device
    prep's kept transforms and map pointers, read where the lighting pass reads them, equal the host prep's byte for
    byte, with its records, model rows, type mask and Z ranges."""
    from granite_b200 import synth, viewer

    if name == "odd-37":
        w, h = 1920, 1080
        proj, view = cases.default_camera(w, h)
        lights = synth.make_lights(37, spot_fraction=0.4)
        lights.position[::5, 2] += 200.0
        lights = cases.shuffled(lights)
    else:
        w, h, proj, view, lights, _ = cases.case(oracle, name)
    n = len(lights.color)
    pool = MapPool(lights, 4, skip_every=0)  # every light has a map of its own: the pointer names the input light
    host = viewer.Viewer(w, h, cuda_device=-1, light_shadows=True, shadow_resolution=4)
    host.set_camera(proj, view)
    host.set_lights(lights)
    host.set_light_shadow_maps(pool.pointers().tolist())
    want = host.light_prep()
    want_t, want_m = host.light_shadow_prep()
    transforms = transforms_in_input_order(oracle, host, lights)
    host.close()
    k = want[0]
    assert len(want_t) == k
    by_pointer = {int(p): i for i, p in enumerate(pool.pointers())}
    order = np.array([by_pointer[int(p)] for p in want_m], np.int64)
    assert transforms[order].tobytes() == want_t.tobytes()

    v, keep, _ = _viewer_with_scene(proj, view, res=4)
    held = _bind(v, cases.to_device(lights), transforms if n else np.zeros((0, 16), np.float32), pool)
    _frame(v, keep, True)
    got = v.light_prep()
    got_t, got_m = v.light_shadow_prep()
    assert got[0] == k
    for a, b in zip(want[1:], got[1:]):
        assert a.tobytes() == b.tobytes()
    assert got_t.tobytes() == want_t.tobytes()
    assert np.array_equal(got_m, want_m)
    if name == "6000-visible":
        assert k == 4096
    if name in ("all-culled", "0-0.0"):
        assert k == 0
    del held
    v.close()


CONFIGS = {
    "no AA": dict(post_aa=_viewer.AA_NONE),
    "TAA High + FXAA": dict(post_aa=_viewer.AA_TAA_HIGH_PLUS_FXAA),
    "resolution_scale 0.75": dict(resolution_scale=0.75),
    "RGBA16F": dict(render_target_fp16=True),
}


@pytest.mark.parametrize("device_gbuffer", [False, True], ids=["host G-buffer", "device G-buffer"])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_frames_equal_host_light_shadowed_frames(cuda, oracle, config, device_gbuffer):
    """Five frames; each frame a torch op moves the lights (their transforms follow) and rewrites texels of the maps.
    The output and HDR-main bit for bit those of a host-light shadowed viewer given the same maps in input order, and
    the maps shadow pixels: HDR-main differs from the same frame with every map null."""
    import torch

    from granite_b200 import synth, viewer

    cfg = CONFIGS[config]
    proj, view = cases.default_camera(W, H)
    lights = synth.make_lights(300, spot_fraction=0.3, aspect=W / H)
    pool = MapPool(lights, RES)
    vh, keep, _ = _viewer_with_scene(proj, view, lights, pool, **cfg)
    vd, _, _ = _viewer_with_scene(proj, view, **cfg)
    d = cases.to_device(lights)
    t, m = _bind(vd, d, transforms_in_input_order(oracle, vh, lights), pool)
    if cfg.get("post_aa") == viewer.AA_TAA_HIGH_PLUS_FXAA:
        keep.append(np.zeros(keep[0].shape[:2], np.uint32))  # still motion vectors
    if device_gbuffer:
        planes = [torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else (a.view(np.int16) if a.dtype == np.uint16 else a)).cuda()
                  for a in keep]
        gb = vd.device_gbuffer(*planes)
    step = torch.tensor([0.3, -0.05, 0.7], device="cuda")
    for f in range(5):
        if f:
            d["position"].add_(step * torch.sin(torch.arange(len(lights.color), device="cuda", dtype=torch.float32))[:, None])
            pool.rewrite(f)
            moved = synth.Lights(lights.color, d["position"].cpu().numpy(), lights.is_point, lights.rot, lights.inner_cone, lights.outer_cone)
            t.copy_(torch.from_numpy(transforms_in_input_order(oracle, vh, moved)))
            vh.set_lights(moved)
            vh.set_light_shadow_maps(pool.pointers().tolist())
        want = _frame(vh, keep, f == 0)
        if device_gbuffer:
            vd.render_frame_device(gb if f == 0 else None)
            got = np.zeros((vd.height, vd.width), np.uint32)
            vd.read_output(got)
        else:
            got = _frame(vd, keep, f == 0)
        assert np.array_equal(want, got), f"frame {f}: {int((want != got).sum())} pixels differ"
        assert np.array_equal(vh.download_image("HDR-main"), vd.download_image("HDR-main")), f"frame {f}: HDR-main"
    lit = vd.download_image("HDR-main")
    m.zero_()
    if device_gbuffer:
        vd.render_frame_device(None)
        vd.read_output(np.zeros((vd.height, vd.width), np.uint32))
    else:
        _frame(vd, keep, False)
    assert (lit != vd.download_image("HDR-main")).mean() > 0.001, "the maps must shadow pixels"
    torch.cuda.synchronize()
    vh.close()
    vd.close()


def _rolled(transforms, is_point, angle=0.5):
    """Spot transforms of a camera rolled about the light's axis by `angle` (bias * roll * bias^-1 * T, in fp32), point
    transforms with the depth terms of a near plane twice as far: matrices that are not the reference's."""
    out = transforms.copy()
    c, s = np.cos(angle), np.sin(angle)
    bias = np.array([[0.5, 0, 0, 0.5], [0, 0.5, 0, 0.5], [0, 0, 1, 0], [0, 0, 0, 1]], np.float64)
    roll = np.array([[c, -s, 0, 0], [s, c, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]], np.float64)
    r = bias @ roll @ np.linalg.inv(bias)
    for i in range(len(out)):
        if is_point[i]:
            out[i, 2] = np.float32(out[i, 2] * 2.0)  # proj[3].z = near-dependent depth term (reverse-Z: near * ...)
        else:
            mt = out[i].reshape(4, 4).T.astype(np.float64)  # column-major storage -> row-major matrix
            out[i] = (r @ mt).T.reshape(-1).astype(np.float32)
    return out


def test_caller_transforms_are_the_ones_sampled(cuda, oracle):
    """Shadow transforms that are not the reference's: HDR-main equals the oracle's shadowed pass with those matrices
    and meets the float64 bar, and differs from the pass with the reference's matrices."""
    from granite_b200 import synth
    from tests import common
    from tests import lighting_ref64 as R
    from tests.test_zy_gpu_shadows import _compare

    res = 32
    scene = synth.make_scene(W, H)
    lights = synth.make_lights(150, spot_fraction=0.4, aspect=W / H)
    pool = MapPool(lights, res)
    v, keep, _ = _viewer_with_scene(scene.projection, scene.view, res=res)
    reference_t = transforms_in_input_order(oracle, v, lights)
    chosen = _rolled(reference_t, lights.is_point)
    assert not np.array_equal(chosen, reference_t)
    held = _bind(v, cases.to_device(lights), chosen, pool)
    _frame(v, keep, True)
    got = v.download_image("HDR-main")

    cam, prep = common.build_case_for_viewer(oracle, v, scene, lights)
    kept = np.flatnonzero(oracle.visible_lights(cam, lights))  # make_lights lists them front to back
    assert len(kept) == prep.n
    clus = oracle.cluster_build(cam, prep)
    maps = pool.host_maps(kept)
    ref = oracle.deferred_lighting_shadowed(scene, cam, prep, clus, chosen[kept], maps, res)
    assert (ref != oracle.deferred_lighting_shadowed(scene, cam, prep, clus, reference_t[kept], maps, res)).mean() > 0.001
    _compare(got, ref, 0.97)
    share = R.assert_meets_bar(got, R.reference(oracle, scene, cam, prep, clus, shadows=(chosen[kept], maps, res)), "caller transforms")
    print(f"caller transforms: within the float64 bar; it admits one code on {share:.4f} of the lit channels")
    del held
    v.close()


def test_maps_ready_and_consumed_events(cuda, oracle):
    """maps_ready: a producer stream sleeps, then writes the maps and records maps_ready; the frame shows the new maps.
    maps_consumed: a stream that overwrites the maps after maps_consumed leaves the frame in flight as it was."""
    import torch

    from granite_b200 import synth

    proj, view = cases.default_camera(W, H)
    lights = synth.make_lights(300, spot_fraction=0.3, aspect=W / H)
    old, new = MapPool(lights, RES, seed=1), MapPool(lights, RES, seed=2)
    new_ref, keep, _ = _viewer_with_scene(proj, view, lights, new)
    want = [_frame(new_ref, keep, True), _frame(new_ref, keep, False)]
    old_ref, _, _ = _viewer_with_scene(proj, view, lights, old)
    assert not np.array_equal(_frame(old_ref, keep, True), want[0]), "the new maps change the frame"

    live = MapPool(lights, RES, seed=1)  # the maps the device viewer samples, first holding the old texels
    vd, _, _ = _viewer_with_scene(proj, view)
    maps_ready, maps_consumed = torch.cuda.Event(), torch.cuda.Event()
    held = _bind(vd, cases.to_device(lights), transforms_in_input_order(oracle, vd, lights), live, maps_ready=maps_ready,
                 maps_consumed=maps_consumed)
    producer = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(producer):
        torch.cuda._sleep(50_000_000)
        live.pool.copy_(new.pool)
        maps_ready.record()
    assert np.array_equal(_frame(vd, keep, True), want[0]), "the frame sampled the maps before maps_ready"

    with torch.cuda.stream(producer):
        maps_ready.record()
    vd.render_frame(None)
    with torch.cuda.stream(producer):
        producer.wait_event(maps_consumed)
        live.pool.copy_(old.pool)
    out = np.zeros((H, W), np.uint32)
    vd.read_output(out)
    assert np.array_equal(out, want[1]), "overwriting the maps after maps_consumed changed the frame"
    torch.cuda.synchronize()
    del held
    for v in (old_ref, new_ref, vd):
        v.close()


def test_lights_ready_covers_the_transform_table(cuda, oracle):
    """The transform table is read under the lights' ready event: written by a producer stream after a sleep, it is
    the table the frame uses."""
    import torch

    from granite_b200 import synth

    proj, view = cases.default_camera(W, H)
    lights = synth.make_lights(300, spot_fraction=0.3, aspect=W / H)
    pool = MapPool(lights, RES)
    ref, keep, _ = _viewer_with_scene(proj, view, lights, pool)
    want = _frame(ref, keep, True)
    vd, _, _ = _viewer_with_scene(proj, view)
    ready = torch.cuda.Event()
    right = torch.from_numpy(transforms_in_input_order(oracle, vd, lights)).cuda()
    t = torch.zeros_like(right)
    held = _bind(vd, cases.to_device(lights), t, pool, ready=ready)
    producer = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(producer):
        torch.cuda._sleep(50_000_000)
        t.copy_(right)
        ready.record()
    assert np.array_equal(_frame(vd, keep, True), want), "the frame read the transforms before `ready`"
    torch.cuda.synchronize()
    del held
    ref.close()
    vd.close()


def test_switching_between_host_and_device_shadowed_lights(cuda, oracle):
    """host shadowed -> device shadowed -> host shadowed lights on one viewer: each frame equals the frame of a viewer
    that only had that kind of lights."""
    from granite_b200 import synth

    proj, view = cases.default_camera(W, H)
    lights = synth.make_lights(300, spot_fraction=0.3, aspect=W / H)
    other = synth.make_lights(200, spot_fraction=0.5, aspect=W / H)
    pool, other_pool = MapPool(lights, RES), MapPool(other, RES, seed=9)
    ref, keep, _ = _viewer_with_scene(proj, view, lights, pool)
    want = [_frame(ref, keep, True), _frame(ref, keep, False)]
    ref.set_lights(other)
    ref.set_light_shadow_maps(other_pool.pointers().tolist())
    want.append(_frame(ref, keep, False))
    dev, _, _ = _viewer_with_scene(proj, view)
    held_dev = _bind(dev, cases.to_device(lights), transforms_in_input_order(oracle, dev, lights), pool)
    dev_frames = [_frame(dev, keep, True), _frame(dev, keep, False)]

    v, _, _ = _viewer_with_scene(proj, view, lights, pool)
    got = [_frame(v, keep, True)]
    held = _bind(v, cases.to_device(lights), transforms_in_input_order(oracle, v, lights), pool)
    got.append(_frame(v, keep, False))
    assert v.light_prep()[0] == 300 and len(v.light_shadow_prep()[0]) == 300
    v.set_lights(other)
    v.set_light_shadow_maps(other_pool.pointers().tolist())
    got.append(_frame(v, keep, False))
    assert v.light_prep()[0] == 200
    assert sorted(v.light_shadow_prep()[1].tolist()) == sorted(int(p) for p in other_pool.pointers())
    for i, (a, b) in enumerate(zip(want, got)):
        assert np.array_equal(a, b), f"frame {i}"
    assert np.array_equal(dev_frames[1], got[1]), "device lights frame"
    del held, held_dev
    for x in (ref, dev, v):
        x.close()


def test_shadow_tables_in_host_memory_are_refused(cuda):
    """Transforms or maps in host memory are refused by the pointer check, each with its message."""
    import ctypes as C

    import torch

    from granite_b200 import synth, viewer

    proj, view = cases.default_camera(W, H)
    v, _, _ = _viewer_with_scene(proj, view)
    d = cases.to_device(synth.make_lights(8))
    l = viewer.GrbhDeviceLights(8, d["color"].data_ptr(), d["position"].data_ptr(), d["is_point"].data_ptr(), d["rotation"].data_ptr(),
                                d["inner_cone"].data_ptr(), d["outer_cone"].data_ptr(), 1e10, None, None)
    t_host, m_host = np.zeros((8, 16), np.float32), np.zeros(8, np.uint64)
    t_dev, m_dev = torch.zeros(8, 16, device="cuda"), torch.zeros(8, dtype=torch.int64, device="cuda")
    for t, m, what in ((t_host.ctypes.data, m_dev.data_ptr(), b"shadow transforms is not device memory"),
                       (t_dev.data_ptr(), m_host.ctypes.data, b"shadow maps is not device memory")):
        sh = viewer.GrbhDeviceLightShadows(t, m, None, None)
        assert viewer.lib().grbh_viewer_set_lights_device_shadowed(v._h, C.byref(l), C.byref(sh)) < 0
        assert what in viewer.lib().grbh_last_error()
    with pytest.raises(ValueError, match="CUDA tensor"):
        v.set_lights_device(**d, shadow_transforms=t_dev.cpu(), shadow_maps=m_dev)
    with pytest.raises(ValueError, match="shadow_maps must be"):
        v.set_lights_device(**d, shadow_transforms=t_dev, shadow_maps=m_dev.to(torch.int32))
    torch.cuda.synchronize()
    v.close()
