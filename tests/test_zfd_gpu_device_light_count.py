"""A device light list whose length lives in device memory, on one GPU (grbh_viewer_set_light_count_device through
Viewer.set_lights_device(..., count=)): the device prep of a capacity-8192 list against the host prep and the device
prep of its first `count` lights, with the entries past the count poisoned; whole frames with the count rewritten on the
device between frames against host-light frames, bit for bit; rebinding; and the refusals that need a device."""
import ctypes as C

import numpy as np
import pytest

from granite_b200 import viewer as _viewer
from tests import device_lights_cases as cases
from tests.device_shadow_cases import MapPool, transforms_in_input_order

pytestmark = pytest.mark.gpu

W, H = 320, 192
CAPACITY = 8192


def _first(lights, k):
    from granite_b200 import synth

    return synth.Lights(lights.color[:k], lights.position[:k], lights.is_point[:k], lights.rot[:k], lights.inner_cone[:k], lights.outer_cone[:k])


def _scene_viewer(proj, view, w=W, h=H, **cfg):
    from granite_b200 import synth, viewer

    v = viewer.Viewer(w, h, cuda_device=0, **cfg)
    rw, rh = v.render_size()
    scene = synth.make_scene(rw, rh)
    v.set_directional(scene.dir_color, scene.dir_direction)
    v.set_camera(proj, view)
    v.bake()
    keep = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, scene.emissive)]
    return v, keep


def _frame(v, keep, first):
    from granite_b200 import viewer

    v.render_frame(viewer.Viewer.host_gbuffer(*keep) if first else None)
    out = np.zeros((v.height, v.width), np.uint32)
    v.read_output(out)
    return out


def _poison(d, clean, k, transforms=None, maps=None, clean_t=None, clean_m=None):
    """Entries [0, k) from the clean copies, entries [k, capacity) NaN positions and colours, NaN transforms and map
    pointers that name no memory (stream-ordered torch ops, no host sync)."""
    for name in ("position", "color"):
        d[name].copy_(clean[name])
        d[name][k:] = float("nan")
    if transforms is not None:
        transforms.copy_(clean_t)
        transforms[k:] = float("nan")
        maps.copy_(clean_m)
        maps[k:] = 0x7FF0_DEAD_BEE8


def _prep_lights():
    """8192 shuffled lights at the default camera, every seventh behind the eye (culled), so that more than 4096 of the
    first 6000 are visible and fewer than 4096 of the first 4096."""
    from granite_b200 import synth

    lights = synth.make_lights(CAPACITY, spot_fraction=0.25)
    lights.position[::7, 2] += 200.0
    return cases.shuffled(lights)


@pytest.mark.parametrize("shadowed", [False, True], ids=["unshadowed", "shadowed"])
def test_counted_prep_equals_prep_of_the_first_count_lights(cuda, oracle, shadowed):
    """For each device count (clamps included): count, records, model rows, type mask and Z ranges (and, shadowed, the
    transforms and map pointers) of the last frame's prep byte for byte the host prep's of the first k lights and the
    device prep's of a list bound with exactly those k lights; entries past k hold NaNs and wild map pointers."""
    import torch

    from granite_b200 import viewer
    from tests import common

    w, h = 1920, 1080
    proj, view = cases.default_camera(w, h)
    lights = _prep_lights()
    cfg = dict(light_shadows=True, shadow_resolution=4) if shadowed else {}
    pool = MapPool(lights, 4, skip_every=0) if shadowed else None
    host = viewer.Viewer(w, h, cuda_device=-1, **cfg)
    host.set_camera(proj, view)
    vis = oracle.visible_lights(common.oracle_camera_from_viewer(oracle, host), lights)
    k_full = next(k for k in range(4096, CAPACITY + 1) if vis[:k].sum() >= 4096)
    assert vis[:4096].sum() < 4096 and k_full < CAPACITY
    transforms = transforms_in_input_order(oracle, host, lights) if shadowed else None

    v, keep = _scene_viewer(proj, view, w=w, h=h, **cfg)
    exact, _ = _scene_viewer(proj, view, w=w, h=h, **cfg)
    d = cases.to_device(lights)
    clean = {k: t.clone() for k, t in d.items()}
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    extra = {}
    if shadowed:
        t_dev, m_dev = torch.from_numpy(transforms).cuda(), pool.device_pointers()
        clean_t, clean_m = t_dev.clone(), m_dev.clone()
        extra = dict(shadow_transforms=t_dev, shadow_maps=m_dev)
    v.set_lights_device(**d, **extra, count=count)
    first = True
    for raw in (0, 1, 37, 4095, 4096, CAPACITY, k_full, -3, 9000):
        k = min(max(raw, 0), CAPACITY)
        count.fill_(raw)
        if shadowed:
            _poison(d, clean, k, t_dev, m_dev, clean_t, clean_m)
        else:
            _poison(d, clean, k)
        torch.cuda.synchronize()
        _frame(v, keep, first)
        got = v.light_prep()

        host.set_lights(_first(lights, k))
        if shadowed:
            host.set_light_shadow_maps(pool.pointers()[:k].tolist())
        want = host.light_prep()
        sub = {n: clean[n][:k].contiguous() for n in clean}
        if shadowed:
            exact.set_lights_device(**sub, shadow_transforms=clean_t[:k].contiguous(), shadow_maps=clean_m[:k].contiguous())
        else:
            exact.set_lights_device(**sub)
        _frame(exact, keep, first)
        first = False
        same_k = exact.light_prep()
        assert got[0] == want[0] == same_k[0], f"count {raw}"
        if raw == k_full or raw >= CAPACITY:
            assert got[0] == 4096
        if raw <= 0:
            assert got[0] == 0
        for a, b, c in zip(want[1:], got[1:], same_k[1:]):
            assert a.tobytes() == b.tobytes() == c.tobytes(), f"count {raw}"
        if shadowed:
            want_t, want_m = host.light_shadow_prep()
            got_t, got_m = v.light_shadow_prep()
            exact_t, exact_m = exact.light_shadow_prep()
            assert want_t.tobytes() == got_t.tobytes() == exact_t.tobytes(), f"count {raw}"
            assert np.array_equal(want_m, got_m) and np.array_equal(want_m, exact_m), f"count {raw}"
        del sub
    host.close()
    torch.cuda.synchronize()
    v.close()
    exact.close()


CONFIGS = {
    "c3-like": dict(),
    "TAA + FXAA": dict(post_aa=_viewer.AA_TAA_HIGH_PLUS_FXAA),
    "resolution_scale 0.75": dict(resolution_scale=0.75),
    "clustered_lights_shadows": dict(light_shadows=True, shadow_resolution=16),
}
# the live count of each frame: a busy frame, then a drop to 10 whose tiles must lose the earlier frames' words
COUNTS = (1500, 6000, 10, 3000, 37)


@pytest.mark.parametrize("config", list(CONFIGS))
def test_frames_with_the_count_rewritten_on_the_device(cuda, oracle, config):
    """Five frames; before each a stream of the caller's waits on `consumed`, rewrites the count and poisons the entries
    past it, then records `ready` -- no host read of the count.  The output and HDR-main bit for bit those of a host-light
    viewer given the first `count` lights; measure_row_cost identical."""
    import torch

    from granite_b200 import synth, viewer

    cfg = CONFIGS[config]
    shadowed = bool(cfg.get("light_shadows"))
    proj, view = cases.default_camera(W, H)
    lights = synth.make_lights(6500, spot_fraction=0.25, aspect=W / H)
    vh, keep = _scene_viewer(proj, view, **cfg)
    vd, _ = _scene_viewer(proj, view, **cfg)
    if cfg.get("post_aa") == viewer.AA_TAA_HIGH_PLUS_FXAA:
        keep.append(np.zeros(keep[0].shape[:2], np.uint32))  # still motion vectors
    d = cases.to_device(lights)
    clean = {k: t.clone() for k, t in d.items()}
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    ready, consumed = torch.cuda.Event(), torch.cuda.Event()
    extra, poison = {}, {}
    if shadowed:
        pool = MapPool(lights, 16)
        t_dev, m_dev = torch.from_numpy(transforms_in_input_order(oracle, vh, lights)).cuda(), pool.device_pointers()
        extra = dict(shadow_transforms=t_dev, shadow_maps=m_dev)
        poison = dict(transforms=t_dev, maps=m_dev, clean_t=t_dev.clone(), clean_m=m_dev.clone())
    vd.set_lights_device(**d, **extra, ready=ready, consumed=consumed, count=count)
    producer = torch.cuda.Stream()
    torch.cuda.synchronize()
    for f, k in enumerate(COUNTS):
        with torch.cuda.stream(producer):
            if f:
                producer.wait_event(consumed)
            count.fill_(k)
            _poison(d, clean, k, **poison)
            ready.record()
        vh.set_lights(_first(lights, k))
        if shadowed:
            vh.set_light_shadow_maps(pool.pointers()[:k].tolist())
        want = _frame(vh, keep, f == 0)
        got = _frame(vd, keep, f == 0)
        assert np.array_equal(want, got), f"frame {f} (count {k}): {int((want != got).sum())} pixels differ"
        assert np.array_equal(vh.download_image("HDR-main"), vd.download_image("HDR-main")), f"frame {f} (count {k}): HDR-main"
    assert np.array_equal(vh.measure_row_cost(), vd.measure_row_cost())
    torch.cuda.synchronize()
    vh.close()
    vd.close()


def test_rebinding_clears_the_count(cuda):
    """A new set_lights_device binding drops the count (every bound entry is live again); set_lights goes back to host
    lights, after which the viewer has no device list to give a count to."""
    import torch

    from granite_b200 import synth, viewer

    proj, view = cases.default_camera(W, H)
    lights = synth.make_lights(1000, spot_fraction=0.25, aspect=W / H)
    # the frames carry exposure and bloom state over, so the reference renders the same sequence of light lists
    sequence = [10, 1000, 10, 1000, 10]
    ref, keep = _scene_viewer(proj, view)
    want = []
    for f, k in enumerate(sequence):
        ref.set_lights(_first(lights, k))
        want.append(_frame(ref, keep, f == 0))
    assert not np.array_equal(want[0], want[1])

    v, _ = _scene_viewer(proj, view)
    d = cases.to_device(lights)
    count = torch.full((1,), 10, dtype=torch.int32, device="cuda")
    v.set_lights_device(**d, count=count)
    torch.cuda.synchronize()
    assert np.array_equal(_frame(v, keep, True), want[0])
    assert v.light_prep()[0] == 10
    v.set_lights_device(**d)
    assert np.array_equal(_frame(v, keep, False), want[1]), "a new binding keeps every entry live"
    assert v.light_prep()[0] == 1000
    v.set_lights_device(**d, count=count)
    assert np.array_equal(_frame(v, keep, False), want[2])
    assert viewer.lib().grbh_viewer_set_light_count_device(v._h, None) == 0  # null: every bound entry live again
    assert np.array_equal(_frame(v, keep, False), want[3])
    v.set_lights(_first(lights, 10))
    assert np.array_equal(_frame(v, keep, False), want[4])
    assert viewer.lib().grbh_viewer_set_light_count_device(v._h, count.data_ptr()) < 0
    assert b"no device light list is bound" in viewer.lib().grbh_last_error()
    assert b"grbh_viewer_set_lights_device" in viewer.lib().grbh_last_error()
    torch.cuda.synchronize()
    ref.close()
    v.close()


def test_set_light_count_device_refusals_on_a_device_viewer(cuda):
    """No device list bound, a count in host memory, a misaligned count: refused by the C call, each with its message;
    a host, non-int32 or multi-element tensor refused in Python; the binding in force is kept."""
    import torch

    from granite_b200 import synth, viewer

    L = viewer.lib()
    proj, view = cases.default_camera(W, H)
    v, keep = _scene_viewer(proj, view)
    buf = torch.zeros(4, dtype=torch.int32, device="cuda")
    assert L.grbh_viewer_set_light_count_device(v._h, buf.data_ptr()) < 0
    assert b"no device light list is bound (grbh_viewer_set_lights_device" in L.grbh_last_error()
    lights = synth.make_lights(64, spot_fraction=0.25, aspect=W / H)
    d = cases.to_device(lights)
    v.set_lights_device(**d)
    host = (C.c_int32 * 2)()
    assert L.grbh_viewer_set_light_count_device(v._h, C.addressof(host)) < 0
    assert b"count is not device memory of the viewer's device" in L.grbh_last_error()
    assert L.grbh_viewer_set_light_count_device(v._h, buf.data_ptr() + 2) < 0
    assert b"not 4-byte aligned" in L.grbh_last_error()
    for bad, match in ((torch.zeros(1, dtype=torch.int32), "CUDA tensor"), (torch.zeros(1, dtype=torch.int64, device="cuda"), "int32"),
                       (torch.zeros(2, dtype=torch.int32, device="cuda"), "one torch.int32 element")):
        with pytest.raises(ValueError, match=match):
            v.set_lights_device(**d, count=bad)
    _frame(v, keep, True)
    assert v.light_prep()[0] == 64
    torch.cuda.synchronize()
    v.close()
