"""Shadowed device lights by map id, on one GPU: grb_light_list_shadowed_to_peers into three slot tensors of one device
(the slots, count words, flags and scratch counter, and the id prep of every slot against the pointer-form prep of the
source list), whole frames of set_lights_device(shadow_map_ids=) against the pointer form and host lights given
table[id] (a permuted table, ids out of range, with and without a device count that changes every frame, a table
replaced between frames), the table's maps_ready / maps_consumed events, and the refusals that need a device."""
import ctypes as C

import numpy as np
import pytest

from tests import device_lights_cases as cases
from tests import test_device_lights_cpu as base
from tests.device_shadow_cases import MapPool, transforms_in_input_order
from tests.test_device_lights_shadowed_cpu import GrbLightShadowList

pytestmark = pytest.mark.gpu

W, H = 320, 192
RES = 16
CAPACITY = 8192
LIGHT_ARRAYS = (("color", 12), ("position", 12), ("is_point", 1), ("rotation", 36), ("inner_cone", 4), ("outer_cone", 4))
INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1


def _ids_and_table(pointers, rng, extra=5):
    """A table holding `pointers` in a random order (plus `extra` null entries) and each light's id into it; some ids out
    of range (-1, the table size, INT32_MIN, INT32_MAX).  Returns (table, ids, effective map per light)."""
    n = len(pointers)
    size = n + extra
    slot = rng.permutation(size)[:n]
    table = np.zeros(size, np.int64)
    table[slot] = pointers
    ids = slot.astype(np.int32)
    ids[::13] = size
    ids[5::29] = -1
    ids[7] = INT32_MIN
    ids[11] = INT32_MAX
    valid = (ids >= 0) & (ids < size)
    eff = np.where(valid, table[np.clip(ids, 0, size - 1)], 0).astype(np.int64)
    return table, ids, eff


def _outputs():
    import torch

    return dict(records=torch.zeros(4096 * 48, dtype=torch.uint8, device="cuda"), model=torch.zeros(4096 * 48, dtype=torch.uint8, device="cuda"),
                mask=torch.zeros(128 * 4, dtype=torch.uint8, device="cuda"), ranges=torch.zeros(4096 * 8, dtype=torch.uint8, device="cuda"),
                transforms=torch.zeros(4096 * 64, dtype=torch.uint8, device="cuda"), maps=torch.zeros(4096 * 8, dtype=torch.uint8, device="cuda"),
                kept=torch.full((1,), -1, dtype=torch.int32, device="cuda"))


def _result(o):
    import torch

    torch.cuda.synchronize()
    return [int(o["kept"].item())] + [o[k].cpu().numpy().tobytes() for k in ("records", "model", "mask", "ranges", "transforms", "maps")]


def _prep_pointers(ll, count_t, transforms_t, maps_t, view, scratch):
    """grb_light_prep_shadowed_counted, the pointer form, into fresh outputs."""
    from granite_b200 import capi

    o = _outputs()
    sh = GrbLightShadowList(transforms_t.data_ptr(), maps_t.data_ptr())
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    rc = capi.lib().grb_light_prep_shadowed_counted(C.byref(ll), p(count_t), C.byref(sh), C.byref(view), p(o["records"]), p(o["model"]), p(o["mask"]),
                                                    p(o["ranges"]), p(o["transforms"]), p(o["maps"]), p(o["kept"]), p(scratch),
                                                    C.c_uint64(scratch.numel()), capi.stream_ptr())
    capi.check(rc, "grb_light_prep_shadowed_counted")
    return _result(o)


def _prep_ids(ll, count_t, transforms_t, ids_t, table_t, view, scratch):
    from granite_b200 import harness

    o = _outputs()
    harness.light_prep_shadow_ids(ll, count_t, transforms_t, ids_t, table_t, view, o["records"], o["model"], o["mask"], o["ranges"], o["transforms"],
                                  o["maps"], o["kept"], scratch)
    return _result(o)


def test_shadowed_push_into_three_slots_and_id_prep_parity(cuda, oracle):
    """For counts 0, 1, 37, 4096, 8192 and the clamps -3 and 9000, with the entries past the count poisoned: each slot
    holds the live bytes of all eight arrays and the live count, every other byte its sentinel; every rank's flag array
    has word 0 at the epoch and the scratch counter is back at 0.  The id prep of each slot equals the id prep of the
    source list and the pointer-form prep given table[id], bit for bit."""
    import torch

    from granite_b200 import capi, harness, synth, viewer

    w, h = 1920, 1080
    proj, view_m = cases.default_camera(w, h)
    lights = synth.make_lights(CAPACITY, spot_fraction=0.25)
    lights.position[::7, 2] += 200.0
    lights = cases.shuffled(lights)
    host = viewer.Viewer(w, h, cuda_device=-1)
    host.set_camera(proj, view_m)
    view = base.prep_view(oracle, host)
    host.close()

    rng = np.random.default_rng(17)
    fake = np.int64(0x7F0000000000) + np.arange(1, 1001, dtype=np.int64) * 0x1000  # never dereferenced by the prep
    table, ids, _ = _ids_and_table(fake, rng)
    ids = ids[rng.integers(0, len(ids), CAPACITY)]
    valid = (ids >= 0) & (ids < len(table))
    eff = np.where(valid, table[np.clip(ids, 0, len(table) - 1)], 0).astype(np.int64)
    d = cases.to_device(lights)
    t = torch.from_numpy(rng.standard_normal((CAPACITY, 16)).astype(np.float32)).cuda()
    ids_t, table_t, eff_t = (torch.from_numpy(a).cuda() for a in (ids, table, eff))
    clean = {k: x.clone() for k, x in d.items()}
    clean_t, clean_ids = t.clone(), ids_t.clone()
    src = harness.light_list(**d)
    _, _, slot_bytes = harness.light_shadow_slot_layout()
    assert slot_bytes == 8978688
    slots = [torch.full((slot_bytes,), 0xA5, dtype=torch.uint8, device="cuda") for _ in range(3)]
    flags = [torch.zeros(16, dtype=torch.int32, device="cuda") for _ in range(3)]
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    scratch = torch.zeros(int(capi.lib().grb_light_prep_scratch_bytes(CAPACITY)), dtype=torch.uint8, device="cuda")
    for epoch, raw in enumerate((0, 1, 37, 4096, CAPACITY, -3, 9000), start=1):
        live = min(max(raw, 0), CAPACITY)
        count.fill_(raw)
        for name in ("color", "position", "inner_cone"):
            d[name].copy_(clean[name])
            d[name][live:] = float("nan")
        t.copy_(clean_t)
        t[live:] = float("nan")
        ids_t.copy_(clean_ids)
        ids_t[live:] = 3  # an id that resolves: a read of a dead entry would show as a map
        for s in slots:
            s.fill_(0xA5)
        harness.light_list_shadowed_to_peers(src, t, ids_t, count, slots, flags, 0, epoch, counter)
        torch.cuda.synchronize()
        assert [int(f[0].item()) for f in flags] == [epoch] * 3
        assert int(counter.item()) == 0
        want = _prep_ids(src, count, t, ids_t, table_t, view, scratch)
        eff_live = eff_t.clone()
        eff_live[live:] = 0
        assert want == _prep_pointers(src, count, t, eff_live, view, scratch), f"count {raw}: the id prep differs from the pointer form's"
        sources = [d[name].reshape(-1).view(torch.uint8).cpu().numpy() for name, _ in LIGHT_ARRAYS]
        sources += [t.reshape(-1).view(torch.uint8).cpu().numpy(), ids_t.view(torch.uint8).cpu().numpy()]
        for s in slots:
            host_slot = s.cpu().numpy()
            written = np.zeros(slot_bytes, bool)
            assert int(host_slot[:4].view(np.int32)[0]) == live
            written[:4] = True
            at = 256
            for (name, elem), source in zip(LIGHT_ARRAYS + (("transforms", 64), ("map_ids", 4)), sources):
                n = live * elem
                assert np.array_equal(host_slot[at:at + n], source[:n]), (raw, name)
                written[at:at + n] = True
                at += (65536 * elem + 255) // 256 * 256
            assert (host_slot[~written] == 0xA5).all(), f"count {raw}: a byte past the live entries was written"
            ll, count_ptr, _ = harness.light_slot_layout(s.data_ptr())
            ll.count, ll.cutoff_range = CAPACITY, 1e10
            slot_t, slot_ids, _ = harness.light_shadow_slot_layout(s.data_ptr())
            got = _prep_ids(ll, _Ptr(count_ptr), _Ptr(slot_t), _Ptr(slot_ids), table_t, view, scratch)
            assert got == want, f"count {raw}: the slot's prep differs from the source's"


class _Ptr:
    """A device address where the harness takes a tensor (it only calls data_ptr())."""

    def __init__(self, p):
        self.p = p

    def data_ptr(self):
        return self.p


def _viewer(proj, view, lights=None, maps=None, **cfg):
    from granite_b200 import synth, viewer

    v = viewer.Viewer(W, H, cuda_device=0, light_shadows=True, shadow_resolution=RES, **cfg)
    scene = synth.make_scene(W, H)
    v.set_directional(scene.dir_color, scene.dir_direction)
    v.set_camera(proj, view)
    if lights is not None:
        v.set_lights(lights)
        v.set_light_shadow_maps([int(m) for m in maps])
    v.bake()
    keep = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, scene.emissive)]
    return v, keep


def _frame(v, keep, first):
    from granite_b200 import viewer

    v.render_frame(viewer.Viewer.host_gbuffer(*keep) if first else None)
    out = np.zeros((v.height, v.width), np.uint32)
    v.read_output(out)
    return out


def _first(lights, k):
    from granite_b200 import synth

    return synth.Lights(lights.color[:k], lights.position[:k], lights.is_point[:k], lights.rot[:k], lights.inner_cone[:k], lights.outer_cone[:k])


@pytest.mark.parametrize("counted", [False, True], ids=["every entry live", "device count"])
def test_frames_by_id_equal_pointer_form_and_host_light_frames(cuda, oracle, counted):
    """Five frames; each frame a torch op moves the lights (their transforms follow) and rewrites texels of the maps,
    and with a device count the count changes (a clamp past the capacity included).  Before frame 3 the table is
    replaced by another permutation with new ids.  The id form's output, HDR-main and shadow prep equal those of the
    pointer form given table[id] (null out of range) and of host lights given the same maps, bit for bit."""
    import torch

    from granite_b200 import synth

    n = 300
    proj, view = cases.default_camera(W, H)
    lights = synth.make_lights(n, spot_fraction=0.3, aspect=W / H)
    pool = MapPool(lights, RES)
    rng = np.random.default_rng(23)
    tables = [_ids_and_table(pool.pointers(), rng), _ids_and_table(pool.pointers(), rng, extra=40)]
    table, ids, eff = tables[0]
    counts = (n, 120, n + 50, 7, 260) if counted else (None,) * 5
    vh, keep = _viewer(proj, view, lights, eff)
    vp, _ = _viewer(proj, view)
    vi, _ = _viewer(proj, view)
    d = cases.to_device(lights)
    t = torch.from_numpy(transforms_in_input_order(oracle, vh, lights)).cuda()
    maps_t = torch.from_numpy(eff).cuda()
    ids_t = torch.from_numpy(ids).cuda()
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    extra = dict(count=count) if counted else {}
    vp.set_lights_device(**d, shadow_transforms=t, shadow_maps=maps_t, **extra)
    vi.set_light_shadow_map_table(table.tolist())
    vi.set_lights_device(**d, shadow_transforms=t, shadow_map_ids=ids_t, **extra)
    step = torch.tensor([0.3, -0.05, 0.7], device="cuda")
    for f in range(5):
        live = n if counts[f] is None else min(counts[f], n)
        if counted:
            count.fill_(counts[f])
        if f:
            d["position"].add_(step * torch.sin(torch.arange(n, device="cuda", dtype=torch.float32))[:, None])
            pool.rewrite(f)
        if f == 3:
            table, ids, eff = tables[1]
            vi.set_light_shadow_map_table(table.tolist())
            ids_t.copy_(torch.from_numpy(ids))
            maps_t.copy_(torch.from_numpy(eff))
        moved = synth.Lights(lights.color, d["position"].cpu().numpy(), lights.is_point, lights.rot, lights.inner_cone, lights.outer_cone)
        t.copy_(torch.from_numpy(transforms_in_input_order(oracle, vh, moved)))
        vh.set_lights(_first(moved, live))
        vh.set_light_shadow_maps([int(m) for m in eff[:live]])
        want = _frame(vh, keep, f == 0)
        for label, v in (("pointer form", vp), ("map ids", vi)):
            got = _frame(v, keep, f == 0)
            assert np.array_equal(want, got), f"frame {f} {label}: {int((want != got).sum())} pixels differ"
            assert np.array_equal(vh.download_image("HDR-main"), v.download_image("HDR-main")), f"frame {f} {label}: HDR-main"
        wt, wm = vh.light_shadow_prep()
        for v in (vp, vi):
            gt, gm = v.light_shadow_prep()
            assert gt.tobytes() == wt.tobytes() and np.array_equal(gm, wm), f"frame {f}: shadow prep"
        assert wm.any() and (wm == 0).any(), "some kept lights have maps and some do not"
    torch.cuda.synchronize()
    for v in (vh, vp, vi):
        v.close()


def test_table_maps_ready_and_consumed_events(cuda, oracle):
    """maps_ready given with the table: a producer stream sleeps, then writes the maps and records it; the frame shows
    the new maps.  maps_consumed: a stream that overwrites the maps after it leaves the frame in flight as it was."""
    import torch

    from granite_b200 import synth

    proj, view = cases.default_camera(W, H)
    lights = synth.make_lights(300, spot_fraction=0.3, aspect=W / H)
    old, new = MapPool(lights, RES, seed=1), MapPool(lights, RES, seed=2)
    new_ref, keep = _viewer(proj, view, lights, new.pointers())
    want = [_frame(new_ref, keep, True), _frame(new_ref, keep, False)]

    live = MapPool(lights, RES, seed=1)
    vd, _ = _viewer(proj, view)
    maps_ready, maps_consumed = torch.cuda.Event(), torch.cuda.Event()
    n = len(lights.color)
    vd.set_light_shadow_map_table(live.pointers()[::-1].tolist(), maps_ready=maps_ready, maps_consumed=maps_consumed)
    ids = torch.arange(n - 1, -1, -1, dtype=torch.int32, device="cuda")
    t = torch.from_numpy(transforms_in_input_order(oracle, vd, lights)).cuda()
    d = cases.to_device(lights)
    vd.set_lights_device(**d, shadow_transforms=t, shadow_map_ids=ids)
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
    for v in (new_ref, vd):
        v.close()


def test_refusals_that_need_a_device(cuda):
    """No table; a table entry or id arrays not in device memory; on a light source rank the pointer form is refused in
    favour of the id form, and on a receiving rank both bindings name the receiving one, which is accepted."""
    import torch

    from granite_b200 import capi, synth, viewer

    proj, view = cases.default_camera(W, H)
    d = cases.to_device(synth.make_lights(8))
    t = torch.zeros(8, 16, device="cuda")
    ids = torch.zeros(8, dtype=torch.int32, device="cuda")
    maps = torch.zeros(8, dtype=torch.int64, device="cuda")
    pool = torch.zeros(64, dtype=torch.int16, device="cuda")
    v = viewer.Viewer(W, H, cuda_device=0, light_shadows=True, shadow_resolution=RES)
    with pytest.raises(capi.GrbError, match="no shadow map table is set on this rank"):
        v.set_lights_device(**d, shadow_transforms=t, shadow_map_ids=ids)
    with pytest.raises(capi.GrbError, match="grbh_viewer_set_light_source_rank: not with clustered_lights_shadows"):
        v.set_light_source_rank(0)
    host_map = np.zeros(64, np.int16)
    with pytest.raises(capi.GrbError, match="map 1 is not device memory of the viewer's device"):
        v.set_light_shadow_map_table([pool.data_ptr(), host_map.ctypes.data])
    v.set_light_shadow_map_table([pool.data_ptr(), 0])
    L = viewer.lib()
    l = viewer.GrbhDeviceLights(8, *[d[k].data_ptr() for k in ("color", "position", "is_point", "rotation", "inner_cone", "outer_cone")], 1e10, None, None)
    t_host, ids_host = np.zeros((8, 16), np.float32), np.zeros(8, np.int32)
    for tp, ip, what in ((t_host.ctypes.data, ids.data_ptr(), b"shadow transforms is not device memory"),
                         (t.data_ptr(), ids_host.ctypes.data, b"map ids is not device memory")):
        assert L.grbh_viewer_set_lights_device_shadow_ids(v._h, C.byref(l), C.byref(viewer.GrbhDeviceLightShadowIds(tp, ip))) < 0
        assert what in L.grbh_last_error()
    v.set_lights_device(**d, shadow_transforms=t, shadow_map_ids=ids)
    v.set_light_source_rank(0)  # unsharded: one band; accepted now that the rank has a table
    with pytest.raises(capi.GrbError, match="binds shadowed device lights by map id.*grbh_viewer_set_lights_device_shadow_ids"):
        v.set_lights_device(**d, shadow_transforms=t, shadow_maps=maps)
    v.set_light_source_rank(-1)
    v.set_lights_device(**d, shadow_transforms=t, shadow_maps=maps)  # off again: the pointer form is back
    v.close()

    r = viewer.Viewer(W, H, cuda_device=0, light_shadows=True, shadow_resolution=RES)
    r.set_row_shards([(0, 48), (48, 96), (96, 144), (144, 192)], 1)
    r.set_light_shadow_map_table([pool.data_ptr()])
    r.set_light_source_rank(0)
    for kw in (dict(shadow_map_ids=ids), dict(shadow_maps=maps)):
        with pytest.raises(capi.GrbError, match="rank 1 receives its device lights from light source rank 0"):
            r.set_lights_device(**d, shadow_transforms=t, **kw)
    r.set_lights_device_from_source(64)
    r.close()
    torch.cuda.synchronize()
