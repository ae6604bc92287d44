"""Device lights pushed from one rank, on one GPU: grb_light_list_to_peers pushes a capacity-8192 list into three slot
tensors of one device (the slots every rank of a row-sharded frame would hold), with counts from 0 to the capacity and
the clamps; the slots, the count words, the flags and the scratch counter are checked, and the counted prep of every
slot must equal the prep of the source list bit for bit.  Also a receiver's credit, and the refusal that needs a
baked viewer."""
import ctypes as C

import numpy as np
import pytest

from tests import device_lights_cases as cases
from tests import test_device_lights_cpu as base

pytestmark = pytest.mark.gpu

CAPACITY = 8192
ARRAYS = (("color", 12), ("position", 12), ("is_point", 1), ("rotation", 36), ("inner_cone", 4), ("outer_cone", 4))


def _prep(ll, count_ptr, view, scratch):
    """grb_light_prep_counted of ll with the device count at count_ptr into fresh outputs: the kept count and the bytes
    of records, model rows, type mask and Z ranges."""
    import torch

    from granite_b200 import capi

    records = torch.zeros(4096 * 48, dtype=torch.uint8, device="cuda")
    model = torch.zeros(4096 * 48, dtype=torch.uint8, device="cuda")
    mask = torch.zeros(128 * 4, dtype=torch.uint8, device="cuda")
    ranges = torch.zeros(4096 * 8, dtype=torch.uint8, device="cuda")
    kept = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    L = capi.lib()
    rc = L.grb_light_prep_counted(C.byref(ll), C.c_void_p(count_ptr), C.byref(view), C.c_void_p(records.data_ptr()), C.c_void_p(model.data_ptr()),
                                  C.c_void_p(mask.data_ptr()), C.c_void_p(ranges.data_ptr()), C.c_void_p(kept.data_ptr()), C.c_void_p(scratch.data_ptr()),
                                  C.c_uint64(scratch.numel()), capi.stream_ptr())
    capi.check(rc, "grb_light_prep_counted")
    torch.cuda.synchronize()
    return [int(kept.item())] + [t.cpu().numpy().tobytes() for t in (records, model, mask, ranges)]


def test_push_into_three_slots_and_prep_parity(cuda, oracle):
    """For counts 0, 1, 37, 4096, 8192 and the clamps -3 and 9000, with the entries past the count NaN: each slot holds
    the live bytes of each array and the live count, every other byte its sentinel; every rank's flag array has word 0
    at the epoch; the scratch counter is back at 0; and the counted prep of each slot (as a list of the receiver's own
    capacity) equals the counted prep of the source list, bit for bit."""
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

    d = cases.to_device(lights)
    clean = {k: t.clone() for k, t in d.items()}
    src = harness.light_list(**d)
    _, _, slot_bytes = harness.light_slot_layout()
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
        for s in slots:
            s.fill_(0xA5)
        harness.light_list_to_peers(src, count, slots, flags, 0, epoch, counter)
        torch.cuda.synchronize()
        assert [int(f[0].item()) for f in flags] == [epoch] * 3
        assert int(counter.item()) == 0
        want = _prep(src, count.data_ptr(), view, scratch)
        for s in slots:
            host_slot = s.cpu().numpy()
            written = np.zeros(slot_bytes, bool)
            assert int(host_slot[:4].view(np.int32)[0]) == live
            written[:4] = True
            at = 256
            for name, elem in ARRAYS:
                n = live * elem
                source = d[name].reshape(-1).view(torch.uint8).cpu().numpy()
                assert np.array_equal(host_slot[at:at + n], source[:n]), (raw, name)
                written[at:at + n] = True
                at += (65536 * elem + 255) // 256 * 256
            assert (host_slot[~written] == 0xA5).all(), f"count {raw}: a byte past the live entries was written"
            ll, count_ptr, _ = harness.light_slot_layout(s.data_ptr())
            ll.count, ll.cutoff_range = CAPACITY, 1e10
            got = _prep(ll, count_ptr, view, scratch)
            assert got[0] == want[0] and got[1:] == want[1:], f"count {raw}: the slot's prep differs from the source's"


def test_no_count_pushes_the_whole_list_and_flags_only_publish_stores_nothing(cuda):
    """Without a device count every entry is live; a receiver's credit, the flags-only publish of grb_peer_publish,
    raises the flags at its epoch and stores nothing."""
    import torch

    from granite_b200 import harness, synth

    lights = synth.make_lights(37, spot_fraction=0.5)
    d = cases.to_device(lights)
    src = harness.light_list(**d)
    _, _, slot_bytes = harness.light_slot_layout()
    slots = [torch.full((slot_bytes,), 0x5A, dtype=torch.uint8, device="cuda") for _ in range(2)]
    flags = [torch.zeros(16, dtype=torch.int32, device="cuda") for _ in range(2)]
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    harness.light_list_to_peers(src, None, slots, flags, 1, 7, counter)
    torch.cuda.synchronize()
    for s in slots:
        assert int(s[:4].view(torch.int32).item()) == 37
        assert torch.equal(s[256 + 16 * 0:256 + 37 * 12], d["color"].reshape(-1).view(torch.uint8))
    before = [s.clone() for s in slots]
    harness.peer_publish(flags, 0, 8, counter)
    torch.cuda.synchronize()
    assert [f[:2].tolist() for f in flags] == [[8, 7], [8, 7]]
    assert int(counter.item()) == 0
    assert all(torch.equal(a, b) for a, b in zip(before, slots))


def test_light_source_rank_is_refused_after_bake_and_changes_nothing_unsharded(cuda):
    """An unsharded viewer accepts source rank 0 before bake and renders the frame it renders without it; after bake
    the call is refused with its message."""
    import torch

    from granite_b200 import capi, synth, viewer

    w, h = 160, 96
    proj, view_m = cases.default_camera(w, h)
    lights = synth.make_lights(300, spot_fraction=0.25)
    scene = synth.make_scene(w, h)
    keep = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, scene.emissive)]
    frames = []
    for source in (-1, 0):
        v = viewer.Viewer(w, h, cuda_device=0)
        v.set_directional(scene.dir_color, scene.dir_direction)
        v.set_camera(proj, view_m)
        v.set_light_source_rank(source)
        d = cases.to_device(lights)
        v.set_lights_device(**d)
        v.bake()
        with pytest.raises(capi.GrbError, match="grbh_viewer_set_light_source_rank: the viewer is baked"):
            v.set_light_source_rank(source)
        v.render_frame(viewer.Viewer.host_gbuffer(*keep))
        out = np.zeros((h, w), np.uint32)
        v.read_output(out)
        frames.append(out)
        torch.cuda.synchronize()
        v.close()
    assert np.array_equal(frames[0], frames[1])
