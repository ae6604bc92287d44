"""Shadowed device lights by map id, without a GPU: the shadowed slot's layout, the shadowed push of
grb_light_list_shadowed_to_peers and the id resolution of grb_light_prep_shadow_ids's pack kernel compiled for the CPU
(granite_b200/csrc/grb_light_prep.cuh through tests/cpp/emulate_light_shadow_ids.cpp), and every refusal of the kernel
entries and the viewer API that comes before any CUDA call."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from granite_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIGHT_ARRAYS = (("color", 12), ("position", 12), ("is_point", 1), ("rotation", 36), ("inner_cone", 4), ("outer_cone", 4))
ARRAYS = LIGHT_ARRAYS + (("transforms", 64), ("map_ids", 4))
LIGHT_SLOT_BYTES = 4522240
SLOT_BYTES = 8978688
CAPACITY = 300
INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1


class GrbLightShadowIdList(C.Structure):
    _fields_ = [("transforms", C.c_void_p), ("map_ids", C.c_void_p)]


class GrbLightShadowList(C.Structure):
    _fields_ = [("transforms", C.c_void_p), ("maps", C.c_void_p)]


@pytest.fixture(scope="module")
def built():
    from granite_b200 import build

    return build.build_all()


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """The id form and, beside it, the pointer form of the pack's shadow part (emulate_light_prep_shadows.cpp)."""
    out = str(tmp_path_factory.mktemp("emu") / "libemu_light_shadow_ids.so")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    srcs = [os.path.join(ROOT, "tests", "cpp", f) for f in ("emulate_light_shadow_ids.cpp", "emulate_light_prep_shadows.cpp")]
    cmd = ["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-x", "c++", f"-I{cuda}/include", *srcs, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(out)
    lib.emu_shadow_push.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32]
    lib.emu_shadow_slot_layout.argtypes = [C.c_void_p]
    lib.emu_pack_shadow_ids.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    lib.emu_pack_shadows.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    return lib


def _offsets():
    at, out = 256, []
    for _, e in ARRAYS:
        out.append(at)
        at += (65536 * e + 255) // 256 * 256
    return out, at


def test_shadow_slot_layout(built, emu):
    """The shadow part starts at the light slot's end: 65536 transforms, then 65536 map ids, each from a multiple of
    256 bytes, 8,978,688 bytes in all; the C entry, the CPU build and this file agree, and the light slot is unchanged."""
    from granite_b200 import harness

    offsets, end = _offsets()
    assert end == SLOT_BYTES == LIGHT_SLOT_BYTES + 65536 * 64 + 65536 * 4
    assert offsets[6] == LIGHT_SLOT_BYTES and all(o % 256 == 0 for o in offsets)
    layout = (C.c_uint64 * 3)()
    emu.emu_shadow_slot_layout(layout)
    assert list(layout) == [offsets[6], offsets[7], SLOT_BYTES]
    base = 0x7F0000000000
    t, m, size = harness.light_shadow_slot_layout(base)
    assert (t, m, size) == (base + offsets[6], base + offsets[7], SLOT_BYTES)
    assert harness.light_shadow_slot_layout(None) == (None, None, SLOT_BYTES)
    assert harness.light_slot_layout(None)[2] == LIGHT_SLOT_BYTES


def test_shadow_slot_layout_refusals(built):
    from granite_b200 import capi

    L = capi.lib()
    size = C.c_uint64()
    assert L.grb_light_shadow_slot_layout(None, None, None, None) == -1
    assert b"grb_light_shadow_slot_layout: a null size pointer" in L.grb_last_error_string()
    assert L.grb_light_shadow_slot_layout(C.c_void_p(0x10008), None, None, C.byref(size)) == -1
    assert b"grb_light_shadow_slot_layout: the slot is not 16-byte aligned" in L.grb_last_error_string()


def _shadows(n, rng, table_size):
    """(transforms (n, 16) float32, ids (n,) int32): ids in range and some out of it, the extremes included."""
    t = rng.standard_normal((n, 16)).astype(np.float32)
    ids = rng.integers(0, table_size, n).astype(np.int32)
    bad = [-1, table_size, INT32_MIN, INT32_MAX]
    ids[3:3 + 4 * len(bad):4] = bad[: len(ids[3:3 + 4 * len(bad):4])]
    return t, ids


def _source(arrays, live_rows, offset):
    """Each array as a buffer whose data starts `offset` bytes into a 64-byte aligned allocation (offset 4: no array
    moves in 16-byte words), entries at or past live_rows poisoned (NaN floats, 0xFF bytes, ids that resolve)."""
    keep, ptrs = [], []
    for (name, _), a in zip(ARRAYS, arrays):
        a = np.ascontiguousarray(a).copy()
        if name == "is_point":
            a[live_rows:] = 0xFF
        elif name == "map_ids":
            a[live_rows:] = 1
        else:
            a[live_rows:] = np.float32(np.nan)
        raw = np.zeros(a.nbytes + 128, np.uint8)
        start = (-raw.ctypes.data) % 64 + offset
        raw[start:start + a.nbytes] = a.reshape(-1).view(np.uint8)
        keep.append((raw, start, a))
        ptrs.append(raw.ctypes.data + start)
    return keep, ptrs


@pytest.mark.parametrize("offset", [0, 4])
@pytest.mark.parametrize("count", [-3, 0, 1, 37, CAPACITY, CAPACITY + 10, None])
def test_shadowed_push_stores_the_live_bytes_of_eight_arrays(built, emu, count, offset):
    """Into three slots filled with a sentinel: bytes [0, live x element size) of all eight arrays equal the source's,
    the count word holds live, and every other byte of every slot still holds the sentinel.  The source's dead entries
    are poisoned, so a read of them would show."""
    from granite_b200 import capi

    rng = np.random.default_rng(5)
    lights = synth.make_lights(CAPACITY, spot_fraction=0.25)
    t, ids = _shadows(CAPACITY, rng, 64)
    live = CAPACITY if count is None else min(max(count, 0), CAPACITY)
    arrays = (np.float32(lights.color), np.float32(lights.position), np.uint8(lights.is_point), np.float32(lights.rot),
              np.float32(lights.inner_cone), np.float32(lights.outer_cone), t, ids)
    keep, ptrs = _source(arrays, live, offset)
    ll = capi.GrbLightList(CAPACITY, *ptrs[:6], 1e10)
    sh = GrbLightShadowIdList(ptrs[6], ptrs[7])
    slots = [np.full(SLOT_BYTES + 16, 0xA5, np.uint8) for _ in range(3)]
    starts = [(-s.ctypes.data) % 16 for s in slots]
    addrs = (C.c_void_p * 3)(*[s.ctypes.data + k for s, k in zip(slots, starts)])
    got = emu.emu_shadow_push(C.byref(ll), C.byref(sh), count is not None, 0 if count is None else count, addrs, 3)
    assert got == live
    offsets, _ = _offsets()
    for s, k in zip(slots, starts):
        slot = s[k:k + SLOT_BYTES]
        written = np.zeros(SLOT_BYTES, bool)
        assert int(slot[:4].view(np.int32)[0]) == live
        written[:4] = True
        for (name, elem), (_, _, a), at in zip(ARRAYS, keep, offsets):
            n = live * elem
            assert np.array_equal(slot[at:at + n], a.reshape(-1).view(np.uint8)[:n]), name
            written[at:at + n] = True
        assert (slot[~written] == 0xA5).all(), "a byte outside the live entries and the count word was written"
        assert (s[:k] == 0xA5).all() and (s[k + SLOT_BYTES:] == 0xA5).all()


def _pack(emu, pointer_form, transforms, ids_or_maps, order, slots, table=None):
    """The shadow tables of `slots` slots from either form, in a buffer with a sentinel around them."""
    n = len(transforms)
    base = 8 * 7  # an offset 8 bytes past a 16-byte boundary, as for odd slot counts
    buf = np.full(base + 72 * slots + 64, 0xA5, np.uint8)
    raw = np.zeros(16 * n + 1, np.float32)[1:]  # the transforms only 4-byte aligned
    raw[:] = transforms.reshape(-1)
    out_t, out_m = C.c_void_p(buf.ctypes.data + base), C.c_void_p(buf.ctypes.data + base + 64 * slots)
    o = np.ascontiguousarray(order, np.uint32)
    if pointer_form:
        sh = GrbLightShadowList(raw.ctypes.data, ids_or_maps.ctypes.data)
        emu.emu_pack_shadows(C.byref(sh), o.ctypes.data, len(o), slots, out_t, out_m)
    else:
        sh = GrbLightShadowIdList(raw.ctypes.data, ids_or_maps.ctypes.data)
        emu.emu_pack_shadow_ids(C.byref(sh), table.ctypes.data if len(table) else None, len(table), o.ctypes.data, len(o), slots, out_t, out_m)
    assert (buf[:base] == 0xA5).all() and (buf[base + 72 * slots:] == 0xA5).all(), "a byte outside the shadow tables was written"
    return buf[base:base + 72 * slots].copy()


@pytest.mark.parametrize("n,kept,table_size", [(300, 211, 64), (37, 37, 37), (5000, 4096, 1000), (12, 5, 0)])
def test_id_resolution_gives_the_pointer_forms_bytes(emu, n, kept, table_size):
    """With maps[i] = table[ids[i]] (null where the id is -1, table_size, INT32_MIN or INT32_MAX) the id form packs the
    pointer form's bytes; a permuted table with null entries.  Entries no slot packs are poisoned (ids that resolve to
    a map, NaN transforms) and none of them reaches the output."""
    rng = np.random.default_rng(n)
    transforms, ids = _shadows(n, rng, max(table_size, 1))
    if table_size == 0:
        ids[:] = rng.integers(-3, 3, n)
    table = (np.uint64(0x7F0000000000) + rng.permutation(max(table_size, 1)).astype(np.uint64) * np.uint64(0x1000))[:table_size]
    table[::9] = 0  # null entries: no shadow either
    order = rng.permutation(n)[:kept]
    dead = np.setdiff1d(np.arange(n), order)
    transforms[dead] = np.nan
    ids[dead] = 0
    valid = (ids >= 0) & (ids < table_size)
    maps = np.where(valid, table[np.clip(ids, 0, max(table_size - 1, 0))] if table_size else 0, 0).astype(np.uint64)
    slots = min(n, 4096)
    by_pointer = _pack(emu, True, transforms, maps, order, slots)
    by_id = _pack(emu, False, transforms, ids, order, slots, table)
    assert by_id.tobytes() == by_pointer.tobytes()
    got_t = by_id[:64 * slots].view(np.float32).reshape(slots, 16)
    got_m = by_id[64 * slots:].view(np.uint64)
    assert not np.isnan(got_t).any(), "a dead entry's transform was packed"
    assert np.array_equal(got_m[:kept], maps[order]) and not got_m[kept:].any()
    for bad in (-1, table_size, INT32_MIN, INT32_MAX):
        hit = np.flatnonzero(ids[order] == bad)
        assert not got_m[hit].any()


def capi_light_list(d, n=4):
    from granite_b200 import capi

    return capi.GrbLightList(n, d, d, d, d, d, d, 1e10)


def test_prep_shadow_ids_refuses_before_any_cuda_call(built):
    """grb_light_prep_shadow_ids refuses, with GRB_ERR_INVALID_ARGUMENT and its message: a null id list, null
    transforms or ids with lights, a null output table, a table size outside 0..65536, a null table with entries,
    misaligned tables or ids, a misaligned input count, and what grb_light_prep refuses."""
    from granite_b200 import capi

    L = capi.lib()
    fn = L.grb_light_prep_shadow_ids
    d = 4096
    ll = capi_light_list(d)
    view = (C.c_uint8 * 256)()
    ids = capi.GrbLightShadowIdList(d, d)

    def call(lights=C.byref(ll), count=None, i=C.byref(ids), table=d, size=8, out_t=d, out_m=d, scratch=d):
        return fn(lights, count, i, table, size, view, d, d, d, d, out_t, out_m, d, scratch, 1 << 40, None)

    def refused(text, **kw):
        assert call(**kw) == -1
        assert text in L.grb_last_error_string(), L.grb_last_error_string()

    refused(b"grb_light_prep_shadow_ids: a null shadow id list", i=None)
    refused(b"grb_light_prep_shadow_ids: a null pointer or a count outside 0..65536", lights=None)
    refused(b"grb_light_prep_shadow_ids: a null pointer or a count outside 0..65536", lights=C.byref(capi_light_list(d, 65537)))
    nulls = b"grb_light_prep_shadow_ids: a null shadow transform or map id array, or a null output table"
    for bad in (capi.GrbLightShadowIdList(None, d), capi.GrbLightShadowIdList(d, None)):
        refused(nulls, i=C.byref(bad))
    refused(nulls, out_t=None)
    refused(nulls, out_m=None)
    table = b"grb_light_prep_shadow_ids: a map table size outside 0..GRB_MAX_LIGHT_LIST or a null map table"
    for size in (-1, 65537, INT32_MIN):
        refused(table, size=size)
    refused(table, table=None, size=1)
    aligned = b"not 8-byte aligned, or the map ids not 4-byte aligned"
    refused(aligned, table=d + 4)
    refused(aligned, out_t=d + 4)
    refused(aligned, out_m=d + 4)
    refused(aligned, i=C.byref(capi.GrbLightShadowIdList(d, d + 2)))
    refused(b"grb_light_prep_shadow_ids: the input count is not 4-byte aligned", count=d + 2)


def test_shadowed_push_refuses_before_any_cuda_call(built):
    """grb_light_list_shadowed_to_peers refuses what grb_light_list_to_peers refuses, under its own name, and a null id
    list or null id arrays with lights."""
    from granite_b200 import capi

    L = capi.lib()
    fn = L.grb_light_list_shadowed_to_peers
    d = C.c_void_p(4096)
    ll = capi_light_list(4096)
    ids = capi.GrbLightShadowIdList(4096, 4096)
    slots = (C.c_void_p * 2)(4096, 4096)
    flags = (C.c_void_p * 2)(64, 64)
    peers = b"grb_light_list_shadowed_to_peers: null pointer, peer_count outside 1..GRB_MAX_PEERS or flag_index outside 0..peer_count-1"
    for args in ((C.byref(ll), C.byref(ids), None, slots, None, 2, 0, 1, d, None),
                 (C.byref(ll), C.byref(ids), None, slots, flags, 2, 0, 1, None, None),
                 (C.byref(ll), C.byref(ids), None, slots, flags, 0, 0, 1, d, None),
                 (C.byref(ll), C.byref(ids), None, slots, flags, 9, 0, 1, d, None),
                 (C.byref(ll), C.byref(ids), None, slots, flags, 2, 2, 1, d, None),
                 (C.byref(ll), C.byref(ids), None, None, flags, 2, 0, 1, d, None)):
        assert fn(*args) == -1
        assert peers in L.grb_last_error_string()
    lists = b"grb_light_list_shadowed_to_peers: a null light list or array, or a count outside 0..GRB_MAX_LIGHT_LIST"
    for bad in (None, C.byref(capi.GrbLightList(4, d, d, None, d, d, d, 1e10)), C.byref(capi_light_list(4096, -1))):
        assert fn(bad, C.byref(ids), None, slots, flags, 2, 0, 1, d, None) == -1
        assert lists in L.grb_last_error_string()
    assert fn(C.byref(ll), C.byref(ids), C.c_void_p(4098), slots, flags, 2, 0, 1, d, None) == -1
    assert b"grb_light_list_shadowed_to_peers: the input count is not 4-byte aligned" in L.grb_last_error_string()
    odd = (C.c_void_p * 2)(4096, 4104)
    assert fn(C.byref(ll), C.byref(ids), None, odd, flags, 2, 0, 1, d, None) == -1
    assert b"grb_light_list_shadowed_to_peers: a slot is not 16-byte aligned" in L.grb_last_error_string()
    no_ids = b"grb_light_list_shadowed_to_peers: a null shadow id list, or null transforms or map ids"
    for bad in (None, C.byref(capi.GrbLightShadowIdList(None, 4096)), C.byref(capi.GrbLightShadowIdList(4096, None))):
        assert fn(C.byref(ll), bad, None, slots, flags, 2, 0, 1, d, None) == -1
        assert no_ids in L.grb_last_error_string()
    empty = capi_light_list(4096, 0)
    assert fn(C.byref(empty), None, None, slots, flags, 2, 0, 1, d, None) == -1  # the id list itself is always needed
    assert no_ids in L.grb_last_error_string()


def _refused(L, rc, text):
    assert rc < 0
    assert text in L.grbh_last_error(), L.grbh_last_error()


def test_viewer_refusals_on_a_host_only_viewer(built):
    """Every refusal of grbh_viewer_set_light_shadow_map_table and grbh_viewer_set_lights_device_shadow_ids that a
    host-only viewer reaches, each with its message; set_light_source_rank on a shadowed viewer keeps its old refusal
    without a table; Viewer.set_lights_device refuses shadow_maps with shadow_map_ids."""
    from granite_b200 import viewer

    L = viewer.lib()
    table = b"grbh_viewer_set_light_shadow_map_table: "
    ids = b"grbh_viewer_set_lights_device_shadow_ids: "
    maps = (C.c_void_p * 2)(4096, None)
    _refused(L, L.grbh_viewer_set_light_shadow_map_table(None, maps, 2, None, None), table + b"null viewer")
    l = viewer.GrbhDeviceLights(4, 16, 16, 16, 16, 16, 16, 1e10, None, None)
    sh = viewer.GrbhDeviceLightShadowIds(16, 16)
    _refused(L, L.grbh_viewer_set_lights_device_shadow_ids(None, C.byref(l), C.byref(sh)), ids + b"null viewer, light list or shadow id list")

    plain = viewer.Viewer(64, 64, cuda_device=-1)
    _refused(L, L.grbh_viewer_set_light_shadow_map_table(plain._h, maps, 2, None, None), table + b"the viewer was created without clustered_lights_shadows")
    _refused(L, L.grbh_viewer_set_lights_device_shadow_ids(plain._h, C.byref(l), C.byref(sh)), ids + b"the viewer was created without clustered_lights_shadows")
    plain.close()

    s = viewer.Viewer(64, 64, cuda_device=-1, light_shadows=True)
    for count in (-1, 65537):
        _refused(L, L.grbh_viewer_set_light_shadow_map_table(s._h, maps, count, None, None), table + f"count {count} is outside 0..65536".encode())
    _refused(L, L.grbh_viewer_set_light_shadow_map_table(s._h, None, 2, None, None), table + b"null map array with count > 0")
    for count in (0, 2):
        _refused(L, L.grbh_viewer_set_light_shadow_map_table(s._h, maps, count, None, None), table + b"host-only viewer")
    _refused(L, L.grbh_viewer_set_lights_device_shadow_ids(s._h, C.byref(l), None), ids + b"null viewer, light list or shadow id list")
    for n in (-1, 65537):
        bad = viewer.GrbhDeviceLights(n, 16, 16, 16, 16, 16, 16, 1e10, None, None)
        _refused(L, L.grbh_viewer_set_lights_device_shadow_ids(s._h, C.byref(bad), C.byref(sh)), ids + f"count {n} is outside 0..65536".encode())
    for t, m in ((None, 16), (16, None)):
        _refused(L, L.grbh_viewer_set_lights_device_shadow_ids(s._h, C.byref(l), C.byref(viewer.GrbhDeviceLightShadowIds(t, m))),
                 ids + b"null shadow transforms or map ids")
    _refused(L, L.grbh_viewer_set_lights_device_shadow_ids(s._h, C.byref(l), C.byref(sh)), ids + b"host-only viewer")
    # without a table (a host-only viewer cannot have one) the light source rank is refused as before
    _refused(L, L.grbh_viewer_set_light_source_rank(s._h, 0), b"grbh_viewer_set_light_source_rank: not with clustered_lights_shadows")
    assert b"unless a shadow map table is set (grbh_viewer_set_light_shadow_map_table)" in L.grbh_last_error()
    with pytest.raises(ValueError, match="shadow_maps and shadow_map_ids together"):
        s.set_lights_device(*([None] * 6), shadow_transforms=object(), shadow_maps=object(), shadow_map_ids=object())
    with pytest.raises(ValueError, match="map events go with the table"):
        s.set_lights_device(*([None] * 6), shadow_transforms=object(), shadow_map_ids=object(), maps_ready=object())
    s.close()
