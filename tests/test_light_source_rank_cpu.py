"""Device lights pushed from one rank, without a GPU: the argument checks of grb_light_list_to_peers and
grb_light_slot_layout that refuse before any CUDA call, the slot layout, the push of grb_light_list_to_peers compiled for
the CPU (lp::light_push, lp::push_light_chunk and lp::live_count of granite_b200/csrc/grb_light_prep.cuh, run for every
thread of the kernel's grid), and every refusal of the light-source-rank API that a host-only viewer reaches."""
import ctypes as C

import numpy as np
import pytest

from tests import test_device_light_count_cpu as counted

ARRAYS = (("color", 12), ("position", 12), ("is_point", 1), ("rotation", 36), ("inner_cone", 4), ("outer_cone", 4))
SLOT_BYTES = 256 + sum((65536 * e + 255) // 256 * 256 for _, e in ARRAYS)
CAPACITY = 300


@pytest.fixture(scope="module")
def built():
    from granite_b200 import build

    return build.build_all()


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = counted._compile(tmp_path_factory, "emulate_light_push.cpp")
    lib.emu_push.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32]
    lib.emu_slot_layout.argtypes = [C.c_void_p]
    return lib


def test_slot_layout(built, emu):
    """The count word at the slot's start, then the six arrays of a GRB_MAX_LIGHT_LIST-entry list in GrbLightList order,
    each from a multiple of 256 bytes; the C entry, the CPU build of the layout and this file agree."""
    from granite_b200 import capi, harness

    assert capi.MAX_LIGHT_LIST == 65536
    offsets = [256]
    for _, e in ARRAYS[:-1]:
        offsets.append(offsets[-1] + (65536 * e + 255) // 256 * 256)
    assert SLOT_BYTES == 4522240  # about 4.5 MB: 69 bytes per entry plus the count word's 256
    layout = (C.c_uint64 * 8)()
    emu.emu_slot_layout(layout)
    assert list(layout) == [0, *offsets, SLOT_BYTES]

    base = 0x7F0000000000
    ll, count, size = harness.light_slot_layout(base)
    assert size == SLOT_BYTES and count == base and ll.count == 65536 and ll.cutoff_range == 0.0
    got = [getattr(ll, name) for name, _ in ARRAYS]
    assert got == [base + o for o in offsets]
    assert all(o % 256 == 0 for o in offsets)
    ll, count, size = harness.light_slot_layout(None)  # size query: null pointers
    assert size == SLOT_BYTES and not count and all(not getattr(ll, name) for name, _ in ARRAYS)


def test_slot_layout_refusals(built):
    from granite_b200 import capi

    L = capi.lib()
    size = C.c_uint64()
    assert L.grb_light_slot_layout(None, None, None, None) == -1
    assert b"grb_light_slot_layout: a null size pointer" in L.grb_last_error_string()
    assert L.grb_light_slot_layout(C.c_void_p(0x10008), None, None, C.byref(size)) == -1
    assert b"grb_light_slot_layout: the slot is not 16-byte aligned" in L.grb_last_error_string()


def _source(lights, live_rows, offset):
    """The six arrays of `lights` as numpy buffers whose data starts `offset` bytes into an allocation aligned to 64
    bytes (offset 4: the float arrays move in 4-byte words and is_point byte by byte), entries at or past live_rows
    NaN (0xFF for is_point)."""
    keep = []
    ptrs = []
    for (name, elem), a in zip(ARRAYS, (lights.color, lights.position, lights.is_point, lights.rot, lights.inner_cone, lights.outer_cone)):
        a = np.ascontiguousarray(a, np.uint8 if name == "is_point" else np.float32).copy()
        a[live_rows:] = 0xFF if name == "is_point" else np.float32(np.nan)
        raw = np.zeros(a.nbytes + 128, np.uint8)
        start = (-raw.ctypes.data) % 64 + offset
        raw[start:start + a.nbytes] = a.reshape(-1).view(np.uint8)
        keep.append((raw, start, a))
        ptrs.append(raw.ctypes.data + start)
    return keep, ptrs


@pytest.mark.parametrize("offset", [0, 4])
@pytest.mark.parametrize("count", [-3, 0, 1, 37, CAPACITY, CAPACITY + 10, None])
def test_push_stores_the_live_bytes_and_the_count_only(built, emu, count, offset):
    """Into three slots filled with a sentinel: bytes [0, live x element size) of each array equal the source's, the
    count word holds live = min(max(count, 0), capacity) (the capacity without a count), and every other byte of every
    slot still holds the sentinel.  The source's dead entries are NaN, so a read of them would show."""
    from granite_b200 import capi, synth

    lights = synth.make_lights(CAPACITY, spot_fraction=0.25)
    live = CAPACITY if count is None else min(max(count, 0), CAPACITY)
    keep, ptrs = _source(lights, live, offset)
    ll = capi.GrbLightList(CAPACITY, *ptrs, 1e10)
    slots = [np.full(SLOT_BYTES + 16, 0xA5, np.uint8) for _ in range(3)]
    starts = [(-s.ctypes.data) % 16 for s in slots]  # the kernel's slots are 16-byte aligned
    addrs = (C.c_void_p * 3)(*[s.ctypes.data + k for s, k in zip(slots, starts)])
    got = emu.emu_push(C.byref(ll), count is not None, 0 if count is None else count, addrs, 3)
    assert got == live
    for s, k in zip(slots, starts):
        slot = s[k:k + SLOT_BYTES]
        written = np.zeros(SLOT_BYTES, bool)
        assert int(slot[:4].view(np.int32)[0]) == live
        written[:4] = True
        at = 256
        for (name, elem), (_, _, a) in zip(ARRAYS, keep):
            n = live * elem
            assert np.array_equal(slot[at:at + n], a.reshape(-1).view(np.uint8)[:n]), name
            written[at:at + n] = True
            at += (65536 * elem + 255) // 256 * 256
        assert (slot[~written] == 0xA5).all(), "a byte outside the live entries and the count word was written"
        assert (s[:k] == 0xA5).all() and (s[k + SLOT_BYTES:] == 0xA5).all()


def _peer_args(n=2):
    flags = (C.c_void_p * n)(*([64] * n))
    slots = (C.c_void_p * n)(*([4096] * n))
    return slots, flags


def test_list_to_peers_refuses_before_any_cuda_call(built):
    """grb_light_list_to_peers refuses, with GRB_ERR_INVALID_ARGUMENT and its message: a null pointer (flag arrays,
    counter, slots, light list, array), peer_count outside 1..8, a flag_index outside 0..peer_count-1, a count outside
    0..65536, a misaligned count and a misaligned slot."""
    from granite_b200 import capi

    L = capi.lib()
    fn = L.grb_light_list_to_peers
    d = C.c_void_p(4096)
    ll = capi.GrbLightList(4, d, d, d, d, d, d, 1e10)
    slots, flags = _peer_args()
    peers = b"grb_light_list_to_peers: null pointer, peer_count outside 1..GRB_MAX_PEERS or flag_index outside 0..peer_count-1"
    for args in ((C.byref(ll), None, slots, None, 2, 0, 1, d, None),  # null flag arrays
                 (C.byref(ll), None, slots, flags, 2, 0, 1, None, None),  # null counter
                 (C.byref(ll), None, slots, flags, 0, 0, 1, d, None),
                 (C.byref(ll), None, slots, flags, 9, 0, 1, d, None),
                 (C.byref(ll), None, slots, flags, 2, -1, 1, d, None),
                 (C.byref(ll), None, slots, flags, 2, 2, 1, d, None),
                 (C.byref(ll), None, None, flags, 2, 0, 1, d, None),  # null slots (the credit is grb_peer_publish)
                 (None, None, None, flags, 2, 2, 1, d, None)):
        assert fn(*args) == -1
        assert peers in L.grb_last_error_string()
    nulls = (C.c_void_p * 2)(4096, None)
    assert fn(C.byref(ll), None, nulls, flags, 2, 0, 1, d, None) == -1
    assert b"grb_light_list_to_peers: null peer pointer" in L.grb_last_error_string()
    lists = b"grb_light_list_to_peers: a null light list or array, or a count outside 0..GRB_MAX_LIGHT_LIST"
    assert fn(None, None, slots, flags, 2, 0, 1, d, None) == -1
    assert lists in L.grb_last_error_string()
    for bad in (capi.GrbLightList(4, d, d, None, d, d, d, 1e10), capi.GrbLightList(-1, d, d, d, d, d, d, 1e10),
                capi.GrbLightList(65537, d, d, d, d, d, d, 1e10)):
        assert fn(C.byref(bad), None, slots, flags, 2, 0, 1, d, None) == -1
        assert lists in L.grb_last_error_string()
    assert fn(C.byref(ll), C.c_void_p(4098), slots, flags, 2, 0, 1, d, None) == -1
    assert b"grb_light_list_to_peers: the input count is not 4-byte aligned" in L.grb_last_error_string()
    odd = (C.c_void_p * 2)(4096, 4104)
    assert fn(C.byref(ll), None, odd, flags, 2, 0, 1, d, None) == -1
    assert b"grb_light_list_to_peers: a slot is not 16-byte aligned" in L.grb_last_error_string()


def _device_lights(viewer, n=4):
    d = C.c_void_p(4096)
    return viewer.GrbhDeviceLights(n, d, d, d, d, d, d, 1e10, None, None)


def _refused(L, rc, text):
    assert rc < 0
    assert text in L.grbh_last_error(), L.grbh_last_error()


def test_light_source_rank_refusals_on_a_host_only_viewer(built):
    """Every refusal of grbh_viewer_set_light_source_rank, grbh_viewer_set_lights_device_from_source and the bindings
    of a non-source rank that a host-only viewer reaches, each with its message; an unsharded viewer accepts 0."""
    from granite_b200 import viewer

    L = viewer.lib()
    _refused(L, L.grbh_viewer_set_light_source_rank(None, 0), b"grbh_viewer_set_light_source_rank: null viewer")
    _refused(L, L.grbh_viewer_set_lights_device_from_source(None, 16, 1e10), b"grbh_viewer_set_lights_device_from_source: null viewer")

    shadowed = viewer.Viewer(64, 64, cuda_device=-1, light_shadows=True)
    _refused(L, L.grbh_viewer_set_light_source_rank(shadowed._h, 0), b"grbh_viewer_set_light_source_rank: not with clustered_lights_shadows")
    shadowed.set_light_source_rank(-1)  # off is always accepted
    shadowed.close()

    v = viewer.Viewer(64, 64, cuda_device=-1)
    for rank in (-2, 1):
        _refused(L, L.grbh_viewer_set_light_source_rank(v._h, rank), b"grbh_viewer_set_light_source_rank: rank must be -1 (off) or within [0, 1)")
    _refused(L, L.grbh_viewer_set_lights_device_from_source(v._h, 16, 1e10),
             b"grbh_viewer_set_lights_device_from_source: the viewer has no light source rank")
    v.set_light_source_rank(0)  # unsharded: one band, rank 0 is the source, nothing changes
    _refused(L, L.grbh_viewer_set_lights_device_from_source(v._h, 16, 1e10),
             b"grbh_viewer_set_lights_device_from_source: rank 0 is the light source rank")
    _refused(L, L.grbh_viewer_set_lights_device(v._h, C.byref(_device_lights(viewer))), b"grbh_viewer_set_lights_device: host-only viewer")
    v.close()

    bands = [(0, 16), (16, 32), (32, 48), (48, 64)]
    for rank in range(4):
        v = viewer.Viewer(64, 64, cuda_device=-1)
        v.set_row_shards(bands, rank)
        _refused(L, L.grbh_viewer_set_light_source_rank(v._h, 4), b"grbh_viewer_set_light_source_rank: rank must be -1 (off) or within [0, 4)")
        v.set_light_source_rank(3)
        _refused(L, L.grbh_viewer_set_row_shards(v._h, (viewer.capi.GrbRows * 2)(*[viewer.capi.GrbRows(0, 32), viewer.capi.GrbRows(32, 64)]), 2, 0),
                 b"grbh_viewer_set_row_shards: the light source rank 3 would have no band among 2")
        if rank == 3:
            _refused(L, L.grbh_viewer_set_lights_device_from_source(v._h, 16, 1e10),
                     b"grbh_viewer_set_lights_device_from_source: rank 3 is the light source rank")
            _refused(L, L.grbh_viewer_set_lights_device(v._h, C.byref(_device_lights(viewer))), b"grbh_viewer_set_lights_device: host-only viewer")
            _refused(L, L.grbh_viewer_set_light_count_device(v._h, None), b"grbh_viewer_set_light_count_device: host-only viewer")
        else:
            receiver = f"rank {rank} receives its device lights from light source rank 3".encode()
            _refused(L, L.grbh_viewer_set_lights_device(v._h, C.byref(_device_lights(viewer))), b"grbh_viewer_set_lights_device: " + receiver)
            _refused(L, L.grbh_viewer_set_light_count_device(v._h, None), b"grbh_viewer_set_light_count_device: " + receiver)
            for capacity in (-1, 65537):
                _refused(L, L.grbh_viewer_set_lights_device_from_source(v._h, capacity, 1e10),
                         f"grbh_viewer_set_lights_device_from_source: capacity {capacity} is outside 0..65536".encode())
            _refused(L, L.grbh_viewer_set_lights_device_from_source(v._h, 16, 1e10), b"grbh_viewer_set_lights_device_from_source: host-only viewer")
        _refused(L, L.grbh_viewer_bake(v._h), b"host-only viewer")  # so "after bake" needs a device: the GPU tests check it
        v.close()
