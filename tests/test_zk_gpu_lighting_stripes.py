"""Lighting in stripes on the GPU, one device: grb_deferred_lighting_stripes must write, on every row of its stripe set,
what the whole-image pass writes there, bit for bit, and leave every other row alone; grb_hdr_rows_to_peers must store
exactly the rows of its stripe set that lie in each other rank's lighting rows into that rank's slot, and raise every
rank's flag.  Local buffers stand in for the ranks' slots and flag arrays."""
import numpy as np
import pytest

from tests import common

pytestmark = pytest.mark.gpu

SENTINEL = 0x2AB5A5A5
# (first, rows, period): several heights, phases and periods; the last stripe of each is cut by the image, and the
# images' heights are not multiples of 4 rows
STRIPE_SETS = [(0, 8, 16), (8, 8, 16), (16, 16, 48), (24, 64, 128), (64, 32, 64), (312, 64, 128)]


def _gbuffer_with_emissive(gb, emissive_img):
    """The G-buffer with its emissive image set, so that the pass writes every pixel it lights into a separate hdr."""
    from granite_b200 import capi

    g = capi.GrbGBuffer.from_buffer_copy(gb.struct)
    g.emissive = emissive_img
    gb.struct = g
    return gb


def _set_rows(h, first, rows, period):
    inside = np.zeros(h, bool)
    for y in range(first, h, period):
        inside[y:y + rows] = True
    return inside


def _check_stripes(whole, run_stripes, sentinel, h):
    for s in STRIPE_SETS:
        got = run_stripes(s)
        inside = _set_rows(h, *s)
        assert inside.any() and not inside.all()
        assert np.array_equal(got[inside], whole[inside]), f"stripes {s}: lit rows differ from the whole-image pass"
        assert (got[~inside] == sentinel).all(), f"stripes {s}: a row outside the set was written"


@pytest.mark.parametrize("form", ["persistent", "rgba16f", "shadowed", "shadowed-rgba16f"])
def test_stripes_equal_whole_image_lighting(cuda, oracle, form):
    import torch

    from granite_b200 import capi, harness
    from tests.test_gpu_parity import _cluster

    if form.startswith("shadowed"):
        from tests.test_oracle_ref_light_shadows import shadow_case
        from tests.test_zy_gpu_shadows import _device_shadows

        w, h = 641, 359
        scene, cam, prep, clus, transforms, maps = shadow_case(oracle, w, h, 300, 0.5, 64)
        t, table, held = _device_shadows(transforms, maps)
        shadows = (t, table, 64)
    else:
        w, h = 640, 358
        scene, cam, _, prep = common.build_case(oracle, w, h, 300, 0.25)
        shadows = None
    dev, gcam = _cluster(cuda, oracle, cam, prep)
    gb = harness.GBufferDevice(scene)
    if form.endswith("rgba16f"):
        em = harness.to_dev(common.random_hdr_f16(np.random.default_rng(3), w, h, scale=0.02, hot=0.001))
        emissive_img = capi.image(em, capi.FORMAT_R16G16B16A16_SFLOAT)
        new_hdr = lambda: torch.full((h, w, 4), 0x2AB5, dtype=torch.int16, device="cuda")
        host = lambda t: harness.to_host(t, np.uint16)
        sentinel = np.uint16(0x2AB5)
    else:
        em = gb.emissive
        emissive_img = capi.image(em, capi.FORMAT_B10G11R11_UFLOAT)
        new_hdr = lambda: torch.full((h, w), SENTINEL, dtype=torch.int32, device="cuda")
        host = lambda t: harness.to_host(t, np.uint32)
        sentinel = np.uint32(SENTINEL)
    _gbuffer_with_emissive(gb, emissive_img)

    whole_t = new_hdr()
    if shadows:
        harness.deferred_lighting_shadowed(gb, gcam, dev, shadows[0], shadows[1], shadows[2], whole_t)
    else:
        harness.deferred_lighting(gb, gcam, dev, whole_t)
    torch.cuda.synchronize()
    whole = host(whole_t)
    schedule = harness.lighting_schedule(h) if form == "persistent" else None

    def run(s):
        out = []
        # with a schedule, the second launch takes its strips in the order the first one measured
        for _ in range(2 if schedule is not None else 1):
            t = new_hdr()
            harness.deferred_lighting_stripes(gb, gcam, dev, t, s, schedule=schedule, shadows=shadows)
            torch.cuda.synchronize()
            out.append(host(t))
        assert all(np.array_equal(o, out[0]) for o in out)
        return out[0]

    _check_stripes(whole, run, sentinel, h)


@pytest.mark.parametrize("texel", ["b10g11r11", "rgba16f", "b10g11r11-odd-width", "b10g11r11-padded-pitch"])
def test_hdr_rows_to_peers_routes_the_push_rows(cuda, texel):
    """Three ranks' slots on one device; rank 1 of 3 lights stripes of 8 rows and pushes.  Each other rank's slot gets
    exactly the rows of rank 1's stripes inside that rank's lighting rows and keeps the sentinel elsewhere; rank 1's own
    slot is not written; every flag array gets the epoch at index 1, and the scratch
    counter is reset.  A rank whose stripes all lie below the image still raises its flags.  Widths: 16-byte stores only;
    a pitch that allows none (4-byte stores); a 16-byte-aligned pitch past a row of 200 bytes (16-byte stores and an
    8-byte tail in the same launch, the padding untouched)."""
    import torch

    from granite_b200 import harness

    h = 100
    w = {"b10g11r11-odd-width": 13, "b10g11r11-padded-pitch": 50}.get(texel, 48)
    rng = np.random.default_rng(w)
    if texel == "b10g11r11-padded-pitch":
        # (h, 52) buffers, the image their first 50 texels: pitch 208 bytes, rows of 200
        src = torch.from_numpy(rng.integers(0, 2**32, (h, 52), dtype=np.uint32).view(np.int32)).cuda()
        new_slot = lambda: torch.full((h, 52), SENTINEL, dtype=torch.int32, device="cuda")
    elif texel == "rgba16f":
        src = torch.from_numpy(rng.integers(-2**15, 2**15, (h, w, 4), dtype=np.int16)).cuda()
        new_slot = lambda: torch.full((h, w, 4), 0x2AB5, dtype=torch.int16, device="cuda")
    else:
        src = torch.from_numpy(rng.integers(0, 2**32, (h, w), dtype=np.uint32).view(np.int32)).cuda()
        new_slot = lambda: torch.full((h, w), SENTINEL, dtype=torch.int32, device="cuda")
    slots = [new_slot() for _ in range(3)]
    sentinel = slots[0].cpu().numpy().copy()
    flags = [torch.zeros(8, dtype=torch.int32, device="cuda") for _ in range(3)]
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    lighting = [(0, 40), (30, 75), (66, 100)]  # overlapping, as lighting rows with halos are
    stripes = (8, 8, 24)
    width = w if texel == "b10g11r11-padded-pitch" else None
    harness.hdr_rows_to_peers(src, slots, flags, lighting, 1, 7, counter, stripes, width=width)
    torch.cuda.synchronize()
    lit = _set_rows(h, *stripes)
    s = src.cpu().numpy().copy()
    if width is not None:
        s[:, w:] = sentinel[:, w:]  # the padding past the image is not copied
    for q in range(3):
        want = sentinel.copy()
        if q != 1:
            rows = lit.copy()
            rows[:lighting[q][0]] = False
            rows[lighting[q][1]:] = False
            assert rows.any()
            want[rows] = s[rows]
        assert np.array_equal(slots[q].cpu().numpy(), want), f"slot of rank {q}"
        assert list(flags[q].cpu().numpy()) == [0, 7, 0, 0, 0, 0, 0, 0]
    assert counter.item() == 0
    # nothing to push: the flags rise all the same
    harness.hdr_rows_to_peers(src, slots, flags, lighting, 2, 8, counter, (h + 8, 8, 24), width=width)
    torch.cuda.synchronize()
    for q in range(3):
        assert list(flags[q].cpu().numpy()[:3]) == [0, 7, 8]
    assert counter.item() == 0
