"""Every form of the lighting pass against the float64 reference (tests/lighting_ref64.py).

launch_deferred_lighting (grb_lighting.cu) runs one of three kernels:
  persistent  deferred_lighting_persistent_kernel: pixel pairs possible (even width, 8-byte aligned bases and pitches),
              <= 4096 lights in <= 128 words, the light table fits in shared memory, not _blocks, no GRB_LIGHTING_V2;
  pairs       deferred_lighting2_kernel: grb_deferred_lighting_blocks, GRB_LIGHTING_V2, or pairs possible but not the
              persistent kernel (> 4096 lights);
  one pixel   deferred_lighting_kernel<false>: odd width, a misaligned base or pitch, GRB_LIGHTING_1PX.
Each case holds its form to the float64 bar and to the oracle's (at most one code, > 97 % of pixels identical), and
shows that it reached the form it names: from the selection condition on its inputs, or by bit-identity with a call
that can only take that form.  Switches read once per process run in tests/kernel_forms_worker.py."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from granite_b200 import synth
from tests import common
from tests import lighting_ref64 as R
from tests.kernel_forms_worker import LIGHTING_CASE, SWITCHES

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 0x2AB5A5A5
FORMS = ("persistent", "pairs", "1px-pitch", "1px-offset")
_CASES = {}


def _case(oracle, name):
    """(scene, cam, prep, oracle cluster, oracle frame, float64 reference) of a named case, computed once."""
    if name not in _CASES:
        if name == "dense-256x144":
            scene, cam, _, prep = R.dense_case(oracle)
        elif name == "grazing-640x360":
            scene, cam, _, prep, _, _ = R.grazing_case(oracle)
        else:
            w, h, n, spots = {"small-640x360": LIGHTING_CASE, "odd-641x359": (641, 359, 300, 0.25),
                              "partial-block-328x184": (328, 184, 300, 0.25), "zero-640x360": (640, 360, 0, 0.0),
                              "boundary-4096": (320, 180, 4096, 0.0), "boundary-4097": (320, 180, 4097, 0.0)}[name]
            scene = synth.make_scene(w, h)
            cam = oracle.camera_setup(scene.projection, scene.view)
            prep = oracle.prepare_lights(cam, synth.make_lights(n, spot_fraction=spots, aspect=w / h), res=synth.CLUSTER_RES, cull=n < 4096)
        clus = oracle.cluster_build(cam, prep)
        got, tile, zi, _ = oracle.deferred_lighting(scene, cam, prep, clus, want_indices=True)
        _CASES[name] = (scene, cam, prep, clus, got, R.reference(oracle, scene, cam, prep, clus, (tile, zi)))
    return _CASES[name]


def _device(scene, cam, prep):
    from granite_b200 import harness

    dev = harness.ClusterDevice(prep.records, prep.model, prep.type_mask, prep.z_ranges, prep.params, prep.res)
    gcam = harness.camera_struct(cam)
    dev.build(gcam)
    torch.cuda.synchronize()
    return harness.GBufferDevice(scene), dev, gcam


class _Strided:
    """A copy of an (H, W) int32 device image at row pitch `pitch` texels, starting `offset` texels into its buffer."""

    def __init__(self, t, fmt, pitch, offset=0):
        from granite_b200 import capi

        h, w = t.shape
        self.buf = torch.full((h * pitch + offset + pitch,), -1, dtype=torch.int32, device="cuda")
        self.buf[offset:offset + h * pitch].view(h, pitch)[:, :w].copy_(t)
        self.img = capi.GrbImage(self.buf.data_ptr() + 4 * offset, w, h, 4 * pitch, fmt)


def _run(form, gb, gcam, dev, hdr, rows=None):
    """Lights hdr in place with `form`; 1px forms read a copy of the albedo at a pitch or base that pairs cannot use."""
    from granite_b200 import capi, harness

    if form == "persistent":
        return harness.deferred_lighting(gb, gcam, dev, hdr, rows=rows)
    if form == "pairs":
        return harness.deferred_lighting_blocks(gb, gcam, dev, hdr, rows=rows)
    w = gb.w
    s = _Strided(gb.albedo, capi.FORMAT_R8G8B8A8_SRGB, w + 1 if form == "1px-pitch" else w + 2, 0 if form == "1px-pitch" else 1)
    assert (s.img.row_pitch % 8 != 0) if form == "1px-pitch" else (s.img.data % 8 != 0), "one-pixel form: pairs need 8-byte alignment"
    g = capi.GrbGBuffer.from_buffer_copy(gb.struct)
    g.albedo = s.img
    saved, gb.struct = gb.struct, g
    try:
        harness.deferred_lighting(gb, gcam, dev, hdr, rows=rows)
        torch.cuda.synchronize()
    finally:
        gb.struct = saved


def _check(got, oracle_frame, ref, what):
    R.assert_meets_bar(got, ref, what)
    assert common.max_code_diff_r11g11b10(got, oracle_frame) <= 1, what
    assert float((got == oracle_frame).mean()) > 0.97, what


def _frames(name, oracle, forms=FORMS):
    from granite_b200 import harness

    scene, cam, prep, clus, ref_frame, ref = _case(oracle, name)
    gb, dev, gcam = _device(scene, cam, prep)
    out = {}
    for form in forms:
        hdr = gb.emissive.clone()
        _run(form, gb, gcam, dev, hdr)
        out[form] = harness.to_host(hdr, np.uint32)
    return scene, ref_frame, ref, gb, dev, gcam, out


@pytest.mark.parametrize("name", ["small-640x360", "dense-256x144", "grazing-640x360", "partial-block-328x184"])
def test_every_form_meets_the_float64_bar(cuda, oracle, name):
    """All three forms in one process.  The two one-pixel calls (row pitch 4 (w + 1) bytes, base 4 bytes past 8-byte
    alignment) can only take the one-pixel kernel and must agree bit for bit; the persistent and pairs forms sum the
    lights in a different order and each meets the bar on its own.  328 is even but not a multiple of 16: the last
    16x4 block of every strip of the persistent form holds 8 pixel columns."""
    scene, ref_frame, ref, gb, dev, gcam, out = _frames(name, oracle)
    for form, got in out.items():
        _check(got, ref_frame, ref, f"{name} {form}")
    assert np.array_equal(out["1px-pitch"], out["1px-offset"])
    if name == "grazing-640x360":
        # the case discriminates only if the grazing pixels carry the specular peak: assert it is lit that brightly
        _, _, _, _, mask, _ = R.grazing_case(oracle)
        assert R.decode(out["persistent"][mask]).max(-1).min() > 8.0


def test_odd_width_takes_the_one_pixel_form(cuda, oracle):
    """641 x 359: odd width, so grb_deferred_lighting and grb_deferred_lighting_blocks both run the one-pixel kernel,
    bit for bit the same frame as a misaligned-pitch call."""
    scene, ref_frame, ref, gb, dev, gcam, out = _frames("odd-641x359", oracle, ("persistent", "pairs", "1px-offset"))
    assert scene.depth.shape[1] % 2 == 1
    _check(out["persistent"], ref_frame, ref, "641x359")
    assert np.array_equal(out["persistent"], out["pairs"]) and np.array_equal(out["persistent"], out["1px-offset"])


def test_padded_pitch_keeps_the_persistent_form(cuda, oracle):
    """A row pitch padded to a multiple of 8 bytes (w + 6 texels) still takes the persistent kernel: its bits."""
    from granite_b200 import capi, harness

    scene, ref_frame, ref, gb, dev, gcam, out = _frames("small-640x360", oracle, ("persistent", "pairs"))
    assert not np.array_equal(out["persistent"], out["pairs"]), "the two pair forms associate the sums differently"
    s = _Strided(gb.albedo, capi.FORMAT_R8G8B8A8_SRGB, gb.w + 6)
    assert s.img.row_pitch % 8 == 0 and s.img.data % 8 == 0
    g = capi.GrbGBuffer.from_buffer_copy(gb.struct)
    g.albedo = s.img
    saved, gb.struct = gb.struct, g
    hdr = gb.emissive.clone()
    harness.deferred_lighting(gb, gcam, dev, hdr)
    torch.cuda.synchronize()
    gb.struct = saved
    assert np.array_equal(harness.to_host(hdr, np.uint32), out["persistent"])


def test_zero_lights_with_null_buffers(cuda, oracle):
    """num_lights 0 with null lights, type mask and bitmask (the ABI allows it): the directional term only, on every
    form."""
    from granite_b200 import harness

    scene, cam, prep, clus, ref_frame, ref = _case(oracle, "zero-640x360")
    assert prep.n == 0 and len(ref.pairs[0]) == 0
    gb, dev, gcam = _device(scene, cam, prep)
    dev.buffers.lights = dev.buffers.type_mask = dev.buffers.bitmask = None
    for form in FORMS:
        hdr = gb.emissive.clone()
        _run(form, gb, gcam, dev, hdr)
        _check(harness.to_host(hdr, np.uint32), ref_frame, ref, f"zero lights {form}")


def test_separate_emissive_equals_in_place(cuda, oracle):
    """GrbGBuffer.emissive set (the viewer's configuration), hdr prefilled with a sentinel: every pixel, sky included,
    equals the in-place call bit for bit, on every form."""
    from granite_b200 import capi, harness

    scene, ref_frame, ref, gb, dev, gcam, out = _frames("small-640x360", oracle)
    assert (scene.depth == 0).any()
    gb.struct.emissive = capi.image(gb.emissive, capi.FORMAT_B10G11R11_UFLOAT)
    try:
        for form in FORMS:
            hdr = torch.full_like(gb.emissive, SENTINEL)
            _run(form, gb, gcam, dev, hdr)
            assert np.array_equal(harness.to_host(hdr, np.uint32), out[form]), form
    finally:
        gb.struct.emissive = capi.GrbImage()


def test_row_bands_equal_the_whole_image(cuda, oracle):
    """Bands whose first rows are not multiples of 4: within one form each band is bit-identical to the whole-image
    call, and rows outside the band keep the sentinel."""
    from granite_b200 import harness

    scene, ref_frame, ref, gb, dev, gcam, out = _frames("small-640x360", oracle)
    h = scene.depth.shape[0]
    for form in FORMS:
        for y0, y1 in ((0, 37), (37, 202), (202, h), (5, 6)):
            hdr = torch.full_like(gb.emissive, SENTINEL)
            hdr[y0:y1] = gb.emissive[y0:y1]
            _run(form, gb, gcam, dev, hdr, rows=(y0, y1))
            got = harness.to_host(hdr, np.uint32)
            assert np.array_equal(got[y0:y1], out[form][y0:y1]), (form, y0, y1)
            assert (got[:y0] == SENTINEL).all() and (got[y1:] == SENTINEL).all(), (form, y0, y1)


@pytest.mark.parametrize("w,h,n", [pytest.param(64, 400, 2, id="few-lights-64x400"), pytest.param(64, 8200, 8, id="tall-64x8200")])
def test_schedule_fallbacks(cuda, oracle, w, h, n):
    """The persistent kernel keeps no schedule when the row costs do not fit the light table's shared memory
    (blocks_y * 4 > rec_total) or the rows exceed kMaxOrderRows (2048 strips): the header's valid word reads 0 and every
    launch on that buffer gives the unscheduled frame."""
    from granite_b200 import harness

    scene = synth.make_scene(w, h)
    cam = oracle.camera_setup(scene.projection, scene.view)
    prep = oracle.prepare_lights(cam, synth.make_lights(n, aspect=w / h), res=synth.CLUSTER_RES, cull=False)
    strips = (h + 3) // 4
    assert strips * 4 > n * 48 + 48 or strips > 2048
    gb, dev, gcam = _device(scene, cam, prep)
    hdr = gb.emissive.clone()
    harness.deferred_lighting(gb, gcam, dev, hdr)
    sched = harness.lighting_schedule(h)
    for _ in range(2):
        hdr_s = gb.emissive.clone()
        harness.deferred_lighting(gb, gcam, dev, hdr_s, schedule=sched)
        assert torch.equal(hdr, hdr_s)
        assert int(sched[2]) == 0, "no schedule is published"
    if h <= 1024:
        clus = oracle.cluster_build(cam, prep)
        got, tile, zi, _ = oracle.deferred_lighting(scene, cam, prep, clus, want_indices=True)
        _check(harness.to_host(hdr, np.uint32), got, R.reference(oracle, scene, cam, prep, clus, (tile, zi)), f"{w}x{h}")


def test_light_count_boundary(cuda, oracle):
    """4096 lights (128 words, a 192 KiB table that still fits the persistent kernel's shared memory) on the persistent
    form; 4097 lights, which grb_cluster_build and the oracle accept through the raw ABI (the host clusterer caps the
    frame at 4096), leave it for the pairs kernel: grb_deferred_lighting then gives grb_deferred_lighting_blocks'
    bits.  Both within the float64 bar."""
    from granite_b200 import harness

    smem = 4096 * 48 + 48 + 1024 + ((16 * 162 * 2 + 15) & ~15) + 32 * 16 * 48 + 16 + 2048 * 2  # launch_deferred_lighting
    assert smem <= torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    frames = {}
    for name in ("boundary-4096", "boundary-4097"):
        scene, cam, prep, clus, ref_frame, ref = _case(oracle, name)
        gb, dev, gcam = _device(scene, cam, prep)
        for form in ("persistent", "pairs"):
            hdr = gb.emissive.clone()
            _run(form, gb, gcam, dev, hdr)
            frames[name, form] = harness.to_host(hdr, np.uint32)
            _check(frames[name, form], ref_frame, ref, f"{name} {form}")
    assert prep.n == 4097 and prep.params.num_lights_32 == 129
    assert not np.array_equal(frames["boundary-4096", "persistent"], frames["boundary-4096", "pairs"])
    assert np.array_equal(frames["boundary-4097", "persistent"], frames["boundary-4097", "pairs"])


# ------------------------------------------------------------------------------------------ run-time switches
def _run_worker(case, out_dir, **switches):
    """tests/kernel_forms_worker.py <case> in a child process whose GRB_* switches are exactly `switches`."""
    env = {k: v for k, v in os.environ.items() if k not in SWITCHES}
    env.update(switches)
    cmd = [sys.executable, "-m", "tests.kernel_forms_worker", case, str(out_dir)]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, f"worker {case} {switches} exited with {r.returncode}:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    seen = next(line for line in r.stdout.splitlines() if line.startswith("switches:"))
    assert seen.split()[1:] == [f"{k}={switches[k]}" for k in SWITCHES if k in switches], seen
    return np.load(os.path.join(out_dir, f"{case}.npz"))


@pytest.fixture(scope="module")
def in_process(oracle):
    """The worker's lighting case in this process: persistent, pairs and one-pixel frames."""
    return _frames("small-640x360", oracle, ("persistent", "pairs", "1px-pitch"))[-1]


def test_lighting_v2_switch_runs_the_pairs_form(cuda, in_process, tmp_path):
    """GRB_LIGHTING_V2=1: grb_deferred_lighting gives grb_deferred_lighting_blocks' frame bit for bit."""
    f = _run_worker("lighting", tmp_path, GRB_LIGHTING_V2="1")
    assert np.array_equal(f["default"], in_process["pairs"])


def test_lighting_1px_switch_runs_the_one_pixel_form(cuda, in_process, tmp_path):
    """GRB_LIGHTING_1PX=1: grb_deferred_lighting gives the frame of a misaligned-pitch copy of the same G-buffer."""
    f = _run_worker("lighting", tmp_path, GRB_LIGHTING_1PX="1")
    assert np.array_equal(f["default"], in_process["1px-pitch"])
