"""Shared helpers for the parity tests (test infrastructure)."""
from __future__ import annotations

import os
import signal
import subprocess
import sys

import numpy as np

from granite_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def free_port() -> int:
    """A TCP port nothing listens on now, for the rendezvous of a torchrun launch.  A fixed port fails with EADDRINUSE
    whenever another run on the same host holds it."""
    import socket

    with socket.socket() as s:
        s.bind(("", 0))
        return s.getsockname()[1]


def run_ranks(worker, args, world, env, timeout):
    """Run tests/<worker> on `world` ranks under torchrun, with `env` added to the environment; returns (returncode,
    stdout, stderr).  The launcher runs in a session of its own, so that a run past `timeout` seconds is killed with
    every rank it started, and the test fails."""
    import pytest

    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(free_port()), os.path.join(ROOT, "tests", worker), *map(str, args)]
    proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, cwd=ROOT, env=dict(os.environ, **env),
                            start_new_session=True)
    try:
        out, err = proc.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        os.killpg(proc.pid, signal.SIGKILL)  # the launcher and every rank
        out, err = proc.communicate()
        pytest.fail(f"the sharded run did not finish in {timeout} s:\n" + out[-3000:] + err[-3000:])
    sys.stdout.write(out[-6000:])
    return proc.returncode, out, err


def build_case(oracle, width, height, n_lights, spot_fraction=0.0):
    """Scene + oracle host prep (camera, light records, cluster params) for one config."""
    scene = synth.make_scene(width, height)
    cam = oracle.camera_setup(scene.projection, scene.view)
    lights = synth.make_lights(n_lights, spot_fraction=spot_fraction, aspect=width / height)
    prep = oracle.prepare_lights(cam, lights, res=synth.CLUSTER_RES)
    return scene, cam, lights, prep


def oracle_camera_from_viewer(oracle, viewer_obj):
    """The camera block the HOST LAYER derived (RenderContext::set_camera), repackaged for the
    oracle: matrices are inputs of the hot path, so both sides must see the same bits (the host
    layer's mat4 inverse is not the reference's cofactor expansion and differs by an ulp)."""
    gcam, proj, inv_proj = viewer_obj.camera()
    cam = oracle.Camera()
    cam.projection[:] = proj.reshape(-1).tolist()
    cam.inv_projection[:] = inv_proj.reshape(-1).tolist()
    cam.view[:] = list(gcam.view)
    cam.view_projection[:] = list(gcam.view_projection)
    cam.inv_view_projection[:] = list(gcam.inv_view_projection)
    cam.camera_position[:] = list(gcam.camera_position)
    cam.camera_front[:] = list(gcam.camera_front)
    cam.z_near, cam.z_far = gcam.z_near, gcam.z_far
    return cam


def build_case_for_viewer(oracle, viewer_obj, scene, lights):
    cam = oracle_camera_from_viewer(oracle, viewer_obj)
    prep = oracle.prepare_lights(cam, lights, res=synth.CLUSTER_RES)
    return cam, prep


def build_lights_case(oracle, aspect, n_lights, spot_fraction=0.0):
    """Camera + lights + oracle host prep only (no G-buffer)."""
    import math

    proj = synth.perspective_inf(math.pi / 4.0, aspect, 1.0 / 16.0)
    view = synth.look_at_view((0.0, 0.0, 8.0), (0.0, 0.0, 0.0))
    cam = oracle.camera_setup(proj, view)
    lights = synth.make_lights(n_lights, spot_fraction=spot_fraction, aspect=aspect)
    prep = oracle.prepare_lights(cam, lights, res=synth.CLUSTER_RES)
    return cam, lights, prep


def r11g11b10_codes(p: np.ndarray):
    """Split packed B10G11R11 into per-channel integer codes (monotone in the decoded value)."""
    p = p.astype(np.uint32)
    return (p & 0x7FF).astype(np.int64), ((p >> 11) & 0x7FF).astype(np.int64), (p >> 22).astype(np.int64)


def max_code_diff_r11g11b10(a, b):
    return max(int(np.abs(x - y).max()) for x, y in zip(r11g11b10_codes(a), r11g11b10_codes(b)))


def f16_ulp_diff(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """ULP distance between two fp16 bit patterns (sign-magnitude -> monotone integer)."""
    def key(u):
        u = u.astype(np.int32)
        return np.where(u & 0x8000, -(u & 0x7FFF), u & 0x7FFF)
    return np.abs(key(a.view(np.uint16)) - key(b.view(np.uint16)))


def f32_ulp_diff(a, b):
    def key(f):
        u = np.asarray(f, np.float32).view(np.int32).astype(np.int64)
        return np.where(u < 0, -(u & 0x7FFFFFFF), u)
    return np.abs(key(a) - key(b))


def rgba8_channel_diff(a, b):
    a = np.ascontiguousarray(a).view(np.uint8).astype(np.int32)
    b = np.ascontiguousarray(b).view(np.uint8).astype(np.int32)
    return np.abs(a - b)


def a2b10g10r10_channel_diff(a, b):
    """|difference| of the three 10-bit channels and of the 2-bit alpha, as one (..., 4) array."""
    a = np.ascontiguousarray(a).astype(np.uint32)
    b = np.ascontiguousarray(b).astype(np.uint32)
    ch = lambda v: np.stack([v & 1023, (v >> 10) & 1023, (v >> 20) & 1023, v >> 30], -1).astype(np.int32)
    return np.abs(ch(a) - ch(b))


def random_hdr(rng, w, h, scale=4.0, hot=0.002):
    """Random B10G11R11 image with a few very bright texels (drives bloom)."""
    rgb = (rng.random((h, w, 3)) ** 3 * scale).astype(np.float32)
    m = rng.random((h, w)) < hot
    rgb[m] = rng.uniform(10.0, 200.0, size=(int(m.sum()), 3)).astype(np.float32)
    return synth.pack_r11g11b10(rgb)


def random_rgba16f(rng, w, h, lo=-2.0, hi=8.0):
    return rng.uniform(lo, hi, size=(h, w, 4)).astype(np.float16).view(np.uint16)


def assert_f16_close(got, ref, what="", min_identical=0.999, abs_floor=0.0):
    """Stored RGBA16F values: at most 1 fp16 ulp apart (or `abs_floor` absolute, for signed values that
    pass through zero), and identical for at least `min_identical` of the values."""
    d = f16_ulp_diff(got, ref)
    if abs_floor > 0.0:
        a = np.abs(got.view(np.float16).astype(np.float32) - ref.view(np.float16).astype(np.float32))
        bad = (d > 1) & ~(a <= abs_floor)
    else:
        bad = d > 1
    assert not bad.any(), f"{what}: {int(bad.sum())} values differ by more than 1 fp16 ulp (max {int(d.max())})"
    ident = float((d == 0).mean())
    assert ident >= min_identical, f"{what}: only {ident:.6f} identical"
    return ident


def unpack_r11g11b10_np(p: np.ndarray) -> np.ndarray:
    """Decode packed B10G11R11_UFLOAT to float32 (..., 3): 5-bit exponent (bias 15), 6 / 6 / 5 mantissa bits."""
    p = p.astype(np.uint32)

    def dec(v, mbits):
        e = (v >> mbits).astype(np.int32)
        m = (v & ((1 << mbits) - 1)).astype(np.float64)
        normal = np.ldexp(1.0 + m / (1 << mbits), e - 15)
        denorm = np.ldexp(m / (1 << mbits), -14)
        return np.where(e == 0, denorm, np.where(e == 31, np.inf, normal)).astype(np.float32)

    return np.stack([dec(p & 0x7FF, 6), dec((p >> 11) & 0x7FF, 6), dec(p >> 22, 5)], -1)


def assert_r11g11b10_close(got, ref, what="", abs_floor=2.0 ** -16, min_identical=0.99):
    """Stored B10G11R11 values: at most 1 code apart per channel, or -- for values so close to zero that a
    code is a few 1e-6 -- within `abs_floor` absolute."""
    d = np.stack([np.abs(a - b) for a, b in zip(r11g11b10_codes(got), r11g11b10_codes(ref))], -1)
    a = np.abs(unpack_r11g11b10_np(got) - unpack_r11g11b10_np(ref))
    bad = (d > 1) & ~(a <= abs_floor)
    assert not bad.any(), f"{what}: {int(bad.sum())} channels differ by more than one code (max {int(d.max())}, max abs {float(a[d > 1].max()) if (d > 1).any() else 0.0:.3e})"
    ident = float((d == 0).mean())
    assert ident >= min_identical, f"{what}: only {ident:.6f} identical"
    return ident


def make_shadow_maps(prep, resolution, seed=0x5AD0, skip_every=7, block=4):
    """Synthetic D16 shadow maps, one per light of prep (cluster order): blocks of block x block texels holding depths spread
    over the range the receivers' reference depths fall in (reverse-Z with near = 0.5 % of the light's range: a
    receiver at 10 % .. 100 % of the range compares 0.045 .. 0 against the map), so footprints come out lit, shadowed
    and partially lit.  Every skip_every-th light has no map (casts no shadow).  Spot: (res, res); point: (6, res, res)."""
    rng = np.random.default_rng(seed + prep.n)
    maps = []
    blocks = (resolution + block - 1) // block
    for i in range(prep.n):
        if skip_every and i % skip_every == skip_every - 1:
            maps.append(None)
            continue
        is_point = (int(prep.type_mask[i >> 5]) >> (i & 31)) & 1
        faces = 6 if is_point else 1
        coarse = rng.integers(0, 3000, (faces, blocks, blocks)).astype(np.uint16)
        coarse[rng.random(coarse.shape) < 0.3] = 0  # open sky: everything in front of the far plane is lit
        m = np.repeat(np.repeat(coarse, block, axis=1), block, axis=2)[:, :resolution, :resolution]
        maps.append(np.ascontiguousarray(m if is_point else m[0]))
    return maps


def random_hdr_f16(rng, w, h, scale=4.0, hot=0.002):
    """Random R16G16B16A16_SFLOAT HDR image ("renderTargetFp16"), a few very bright texels, alpha 1: (h, w, 4) uint16."""
    rgb = (rng.random((h, w, 3)) ** 3 * scale).astype(np.float32)
    m = rng.random((h, w)) < hot
    rgb[m] = rng.uniform(10.0, 200.0, size=(int(m.sum()), 3)).astype(np.float32)
    img = np.ones((h, w, 4), np.float16)
    img[..., :3] = rgb
    return np.ascontiguousarray(img).view(np.uint16)
