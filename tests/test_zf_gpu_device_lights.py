"""Lights from device memory on one GPU (grbh_viewer_set_lights_device): the device prep against the host prep and the
oracle, the cluster it bins against the host-light cluster, and whole frames against host-light frames, bit for bit;
the `ready` / `consumed` events and switching between host and device lights."""
import numpy as np
import pytest

from granite_b200 import viewer as _viewer
from tests import device_lights_cases as cases

pytestmark = pytest.mark.gpu

W, H = 320, 192


def _scene_viewer(proj, view, lights=None, w=W, h=H, **cfg):
    from granite_b200 import synth, viewer

    v = viewer.Viewer(w, h, cuda_device=0, **cfg)
    rw, rh = v.render_size()
    scene = synth.make_scene(rw, rh)
    v.set_directional(scene.dir_color, scene.dir_direction)
    v.set_camera(proj, view)
    if lights is not None:
        v.set_lights(lights)
    v.bake()
    keep = [np.ascontiguousarray(a) for a in (scene.albedo, scene.normal, scene.pbr, scene.depth, scene.emissive)]
    return v, keep


def _frame(v, keep, first):
    from granite_b200 import viewer

    v.render_frame(viewer.Viewer.host_gbuffer(*keep) if first else None)
    out = np.zeros((v.height, v.width), np.uint32)
    v.read_output(out)
    return out


@pytest.mark.parametrize("name", cases.HOST_PREP_CASES + cases.TIE_CASES + cases.LIMIT_CASES)
def test_device_prep_equals_host_prep_and_oracle(cuda, oracle, name):
    """Count, records, model rows, type mask and Z ranges of the device prep byte for byte the host prep's of the same
    shuffled list, and the oracle's where the case has a front-to-back order."""
    from granite_b200 import viewer
    from tests import common

    w, h, proj, view, lights, ordered = cases.case(oracle, name)
    host = viewer.Viewer(w, h, cuda_device=-1)
    host.set_camera(proj, view)
    host.set_lights(lights)
    want = host.light_prep()
    host.close()
    v, keep = _scene_viewer(proj, view)
    v.set_lights_device(**cases.to_device(lights))
    _frame(v, keep, True)
    got = v.light_prep()
    k = want[0]
    assert got[0] == k
    if name == "6000-visible":
        assert k == 4096
    if name in ("all-culled", "0-0.0"):
        assert k == 0
    for a, b in zip(want[1:], got[1:]):
        assert a.tobytes() == b.tobytes()
    if ordered is not None:
        prep = oracle.prepare_lights(common.oracle_camera_from_viewer(oracle, v), ordered)
        assert got[1].tobytes() == prep.records[:k].tobytes()
        assert np.array_equal(got[2].view(np.uint32), prep.model[:k].view(np.uint32))
        if k:
            assert np.array_equal(got[4], prep.z_ranges[:k])
    v.close()


def _cluster(v):
    p, _ = v.cluster()
    n32 = p.num_lights_32
    bm = v.download_buffer("cluster-bitmask", np.uint32, 128 * 64 * n32).reshape(64 * 128, n32) if n32 else np.zeros((64 * 128, 0), np.uint32)
    cr = v.download_buffer("cluster-range", np.uint32, 4096 * 2)
    return bm, cr


def test_cluster_equals_host_cluster_after_a_busier_frame(cuda):
    """cluster-range identical, each tile's bitmask equal in words [0, ceil(count / 32)) and zero after them, on the
    frames after a frame with more visible lights (both copies of the ping-pong buffers)."""
    import torch

    from granite_b200 import synth

    proj, view = cases.default_camera(W, H)
    lights = synth.make_lights(1500, spot_fraction=0.25, aspect=W / H)
    d = cases.to_device(lights)
    vd, keep = _scene_viewer(proj, view)
    vh, _ = _scene_viewer(proj, view, lights)
    vd.set_lights_device(**d)
    for f in range(4):
        if f == 1:
            # most lights go behind the eye: far fewer kept than in frame 0
            lights.position[200:, 2] += 300.0
            d["position"].copy_(torch.from_numpy(lights.position))
            vh.set_lights(lights)
        _frame(vd, keep, f == 0)
        _frame(vh, keep, f == 0)
        k = vh.light_prep()[0]
        assert vd.light_prep()[0] == k
        bm_h, cr_h = _cluster(vh)
        bm_d, cr_d = _cluster(vd)
        assert np.array_equal(cr_h, cr_d), f"frame {f}"
        w32 = (k + 31) // 32
        assert np.array_equal(bm_h[:, :w32], bm_d[:, :w32]), f"frame {f}"
        assert not bm_d[:, w32:].any(), f"frame {f}"
        assert bm_h[:, :w32].any()
    vd.close()
    vh.close()


CONFIGS = {
    "c3-like": dict(),
    "TAA + FXAA": dict(post_aa=_viewer.AA_TAA_HIGH_PLUS_FXAA),
    "resolution_scale 0.75": dict(resolution_scale=0.75),
}


@pytest.mark.parametrize("device_gbuffer", [False, True], ids=["host G-buffer", "device G-buffer"])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_frames_equal_host_light_frames(cuda, config, device_gbuffer):
    """Five frames, the lights moved every frame by a torch op on the device (the host viewer gets the same bytes back):
    the output and HDR-main bit for bit the host-light viewer's; measure_row_cost identical."""
    import torch

    from granite_b200 import synth, viewer

    cfg = CONFIGS[config]
    proj, view = cases.default_camera(W, H)
    lights = synth.make_lights(700, spot_fraction=0.25, aspect=W / H)
    d = cases.to_device(lights)
    vh, keep = _scene_viewer(proj, view, lights, **cfg)
    vd, _ = _scene_viewer(proj, view, **cfg)
    vd.set_lights_device(**d)
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
            moved = synth.Lights(lights.color, d["position"].cpu().numpy(), lights.is_point, lights.rot, lights.inner_cone, lights.outer_cone)
            vh.set_lights(moved)
        want = _frame(vh, keep, f == 0)
        if device_gbuffer:
            vd.render_frame_device(gb if f == 0 else None)
            got = np.zeros((vd.height, vd.width), np.uint32)
            vd.read_output(got)
        else:
            got = _frame(vd, keep, f == 0)
        assert np.array_equal(want, got), f"frame {f}: {int((want != got).sum())} pixels differ"
        assert np.array_equal(vh.download_image("HDR-main"), vd.download_image("HDR-main")), f"frame {f}: HDR-main"
    assert np.array_equal(vh.measure_row_cost(), vd.measure_row_cost())
    vh.close()
    vd.close()


def test_ready_and_consumed_events(cuda):
    """ready: a producer stream sleeps, then writes new positions and records `ready`; the frame shows them.  consumed:
    a stream that overwrites the positions after `consumed` leaves the frame as it was."""
    import torch

    from granite_b200 import synth

    proj, view = cases.default_camera(W, H)
    lights = synth.make_lights(400, spot_fraction=0.25, aspect=W / H)
    new = synth.Lights(lights.color, lights.position + np.float32(1.5), lights.is_point, lights.rot, lights.inner_cone, lights.outer_cone)
    old_ref, keep = _scene_viewer(proj, view, lights)
    new_ref, _ = _scene_viewer(proj, view, new)
    want = [_frame(new_ref, keep, True), _frame(new_ref, keep, False)]
    assert not np.array_equal(_frame(old_ref, keep, True), want[0]), "the moved lights change the frame"

    vd, _ = _scene_viewer(proj, view)
    d = cases.to_device(lights)
    ready, consumed = torch.cuda.Event(), torch.cuda.Event()
    vd.set_lights_device(**d, ready=ready, consumed=consumed)
    producer = torch.cuda.Stream()
    new_t = torch.from_numpy(new.position).cuda()
    old_t = torch.from_numpy(lights.position).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(producer):
        torch.cuda._sleep(50_000_000)
        d["position"].copy_(new_t)
        ready.record()
    assert np.array_equal(_frame(vd, keep, True), want[0]), "the frame read the positions before `ready`"

    # overwrite right after `consumed`: the frame in flight keeps the positions it read
    with torch.cuda.stream(producer):
        ready.record()
    vd.render_frame(None)
    with torch.cuda.stream(producer):
        producer.wait_event(consumed)
        d["position"].copy_(old_t)
    out = np.zeros((H, W), np.uint32)
    vd.read_output(out)
    assert np.array_equal(out, want[1]), "overwriting after `consumed` changed the frame"
    torch.cuda.synchronize()
    for v in (old_ref, new_ref, vd):
        v.close()


def test_switching_between_host_and_device_lights(cuda):
    """host -> device -> host lights on one viewer: each frame equals the frame of a viewer that only had that kind."""
    from granite_b200 import synth

    proj, view = cases.default_camera(W, H)
    lights = synth.make_lights(300, spot_fraction=0.25, aspect=W / H)
    other = synth.make_lights(200, spot_fraction=0.5, aspect=W / H)
    ref, keep = _scene_viewer(proj, view, lights)
    want = [_frame(ref, keep, True), _frame(ref, keep, False)]
    ref.set_lights(other)
    want.append(_frame(ref, keep, False))
    v, _ = _scene_viewer(proj, view, lights)
    got = [_frame(v, keep, True)]
    d = cases.to_device(lights)
    v.set_lights_device(**d)
    got.append(_frame(v, keep, False))
    assert v.light_prep()[0] == 300
    v.set_lights(other)
    got.append(_frame(v, keep, False))
    assert v.light_prep()[0] == 200
    for i, (a, b) in enumerate(zip(want, got)):
        assert np.array_equal(a, b), f"frame {i}"
    ref.close()
    v.close()


def test_set_lights_device_refuses_foreign_memory(cuda):
    """Host tensors and tensors that are not contiguous are refused in Python; host memory behind the C call is refused
    by the pointer check."""
    import ctypes as C

    import torch

    from granite_b200 import capi, synth, viewer

    proj, view = cases.default_camera(W, H)
    v, _ = _scene_viewer(proj, view)
    d = cases.to_device(synth.make_lights(8))
    with pytest.raises(ValueError, match="CUDA tensor"):
        v.set_lights_device(**dict(d, color=d["color"].cpu()))
    with pytest.raises(ValueError, match="contiguous"):
        v.set_lights_device(**dict(d, rotation=d["rotation"].transpose(1, 2)))
    host = np.zeros((8, 3), np.float32)
    l = viewer.GrbhDeviceLights(8, host.ctypes.data, d["position"].data_ptr(), d["is_point"].data_ptr(), d["rotation"].data_ptr(),
                                d["inner_cone"].data_ptr(), d["outer_cone"].data_ptr(), 1e10, None, None)
    assert viewer.lib().grbh_viewer_set_lights_device(v._h, C.byref(l)) < 0
    assert b"color is not device memory" in viewer.lib().grbh_last_error()
    with pytest.raises(capi.GrbError, match="no frame has been rendered"):
        v.set_lights_device(**d)
        v.light_prep()
    torch.cuda.synchronize()
    v.close()
