"""Light lists for the device light prep tests (test infrastructure): the cases the host prep is held to the oracle on,
handed over in a shuffled order, plus lists that only the sort and the count limit can tell apart.

case(oracle, name) returns (width, height, projection, view, lights, ordered) for one named case: `lights` shuffled,
`ordered` the same lights in the host clusterer's order where the case has one (the oracle's prep takes them so), else
None."""
from __future__ import annotations

import numpy as np

from granite_b200 import synth

HOST_PREP_CASES = ["0-0.0", "16-0.0", "300-0.25", "4096-0.25", "turned", "around-eye", "spots-at-eye", "finite-far", "tall"]
# ties: pairs of lights at identical positions; signed-zero: keys of -0.0 and +0.0 (lights in the plane z = 0 of the
# default view, whose front is (0, 0, -1)), which compare equal and so must keep input order
TIE_CASES = ["ties", "signed-zero"]
# more visible lights than the cluster holds, every light culled, no light at all
LIMIT_CASES = ["6000-visible", "all-culled"]


def default_camera(w=1920, h=1080):
    return synth.perspective_inf(np.pi / 4, w / h, 1 / 16), synth.look_at_view((0, 0, 8), (0, 0, 0))


def shuffled(lights, seed=1):
    perm = np.random.default_rng(seed).permutation(len(lights.color))
    return synth.Lights(lights.color[perm], lights.position[perm], lights.is_point[perm], lights.rot[perm], lights.inner_cone[perm],
                        lights.outer_cone[perm])


def case(oracle, name):
    w, h = 1920, 1080
    proj, view = default_camera(w, h)
    if name in ("turned", "around-eye", "spots-at-eye", "finite-far", "tall"):
        from tests import cluster_cases

        scene, _, lights, _ = cluster_cases.build(oracle, name, check=False)
        return scene.width, scene.height, scene.projection, scene.view, shuffled(lights), lights
    if name == "ties":
        lights = synth.make_lights(96, spot_fraction=0.5)
        lights.position[1::2] = lights.position[0::2]
        lights.position[2::3] = lights.position[0]
    elif name == "signed-zero":
        lights = synth.make_lights(12, spot_fraction=0.5)
        xy = np.array([[-1, -1], [1, 1], [-2, 0.5], [0.5, -2], [3, 1], [-3, -1], [1, -1], [-1, 1], [2, 2], [-2, -2], [0, 0], [0.25, -0.25]],
                      np.float32)
        lights.position[:] = np.concatenate([xy, np.zeros((12, 1), np.float32)], 1)
    elif name == "6000-visible":
        lights = synth.make_lights(6000, spot_fraction=0.25)
    elif name == "all-culled":
        lights = synth.make_lights(200, spot_fraction=0.25)
        lights.position[:, 2] += 200.0  # behind the eye at z = 8, out of reach of every light
    else:
        n, frac = name.split("-")
        lights = synth.make_lights(int(n), spot_fraction=float(frac))
    ordered = None if name in TIE_CASES or name == "all-culled" else lights  # make_lights lists them front to back
    return w, h, proj, view, shuffled(lights), ordered


def to_device(lights, device="cuda"):
    """The light list as the torch tensors Viewer.set_lights_device takes."""
    import torch

    return dict(color=torch.from_numpy(np.ascontiguousarray(lights.color, np.float32)).to(device),
                position=torch.from_numpy(np.ascontiguousarray(lights.position, np.float32)).to(device),
                is_point=torch.from_numpy(np.ascontiguousarray(lights.is_point, np.uint8)).to(device),
                rotation=torch.from_numpy(np.ascontiguousarray(lights.rot, np.float32)).to(device),
                inner_cone=torch.from_numpy(np.ascontiguousarray(lights.inner_cone, np.float32)).to(device),
                outer_cone=torch.from_numpy(np.ascontiguousarray(lights.outer_cone, np.float32)).to(device))
