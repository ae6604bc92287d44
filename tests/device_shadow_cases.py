"""Shadows for device lights in the GPU tests (test infrastructure): the caller's shadow transforms in input order, and
one synthetic D16 shadow map per input light held in a single device tensor, so that a torch op can rewrite texels of
every map and the host-light viewers can be handed the same maps by pointer."""
from __future__ import annotations

import types

import numpy as np


def transforms_in_input_order(oracle, v, lights):
    """The reference's shadow camera of every input light (ClustererBindlessTransforms::shadow, clusterer.cpp:467-474,
    518-521), culled lights included: (N, 16) float32, column-major.  The transform depends on the light alone."""
    from tests import common

    cam = common.oracle_camera_from_viewer(oracle, v)
    return np.ascontiguousarray(oracle.shadow_transforms(oracle.prepare_lights(cam, lights, cull=False)), np.float32).reshape(-1, 16)


class MapPool:
    """Light i's map at texel offsets[i] of one int16 CUDA tensor: res^2 texels for a spot light, 6 res^2 for a point
    light, the texels of tests.common.make_shadow_maps.  Every skip_every-th light has no map (a null pointer)."""

    def __init__(self, lights, res, seed=0x5AD0, skip_every=7):
        import torch

        from tests import common

        n = len(lights.color)
        mask = np.zeros(max((n + 31) // 32, 1), np.uint32)
        for i in np.flatnonzero(lights.is_point):
            mask[i >> 5] |= np.uint32(1 << (i & 31))
        maps = common.make_shadow_maps(types.SimpleNamespace(n=n, type_mask=mask), res, seed=seed, skip_every=skip_every)
        self.res, self.n = res, n
        self.has = np.array([m is not None for m in maps], bool)
        sizes = np.where(np.asarray(lights.is_point, bool), 6, 1) * res * res
        self.offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        host = np.zeros(max(int(self.offsets[-1]), 1), np.uint16)
        for i, m in enumerate(maps):
            if m is not None:
                host[self.offsets[i]:self.offsets[i + 1]] = m.reshape(-1)
        self.pool = torch.from_numpy(host.view(np.int16)).cuda()

    def pointers(self):
        """(N,) int64 map pointers by input light, 0 where the light has no map."""
        p = self.pool.data_ptr() + 2 * self.offsets[:-1]
        return np.where(self.has, p, 0).astype(np.int64)

    def device_pointers(self):
        import torch

        return torch.from_numpy(self.pointers()).cuda()

    def host_maps(self, indices):
        """The maps of input lights `indices` as the oracle takes them: (res, res) or (6, res, res) uint16, None = none."""
        host = self.pool.cpu().numpy().view(np.uint16)
        out = []
        for i in indices:
            if not self.has[i]:
                out.append(None)
                continue
            m = host[self.offsets[i]:self.offsets[i + 1]]
            out.append(m.reshape(-1, self.res, self.res) if m.size > self.res * self.res else m.reshape(self.res, self.res))
        return out

    def rewrite(self, frame):
        """A torch op that changes texels of many maps: every 11th texel from `frame` moves by 700 (mod 3000)."""
        t = self.pool[frame % 11::11]
        t.copy_((t + 700) % 3000)
