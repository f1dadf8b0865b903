"""Level table of the multiresolution hash grid, computed the way tiny-cuda-nn does (grid.h: grid_scale,
grid_resolution, params_in_level) from the constructor arguments of `NeuralFeatureField`
(reference dvt/models/neural_feature_field.py:25-39).  Host-side numpy, fp32 arithmetic where tcnn uses float."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np


@dataclass
class HashGridMeta:
    n_levels: int
    n_features: int
    per_level_scale: float
    scale: np.ndarray      # float32 [L]
    res: np.ndarray        # uint32 [L]
    size: np.ndarray       # uint32 [L]   entries per level
    offset: np.ndarray     # uint32 [L+1] entry offsets
    hashed: np.ndarray     # uint32 [L]   1 = level uses the spatial hash

    @property
    def n_entries(self) -> int:
        return int(self.offset[-1])

    @property
    def n_params(self) -> int:
        return self.n_entries * self.n_features

    @property
    def n_output_dims(self) -> int:
        return self.n_levels * self.n_features

    def c_args(self):
        """(n_levels, scale*, res*, size*, offset*, hashed*) for the C ABI (host pointers)."""
        import ctypes
        f = lambda a, t: a.ctypes.data_as(ctypes.POINTER(t))
        return (self.n_levels, f(self.scale, ctypes.c_float), f(self.res, ctypes.c_uint32),
                f(self.size, ctypes.c_uint32), f(self.offset, ctypes.c_uint32), f(self.hashed, ctypes.c_uint32))


def make_meta(n_levels: int, base_resolution: int = 16, max_resolution: int = 1024, n_features_per_level: int = 8,
              log2_hashmap_size: int = 20) -> HashGridMeta:
    if n_features_per_level != 8:
        raise NotImplementedError("the H100 hash grid implements n_features_per_level == 8 (the value DVT uses)")
    if not 1 <= n_levels <= 16:
        raise NotImplementedError("n_levels must be in [1, 16]")
    pls64 = float(np.exp((np.log(max_resolution) - np.log(base_resolution)) / (n_levels - 1))) if n_levels > 1 else 1.0
    log2_pls = np.log2(np.float32(pls64)).astype(np.float32)
    scale = np.zeros(n_levels, np.float32)
    res = np.zeros(n_levels, np.uint32)
    size = np.zeros(n_levels, np.uint32)
    hashed = np.zeros(n_levels, np.uint32)
    offset = np.zeros(n_levels + 1, np.uint32)
    cap = 1 << log2_hashmap_size
    for l in range(n_levels):
        s = np.float32(np.exp2(np.float32(l) * log2_pls)) * np.float32(base_resolution) - np.float32(1.0)
        scale[l] = s
        r = int(np.ceil(s)) + 1
        res[l] = r
        dense = r * r
        n = min((dense + 7) // 8 * 8, cap)
        size[l] = n
        hashed[l] = 1 if dense > n else 0
        offset[l + 1] = offset[l] + n
    return HashGridMeta(n_levels, n_features_per_level, pls64, scale, res, size, offset, hashed)
