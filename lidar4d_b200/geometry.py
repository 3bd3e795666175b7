"""Host-side geometry and per-frame constants for the LiDAR4D hot path.

Everything here is *data* handed identically to the CUDA kernels (through the
C-ABI structs in ``include/lidar4d_b200.h``) and to the oracle, so that integer
work (hash indices, slice indices, frame branches) is bit-exact between them.

Reference semantics restated (citations are into /root/reference):
  * hash-grid level geometry: tiny-cuda-nn ``grid_scale`` / ``grid_resolution``
    / ``params_in_level`` (external, un-vendored; spec in SURVEY.md §8(c)),
    constructor call sites model/hash_field.py:43-57,105-117 and
    model/flow_field.py:66-77.
  * frame logic: model/lidar4d.py:143,157-159,166-168.
  * time-slice blend: model/hash_field.py:76-86.
  * Lagrange basis: model/hash_field.py:65-74, model/flow_field.py:102-111.
"""
from __future__ import annotations

import ctypes
import ctypes.util
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

f32 = np.float32

# ----------------------------------------------------------------------------
# float32 libm (glibc) - tcnn computes level scales on the host with
# std::log2(float) / exp2f.  numpy's SIMD float32 exp2/log2 differ by an ulp,
# which moves the top-level resolution across an integer (SURVEY.md §7 "hard
# parts"), so use the C library when it is there.
# ----------------------------------------------------------------------------
_libm = None
try:  # pragma: no cover - platform dependent
    _name = ctypes.util.find_library("m") or "libm.so.6"
    _libm = ctypes.CDLL(_name)
    _libm.exp2f.restype = ctypes.c_float
    _libm.exp2f.argtypes = [ctypes.c_float]
    _libm.log2f.restype = ctypes.c_float
    _libm.log2f.argtypes = [ctypes.c_float]
except Exception:  # pragma: no cover
    _libm = None


def _log2f(x: float) -> np.float32:
    if _libm is not None:
        return f32(_libm.log2f(float(f32(x))))
    return f32(np.log2(f32(x)))


def _exp2f(x: float) -> np.float32:
    if _libm is not None:
        return f32(_libm.exp2f(float(f32(x))))
    return f32(np.exp2(f32(x)))


MAX_LEVELS = 16
HASH_PRIMES = (1, 2654435761, 805459861)


@dataclass
class GridGeometry:
    """One multi-resolution hash grid (one tcnn ``HashGrid`` encoding)."""

    n_dims: int
    n_levels: int
    n_features: int
    log2_hashmap_size: int
    base_resolution: int
    per_level_scale: float
    scale: np.ndarray = field(default=None)      # float32 [L]
    resolution: np.ndarray = field(default=None)  # uint32  [L]
    entries: np.ndarray = field(default=None)     # uint32  [L] (hashmap_size of the level)
    offset: np.ndarray = field(default=None)      # uint32  [L+1] (in entries)

    @property
    def n_params(self) -> int:
        return int(self.offset[-1]) * self.n_features

    @property
    def n_output_dims(self) -> int:
        return self.n_levels * self.n_features


def per_level_scale(base_resolution: int, max_resolution: int, n_levels: int) -> float:
    """np.exp2(np.log2(max/base)/(L-1)) exactly as the reference computes it
    (model/hash_field.py:43, :105; model/flow_field.py:66)."""
    if n_levels <= 1:
        return 1.0
    return float(np.exp2(np.log2(max_resolution / base_resolution) / (n_levels - 1)))


def make_grid(n_dims: int, n_levels: int, n_features: int, log2_hashmap_size: int,
              base_resolution: int, pls: float) -> GridGeometry:
    """tcnn GridEncoding constructor arithmetic [tcnn-ext], float32 on the host."""
    assert 1 <= n_levels <= MAX_LEVELS
    g = GridGeometry(n_dims, n_levels, n_features, log2_hashmap_size, base_resolution, pls)
    log2s = _log2f(f32(pls))
    scale = np.zeros(n_levels, dtype=np.float32)
    res = np.zeros(n_levels, dtype=np.uint32)
    ent = np.zeros(n_levels, dtype=np.uint32)
    off = np.zeros(n_levels + 1, dtype=np.uint32)
    max_params = np.iinfo(np.uint32).max // 2
    acc = 0
    for l in range(n_levels):
        s = f32(_exp2f(f32(l) * log2s) * f32(base_resolution)) - f32(1.0)
        r = int(np.ceil(s)) + 1
        dense = float(f32(r)) ** n_dims
        n = max_params if dense > float(max_params) else r ** n_dims
        n = (n + 7) // 8 * 8                      # next_multiple(., 8)
        n = min(n, 1 << log2_hashmap_size)        # GridType::Hash
        scale[l], res[l], ent[l], off[l] = s, r, n, acc
        acc += n
    off[n_levels] = acc
    g.scale, g.resolution, g.entries, g.offset = scale, res, ent, off
    return g


# ----------------------------------------------------------------------------
# Lagrange basis with the reference's exact float32 op order
# ----------------------------------------------------------------------------
def lagrange_basis(t: np.float32, num_basis: int = 4) -> np.ndarray:
    """L_i(t) for nodes T_i=i/(nb-1), evaluated like hash_field.py:70-72:
    each factor is (t - T[m]) / (T[j] - T[m]) in float32 (python-double nodes
    rounded to float32 when they meet the float32 tensor), multiplied left to
    right by math.prod."""
    t = f32(t)
    T = [i / (num_basis - 1) for i in range(num_basis)]
    out = np.zeros(num_basis, dtype=np.float32)
    for j in range(num_basis):
        p = None
        for m in range(num_basis):
            if m == j:
                continue
            fac = f32(f32(t - f32(T[m])) / f32(T[j] - T[m]))
            p = fac if p is None else f32(p * fac)
        out[j] = p
    return out


@dataclass
class TimeQuery:
    """One (·, tau) query of the dynamic hash planes / time planes."""

    tau: np.float32
    slice_lo: int
    slice_hi: int
    w_lo: np.float32       # (idx2 - idx)
    w_hi: np.float32       # (idx - idx1)
    single: bool           # idx1 == idx2  -> feature = G_lo only
    basis: np.ndarray      # float32 [4]


def make_time_query(tau, time_resolution: int) -> TimeQuery:
    """HashGridT.forward slice selection (hash_field.py:79-85) in float32."""
    tau = f32(tau)
    idx = f32(tau * f32(time_resolution - 1))
    lo = int(np.floor(idx))
    hi = int(np.ceil(idx))
    # the reference indexes a python ModuleList: negative indices wrap, too
    # large ones raise.  Frame times are in [0,1] so this cannot happen; clamp
    # defensively so that the kernel never reads out of bounds.
    lo_c = min(max(lo, 0), time_resolution - 1)
    hi_c = min(max(hi, 0), time_resolution - 1)
    return TimeQuery(
        tau=tau, slice_lo=lo_c, slice_hi=hi_c,
        w_lo=f32(f32(hi) - idx), w_hi=f32(idx - f32(lo)),
        single=(lo == hi), basis=lagrange_basis(tau),
    )


@dataclass
class FrameConstants:
    """Everything LiDAR4D.density() decides on the host from the frame time."""

    time: np.float32
    frame_idx: int
    has_fwd: bool
    has_bwd: bool
    cur: TimeQuery
    fwd: Optional[TimeQuery]
    bwd: Optional[TimeQuery]
    flow_basis: np.ndarray  # Lagrange basis at `time` for the flow grid


def make_frame(time, num_frames: int, time_resolution: int) -> FrameConstants:
    """lidar4d.py:143 frame_idx=int(t*(F-1)); :157-159 t1=(k+1)/F; :166-168 t2=(k-1)/F."""
    t = f32(time)
    k = int(f32(t * f32(num_frames - 1)))
    has_fwd = k < num_frames - 1
    has_bwd = k > 0
    cur = make_time_query(t, time_resolution)
    fwd = make_time_query(f32((k + 1) / num_frames), time_resolution) if has_fwd else None
    bwd = make_time_query(f32((k - 1) / num_frames), time_resolution) if has_bwd else None
    return FrameConstants(t, k, has_fwd, has_bwd, cur, fwd, bwd, lagrange_basis(t))


# ----------------------------------------------------------------------------
# model-level configuration (mirrors LiDAR4D.__init__ kwargs, lidar4d.py:23-45)
# ----------------------------------------------------------------------------
@dataclass
class FieldConfig:
    min_resolution: int = 32
    base_resolution: int = 512
    max_resolution: int = 32768
    time_resolution: int = 8
    n_levels_plane: int = 4
    n_features_per_level_plane: int = 8
    n_levels_hash: int = 8
    n_features_per_level_hash: int = 4
    log2_hashmap_size: int = 19
    hash_size_dynamic: tuple = (15, 13, 13)      # hash_field.py:100
    num_layers_flow: int = 3
    hidden_dim_flow: int = 64
    num_layers_sigma: int = 2
    hidden_dim_sigma: int = 64
    geo_feat_dim: int = 15
    num_layers_lidar: int = 3
    hidden_dim_lidar: int = 64
    out_lidar_dim: int = 2
    num_frames: int = 51
    bound: float = 1.0
    near_lidar: float = 0.01
    far_lidar: float = 0.81
    density_scale: float = 1.0
    active_sensor: bool = False
    # flow field defaults, flow_field.py:41-54
    flow_n_levels: int = 8
    flow_n_features: int = 8
    flow_base_resolution: int = 32
    flow_max_resolution: int = 8192
    flow_log2_hashmap_size: int = 18
    view_degree: int = 12                        # lidar4d.py:72

    # ---- derived ----
    def static_grid(self) -> GridGeometry:
        pls = per_level_scale(self.base_resolution, self.max_resolution, self.n_levels_hash)
        return make_grid(3, self.n_levels_hash, self.n_features_per_level_hash,
                         self.log2_hashmap_size, self.base_resolution, pls)

    def dynamic_grid(self, plane: int) -> GridGeometry:
        pls = per_level_scale(self.base_resolution, self.max_resolution, self.n_levels_hash)
        return make_grid(2, self.n_levels_hash, self.n_features_per_level_hash,
                         self.hash_size_dynamic[plane], self.base_resolution, pls)

    def flow_grid(self) -> GridGeometry:
        pls = per_level_scale(self.flow_base_resolution, self.flow_max_resolution, self.flow_n_levels)
        return make_grid(3, self.flow_n_levels, self.flow_n_features,
                         self.flow_log2_hashmap_size, self.flow_base_resolution, pls)

    @property
    def plane_scales(self) -> List[int]:
        return [2 ** n for n in range(self.n_levels_plane)]

    @property
    def plane_dim(self) -> int:                  # static (== dynamic) plane feature width
        return self.n_levels_plane * self.n_features_per_level_plane

    @property
    def hash_static_dim(self) -> int:
        return self.n_levels_hash * self.n_features_per_level_hash

    @property
    def hash_dynamic_dim(self) -> int:           # 3 planes x L x F/num_basis
        return 3 * self.n_levels_hash * self.n_features_per_level_hash // 4

    @property
    def sigma_in_dim(self) -> int:
        return 2 * self.plane_dim + self.hash_static_dim + self.hash_dynamic_dim

    @property
    def sigma_in_pad(self) -> int:
        return (self.sigma_in_dim + 15) // 16 * 16

    @property
    def view_dim(self) -> int:
        return 3 * 2 * self.view_degree

    @property
    def attr_in_dim(self) -> int:
        return self.view_dim + self.geo_feat_dim

    @property
    def attr_in_pad(self) -> int:
        return (self.attr_in_dim + 15) // 16 * 16

    def mlp_param_count(self, n_in_pad: int, hidden: int, n_hidden_layers: int, n_out_pad: int = 16) -> int:
        """tcnn FullyFusedMLP: [hidden,in_pad] + (n_hidden_layers-1)x[hidden,hidden] + [out_pad,hidden]."""
        return hidden * n_in_pad + (n_hidden_layers - 1) * hidden * hidden + n_out_pad * hidden

    def validate(self) -> None:
        """The sm_90a kernels are specialised for the reference defaults that
        its CLI never changes in the shipped run scripts (run_kitti_lidar4d.sh);
        n_levels_hash / hashmap sizes / resolutions / num_frames stay runtime."""
        assert self.n_features_per_level_hash == 4, "time basis needs F=4 (hash_field.py:38,62)"
        assert self.n_features_per_level_plane == 8
        assert 1 <= self.n_levels_plane <= 4
        assert 1 <= self.n_levels_hash <= MAX_LEVELS
        assert self.hidden_dim_sigma == 64 and self.hidden_dim_lidar == 64 and self.hidden_dim_flow == 64
        assert self.num_layers_sigma == 2 and self.num_layers_lidar == 3 and self.num_layers_flow == 3
        assert self.geo_feat_dim == 15 and self.out_lidar_dim == 2
        assert self.flow_n_features == 8 and self.flow_n_levels == 8
        assert self.time_resolution >= 2
