"""ctypes mirror of include/lidar4d_b200.h and the loader of
csrc/liblidar4d_b200.so.  There is no fallback: a missing library raises."""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

from .geometry import FieldConfig, FrameConstants, GridGeometry, TimeQuery

MAX_LEVELS = 16
MAX_PLANE_SCALES = 4
MAX_TIME_SLICES = 16
ABI_VERSION = 1
STAGE_TABLES, STAGE_SMALL = 1, 2        # l4d_stage_params_ex `what`
ADAM_CHUNK, ADAM_MAX_SEGMENTS = 1024, 64
FLOW_PARTS = 2048                       # L4D_FLOW_PARTS: per-launch slots of the flow loss's partial sums

c_float_p = C.POINTER(C.c_float)


class L4DGrid(C.Structure):
    _fields_ = [("n_dims", C.c_uint32), ("n_levels", C.c_uint32), ("n_features", C.c_uint32),
                ("reserved", C.c_uint32),
                ("scale", C.c_float * MAX_LEVELS), ("resolution", C.c_uint32 * MAX_LEVELS),
                ("entries", C.c_uint32 * MAX_LEVELS), ("offset", C.c_uint32 * (MAX_LEVELS + 1))]


class L4DConfig(C.Structure):
    _fields_ = [("hash_static", L4DGrid), ("hash_dynamic", L4DGrid * 3), ("flow", L4DGrid),
                ("n_plane_scales", C.c_uint32), ("plane_res", C.c_uint32 * MAX_PLANE_SCALES),
                ("time_resolution", C.c_uint32), ("num_frames", C.c_uint32),
                ("active_sensor", C.c_uint32), ("view_degree", C.c_uint32),
                ("sigma_in_dim", C.c_uint32), ("sigma_in_pad", C.c_uint32),
                ("attr_in_dim", C.c_uint32), ("attr_in_pad", C.c_uint32),
                ("bound", C.c_float), ("near_lidar", C.c_float), ("far_lidar", C.c_float),
                ("density_scale", C.c_float), ("mlp_fp16", C.c_uint32), ("reserved", C.c_uint32)]


class L4DTimeQuery(C.Structure):
    _fields_ = [("tau", C.c_float), ("slice_lo", C.c_uint32), ("slice_hi", C.c_uint32),
                ("w_lo", C.c_float), ("w_hi", C.c_float), ("single", C.c_uint32),
                ("basis", C.c_float * 4)]


class L4DFrame(C.Structure):
    _fields_ = [("time", C.c_float), ("frame_idx", C.c_uint32), ("has_fwd", C.c_uint32),
                ("has_bwd", C.c_uint32), ("cur", L4DTimeQuery), ("fwd", L4DTimeQuery),
                ("bwd", L4DTimeQuery), ("flow_basis", C.c_float * 4)]


class L4DMasterParams(C.Structure):
    _fields_ = [("hash_static", C.c_void_p),
                ("hash_dynamic", (C.c_void_p * MAX_TIME_SLICES) * 3),
                ("flow_grid", C.c_void_p),
                ("planes", (C.c_void_p * 6) * MAX_PLANE_SCALES),
                ("sigma_net", C.c_void_p), ("intensity_net", C.c_void_p), ("raydrop_net", C.c_void_p),
                ("flow_mlp", C.c_void_p * 3)]


class L4DMasterGrads(C.Structure):
    _fields_ = L4DMasterParams._fields_


class L4DAdamGroup(C.Structure):
    _fields_ = [("begin", C.c_uint64), ("end", C.c_uint64), ("lr", C.c_float), ("reserved", C.c_uint32)]


class L4DRays(C.Structure):
    _fields_ = [("rays_o", C.c_void_p), ("rays_d", C.c_void_p), ("n_rays", C.c_uint32),
                ("n_steps", C.c_uint32), ("perturb", C.c_uint32), ("reserved", C.c_uint32),
                ("seed", C.c_uint64), ("ray_offset", C.c_uint64)]


# ----------------------------------------------------------------------------
# struct builders
# ----------------------------------------------------------------------------
def _grid(g: GridGeometry) -> L4DGrid:
    s = L4DGrid()
    s.n_dims, s.n_levels, s.n_features = g.n_dims, g.n_levels, g.n_features
    for l in range(g.n_levels):
        s.scale[l] = float(g.scale[l])
        s.resolution[l] = int(g.resolution[l])
        s.entries[l] = int(g.entries[l])
        s.offset[l] = int(g.offset[l])
    s.offset[g.n_levels] = int(g.offset[g.n_levels])
    return s


def make_config(cfg: FieldConfig, mlp_fp16: bool = False) -> L4DConfig:
    cfg.validate()
    c = L4DConfig()
    c.mlp_fp16 = int(bool(mlp_fp16))
    c.hash_static = _grid(cfg.static_grid())
    for p in range(3):
        c.hash_dynamic[p] = _grid(cfg.dynamic_grid(p))
    c.flow = _grid(cfg.flow_grid())
    c.n_plane_scales = cfg.n_levels_plane
    for i, m in enumerate(cfg.plane_scales):
        c.plane_res[i] = cfg.min_resolution * m
    c.time_resolution = cfg.time_resolution
    c.num_frames = cfg.num_frames
    c.active_sensor = int(bool(cfg.active_sensor))
    c.view_degree = cfg.view_degree
    c.sigma_in_dim, c.sigma_in_pad = cfg.sigma_in_dim, cfg.sigma_in_pad
    c.attr_in_dim, c.attr_in_pad = cfg.attr_in_dim, cfg.attr_in_pad
    c.bound = float(cfg.bound)
    c.near_lidar = float(np.float32(cfg.near_lidar))
    c.far_lidar = float(np.float32(cfg.far_lidar))
    c.density_scale = float(cfg.density_scale)
    return c


def _tq(q: Optional[TimeQuery]) -> L4DTimeQuery:
    s = L4DTimeQuery()
    if q is None:
        return s
    s.tau = float(q.tau)
    s.slice_lo, s.slice_hi = q.slice_lo, q.slice_hi
    s.w_lo, s.w_hi = float(q.w_lo), float(q.w_hi)
    s.single = int(q.single)
    for i in range(4):
        s.basis[i] = float(q.basis[i])
    return s


def make_frame_struct(fr: FrameConstants) -> L4DFrame:
    f = L4DFrame()
    f.time = float(fr.time)
    f.frame_idx = fr.frame_idx
    f.has_fwd, f.has_bwd = int(fr.has_fwd), int(fr.has_bwd)
    f.cur, f.fwd, f.bwd = _tq(fr.cur), _tq(fr.fwd), _tq(fr.bwd)
    for i in range(4):
        f.flow_basis[i] = float(fr.flow_basis[i])
    return f


# ----------------------------------------------------------------------------
# library loading
# ----------------------------------------------------------------------------
_LIB = None
LIB_NAME = "liblidar4d_b200.so"
EXPORTS = [
    "l4d_abi_version", "l4d_last_error", "l4d_staged_bytes", "l4d_stage_params", "l4d_saved_bytes",
    "l4d_render_forward", "l4d_grad_work_bytes", "l4d_render_backward", "l4d_unstage_grads",
    "l4d_flow_forward", "l4d_flow_backward", "l4d_hash_indices", "l4d_density_forward", "l4d_attribute_forward", "l4d_chamfer_work_bytes", "l4d_chamfer_forward", "l4d_chamfer_backward", "l4d_tc_selftest", "l4d_tc_selftest2", "l4d_profile_start", "l4d_profile_stop",
    "l4d_stage_params_ex", "l4d_adam_step", "l4d_launch_count", "l4d_render_backward_ex", "l4d_lidar_rays", "l4d_lidar_loss",
    "l4d_density_saved_bytes", "l4d_density_forward_ex", "l4d_density_backward", "l4d_attribute_backward",
    "l4d_pano_project_work_bytes", "l4d_pano_project", "l4d_pano_unproject_work_bytes", "l4d_pano_unproject",
    "l4d_point_metrics",
    "l4d_range_filter_work_bytes", "l4d_range_filter", "l4d_knn_mean_dist", "l4d_outlier_select_work_bytes",
    "l4d_outlier_select", "l4d_plane_scores", "l4d_plane_mask", "l4d_ground_split_work_bytes", "l4d_ground_split",
    "l4d_pose_transform",
    "l4d_patch_loss", "l4d_patch_loss_backward", "l4d_los_work_bytes", "l4d_los_loss", "l4d_los_loss_backward",
    "l4d_nn_grid_bytes", "l4d_nn_grid_work_bytes", "l4d_nn_grid_build", "l4d_nn_grid_query", "l4d_flow_warp_query",
    "l4d_flow_term_backward", "l4d_flow_ground", "l4d_flow_ground_backward", "l4d_flow_loss_finish",
    "l4d_image_metrics_work_bytes", "l4d_image_metrics", "l4d_raydrop_metrics",
    "l4d_sweep_images",
    "l4d_box_mask", "l4d_bce_loss_work_bytes", "l4d_bce_loss", "l4d_bce_loss_backward",
]
SWEEP_SIM, SWEEP_TEST, SWEEP_EVAL = 0, 1, 2     # L4D_SWEEP_* layouts of l4d_sweep_images
SWEEP_F32, SWEEP_F16 = 0, 1                     # L4D_SWEEP_* ray-drop dtypes
MAX_BOXES = 32                                  # L4D_MAX_BOXES of l4d_box_mask
DTYPE_F32, DTYPE_F16, DTYPE_BF16 = 0, 1, 2      # L4D_DTYPE_* of l4d_bce_loss
EINVAL = -1                                     # L4D_EINVAL


def lib_path() -> str:
    # L4D_LIB_PATH: developer override to A/B test differently compiled builds of the same library
    return os.environ.get("L4D_LIB_PATH") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", LIB_NAME)


def declare(lib, prefix: str = "l4d_", host_sim: bool = False):
    """Attach argtypes/restypes.  The host-sim test library exports the same
    entry points with an `hs_` prefix and without size/stream arguments."""
    P, V, U32, SZ = C.POINTER, C.c_void_p, C.c_uint32, C.c_size_t
    f = lambda n: getattr(lib, prefix + n)
    f("last_error").restype = C.c_char_p
    f("last_error").argtypes = []
    f("staged_bytes").restype = SZ
    f("staged_bytes").argtypes = [P(L4DConfig)]
    f("grad_work_bytes").restype = SZ
    f("grad_work_bytes").argtypes = [P(L4DConfig)]
    f("saved_bytes").restype = SZ
    f("saved_bytes").argtypes = [P(L4DConfig), U32, U32]
    if not host_sim:
        lib.l4d_abi_version.restype = C.c_int
        lib.l4d_abi_version.argtypes = []
        f("stage_params").argtypes = [P(L4DConfig), P(L4DMasterParams), V, SZ, V]
        f("render_forward").argtypes = [P(L4DConfig), V, P(L4DFrame), P(L4DRays), V, V, V, V, V, V, SZ, V]
        f("render_backward").argtypes = [P(L4DConfig), V, P(L4DFrame), P(L4DRays), V, SZ, V, V, V, V,
                                         P(L4DMasterGrads), V, SZ, V]
        lib.l4d_render_backward_ex.argtypes = [P(L4DConfig), V, P(L4DFrame), P(L4DRays), V, SZ, V, V, V, V,
                                               P(L4DMasterGrads), V, SZ, V, V]
        lib.l4d_render_backward_ex.restype = C.c_int
        f("unstage_grads").argtypes = [P(L4DConfig), V, SZ, P(L4DMasterGrads), V]
        f("flow_forward").argtypes = [P(L4DConfig), V, P(L4DFrame), V, U32, V, V, V]
        f("flow_backward").argtypes = [P(L4DConfig), V, P(L4DFrame), V, U32, V, V, P(L4DMasterGrads), V, SZ, V]
        f("hash_indices").argtypes = [P(L4DConfig), U32, U32, V, U32, V, V, V]
        f("density_forward").argtypes = [P(L4DConfig), V, P(L4DFrame), V, U32, V, V, V, V, V]
        # explicit-point density / attribute with a backward: saved = l4d_density_saved_bytes(cfg, n) bytes, the
        # backwards accumulate into `grads` / grad_work like l4d_render_backward (then l4d_unstage_grads)
        lib.l4d_density_saved_bytes.argtypes = [P(L4DConfig), U32]
        lib.l4d_density_saved_bytes.restype = SZ
        lib.l4d_density_forward_ex.argtypes = [P(L4DConfig), V, P(L4DFrame), V, U32, V, V, V, V, V, SZ, V]
        lib.l4d_density_backward.argtypes = [P(L4DConfig), V, P(L4DFrame), V, U32, V, SZ, V, V, P(L4DMasterGrads), V, SZ, V]
        lib.l4d_attribute_backward.argtypes = [P(L4DConfig), V, V, V, V, U32, V, V, P(L4DMasterGrads), V, SZ, V]
        for n in ("l4d_density_forward_ex", "l4d_density_backward", "l4d_attribute_backward"):
            getattr(lib, n).restype = C.c_int
        lib.l4d_attribute_forward.argtypes = [P(L4DConfig), V, V, V, V, U32, V, V]
        lib.l4d_attribute_forward.restype = C.c_int
        lib.l4d_chamfer_work_bytes.argtypes = [U32, U32, U32]
        lib.l4d_chamfer_work_bytes.restype = SZ
        lib.l4d_chamfer_forward.argtypes = [V, V, U32, U32, U32, V, V, V, V, V, SZ, V]
        lib.l4d_chamfer_forward.restype = C.c_int
        lib.l4d_chamfer_backward.argtypes = [V, V, U32, U32, U32, V, V, V, V, V, V, V]
        lib.l4d_chamfer_backward.restype = C.c_int
        lib.l4d_tc_selftest.argtypes = [V, V, V, U32, U32, V]
        lib.l4d_tc_selftest.restype = C.c_int
        lib.l4d_tc_selftest2.argtypes = [V, V, V, U32, U32, U32, U32, U32, V]
        lib.l4d_tc_selftest2.restype = C.c_int
        lib.l4d_stage_params_ex.argtypes = [P(L4DConfig), P(L4DMasterParams), V, SZ, U32, V]
        lib.l4d_stage_params_ex.restype = C.c_int
        lib.l4d_adam_step.argtypes = [P(L4DConfig), V, V, V, V, C.c_uint64, P(L4DAdamGroup), U32, C.c_float, C.c_float,
                                      C.c_float, U32, C.c_float, U32, P(L4DMasterParams), V, SZ, V]
        lib.l4d_adam_step.restype = C.c_int
        lib.l4d_lidar_rays.argtypes = [V, C.c_float, C.c_float, U32, U32, V, U32, V, U32, V, V, V, V]
        lib.l4d_lidar_rays.restype = C.c_int
        lib.l4d_lidar_loss.argtypes = [V, V, V, U32, C.c_float, C.c_float, C.c_float, C.c_float, V, V, V, V]
        lib.l4d_lidar_loss.restype = C.c_int
        F = C.c_float
        lib.l4d_patch_loss.argtypes = [V, V, U32, U32, U32, F, U32, U32, F, F, F, F, V, V, V]
        lib.l4d_patch_loss_backward.argtypes = [V, V, U32, V, V]
        lib.l4d_los_work_bytes.argtypes = []
        lib.l4d_los_work_bytes.restype = SZ
        lib.l4d_los_loss.argtypes = [V, V, V, U32, U32, C.c_double, V, V, SZ, V]
        lib.l4d_los_loss_backward.argtypes = [V, V, V, U32, U32, C.c_double, V, V, V, V]
        for n in ("patch_loss", "patch_loss_backward", "los_loss", "los_loss_backward"):
            getattr(lib, f"l4d_{n}").restype = C.c_int
        for n in ("nn_grid_bytes", "nn_grid_work_bytes"):
            getattr(lib, f"l4d_{n}").argtypes = [U32]
            getattr(lib, f"l4d_{n}").restype = SZ
        lib.l4d_nn_grid_build.argtypes = [V, U32, V, SZ, V, SZ, V]
        lib.l4d_nn_grid_query.argtypes = [V, SZ, U32, V, U32, V, V, V, V]
        lib.l4d_flow_warp_query.argtypes = [V, V, U32, U32, F, V, SZ, U32, V, V, V, V]
        lib.l4d_flow_term_backward.argtypes = [V, U32, V, U32, V, V, U32, F, V, V, V]
        lib.l4d_flow_ground.argtypes = [V, U32, V, V]
        lib.l4d_flow_ground_backward.argtypes = [V, U32, V, V, V]
        lib.l4d_flow_loss_finish.argtypes = [V, U32, U32, V, V]
        for n in ("nn_grid_build", "nn_grid_query", "flow_warp_query", "flow_term_backward", "flow_ground",
                  "flow_ground_backward", "flow_loss_finish"):
            getattr(lib, f"l4d_{n}").restype = C.c_int
        lib.l4d_pano_project_work_bytes.argtypes = [U32, U32]
        lib.l4d_pano_project_work_bytes.restype = SZ
        lib.l4d_pano_project.argtypes = [V, U32, U32, C.c_double, C.c_double, U32, U32, C.c_float, V, V, V, SZ, V]
        lib.l4d_pano_project.restype = C.c_int
        lib.l4d_pano_unproject_work_bytes.argtypes = [U32, U32]
        lib.l4d_pano_unproject_work_bytes.restype = SZ
        lib.l4d_pano_unproject.argtypes = [V, V, U32, U32, C.c_float, C.c_float, V, V, V, SZ, V]
        lib.l4d_pano_unproject.restype = C.c_int
        lib.l4d_point_metrics.argtypes = [V, U32, V, U32, C.c_float, V, V]
        lib.l4d_point_metrics.restype = C.c_int
        lib.l4d_image_metrics_work_bytes.argtypes = [U32, U32]
        lib.l4d_image_metrics_work_bytes.restype = SZ
        lib.l4d_image_metrics.argtypes = [V, V, U32, U32, C.c_float, C.c_float, C.c_float, V, V, SZ, V]
        lib.l4d_image_metrics.restype = C.c_int
        lib.l4d_raydrop_metrics.argtypes = [V, V, U32, C.c_float, V, V]
        lib.l4d_raydrop_metrics.restype = C.c_int
        lib.l4d_sweep_images.argtypes = [V, V, V, U32, U32, U32, U32, C.c_float, U32, V, V, V, V, V, V]
        lib.l4d_sweep_images.restype = C.c_int
        lib.l4d_box_mask.argtypes = [V, V, U32, U32, U32, U32, V, U32, V]
        lib.l4d_bce_loss_work_bytes.argtypes = []
        lib.l4d_bce_loss_work_bytes.restype = SZ
        lib.l4d_bce_loss.argtypes = [V, U32, V, U32, V, V, SZ, V]
        lib.l4d_bce_loss_backward.argtypes = [V, U32, V, U32, V, V, V]
        for n in ("box_mask", "bce_loss", "bce_loss_backward"):
            getattr(lib, f"l4d_{n}").restype = C.c_int
        D, F = C.c_double, C.c_float
        for n in ("range_filter", "outlier_select", "ground_split"):
            getattr(lib, f"l4d_{n}_work_bytes").argtypes = [U32]
            getattr(lib, f"l4d_{n}_work_bytes").restype = SZ
        lib.l4d_range_filter.argtypes = [V, U32, U32, F, F, F, F, V, V, V, SZ, V]
        lib.l4d_knn_mean_dist.argtypes = [V, U32, U32, V, V]
        lib.l4d_outlier_select.argtypes = [V, U32, V, D, V, V, V, V, V, SZ, V]
        lib.l4d_plane_scores.argtypes = [V, U32, V, U32, D, V, V]
        lib.l4d_plane_mask.argtypes = [V, U32, D, D, D, D, D, D, V, V]
        lib.l4d_ground_split.argtypes = [V, U32, V, D, V, V, V, V, V, V, SZ, V]
        lib.l4d_pose_transform.argtypes = [V, U32, D, V, V, V]
        for n in ("range_filter", "knn_mean_dist", "outlier_select", "plane_scores", "plane_mask", "ground_split",
                  "pose_transform"):
            getattr(lib, f"l4d_{n}").restype = C.c_int
        lib.l4d_launch_count.argtypes = []
        lib.l4d_launch_count.restype = C.c_uint64
        lib.l4d_profile_start.argtypes = []
        lib.l4d_profile_start.restype = C.c_int
        lib.l4d_profile_stop.argtypes = [P(C.c_char_p), P(C.c_float), C.c_int]
        lib.l4d_profile_stop.restype = C.c_int
    else:
        f("stage_params").argtypes = [P(L4DConfig), P(L4DMasterParams), V]
        f("render_forward").argtypes = [P(L4DConfig), V, P(L4DFrame), P(L4DRays), V, V, V, V, V, V]
        f("render_backward").argtypes = [P(L4DConfig), V, P(L4DFrame), P(L4DRays), V, V, V, V, V,
                                         P(L4DMasterGrads), V]
        f("unstage_grads").argtypes = [P(L4DConfig), V, P(L4DMasterGrads)]
        f("flow_forward").argtypes = [P(L4DConfig), V, P(L4DFrame), V, U32, V, V]
        f("flow_backward").argtypes = [P(L4DConfig), V, P(L4DFrame), V, U32, V, V, P(L4DMasterGrads), V]
        f("hash_indices").argtypes = [P(L4DConfig), U32, U32, V, U32, V, V]
        f("density_forward").argtypes = [P(L4DConfig), V, P(L4DFrame), V, U32, V, V, V, V]
    for n in ("stage_params", "render_forward", "render_backward", "unstage_grads", "flow_forward",
              "flow_backward", "hash_indices", "density_forward"):
        f(n).restype = C.c_int
    return lib


def load_library():
    """Load liblidar4d_b200.so (built by __graft_entry__.build()).  Raises if absent."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if not os.path.exists(path):
        raise RuntimeError(
            f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  lidar4d_b200 has no CPU fallback.")
    lib = C.CDLL(path)
    declare(lib)
    if lib.l4d_abi_version() != ABI_VERSION:
        raise RuntimeError("liblidar4d_b200.so ABI version mismatch; rebuild")
    _LIB = lib
    return lib


def check(lib, rc: int, what: str, prefix: str = "l4d_") -> None:
    if rc != 0:
        msg = getattr(lib, prefix + "last_error")().decode()
        raise RuntimeError(f"{what} failed (code {rc}): {msg}")


# ----------------------------------------------------------------------------
# parameter / gradient pointer tables (reference state_dict names, SURVEY.md 8(b))
# ----------------------------------------------------------------------------
def param_names(cfg: FieldConfig):
    """Reference state_dict keys of every tensor the hot path reads, in arena order."""
    names = []
    for s in range(cfg.n_levels_plane):
        for ci in range(6):
            names.append(f"planes_encoder.planes.{s}.{ci}")
    names.append("hash_encoder.hash_static.params")
    for p in range(3):
        for s in range(cfg.time_resolution):
            names.append(f"hash_encoder.hash_dynamic.{p}.hash_t.{s}.params")
    names.append("flow_net.grid_enc.params")
    names += ["flow_net.mlp.0.weight", "flow_net.mlp.2.weight", "flow_net.mlp.4.weight"]
    names += ["sigma_net.params", "intensity_net.params", "raydrop_net.params"]
    return names


def fill_pointer_table(table, cfg: FieldConfig, ptr_of):
    """Fill an L4DMasterParams / L4DMasterGrads from `ptr_of(name) -> int address`."""
    for s in range(cfg.n_levels_plane):
        for ci in range(6):
            table.planes[s][ci] = ptr_of(f"planes_encoder.planes.{s}.{ci}")
    table.hash_static = ptr_of("hash_encoder.hash_static.params")
    for p in range(3):
        for s in range(cfg.time_resolution):
            table.hash_dynamic[p][s] = ptr_of(f"hash_encoder.hash_dynamic.{p}.hash_t.{s}.params")
    table.flow_grid = ptr_of("flow_net.grid_enc.params")
    for i, k in enumerate((0, 2, 4)):
        table.flow_mlp[i] = ptr_of(f"flow_net.mlp.{k}.weight")
    table.sigma_net = ptr_of("sigma_net.params")
    table.intensity_net = ptr_of("intensity_net.params")
    table.raydrop_net = ptr_of("raydrop_net.params")
    return table


def profile_kernels(fn, cap: int = 256):
    """Run fn() with per-kernel CUDA-event timing enabled; returns {kernel name: [ms, ...]}."""
    lib = load_library()
    lib.l4d_profile_start()
    try:
        fn()
    finally:
        names = (C.c_char_p * cap)()
        ms = (C.c_float * cap)()
        n = lib.l4d_profile_stop(names, ms, cap)
    if n < 0:
        raise RuntimeError(lib.l4d_last_error().decode())
    out = {}
    for i in range(n):
        out.setdefault(names[i].decode(), []).append(float(ms[i]))
    return out
