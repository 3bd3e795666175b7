"""CPU: the multi-frame render entry points (l4d_render_forward_frames / l4d_render_backward_frames) - exports, the
ctypes mirror of L4DFrameTable, argument checking before any launch, the per-frame buffer sizes, and the per-row frame
constants the Python layer builds for a render over rows of different times."""
import ctypes as C
import os
import re

import pytest
import torch

from lidar4d_b200 import _capi
from lidar4d_b200.geometry import FieldConfig, make_frame
from lidar4d_b200.model import LiDAR4D, row_frame_groups

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("l4d_saved_bytes_frames", "l4d_grad_work_bytes_frames", "l4d_render_forward_frames", "l4d_render_backward_frames")


def header_define(name: str) -> int:
    src = open(os.path.join(ROOT, "include", "lidar4d_b200.h")).read()
    return int(re.search(rf"#define\s+{name}\s+(\d+)", src).group(1))


def test_new_symbols_are_exported():
    lib = _capi.load_library()
    for n in NEW:
        assert n in _capi.EXPORTS
        assert hasattr(lib, n), n


def test_frame_table_mirror_matches_header():
    assert _capi.MAX_FRAMES == header_define("L4D_MAX_FRAMES")
    # four uint32 then L4D_MAX_FRAMES L4DFrame records (152 bytes each, 4-byte aligned)
    assert C.sizeof(_capi.L4DFrame) == 152
    assert C.sizeof(_capi.L4DFrameTable) == 16 + _capi.MAX_FRAMES * 152
    assert _capi.L4DFrameTable.frames.offset == 16


def _table(n_frames, rpf, phase):
    t = _capi.L4DFrameTable()
    t.n_frames, t.rays_per_frame, t.first_ray_phase = n_frames, rpf, phase
    for i in range(min(n_frames, _capi.MAX_FRAMES)):
        t.frames[i] = _capi.make_frame_struct(make_frame(0.1 * i, 51, 8))
    return t


def _call_forward(lib, cfg, tab, n_rays):
    ro = (C.c_float * 3)()
    rays = _capi.L4DRays()
    rays.rays_o, rays.rays_d = C.addressof(ro), C.addressof(ro)
    rays.n_rays, rays.n_steps = n_rays, 16
    out = (C.c_float * 8)()
    p = C.addressof(out)
    return lib.l4d_render_forward_frames(C.byref(cfg), p, C.byref(tab), C.byref(rays), p, p, p, None, None, None, 0, None)


def _call_backward(lib, cfg, tab, n_rays):
    ro = (C.c_float * 3)()
    rays = _capi.L4DRays()
    rays.rays_o, rays.rays_d = C.addressof(ro), C.addressof(ro)
    rays.n_rays, rays.n_steps = n_rays, 16
    buf = (C.c_float * 8)()
    p = C.addressof(buf)
    grads = _capi.L4DMasterGrads()
    return lib.l4d_render_backward_frames(C.byref(cfg), p, C.byref(tab), C.byref(rays), p, 1 << 40, p, p, None, None,
                                          C.byref(grads), p, 1 << 40, None, None)


@pytest.mark.parametrize("n_frames,rpf,phase,n_rays,what", [
    (0, 8, 0, 8, b"n_frames"),
    (_capi.MAX_FRAMES + 1, 8, 0, 8, b"n_frames"),
    (2, 0, 0, 8, b"rays_per_frame"),
    (2, 8, 8, 8, b"first_ray_phase"),
    (2, 8, 1, 16, b"does not cover"),
    (3, 5, 0, 16, b"does not cover"),
])
def test_bad_frame_tables_are_rejected(n_frames, rpf, phase, n_rays, what):
    """Every malformed table is an argument error of both entry points, before anything touches the device."""
    lib = _capi.load_library()
    cfg = _capi.make_config(FieldConfig())
    tab = _table(n_frames, rpf, phase)
    assert _call_forward(lib, cfg, tab, n_rays) == _capi.EINVAL
    assert what in lib.l4d_last_error()
    assert _call_backward(lib, cfg, tab, n_rays) == _capi.EINVAL
    assert what in lib.l4d_last_error()


def test_null_frame_table_is_rejected():
    lib = _capi.load_library()
    cfg = _capi.make_config(FieldConfig())
    ro = (C.c_float * 3)()
    rays = _capi.L4DRays()
    rays.rays_o, rays.rays_d, rays.n_rays, rays.n_steps = C.addressof(ro), C.addressof(ro), 1, 16
    out = (C.c_float * 8)()
    p = C.addressof(out)
    assert lib.l4d_render_forward_frames(C.byref(cfg), p, None, C.byref(rays), p, p, p, None, None, None, 0, None) == -1


@pytest.mark.parametrize("L", [8, 16])
def test_per_frame_bytes(L):
    """One frame is the single-frame layout; every further frame adds the same per-frame block."""
    lib = _capi.load_library()
    cfg = _capi.make_config(FieldConfig(n_levels_hash=L))
    for n, S in ((1, 2), (1024, 768), (4096, 768)):
        one = lib.l4d_saved_bytes(C.byref(cfg), n, S)
        sizes = [lib.l4d_saved_bytes_frames(C.byref(cfg), n, S, k) for k in range(1, _capi.MAX_FRAMES + 1)]
        assert sizes[0] == one
        steps = {b - a for a, b in zip(sizes, sizes[1:])}
        assert len(steps) == 1 and steps.pop() > 0
    gw = [lib.l4d_grad_work_bytes_frames(C.byref(cfg), k) for k in range(1, _capi.MAX_FRAMES + 1)]
    assert gw[0] == lib.l4d_grad_work_bytes(C.byref(cfg))
    steps = {b - a for a, b in zip(gw, gw[1:])}
    assert len(steps) == 1 and steps.pop() > 0
    for k in (0, _capi.MAX_FRAMES + 1):
        assert lib.l4d_saved_bytes_frames(C.byref(cfg), 16, 768, k) == 0
        assert lib.l4d_grad_work_bytes_frames(C.byref(cfg), k) == 0


def _fields(f):
    q = lambda t: (t.tau, t.slice_lo, t.slice_hi, t.w_lo, t.w_hi, t.single, tuple(t.basis))
    return (f.time, f.frame_idx, f.has_fwd, f.has_bwd, q(f.cur), q(f.fwd), q(f.bwd), tuple(f.flow_basis))


def test_row_frames_are_make_frame_of_each_row():
    cfg = FieldConfig(num_frames=6)
    times = [0.0, 1.0, 0.5, 0.5, 0.2, 0.37, 0.8] * 3
    groups = row_frame_groups(cfg, times)
    assert [b0 for b0, _ in groups] == [0, _capi.MAX_FRAMES]
    rows = [f for _, fs in groups for f in fs]
    assert len(rows) == len(times)
    for t, f in zip(times, rows):
        assert _fields(f) == _fields(_capi.make_frame_struct(make_frame(t, cfg.num_frames, cfg.time_resolution)))
    tab = _capi.make_frame_table(groups[0][1], 100)
    assert (tab.n_frames, tab.rays_per_frame, tab.first_ray_phase) == (_capi.MAX_FRAMES, 100, 0)
    assert _fields(tab.frames[3]) == _fields(rows[3])


def test_render_frames_grouping_and_bad_time_shapes():
    """The engine's view of a render call's `time`: one frame for one value or equal rows, per-row tables otherwise,
    ValueError for any other shape (no device needed: nothing is launched)."""
    m = LiDAR4D(num_frames=6, n_levels_hash=4, log2_hashmap_size=12)
    eng = m._engine
    B, N = 3, 5
    shape = (B, N, 3)
    for t in (0.4, torch.tensor([0.4]), torch.tensor([[0.4]]), torch.full((B, 1), 0.4), torch.full((B,), 0.4)):
        g = eng.render_frames(t, shape)
        assert len(g) == 1 and g[0][1] is None and isinstance(g[0][2], _capi.L4DFrame)
    g = eng.render_frames(torch.tensor([[0.0], [0.4], [1.0]]), shape)
    assert len(g) == 1 and g[0][:2] == (0, B) and g[0][2].n_frames == B and g[0][2].rays_per_frame == N
    big = torch.linspace(0, 1, _capi.MAX_FRAMES + 3).view(-1, 1)
    g = eng.render_frames(big, (big.shape[0], N, 3))
    assert [(b0, k) for b0, k, _ in g] == [(0, _capi.MAX_FRAMES), (_capi.MAX_FRAMES, 3)]
    for bad, rs in ((torch.zeros(2, 1), shape), (torch.zeros(B, 2), shape), (torch.zeros(1, B), shape),
                    (torch.zeros(B, 1, 1), shape), (torch.zeros(0), shape), (torch.zeros(B, 1), (B * N, 3))):
        with pytest.raises(ValueError):
            eng.render_frames(bad, rs)
