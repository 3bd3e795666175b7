"""CPU: the C-ABI library loads and exports every symbol the header declares,
argument checking works without a GPU, and the host-side mirror of the
reference interface (module names, state_dict, frame logic) is right."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from lidar4d_b200 import _capi
from lidar4d_b200.geometry import FieldConfig, make_frame, lagrange_basis, make_time_query
from lidar4d_b200.rays import lidar_rays, synthetic_sweep

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, "include", "lidar4d_b200.h")).read()
    return sorted(set(re.findall(r"\b(l4d_[a-z_0-9]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = _capi.load_library()
    names = header_functions()
    assert len(names) >= 13
    assert set(names) == set(_capi.EXPORTS)
    for n in names:
        assert hasattr(lib, n), n
    assert lib.l4d_abi_version() == _capi.ABI_VERSION


def test_struct_sizes_match_header_layout():
    assert C.sizeof(_capi.L4DGrid) == 16 + 4 * (16 * 3 + 17)
    assert C.sizeof(_capi.L4DTimeQuery) == 40
    assert C.sizeof(_capi.L4DFrame) == 16 + 3 * 40 + 16
    assert C.sizeof(_capi.L4DRays) == 48


def test_argument_errors_return_codes():
    """Bad configurations and null arguments give error codes, and the saved buffer of a launch is sized for the
    smallest valid one (1 ray, 2 samples: one-sample rays are themselves an argument error)."""
    lib = _capi.load_library()
    cfg = _capi.make_config(FieldConfig())
    assert lib.l4d_staged_bytes(C.byref(cfg)) > 0
    assert lib.l4d_grad_work_bytes(C.byref(cfg)) > 0
    assert lib.l4d_saved_bytes(C.byref(cfg), 16, 768) > 16 * 768 * 4 * 139
    bad = _capi.make_config(FieldConfig())
    bad.sigma_in_dim = 7
    assert lib.l4d_staged_bytes(C.byref(bad)) == 0
    assert b"sigma_in_dim" in lib.l4d_last_error()
    # the scalar per-entry accumulators / contracted tables of the dynamic hash are addressed as aligned quads of entries
    odd = _capi.make_config(FieldConfig())
    odd.hash_dynamic[1].offset[3] += 4
    assert lib.l4d_saved_bytes(C.byref(odd), 16, 768) == 0
    assert b"multiples of 8" in lib.l4d_last_error()
    # the saved buffer of a launch carries the contracted dynamic tables (3 queries x entries x 4 B) and time-plane rows
    c16 = FieldConfig(n_levels_hash=16)
    n_dyn = sum(int(c16.dynamic_grid(p).offset[-1]) for p in range(3))
    small, big = lib.l4d_saved_bytes(C.byref(_capi.make_config(c16)), 1, 2), 3 * n_dyn * 4
    assert small > big + 3 * 3 * 8 * 4 * sum(c16.min_resolution * m for m in c16.plane_scales)
    fr = _capi.make_frame_struct(make_frame(0.3, 51, 8))
    rays = _capi.L4DRays()
    rc = lib.l4d_render_forward(C.byref(cfg), None, C.byref(fr), C.byref(rays), None, None, None, None, None, None, 0, None)
    assert rc == -1 and lib.l4d_last_error()
    rc = lib.l4d_hash_indices(C.byref(cfg), 9, 0, None, 0, None, None, None)
    assert rc == -1


@pytest.mark.parametrize("S", [0, 1, 8193])
def test_sample_count_out_of_range_is_rejected(S):
    """The reference renders nothing at num_steps = 1 (its deltas z[1:] - z[:-1] are empty, renderer.py:98-104), and the
    kernels hold at most L4D_MAX_TILES x 128 samples per ray: both ends are argument errors, before any launch, with
    every other argument valid (the check is the first thing that fails)."""
    from lidar4d_b200 import LiDAR4D
    lib = _capi.load_library()
    cfg = _capi.make_config(FieldConfig())
    assert lib.l4d_saved_bytes(C.byref(cfg), 16, S) == 0
    assert b"n_steps out of range [2, 8192]" in lib.l4d_last_error()
    for ok in (2, 8192):
        assert lib.l4d_saved_bytes(C.byref(cfg), 16, ok) > 0
    fr = _capi.make_frame_struct(make_frame(0.3, 51, 8))
    fake = 256                                    # never dereferenced: the argument check returns first
    rays = _capi.L4DRays()
    rays.rays_o = rays.rays_d = fake
    rays.n_rays, rays.n_steps = 4, S
    lib.l4d_last_error()
    rc = lib.l4d_render_forward(C.byref(cfg), fake, C.byref(fr), C.byref(rays), fake, fake, fake, None, None, None, 0, None)
    assert rc == -1 and b"n_steps out of range" in lib.l4d_last_error()
    rc = lib.l4d_render_backward(C.byref(cfg), fake, C.byref(fr), C.byref(rays), fake, 1 << 40, fake, fake, None, None,
                                 C.byref(_capi.L4DMasterGrads()), fake, 1 << 40, None)
    assert rc == -1 and b"n_steps out of range" in lib.l4d_last_error()
    m = LiDAR4D(min_resolution=8, base_resolution=16, max_resolution=64, n_levels_hash=2, log2_hashmap_size=8,
                hash_size_dynamic=(6, 6, 6), flow_base_resolution=4, flow_max_resolution=32, flow_log2_hashmap_size=8)
    ro = torch.zeros(1, 4, 3)
    with pytest.raises(ValueError, match="num_steps"):
        m.render(ro, ro + 1, torch.tensor([[0.1]]), num_steps=S)


def test_product_has_no_cpu_path():
    from lidar4d_b200 import LiDAR4D
    m = LiDAR4D(min_resolution=8, base_resolution=16, max_resolution=64, n_levels_hash=2, log2_hashmap_size=8,
                hash_size_dynamic=(6, 6, 6), flow_base_resolution=4, flow_max_resolution=32, flow_log2_hashmap_size=8)
    ro = torch.zeros(1, 4, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.render(ro, ro + 1, torch.tensor([[0.1]]), num_steps=8)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.flow(torch.zeros(3, 3), torch.tensor([[0.1]]))
    import lidar4d_b200.model as mod
    src = open(mod.__file__).read()
    assert "oracle" not in src.replace("oracle's", "")      # the product never imports the oracle


def test_state_dict_surface_matches_reference():
    """SURVEY.md 8(b): keys and shapes of LiDAR4D.state_dict() (unet.* excluded: out of scope)."""
    from lidar4d_b200 import LiDAR4D
    m = LiDAR4D()
    sd = m.state_dict()
    expect = {"aabb": (6,), "hash_encoder.hash_static.params": (16777216,), "view_encoder.params": (0,),
              "flow_net.grid_enc.params": (14942208,), "flow_net.mlp.0.weight": (64, 16),
              "flow_net.mlp.2.weight": (64, 64), "flow_net.mlp.4.weight": (6, 64), "sigma_net.params": (9216,),
              "intensity_net.params": (11264,), "raydrop_net.params": (11264,)}
    for s, r in enumerate([32, 64, 128, 256]):
        for ci, shp in enumerate([(r, r), (r, r), (8, r), (r, r), (8, r), (8, r)]):
            expect[f"planes_encoder.planes.{s}.{ci}"] = (1, 8) + shp
    for p, n in enumerate([1048576, 262144, 262144]):
        for t in range(8):
            expect[f"hash_encoder.hash_dynamic.{p}.hash_t.{t}.params"] = (n,)
    assert {k: tuple(v.shape) for k, v in sd.items()} == expect
    groups = m.get_params(1e-2)
    assert [g["lr"] for g in groups] == [1e-2, 1e-2, 1e-2, 1e-3, 1e-3, 1e-3, 1e-3]
    n_opt = sum(p.numel() for g in m.get_params(1e-2) for p in g["params"])
    assert n_opt == sum(v.numel() for k, v in sd.items() if k != "aabb")
    assert m.out_lidar_dim == 2 and m.num_frames == 51 and m.bound == 1
    assert m.planes_encoder.n_output_dims + m.hash_encoder.n_output_dims == 120
    assert m.view_encoder.n_output_dims + 15 == 87


def test_frame_logic_matches_reference_for_whole_sequences():
    """int(float32(t)*(F-1)) equals the frame index for every frame of the 51- and
    64-frame sequences (lidar4d.py:143; kitti360_dataset.py:125 t=k/(F-1))."""
    for F in (51, 64, 6, 2):
        for k in range(F):
            t = np.float32(k / (F - 1))
            fr = make_frame(t, F, 8)
            assert fr.frame_idx == k
            assert fr.has_fwd == (k < F - 1) and fr.has_bwd == (k > 0)
            if fr.has_fwd:
                assert fr.fwd.tau == np.float32((k + 1) / F)       # divides by F, not F-1 (lidar4d.py:159)
            if fr.has_bwd:
                assert fr.bwd.tau == np.float32((k - 1) / F)


def test_time_query_and_lagrange_basis():
    for t in np.linspace(0, 1, 29, dtype=np.float32):
        q = make_time_query(t, 8)
        assert 0 <= q.slice_lo <= q.slice_hi <= 7 and q.slice_hi - q.slice_lo <= 1
        if not q.single:
            assert abs(float(q.w_lo) + float(q.w_hi) - 1.0) < 1e-6
        b = lagrange_basis(t)
        assert abs(float(b.sum()) - 1.0) < 1e-5
    for i in range(4):                        # interpolation property at the nodes
        b = lagrange_basis(np.float32(i / 3))
        assert abs(float(b[i]) - 1.0) < 1e-5 and abs(float(np.delete(b, i)).__abs__().max() if False else float(np.abs(np.delete(b, i)).max())) < 1e-5
    assert make_time_query(np.float32(0.0), 8).single and make_time_query(np.float32(1.0), 8).single


def test_ray_model_matches_reference_formula():
    """data/base_dataset.py:82-97 evaluated with torch for a few pixels."""
    H, W = 6, 16
    pose = np.eye(4, dtype=np.float32)
    pose[:3, :3] = np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1]], np.float32)
    pose[:3, 3] = [0.2, 0.1, -0.3]
    ro, rd = lidar_rays(pose, H, W, 2.0, 26.9)
    i, j = torch.meshgrid(torch.linspace(0, W - 1, W), torch.linspace(0, H - 1, H), indexing="ij")
    i, j = i.t().reshape(-1), j.t().reshape(-1)
    beta = -(i - W / 2) / W * 2 * np.pi
    alpha = (2.0 - j / H * 26.9) / 180 * np.pi
    d = torch.stack([torch.cos(alpha) * torch.cos(beta), torch.cos(alpha) * torch.sin(beta), torch.sin(alpha)], -1)
    d = d @ torch.from_numpy(pose[:3, :3]).t()
    assert np.allclose(rd, d.numpy(), atol=1e-6)
    assert np.allclose(ro, pose[:3, 3][None].repeat(H * W, 0))
    ro2, rd2, t = synthetic_sweep(0)
    assert ro2.shape == (65536, 3) and t == 0.0 and np.allclose(np.linalg.norm(rd2, axis=1), 1, atol=1e-5)
