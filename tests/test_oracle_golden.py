"""CPU: the oracle against the committed golden vectors that were produced by the
UNMODIFIED reference modules on the tcnn shim (tests/golden/make_golden.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import lidar4d_oracle as O
from lidar4d_b200.geometry import FieldConfig
from parity_util import small_config, rel_err, full_oracle

GOLD = os.path.join(os.path.dirname(__file__), "golden")
CASES = ["ref_small_interior", "ref_small_first", "ref_small_last", "ref_small_active"]


def load(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


FULL_CASES = ["ref_full_L16_interior", "ref_full_L16_smooth", "ref_full_L8_smooth", "ref_full_L16_first", "ref_full_L8_last"]


def oracle_case(fx):
    if "levels" in fx.files:
        orc = full_oracle(int(fx["levels"]), int(fx["seed"]), bool(int(fx["smooth"])))
    else:
        import ast
        extra = ast.literal_eval(str(fx["extra"])) if "extra" in fx.files else {}      # renderer options of the case
        orc = O.build_seeded(small_config(**extra), int(fx["seed"]), flow_last_std=0.02)
    chk = sum(float(v.double().sum()) for v in orc.ref_state_dict().values())
    assert abs(chk - float(fx["param_checksum"])) < 1e-6 * abs(float(fx["param_checksum"])), "seeded parameters drifted"
    return orc


@pytest.mark.parametrize("name", CASES + FULL_CASES)
def test_oracle_reproduces_reference_outputs(name):
    fx = load(name)
    orc = oracle_case(fx)
    S = int(fx["num_steps"])
    # small cases: the reference's CPU z grid (renderer.py:69); full-size cases were generated on the CUDA grid
    lin = O.sample_lin(S) if "levels" in fx.files else torch.linspace(0.0, 1.0, S).numpy()
    out = orc.render(torch.from_numpy(fx["rays_o"]), torch.from_numpy(fx["rays_d"]), float(fx["time"]),
                     num_steps=S, perturb=bool(fx["perturb"]), seed=int(fx["seed"]), lin=lin)
    assert rel_err(out["depth_lidar"], fx["ref_depth_lidar"]) < 1e-5
    assert rel_err(out["image_lidar"], fx["ref_image_lidar"]) < 1e-5
    assert rel_err(out["weights_sum_lidar"], fx["ref_weights_sum_lidar"]) < 1e-5
    assert rel_err(out["weights"], fx["ref_weights"]) < 1e-5
    loss = (out["depth_lidar"] * torch.from_numpy(fx["g_depth"])).sum() + \
           (out["image_lidar"] * torch.from_numpy(fx["g_image"])).sum()
    loss.backward()
    grads = orc.ref_named_grads()
    rng = np.random.default_rng(1234)
    for k, g in grads.items():      # same iteration order as the generator: named_parameters of the reference
        pass
    keys = [k[len("gradnorm:"):] for k in fx.files if k.startswith("gradnorm:")]
    for k in keys:
        gv = grads[k].double().numpy().reshape(-1)
        proj = rng.standard_normal(gv.shape[0])
        n_ref = float(fx["gradnorm:" + k])
        assert abs(np.linalg.norm(gv) - n_ref) <= 1e-4 * max(n_ref, 1e-12) + 1e-12, k
        p_ref = float(fx["gradproj:" + k])
        assert abs(gv @ proj - p_ref) <= 2e-4 * max(n_ref * np.sqrt(gv.shape[0]) * 0.05, abs(p_ref)) + 1e-12, k
        if ("grad:" + k) in fx.files:
            assert rel_err(grads[k], fx["grad:" + k]) < 1e-4, k
        if ("gradidx:" + k) in fx.files:          # full-size tables: sampled entries (largest / touched / untouched)
            idx = fx["gradidx:" + k].astype(np.int64)
            ref = fx["gradval:" + k]
            assert np.abs(gv[idx] - ref).max() <= 1e-5 * np.abs(ref).max() + 1e-30, k
            assert np.all(gv[idx][ref == 0] == 0), k
            p2 = float(fx["gradproj2:" + k])
            assert abs(gv @ O.projection_vector(gv.shape[0]) - p2) <= 1e-4 * (abs(p2) + n_ref), k


@pytest.mark.parametrize("name", CASES)
def test_oracle_flow_matches_reference(name):
    fx = load(name)
    orc = oracle_case(fx)
    fl = orc.flow(torch.from_numpy(fx["flow_pts"]), float(fx["time"]))
    assert rel_err(fl["forward"], fx["flow_forward"]) < 1e-5
    assert rel_err(fl["backward"], fx["flow_backward"]) < 1e-5


def test_oracle_hash_indices_known_answers():
    fx = load("hash_indices")
    cfg, cfg16 = FieldConfig(), FieldConfig(n_levels_hash=16)
    grids = {"static3d": cfg.static_grid(), "dyn2d_xy": cfg.dynamic_grid(0), "dyn2d_xz": cfg.dynamic_grid(1),
             "flow3d": cfg.flow_grid(), "static3d_L16": cfg16.static_grid(), "dyn2d_xy_L16": cfg16.dynamic_grid(0),
             "dyn2d_yz_L16": cfg16.dynamic_grid(2)}
    assert int(cfg16.static_grid().resolution[-1]) == 32769      # the L=16 rounding cliff (SURVEY.md 7)
    for name, geo in grids.items():
        # geometry itself is data: it must be reproduced bit-exactly on this machine
        assert np.array_equal(geo.resolution, fx[name + ":resolution"])
        assert np.array_equal(geo.entries, fx[name + ":entries"])
        assert np.array_equal(geo.scale, fx[name + ":scale"])
        x = torch.from_numpy(fx[name + ":x"])
        for l in range(geo.n_levels):
            idx, w = O.hash_indices(x, geo, l)
            assert np.array_equal(idx.numpy().astype(np.uint32), fx[f"{name}:idx{l}"])
            assert np.array_equal(w.numpy(), fx[f"{name}:w{l}"])


def test_planes_restatement_matches_grid_sample_directly():
    """SURVEY.md 8(c) golden (4): the oracle's plane path is F.grid_sample itself;
    check the product rule / concat order against a by-hand evaluation."""
    orc = O.build_seeded(small_config(), 2)
    xt = torch.rand(50, 4)
    st = orc.planes(xt, "static")
    s0 = orc.cfg.min_resolution
    p01 = orc.p("planes_encoder.planes.0.0")[0]          # [8,H(y),W(x)]
    # nearest check at texel centres: sample exactly on a texel -> value equals the texel product
    ix, iy, iz = 3, 5, 2
    pt = torch.tensor([[ix / (s0 - 1), iy / (s0 - 1), iz / (s0 - 1), 0.3]])
    v = orc.planes(pt, "static")[0, :8]
    expect = p01[:, iy, ix] * orc.p("planes_encoder.planes.0.1")[0][:, iz, ix] * orc.p("planes_encoder.planes.0.3")[0][:, iz, iy]
    assert torch.allclose(v, expect, rtol=1e-5, atol=1e-6)
    assert st.shape == (50, 32)


def test_z_grid_restatement_matches_cuda_linspace_dump():
    """tests/golden/cuda_linspace.npz = torch.linspace(0, 1, S, device="cuda") dumped on a GPU (scripts/diag_fullsize.py):
    the oracle's (and, through tests/test_hostsim_parity.py, the kernels') z grid is bit-exact with the grid the reference
    gets on its GPU path (renderer.py:77)."""
    fx = load("cuda_linspace")
    for S in fx.files:
        assert np.array_equal(O.sample_lin(int(S)), fx[S]), S
