"""GPU parity at the BENCHMARKED configuration (BASELINE.json configs[1]): default tables (2^19 static, 2^15/2^13/2^13
x 8 time slices, 2^18 flow), n_levels_hash 8 and 16 (sigma_in_dim 120 / 176), S = 768, jitter on, 12-16 rays.

Two anchors:
  * tests/golden/ref_full_*.npz - the UNMODIFIED reference modules on the tcnn shim (tests/golden/make_golden.py);
  * the oracle, run here on the host cores with the same seeded parameters, for EVERY gradient tensor in full.
Both CUDA modes (wgmma tensor-core kernels with fp16 working weights; fp32-FMA kernels) and both pipelines are held to:

  forward   z_vals / hash indices bit-exact; depth, image, weights <= 1e-4 (rel-to-max, fp32) against the reference
            fixture and the oracle - on white-noise tables AND on band-limited ("trained-like") tables;
  backward  the network is piecewise linear (ReLU x 7 layers, bilinear texels, the w > 1e-4 mask): a sample whose
            pre-activation lies within fp32 rounding of zero gets a different - equally correct - sub-gradient in two
            fp32 implementations, and that sample's whole contribution to the sparse tables changes.  The oracle itself
            counts them (12,288 samples, L=16: 6 flow-MLP pre-activations within 1e-7 of zero, 57 within 1e-6).  Hence
              - band-limited tables (forward noise ~1e-5): every gradient tensor in full:  >= 99.9 % of the entries
                within 1e-4 of max, ||diff|| / ||ref|| <= 1e-3 (flow net: 5e-3), and for the big tables the set of
                touched entries must be IDENTICAL (a wrong index cannot hide) and norm / projection within 1e-3;
              - white-noise tables (one ulp of a warped coordinate = a 1e-3 feature change at 32769 cells; forward noise
                5e-5, tens of ReLU flips): touched-entry sets identical, norms within 1e-2, ||diff||/||ref|| <= 5e-2.
            Measured evidence for this reading: profiles/r02_parity_diag_*.txt (the same kernels agree with the oracle to
            1e-5 on every tensor once the tables are band-limited).  The small-configuration tests
            (tests/test_gpu_parity.py) keep the strict 1e-4-everywhere bar with a ReLU-margin guard.
Also: GradScaler-sized upstream gradients (x65536, runner.py:506-508) and an outer fp16 autocast (runner.py:497)."""
import os

import numpy as np
import pytest
import torch

from oracle import lidar4d_oracle as O
from parity_util import rel_err, grad_errors, full_oracle, cuda_model_from_oracle

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 1e-4
FULL_CASES = ["ref_full_L16_smooth", "ref_full_L8_smooth", "ref_full_L16_interior", "ref_full_L16_first", "ref_full_L8_last"]
FLOW = ("flow_net.grid_enc.params", "flow_net.mlp.0.weight", "flow_net.mlp.2.weight", "flow_net.mlp.4.weight")
MODES = [("tc", "split"), ("fp32", "split"), ("tc", "fused")]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


_cache = {}


def case(name):
    """(fixture, oracle with gradients of the fixture's loss) - computed once per module on the host cores."""
    if name not in _cache:
        fx = np.load(os.path.join(GOLD, name + ".npz"))
        orc = full_oracle(int(fx["levels"]), int(fx["seed"]), bool(int(fx["smooth"])))
        S = int(fx["num_steps"])
        ref = orc.render(torch.from_numpy(fx["rays_o"]), torch.from_numpy(fx["rays_d"]), float(fx["time"]), num_steps=S,
                         perturb=bool(fx["perturb"]), seed=int(fx["seed"]))
        ((ref["depth_lidar"] * torch.from_numpy(fx["g_depth"])).sum() +
         (ref["image_lidar"] * torch.from_numpy(fx["g_image"])).sum()).backward()
        _cache.clear()                 # one full-size oracle resident at a time
        _cache[name] = (fx, orc, {k: v.detach() for k, v in ref.items()}, orc.ref_named_grads())
    return _cache[name]


def cuda_run(fx, orc, dev, mode, pipeline, scale=1.0, autocast=False):
    m = cuda_model_from_oracle(orc).set_mlp_fp16(mode == "tc")
    m.pipeline = pipeline
    m.jitter_seed = int(fx["seed"])
    ro, rd = torch.from_numpy(fx["rays_o"])[None].to(dev), torch.from_numpy(fx["rays_d"])[None].to(dev)
    gd, gi = torch.from_numpy(fx["g_depth"]).to(dev), torch.from_numpy(fx["g_image"]).to(dev)
    with torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
        out = m.render(ro, rd, torch.tensor([[float(fx["time"])]]), num_steps=int(fx["num_steps"]),
                       perturb=bool(fx["perturb"]))
        loss = (out["depth_lidar"][0] * gd).sum() + (out["image_lidar"][0] * gi).sum()
    (loss * scale).backward()
    torch.cuda.synchronize()
    return m, out, {k: p.grad for k, p in m.named_parameters()}


@pytest.mark.parametrize("S", [768, 767, 129, 2, 1000])
def test_z_grid_matches_cuda_linspace(dev, S):
    """The kernel's / oracle's restatement of torch.linspace(0,1,S) on CUDA (renderer.py:69; the reference renders on
    the GPU) is bit-exact - the full-size goldens were generated on this grid."""
    assert np.array_equal(torch.linspace(0.0, 1.0, S, device=dev).cpu().numpy(), O.sample_lin(S))


def test_hash_indices_bit_exact_L16(dev):
    from lidar4d_b200 import LiDAR4D
    fx = np.load(os.path.join(GOLD, "hash_indices.npz"))
    m = LiDAR4D(n_levels_hash=16).to(dev)
    for gid, name in [(0, "static3d_L16"), (1, "dyn2d_xy_L16"), (3, "dyn2d_yz_L16")]:
        x = torch.from_numpy(fx[name + ":x"]).to(dev)
        for l in range(16):
            idx, w = m.hash_indices(gid, l, x)
            assert np.array_equal(idx.cpu().numpy().view(np.uint32), fx[f"{name}:idx{l}"]), (name, l)
            assert np.array_equal(w.cpu().numpy(), fx[f"{name}:w{l}"]), (name, l)


@pytest.mark.parametrize("mode,pipeline", MODES)
@pytest.mark.parametrize("name", FULL_CASES)
def test_full_size_vs_reference_golden_and_oracle(dev, name, mode, pipeline):
    fx, orc, ref, og = case(name)
    smooth = bool(int(fx["smooth"]))
    m, out, got = cuda_run(fx, orc, dev, mode, pipeline)
    # ---- forward: the reference's own numbers, then the oracle's ----
    assert np.array_equal(out["z_vals"].cpu().numpy(), ref["z_vals"].numpy())
    assert rel_err(out["depth_lidar"], fx["ref_depth_lidar"]) < TOL
    assert rel_err(out["image_lidar"], fx["ref_image_lidar"]) < TOL
    assert rel_err(out["weights"], fx["ref_weights"]) < TOL
    for k in ("depth_lidar", "image_lidar", "weights_sum_lidar", "weights"):
        assert rel_err(out[k], ref[k]) < TOL, k
    # the attribute mask (renderer.py:110) is decided identically (the fixtures keep >= 5e-7 from the threshold)
    assert torch.equal(out["weights"].cpu() > 1e-4, torch.from_numpy(fx["ref_weights"]) > 1e-4)
    # ---- gradients: see the module docstring for the criteria ----
    frac_tol, l2_tol, l2_flow, norm_tol = (1e-3, 1e-3, 5e-3, 1e-3) if smooth else (1.0, 5e-2, 1e-1, 1e-2)
    report, bad = {}, {}
    for k, g_ref in og.items():
        if not g_ref.numel():
            continue
        if got.get(k) is None:
            assert float(g_ref.abs().max()) == 0.0, k
            continue
        e_max, e_l2, e_frac = grad_errors(got[k], g_ref)
        report[k] = (e_max, e_l2, e_frac)
        ok = e_l2 <= (l2_flow if k in FLOW else l2_tol) and e_frac <= (1.0 if k in FLOW else frac_tol)
        n_ref, n_got = float(g_ref.double().norm()), float(got[k].double().norm())
        ok = ok and abs(n_got - n_ref) <= norm_tol * n_ref + 1e-30
        if g_ref.numel() > 70000:          # the touched-entry set is index arithmetic: exact, whatever the values do
            a, b = got[k].cpu().reshape(-1), g_ref.reshape(-1)
            diff = (a != 0) != (b != 0)
            if bool(diff.any()):           # only entries whose value is a rounding-level cancellation may differ in being exactly 0
                lim = 1e-6 * float(b.abs().max())
                same = float(a[diff].abs().max()) <= lim and float(b[diff].abs().max()) <= lim and int(diff.sum()) <= 1e-4 * int((b != 0).sum()) + 2
                if not same:
                    report[k] += (f"support: {int(diff.sum())} entries differ, max |cuda| {float(a[diff].abs().max()):.2e} "
                                  f"|oracle| {float(b[diff].abs().max()):.2e} of {float(b.abs().max()):.2e}",)
                ok = ok and same
        if not ok:
            bad[k] = report[k]
    assert not bad, f"failing (max-rel, l2-rel, outlier fraction): {bad}"
    # ---- gradients against the reference fixture (full small tensors, sampled entries + projection of the tables) ----
    for k in [k[5:] for k in fx.files if k.startswith("grad:")]:
        if fx["grad:" + k].size:
            e_max, e_l2, e_frac = grad_errors(got[k], fx["grad:" + k])
            assert e_l2 <= (l2_flow if k in FLOW else l2_tol) and e_frac <= (1.0 if k in FLOW else max(frac_tol, 1.5 / fx["grad:" + k].size)), (k, e_max, e_l2, e_frac)
    for k in [k[8:] for k in fx.files if k.startswith("gradidx:")]:
        g = got[k].reshape(-1)
        n_ref = float(fx["gradnorm:" + k])
        idx = torch.from_numpy(fx["gradidx:" + k].astype(np.int64)).to(dev)
        refv = fx["gradval:" + k]
        gv = g[idx].cpu().numpy()
        assert np.all(gv[refv == 0] == 0), k                  # untouched entries stay untouched
        assert np.mean(np.abs(gv - refv) > TOL * np.abs(refv).max()) <= (2e-3 if smooth else 1.0), k
        proj = torch.cos(torch.arange(g.numel(), device=dev, dtype=torch.float64) * 0.6180339887498949 + 0.25)
        p2 = float(fx["gradproj2:" + k])
        assert abs(float(g.double() @ proj) - p2) <= (norm_tol if k not in FLOW else 10 * norm_tol) * (abs(p2) + n_ref), k


@pytest.mark.parametrize("mode", ["tc", "fp32"])
def test_loss_scaled_upstream_gradients(dev, mode):
    """GradScaler multiplies the loss by 65536 (torch default init_scale; runner.py:102,506-508).  The forward - hence
    every ReLU / mask decision - does not depend on the upstream gradient, so the backward must be exactly linear in
    it: grads(65536 g) / 65536 == grads(g) to fp32 rounding (no overflow of the fp16 delta tiles of the tensor-core
    backward, no flush of small entries), and likewise for a tiny scale."""
    fx, orc, ref, og = case("ref_full_L16_smooth")
    _, _, base = cuda_run(fx, orc, dev, mode, "split")
    for scale in (65536.0, 2.0 ** -20):
        _, _, got = cuda_run(fx, orc, dev, mode, "split", scale=scale)
        for k, g in base.items():
            if g is None or not g.numel():
                continue
            assert torch.isfinite(got[k]).all(), k
            e_max, e_l2, _ = grad_errors(got[k] / scale, g)
            assert e_max < 2e-5 and e_l2 < 2e-5, (k, scale, e_max, e_l2)       # atomics re-order fp32 sums run to run
    # and against the oracle, in aggregate
    for k in ("sigma_net.params", "hash_encoder.hash_static.params", "planes_encoder.planes.3.0"):
        e_max, e_l2, e_frac = grad_errors(got[k] / scale, og[k])
        assert e_l2 < 1e-3 and e_frac < 1e-3, (k, e_max, e_l2, e_frac)


def test_outer_autocast_and_grad_scaler_step(dev):
    """Trainer.train_step runs the model under torch.cuda.amp.autocast and steps through a GradScaler
    (runner.py:497,506-511): outputs stay fp32 and equal to the plain call, scaled grads unscale to the oracle's."""
    fx, orc, ref, og = case("ref_full_L16_smooth")
    m, out, got = cuda_run(fx, orc, dev, "tc", "split", autocast=True)
    assert out["depth_lidar"].dtype == torch.float32 and out["image_lidar"].dtype == torch.float32
    for k in ("depth_lidar", "image_lidar"):
        assert rel_err(out[k], ref[k]) < TOL, k
    for k in ("sigma_net.params", "intensity_net.params", "hash_encoder.hash_static.params", "planes_encoder.planes.0.3"):
        e_max, e_l2, e_frac = grad_errors(got[k], og[k])
        assert e_l2 < 1e-3 and e_frac < 1e-3, (k, e_max, e_l2, e_frac)
    # one real scaler step
    m.zero_grad(set_to_none=True)
    opt = torch.optim.Adam(m.get_params(1e-2), betas=(0.9, 0.99), eps=1e-15)
    scaler = torch.amp.GradScaler("cuda")
    before = m.sigma_net.params.detach().clone()
    ro, rd = torch.from_numpy(fx["rays_o"])[None].to(dev), torch.from_numpy(fx["rays_d"])[None].to(dev)
    with torch.autocast("cuda", dtype=torch.float16):
        o = m.render(ro, rd, torch.tensor([[float(fx["time"])]]), num_steps=768, perturb=True)
        loss = (o["depth_lidar"] - 0.3).abs().mean() + ((o["image_lidar"] - 0.5) ** 2).mean()
    scaler.scale(loss).backward()
    scaler.step(opt)
    scaler.update()
    assert scaler.get_scale() == 65536.0                       # no inf/nan was found in the scaled gradients
    assert not torch.equal(before, m.sigma_net.params.detach())
