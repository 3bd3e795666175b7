"""The float64 compositing reference (tests/compositing_ref.py) against autograd, and the kernels' per-sample compositing
code compiled for the CPU against it.

  a. composite() == the float64 oracle (O.to_float64) on the oracle's own σ and attributes: weights, depth, image, Σw,
     dL/dσ (autograd through the oracle's render) and dL/d(attribute) inside the attribute mask (outside it the
     attributes are constants, not outputs of the heads), at S = 2, 129 and 8192, with and without
     active_sensor.
  b. tests/hostsim (l4d_alpha and the transmittance product of the kernels, compiled for the CPU) at S = 8192, on the σ it
     saved itself: the weights within 5e-6 of their max, each weight within its per-sample bound, the depth within the
     bound of its sum.  With α formed as 1 - expf(e), α of the far samples (4.5e-6 ... 7e-4) loses most of its bits to
     the cancellation: the weights are 5.3e-5 off, 380 times their bound; with α = -expm1f(e) they are 1.3e-6 off,
     within a quarter of the bound."""
import numpy as np
import pytest
import torch

import compositing_ref as CR
from oracle import lidar4d_oracle as O
from parity_util import small_config, rel_err, test_rays as _rays


def sample_dist(cfg, S):
    near, far = np.float32(cfg.near_lidar), np.float32(cfg.far_lidar)
    return float(np.float32((far - near) / np.float32(S)))


def upstream(N, S, seed):
    g = torch.Generator().manual_seed(seed)
    return {"depth_lidar": torch.randn(N, generator=g), "image_lidar": torch.randn(N, 2, generator=g),
            "weights_sum_lidar": torch.randn(N, generator=g) * 0.1, "weights": torch.randn(N, S, generator=g) * 0.01}


@pytest.mark.parametrize("active", [False, True], ids=["passive", "active"])
@pytest.mark.parametrize("S", [2, 129, 8192])
def test_reference_matches_float64_autograd(S, active):
    cfg = small_config(active_sensor=active)
    orc = O.build_seeded(cfg, 3, flow_last_std=0.02).to_float64()
    ro, rd = _rays(1, 2) if S == 8192 else _rays(3, 8)
    ro, rd = torch.from_numpy(ro), torch.from_numpy(rd)
    st = orc.render(ro, rd, 0.4, num_steps=S, perturb=True, seed=3, return_stages=True)
    st["sigma"].retain_grad()
    st["attr"].retain_grad()
    N = ro.shape[0]
    U = upstream(N, S, 5)
    torch.autograd.backward([st[k] for k in U], [U[k].double() for k in U])
    sig, attr = st["sigma"].detach(), st["attr"].detach().permute(2, 0, 1)
    ref = CR.composite(sig, attr, st["z_vals"].float(), sample_dist(cfg, S), cfg.density_scale, active, U)
    assert torch.equal(ref["mask"], st["mask"].view(N, S))
    errs = {"weights": rel_err(ref["weights"], st["weights"]), "depth": rel_err(ref["depth"], st["depth_lidar"]),
            "image": rel_err(ref["image"], st["image_lidar"]), "wsum": rel_err(ref["wsum"], st["weights_sum_lidar"]),
            "dsigma": rel_err(ref["dsigma"], st["sigma"].grad), "dattr": rel_err(ref["dattr"], st["attr"].grad.permute(2, 0, 1) * st["mask"].view(1, N, S))}
    # the float64 oracle forms α as 1 - exp(e): ~1e-16 absolute, 2e-11 relative at α = 5e-6 (S = 8192)
    bad = {k: v for k, v in errs.items() if not v < 1e-12}
    assert not bad, (S, active, errs)
    assert float(st["sigma"].grad.abs().max()) > 0 and float(ref["alpha"].min()) > 0
    print(f"[compositing-ref] S={S} active={active}: {', '.join(f'{k} {v:.1e}' for k, v in errs.items())}, "
          f"alpha {float(ref['alpha'].min()):.1e} ... {float(ref['alpha'].max()):.1e}")


def test_host_build_long_ray_against_reference():
    from hostsim_util import HostSim
    S = 8192
    cfg = small_config()
    orc = O.build_seeded(cfg, 3, flow_last_std=0.02)
    hs = HostSim(orc)
    ro, rd = _rays(1, 2)
    out = hs.render(ro, rd, 0.4, S, perturb=True, seed=3, train=True)
    sv = hs.saved_compositing_inputs()
    ref = CR.composite(sv["sigma"], sv["attr"], out["z_vals"], sample_dist(cfg, S), cfg.density_scale, cfg.active_sensor)
    e_w, e_d = rel_err(out["weights"], ref["weights"]), rel_err(out["depth"], ref["depth"])
    over = (out["weights"].double() - ref["weights"]).abs() / CR.weight_bound(ref)
    print(f"[compositing-ref] host build S={S}: weights {e_w:.2e}, depth {e_d:.2e}, worst {float(over.max()):.3f} of "
          f"the per-sample bound, alpha {float(ref['alpha'].min()):.1e} ... {float(ref['alpha'].max()):.1e}")
    assert e_w < 5e-6, e_w
    assert float(over.max()) <= 1.0
    z = out["z_vals"].double()
    assert float((out["depth"].double() - ref["depth"]).abs().max()) <= float(CR.sum_bound(ref, ref["weights"] * z).min())
