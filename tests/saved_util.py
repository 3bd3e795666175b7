"""Training steps that keep the saved buffer the backward consumed, and its sigma-MLP features (test infrastructure)."""
import torch

import scatter_ref as SR
from lidar4d_b200.model import _RenderFn


def train_step(m, ro, rd, S, U, monkeypatch, t: float = 0.4, keep_flow_in: bool = False, prefill: dict = None):
    """Render + backward; returns (outputs, saved buffer).  keep_flow_in: also return a copy of the flow-MLP inputs
    [16, P] taken before the backward (tensor-core mode writes dL/d(flow-MLP input) over them).  prefill: parameter
    name -> values the gradients hold when the backward starts (otherwise they are zeroed)."""
    captured = {}
    orig = _RenderFn.backward
    N = ro.shape[0]

    def keep_saved(ctx, *g):
        captured["saved"] = ctx.saved             # the backward drops it when it is done
        if keep_flow_in:
            captured["flow_in"] = SR.decode_saved(m.cfg, ctx.saved, N, S)["flow_in"].clone()
        return orig(ctx, *g)
    monkeypatch.setattr(_RenderFn, "backward", staticmethod(keep_saved))
    m.zero_grad(set_to_none=False)
    if prefill:
        for k, p in m.named_parameters():
            if k in prefill:
                if p.grad is None:
                    p.grad = torch.zeros_like(p)
                p.grad.copy_(prefill[k])
    m._jitter_calls = 0
    dev = next(iter(U.values())).device
    out = m.render(ro[None].to(dev), rd[None].to(dev), torch.tensor([[t]]), num_steps=S, perturb=True)
    outs = {"depth_lidar": out["depth_lidar"][0], "image_lidar": out["image_lidar"][0],
            "weights_sum_lidar": out["weights_sum_lidar"], "weights": out["weights"]}
    torch.autograd.backward([outs[k] for k in U], [U[k] for k in U])
    torch.cuda.synchronize()
    monkeypatch.undo()
    out = {k: v.detach() for k, v in out.items()}
    if keep_flow_in:
        out["flow_in"] = captured["flow_in"]
    return out, captured["saved"]


def saved_features(cfg, saved: torch.Tensor, N: int, S: int, mode: str) -> torch.Tensor:
    """The sigma MLP's input features [P, K] the dense kernels read, float32 (exact): fp32 [K][P] (fp32 mode) or fp16
    hi + lo tiles [ray][tile][hi|lo][K/8][128][8] (tensor-core mode; hi + lo is exact in float32)."""
    L = SR.saved_layout(cfg, N, S)
    K, P = cfg.sigma_in_dim, N * S
    if mode == "fp32":
        return saved[L["feat"]:L["feat"] + 4 * K * P].view(torch.float32).view(K, P).t()
    nt, xc = (S + 127) // 128, (K + 7) // 8
    t = saved[L["feat"]:L["feat"] + N * nt * xc * 4096].view(torch.float16).view(N, nt, 2, xc, 128, 8)
    x = t[:, :, 0].float() + t[:, :, 1].float()
    x = x.permute(0, 1, 3, 2, 4).reshape(N, nt * 128, xc * 8)
    return x[:, :S, :K].reshape(P, K)
