"""Generate tests/golden/train_losses.npz: the losses that the UNMODIFIED reference Trainer.train_step adds after the flow
loss (model/runner.py:255-369: URF's line-of-sight loss and the patch branch), with their gradients with respect to the
render outputs depth_lidar and weights, on the reference model-on-shim on the CPU.

Run in the build container only (needs /root/reference, read-only):
    python tests/golden/make_loss_golden.py

The batch is 16 patches of 2 x 8 rays of the 8 x 32 synthetic sweep, in get_lidar_rays' patch order
(data/base_dataset.py:47-72), with a ground-truth image whose depth is constant over runs of columns, so that the
|Δgt| < 0.01 mask of the depth-gradient loss is on for part of the differences (a little noise keeps those differences
nonzero, so the cosine criterion sees more than zero vectors).  To isolate these losses, the main-loss
criteria are passed in as zero criteria and the chamfer function is replaced by one returning zero distances (both are
constructor arguments / attributes of the Trainer; no reference code is edited), and the flow loss is off.  The render
outputs are captured from outside, by wrapping the model's `render` with `retain_grad`; the gradient stored for `weights`
is therefore the whole one, including the path through depth_lidar = sum(weights * z_vals)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.dont_write_bytecode = True

import make_golden as MG  # noqa: E402
from oracle import lidar4d_oracle as O  # noqa: E402
from lidar4d_b200.rays import lidar_rays  # noqa: E402
import loss_ref  # noqa: E402

SEED, S, H, W, PX, PY, N_PATCH = 31, 48, 8, 32, 2, 8, 16
GLOBAL_STEP, ITERS = 1500, 30000


def patch_batch(seed=5, frame=2, num_frames=6):
    """rays / gt of N_PATCH random 2 x 8 patches: pixel (ix + i, (iy + j) % W), ix < H - PX (base_dataset.py:47-72)."""
    g = np.random.default_rng(seed)
    pose = np.eye(4, dtype=np.float32)
    pose[:3, 3] = [-0.25 + 0.5 * frame / (num_frames - 1), 0.0, 0.0]
    ro, rd = lidar_rays(pose, H, W)
    depth = 0.05 + 0.6 * g.random((H, 1)) + np.cumsum((g.random((H, W)) > 0.6) * g.normal(0, 2e-2, (H, W)), axis=1)
    depth = depth + g.normal(0, 2e-5, (H, W))
    img = np.stack([(g.random((H, W)) > 0.15), g.random((H, W)) * 0.5, depth], -1).astype(np.float32).reshape(H * W, 3)
    ix, iy = g.integers(0, H - PX, N_PATCH), g.integers(0, W, N_PATCH)
    pi, pj = np.meshgrid(np.arange(PX), np.arange(PY), indexing="ij")
    rows = (ix[:, None] + pi.reshape(1, -1)).reshape(-1)
    cols = ((iy[:, None] + pj.reshape(1, -1)) % W).reshape(-1)
    inds = rows * W + cols
    t = torch.tensor([[frame / (num_frames - 1)]], dtype=torch.float32)
    return {"rays_o_lidar": torch.from_numpy(ro[inds])[None], "rays_d_lidar": torch.from_numpy(rd[inds])[None],
            "time": t, "images_lidar": torch.from_numpy(img[inds])[None]}, inds


def zero_criterion(a, b):
    return a * 0.0


def main():
    import ref_stubs
    from trainer_mirror import default_opt
    runner = ref_stubs.import_reference_runner()
    orc = MG.oracle_for(MG.SMALL, SEED)
    batch, inds = patch_batch()
    N = batch["rays_o_lidar"].shape[1]
    u = torch.from_numpy(O.jitter_uniform(SEED, np.arange(N), S))
    out = {"seed": SEED, "num_steps": S, "global_step": GLOBAL_STEP, "iters": ITERS, "inds": inds,
           "rays_o": batch["rays_o_lidar"].numpy(), "rays_d": batch["rays_d_lidar"].numpy(),
           "time": batch["time"].numpy(), "images": batch["images_lidar"].numpy(), "names": np.array(list(loss_ref.OPTION_SETS))}
    for name, over in loss_ref.OPTION_SETS.items():
        ref = MG.build_reference(MG.SMALL)
        ref.load_state_dict(orc.ref_state_dict(), strict=False)
        kw = dict(num_frames=6, num_steps=S, near_lidar=0.0105, far_lidar=0.851, fp16=False, iters=ITERS,
                  patch_size_lidar=[PX, PY], flow_loss=False, depth_grad_loss="l1", alpha_grad=0.1, alpha_grad_norm=0.1,
                  alpha_spatial=0.1, alpha_tv=0.1)
        kw.update(over)
        opt = default_opt(**kw)
        crit = {"depth": zero_criterion, "raydrop": zero_criterion, "intensity": zero_criterion,
                "grad": loss_ref.grad_criterion(opt.depth_grad_loss, opt.scale)}
        tr = runner.Trainer("t", opt, ref, criterion=crit, device=torch.device("cpu"), workspace=None, mute=True, fp16=False,
                            use_checkpoint="scratch")
        tr.cham_fn = lambda a, b: (a[..., 0] * 0.0, b[..., 0] * 0.0, None, None)
        tr.global_step = GLOBAL_STEP
        cap = {}
        render = ref.render

        def capture(*a, **k):
            res = render(*a, **k)
            for key in ("depth_lidar", "weights"):
                res[key].retain_grad()
            cap.update(res)
            return res
        ref.render = capture
        orig_rand, orig_cuda = torch.rand, torch.Tensor.cuda

        def rand(*a, **k):       # the jitter of renderer.py:84 from the repo's counter-based stream, as make_golden.py
            shape = tuple(a[0]) if (len(a) == 1 and not isinstance(a[0], int)) else tuple(a)
            return u.clone() if shape == (N, S) else orig_rand(*a, **k)
        torch.rand = rand
        torch.Tensor.cuda = lambda self, *a, **k: self
        try:
            torch.manual_seed(3)
            loss = tr.train_step(batch)[4]
            loss.backward()
        finally:
            torch.rand, torch.Tensor.cuda = orig_rand, orig_cuda
        gw = cap["weights"].grad
        out[f"{name}/loss"] = np.float64(loss.item())
        out[f"{name}/g_depth"] = cap["depth_lidar"].grad.numpy()
        out[f"{name}/g_weights"] = np.zeros(cap["weights"].shape, np.float32) if gw is None else gw.numpy()
        if name == "defaults":
            out["depth_lidar"] = cap["depth_lidar"].detach().numpy()
            out["weights"] = cap["weights"].detach().numpy()
            out["z_vals"] = cap["z_vals"].detach().numpy()
        print(f"{name:9s} loss {loss.item():.6e}  |g_depth| {np.abs(out[f'{name}/g_depth']).max():.3e}  "
              f"|g_weights| {np.abs(out[f'{name}/g_weights']).max():.3e}")
    p = os.path.join(HERE, "train_losses.npz")
    np.savez_compressed(p, **out)
    print("wrote", p, os.path.getsize(p), "bytes")


if __name__ == "__main__":
    torch.set_num_threads(8)
    main()
