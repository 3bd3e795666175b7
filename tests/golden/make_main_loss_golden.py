"""Generate tests/golden/main_loss_ref.npz: the main LiDAR loss that the UNMODIFIED reference Trainer.train_step computes
(model/runner.py:193-220, with its chamfer term) and eval_step's loss (:409-421), with the training loss's gradients
with respect to the render outputs depth_lidar and image_lidar, on the CPU.

Run in the build container only (needs /root/reference, read-only):
    python tests/golden/make_main_loss_golden.py

The model is a stub whose `render` returns seeded leaf tensors (tests/main_loss_ref.py: train_inputs / eval_inputs), so
the stored gradients are d loss / d (depth_lidar, image_lidar).  The criteria are built as main_lidar4d.py:183-195
builds them; the chamfer function is the reference kernel's rule restated in oracle/chamfer_oracle.py; flow, URF and
patch-gradient losses are off.  For eval with refinement the stub U-Net returns a seeded float16 map that holds values
of exactly 0.5 and NaN.  Inputs are not stored: the tests rebuild them from the seeds and check their SHA-256."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.dont_write_bytecode = True

import main_loss_ref as R  # noqa: E402
from oracle import chamfer_oracle  # noqa: E402


class _OracleChamfer(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b):
        d1, d2, i1, i2 = chamfer_oracle.chamfer_forward(a.detach().numpy(), b.detach().numpy())
        ctx.save_for_backward(a, b)
        ctx.idx = (i1, i2)
        return torch.from_numpy(d1), torch.from_numpy(d2), torch.from_numpy(i1), torch.from_numpy(i2)

    @staticmethod
    def backward(ctx, g1, g2, *_):
        a, b = ctx.saved_tensors
        ga, gb = chamfer_oracle.chamfer_backward(a.detach().numpy(), b.detach().numpy(), g1.numpy(), g2.numpy(), *ctx.idx)
        return torch.from_numpy(ga), torch.from_numpy(gb)


def oracle_cham_fn(a, b):
    return _OracleChamfer.apply(a.contiguous(), b.contiguous())


class StubModel(torch.nn.Module):
    """render returns the leaves it holds; unet returns the held U-Net output."""

    def __init__(self):
        super().__init__()
        self.p = torch.nn.Parameter(torch.zeros(1))
        self.out, self.unet_out = None, None

    def render(self, *a, **k):
        return self.out

    def unet(self, x):
        return self.unet_out


def main():
    import ref_stubs
    from trainer_mirror import default_opt
    runner = ref_stubs.import_reference_runner()
    out = {"names": []}
    for name, kind, combo, scale, size, patch, seed, extra in R.case_list():
        opt = default_opt(depth_loss=combo[0], raydrop_loss=combo[1], intensity_loss=combo[2], scale=scale, flow_loss=False,
                          urf_loss=False, grad_loss=False, fp16=False, patch_size_lidar=list(patch) if patch else 1)
        crit = {"depth": R.criterion(combo[0], scale), "raydrop": R.criterion(combo[1], scale),
                "intensity": R.criterion(combo[2], scale), "grad": R.criterion("l1", scale)}
        model = StubModel()
        tr = runner.Trainer("t", opt, model, criterion=crit, device=torch.device("cpu"), workspace=None, mute=True,
                            fp16=False, use_checkpoint="scratch")
        tr.cham_fn = oracle_cham_fn
        if kind == "train":
            depth, image, gt, rays_d = R.train_inputs(size, seed, ties=extra == "ties")
            d = torch.from_numpy(depth).requires_grad_(True)
            im = torch.from_numpy(image).requires_grad_(True)
            model.out = {"depth_lidar": d, "image_lidar": im}
            n = size
            batch = {"rays_o_lidar": torch.zeros(1, n, 3), "rays_d_lidar": torch.from_numpy(rays_d),
                     "time": torch.zeros(1, 1), "images_lidar": torch.from_numpy(gt)}
            loss = tr.train_step(batch)[4]
            loss.backward()
            out[f"{name}/loss"] = np.float32(loss.item())
            out[f"{name}/g_depth"] = d.grad.numpy()
            out[f"{name}/g_image"] = im.grad.numpy()
            out[f"{name}/sha"] = R.sha(depth, image, gt, rays_d)
        else:
            B, H, W = size
            depth, image, gt, r = R.eval_inputs(B, H, W, seed, torch.float16 if extra else None, nan=extra == "unet_nan")
            model.out = {"depth_lidar": torch.from_numpy(depth).reshape(B, H * W),
                         "image_lidar": torch.from_numpy(image).reshape(B, H * W, 2)}
            tr.use_refine = extra is not None
            if tr.use_refine:
                model.unet_out = r.reshape(1, B, H, W)      # unet([1, 3B, H, W]).squeeze(0) is [B, H, W]
            batch = {"rays_o_lidar": torch.zeros(1, B * H * W, 3), "rays_d_lidar": torch.zeros(1, B * H * W, 3),
                     "time": torch.zeros(1, 1), "images_lidar": torch.from_numpy(gt), "H_lidar": H, "W_lidar": W}
            with torch.no_grad():
                loss = tr.eval_step(batch)[-1]
            out[f"{name}/loss"] = np.float32(loss.item())
            out[f"{name}/sha"] = R.sha(depth, image, gt, *(() if r is None else (r.float().numpy(),)))
        out["names"].append(name)
        print(f"{name:36s} loss {float(out[f'{name}/loss']):.9e}")
    out["names"] = np.array(out["names"])
    p = os.path.join(HERE, "main_loss_ref.npz")
    np.savez_compressed(p, **out)
    print("wrote", p, os.path.getsize(p), "bytes")


if __name__ == "__main__":
    torch.set_num_threads(8)
    main()
