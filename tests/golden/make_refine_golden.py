"""Generate tests/golden/refine_ref.npz: the reference's own, unmodified Trainer.refine (model/runner.py:818-922) run on
the CPU, for tests/test_refine_oracle.py (draw_boxes and the in-file refine mirror against it, bit for bit).

Run where the reference checkout exists (CPU only, a few minutes):
    python tests/golden/make_refine_golden.py [OUT.npz]

Stand-ins (tests/ref_stubs.py, tests/refine_cases.py): a Trainer built without its constructor carrying only what refine
reads (ema None, opt.fp16 False, log, ckpt_path, name, epoch, bce_fn); a model whose render() returns the seeded frames
of refine_cases.frames() and whose `unet` is the reference's model/unet.py UNet(in_channels=3, out_channels=1) with parity_util.fill_state_dict
weights; a loader of refine_cases.F frames of refine_cases.H x W, once with float16 and once with float32 images.
``Tensor.cuda`` is the identity during the run (the reference moves the packed inputs with ``.cuda()``).  All 1,000
hard-coded iterations run, with np.random seeded with NP_SEED and torch with TORCH_SEED before the call.

Recorded, per case f16 / f32:
  <case>_inputs [F, 3, H, W], <case>_gt [F, 1, H, W]      the packed inputs and targets (from the final cat)
  <case>_draws                                            every np.random.randint result in call order (int64)
  <case>_boxes_count [1000], <case>_boxes [sum, 4]        each iteration's boxes (y0, x0, h, w), parsed from the draws
  <case>_losses [1000] float32                            every iteration's BCE loss
  <case>_rng_keys [624] uint32, <case>_rng_pos            np.random's final MT19937 state
  <case>_ckpt_keys, <case>_ckpt_epoch, <case>_ckpt_name   the checkpoint torch.save wrote
  <case>_unet_sha256                                      refine_cases.unet_digest of the final U-Net state_dict"""
import os
import sys
import tempfile
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
ROOT = os.path.dirname(TESTS)
sys.path.insert(0, ROOT)
sys.path.insert(0, TESTS)

import ref_stubs  # noqa: E402
import refine_cases as RC  # noqa: E402
from parity_util import fill_state_dict  # noqa: E402


class _LossRecorder(torch.nn.Module):
    def __init__(self, fn):
        super().__init__()
        self.fn, self.losses = fn, []

    def forward(self, a, b):
        loss = self.fn(a, b)
        self.losses.append(loss.item())
        return loss


def run_case(runner, unet_cls, dtype):
    fr = RC.frames()
    unet = fill_state_dict(unet_cls(in_channels=3, out_channels=1))     # model/lidar4d.py:119
    model = RC.StubModel(fr, unet)
    ws = tempfile.mkdtemp()
    tr = runner.Trainer.__new__(runner.Trainer)
    tr.ema, tr.model, tr.ckpt_path, tr.name, tr.epoch, tr.log_ptr = None, model, ws, "lidar4d", 3, None
    import argparse
    tr.opt = argparse.Namespace(fp16=False)
    lines = []
    tr.log = lambda *a, **k: lines.append(" ".join(str(x) for x in a))
    tr.bce_fn = _LossRecorder(torch.nn.BCELoss())

    draws = []
    orig_randint = np.random.randint

    def randint(*a, **k):
        v = orig_randint(*a, **k)
        draws.append(int(v))
        return v

    packed = {}
    orig_cat = torch.cat

    def cat(ts, dim=0, **k):           # the reference's final cat of the input / gt lists (runner.py:862-863)
        out = orig_cat(ts, dim, **k)
        if isinstance(ts, list) and len(ts) == len(fr) and out.dim() == 4:
            packed["inputs" if out.shape[1] == 3 else "gt"] = out.detach().clone().float()
        return out

    np.random.seed(RC.NP_SEED)
    torch.manual_seed(RC.TORCH_SEED)
    cuda = torch.Tensor.cuda
    np.random.randint, torch.Tensor.cuda, torch.cat = randint, lambda self, *a, **k: self, cat
    try:
        tr.refine(RC.Loader(fr, dtype))
    finally:
        np.random.randint, torch.Tensor.cuda, torch.cat = orig_randint, cuda, orig_cat
    state = np.random.get_state()
    ck_name = f"lidar4d_ep{3:04d}_refine.pth"
    ck = torch.load(os.path.join(ws, ck_name), weights_only=False)
    unet_state = {k[len("unet."):]: v for k, v in ck["model"].items() if k.startswith("unet.")}
    # parse the draws into box lists: randint(32) -> k, then k x (h, w, y0, x0)
    counts, boxes, p = [], [], 0
    while p < len(draws):
        k = draws[p]
        p += 1
        counts.append(k)
        for _ in range(k):
            h, w, y0, x0 = draws[p:p + 4]
            boxes.append((y0, x0, h, w))
            p += 4
    assert len(counts) == 1000 and len(tr.bce_fn.losses) == 1000
    return {"inputs": packed["inputs"].numpy(), "gt": packed["gt"].numpy(), "draws": np.array(draws, np.int64),
            "boxes_count": np.array(counts, np.int64), "boxes": np.array(boxes, np.int64).reshape(-1, 4),
            "losses": np.array(tr.bce_fn.losses, np.float32), "rng_keys": np.asarray(state[1], np.uint32),
            "rng_pos": np.array(state[2]), "ckpt_keys": np.array(sorted(ck.keys())), "ckpt_epoch": np.array(ck["epoch"]),
            "ckpt_name": np.array(ck_name), "unet_sha256": np.array(RC.unet_digest(unet_state)),
            "log": np.array(lines)}


def main(out_path):
    warnings.simplefilter("ignore")
    runner = ref_stubs.import_reference_runner()
    from model.unet import UNet
    torch.set_num_threads(RC.CPU_THREADS)      # a fixed thread count: the CPU kernels split their work the same way
    fx = {"numpy_version": np.array(np.__version__), "torch_version": np.array(torch.__version__)}
    for case, dtype in (("f16", torch.float16), ("f32", torch.float32)):
        for k, v in run_case(runner, UNet, dtype).items():
            fx[f"{case}_{k}"] = v
        print(case, "losses", fx[f"{case}_losses"][[0, 1, 500, 999]], flush=True)
    np.savez_compressed(out_path, **fx)
    print(f"wrote {out_path} ({os.path.getsize(out_path)} bytes)")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 and not sys.argv[1].startswith("-") else os.path.join(HERE, "refine_ref.npz"))
