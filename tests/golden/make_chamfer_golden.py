"""Generate tests/golden/chamfer_ref.npz: outputs of the reference's own chamfer kernels (chamfer3D.cu NmDistanceKernel and
NmDistanceGradKernel, built by oracle/build_ref.py into oracle/_ref/) for the cases of tests/test_chamfer.py.

    python tests/golden/make_chamfer_golden.py OUT.npz        # needs a GPU and the built oracle/_ref extension

Per case and direction a fixed, seeded sample of at most 2048 query points is stored: distance, index and the gradient
of sum(d1 * g1) + sum(d2 * g2) with respect to those points (g1, g2 drawn from torch.Generator().manual_seed(seed))."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import build_ref  # noqa: E402
from test_chamfer import REF_CASES, _clouds, golden_sample  # noqa: E402


def main(out_path):
    ext = build_ref.load()
    dev = torch.device("cuda:0")
    fx = {}
    for b, n, m, seed, dup in REF_CASES:
        key = f"{b}_{n}_{m}_{seed}_{int(dup)}"
        x1, x2 = _clouds(b, n, m, seed, dup)
        t1, t2 = torch.from_numpy(x1).to(dev), torch.from_numpy(x2).to(dev)
        r1, r2 = torch.zeros(b, n, device=dev), torch.zeros(b, m, device=dev)
        j1, j2 = torch.zeros(b, n, dtype=torch.int32, device=dev), torch.zeros(b, m, dtype=torch.int32, device=dev)
        assert ext.forward(t1, t2, r1, r2, j1, j2) == 1
        g = torch.Generator().manual_seed(seed)
        g1, g2 = torch.randn(b, n, generator=g).to(dev), torch.randn(b, m, generator=g).to(dev)
        gx1, gx2 = torch.zeros_like(t1), torch.zeros_like(t2)
        assert ext.backward(t1, t2, gx1, gx2, g1, g2, j1, j2) == 1
        torch.cuda.synchronize()
        for side, (d, j, gx) in enumerate(((r1, j1, gx1), (r2, j2, gx2))):
            sel = golden_sample(d.numel(), seed + side)
            fx[f"{key}_sel{side}"] = sel
            fx[f"{key}_d{side}"] = d.reshape(-1).cpu().numpy()[sel]
            fx[f"{key}_i{side}"] = j.reshape(-1).cpu().numpy()[sel]
            fx[f"{key}_g{side}"] = gx.reshape(-1, 3).cpu().numpy()[sel]
    np.savez_compressed(out_path, **fx)
    print(f"wrote {out_path} ({os.path.getsize(out_path)} bytes, {len(REF_CASES)} cases)")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "chamfer_ref.npz"))
