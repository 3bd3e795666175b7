"""Test infrastructure: the two third-party modules the reference's utils/metrics.py imports at module level and that
this project does not depend on, so that the UNMODIFIED utils/metrics.py imports and runs:
  skimage.metrics.structural_similarity  oracle/image_metrics_oracle.py's restatement ([skimage-ext], powf constants);
  lpips.LPIPS                            a stand-in whose call returns the fixed SENTINEL (AlexNet weights are a download).
`install()` puts both in sys.modules; `reference_metrics()` also installs the reference stubs (chamfer wrapper etc.)
and imports utils.metrics from the reference checkout."""
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle import image_metrics_oracle as IO  # noqa: E402

SENTINEL = 0.125
calls = []          # (pred shape, gt shape, normalize) of every LPIPS call


class LPIPS(torch.nn.Module):
    def __init__(self, net="alex", **kw):
        super().__init__()
        self.net = net

    def forward(self, pred, gt, normalize=False):
        calls.append((tuple(pred.shape), tuple(gt.shape), normalize))
        return torch.tensor(SENTINEL)


def structural_similarity(im1, im2, *, data_range=None, **kw):
    if kw or data_range is None:
        raise NotImplementedError("only structural_similarity(im1, im2, data_range=R) is restated")
    return IO.structural_similarity(im1, im2, data_range=data_range)


def install():
    sk = types.ModuleType("skimage")
    skm = types.ModuleType("skimage.metrics")
    skm.structural_similarity = structural_similarity
    sk.metrics = skm
    sys.modules["skimage"], sys.modules["skimage.metrics"] = sk, skm
    lp = types.ModuleType("lpips")
    lp.LPIPS = LPIPS
    sys.modules["lpips"] = lp


def reference_metrics():
    """The reference's own utils/metrics.py (build container only: needs the reference checkout)."""
    from ref_stubs import install_reference_stubs
    install()
    install_reference_stubs()
    sys.dont_write_bytecode = True
    import utils.metrics as M
    return M
