"""The reference's point-cloud metric (``utils/metrics.py``: ``fscore`` :13-27 and ``PointsMeter`` :229-279) on the GPU.

The reference copies both range images to the host, unprojects them with numpy, copies the clouds back and reduces
with torch, for every frame.  Here the whole chain stays on the device: ``pano_to_lidar`` (l4d_pano_unproject), the
chamfer op (l4d_chamfer_forward) and one reduction launch (l4d_point_metrics).  Unlike ``utils/metrics.py`` this
module needs neither lpips nor skimage.
"""
import os

import torch

from . import _capi
from .chamfer import chamfer_3DDist
from .convert import pano_to_lidar


def point_metrics(pred_pano, gt_pano, lidar_K, threshold=0.05):
    """Chamfer distance and F-score between the clouds of two range images, as PointsMeter.update computes them:
    pred_pano, gt_pano [H, W] CUDA -> (cd, fscore, precision, recall), 0-dim float32 device tensors, with
    dist1 / dist2 the SQUARED nearest-neighbour distances of the predicted / ground-truth points,
    cd = mean(dist1) + mean(dist2), precision = mean(dist1 < threshold), recall = mean(dist2 < threshold) and
    fscore = 2 p r / (p + r), or 0 where that is NaN.  The threshold applies to squared distances, as in the reference.
    Raises ValueError when either image has no point (the chamfer op is undefined on an empty cloud)."""
    pred = pano_to_lidar(pred_pano, lidar_K)
    gt = pano_to_lidar(gt_pano, lidar_K)
    with torch.no_grad():
        dist1, dist2, _, _ = chamfer_3DDist()(pred[None], gt[None])
    lib = _capi.load_library()
    dev = pred.device
    out = torch.empty(5, device=dev)
    with torch.cuda.device(dev):
        rc = lib.l4d_point_metrics(dist1.data_ptr(), dist1.shape[1], dist2.data_ptr(), dist2.shape[1], float(threshold),
                                   out.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
    _capi.check(lib, rc, "l4d_point_metrics")
    return out[0], out[1], out[2], out[3]


class PointsMeter:
    """Drop-in for utils/metrics.py:229-279.  update(preds, truths) takes [B, H, W] range images (frame 0 is measured,
    as in the reference), divides them by `scale` on the device and keeps (CD, F-score) as device tensors; measure()
    reads all frames back at once and returns their mean, a float32 numpy array [CD, F-score]."""

    def __init__(self, scale, intrinsics):
        self.V = []
        self.N = 0
        self.scale = scale
        self.intrinsics = intrinsics

    def clear(self):
        self.V = []
        self.N = 0

    def update(self, preds, truths):
        preds = preds.detach() / self.scale
        truths = truths.detach() / self.scale
        cd, fscore, _, _ = point_metrics(preds[0], truths[0], self.intrinsics, threshold=0.05)   # monoSDF threshold
        self.V.append(torch.stack([cd, fscore]))
        self.N += 1

    def measure(self):
        assert self.N == len(self.V)
        return torch.stack(self.V).cpu().numpy().mean(0)

    def write(self, writer, global_step, prefix="", suffix=""):
        writer.add_scalar(os.path.join(prefix, "CD"), self.measure()[0], global_step)

    def report(self):
        return f"Point_error (CD, F-score) = {self.measure()}"
