"""Chamfer / nearest-neighbour distance op (SURVEY.md 8(f) rank 1).

Drop-in for the reference's ``utils/chamfer3D/dist_chamfer_3D.py``: same class names, same call
(``chamfer_3DDist()(xyz1[B,N,3], xyz2[B,M,3]) -> dist1[B,N], dist2[B,M], idx1[B,N], idx2[B,M]``), same
autograd contract (``chamfer_3DFunction``, dist_chamfer_3D.py:31-73), backed by ``l4d_chamfer_forward`` /
``l4d_chamfer_backward`` of the C-ABI library.  Differences that SURVEY.md 5 lists as reference defects:
the kernels run on torch's *current* stream (the reference launches on the default stream,
chamfer3D.cu:141-142) and return codes are checked (dist_chamfer_3D.py:54 ignores them).
"""

import torch
from torch import nn
from torch.autograd import Function

from . import _capi


def _check_cloud(x, name):
    if x.dim() != 3 or x.shape[-1] != 3:
        raise ValueError(f"{name}: expected [B, N, 3], got {tuple(x.shape)}")     # dist_chamfer_3D.py:35-38
    if not x.is_cuda:
        raise RuntimeError("chamfer_3DDist needs CUDA tensors (no CPU fallback)")
    if x.shape[1] == 0:
        raise ValueError(f"{name}: empty point cloud")


class chamfer_3DFunction(Function):
    @staticmethod
    def forward(ctx, xyz1, xyz2):
        _check_cloud(xyz1, "xyz1")
        _check_cloud(xyz2, "xyz2")
        if xyz1.shape[0] != xyz2.shape[0]:
            raise ValueError("batch sizes differ")
        lib = _capi.load_library()
        ctx.in_dtypes = (xyz1.dtype, xyz2.dtype)
        xyz1 = xyz1.contiguous().float()
        xyz2 = xyz2.contiguous().float()
        b, n, _ = xyz1.shape
        m = xyz2.shape[1]
        dev = xyz1.device
        dist1 = torch.empty(b, n, device=dev)
        dist2 = torch.empty(b, m, device=dev)
        idx1 = torch.empty(b, n, dtype=torch.int32, device=dev)
        idx2 = torch.empty(b, m, dtype=torch.int32, device=dev)
        nwork = lib.l4d_chamfer_work_bytes(b, n, m)
        work = torch.empty(nwork, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            rc = lib.l4d_chamfer_forward(xyz1.data_ptr(), xyz2.data_ptr(), b, n, m, dist1.data_ptr(), dist2.data_ptr(),
                                         idx1.data_ptr(), idx2.data_ptr(), work.data_ptr(), nwork,
                                         torch.cuda.current_stream(dev).cuda_stream)
        _capi.check(lib, rc, "l4d_chamfer_forward")
        ctx.save_for_backward(xyz1, xyz2, idx1, idx2)
        ctx.mark_non_differentiable(idx1, idx2)
        return dist1, dist2, idx1, idx2

    @staticmethod
    def backward(ctx, graddist1, graddist2, gradidx1, gradidx2):
        xyz1, xyz2, idx1, idx2 = ctx.saved_tensors
        lib = _capi.load_library()
        b, n, _ = xyz1.shape
        m = xyz2.shape[1]
        dev = xyz1.device
        g1 = torch.zeros(b, n, device=dev) if graddist1 is None else graddist1.contiguous().float()
        g2 = torch.zeros(b, m, device=dev) if graddist2 is None else graddist2.contiguous().float()
        gx1 = torch.zeros_like(xyz1)
        gx2 = torch.zeros_like(xyz2)
        with torch.cuda.device(dev):
            rc = lib.l4d_chamfer_backward(xyz1.data_ptr(), xyz2.data_ptr(), b, n, m, g1.data_ptr(), g2.data_ptr(),
                                          idx1.data_ptr(), idx2.data_ptr(), gx1.data_ptr(), gx2.data_ptr(),
                                          torch.cuda.current_stream(dev).cuda_stream)
        _capi.check(lib, rc, "l4d_chamfer_backward")
        return gx1.to(ctx.in_dtypes[0]), gx2.to(ctx.in_dtypes[1])      # gradients in the inputs' dtype (fp16 clouds under autocast)


class chamfer_3DDist(nn.Module):
    def forward(self, input1, input2):
        return chamfer_3DFunction.apply(input1.contiguous(), input2.contiguous())


# ----------------------------------------------------------------------------------------------------------------------
# the same op through a uniform-grid index: for clouds that are searched many times (the flow loss's frame clouds)
# ----------------------------------------------------------------------------------------------------------------------
def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


class PointGrid:
    """A cloud ``points[n, 3]`` (or [1, n, 3]) on the GPU with its nearest-neighbour index (l4d_nn_grid_build): built once,
    queried by ``chamfer_3DGrid`` and by the flow loss.  The index holds its own copy of the coordinates; ``points`` is the
    float32 cloud in its original order.  b = 1 only."""

    def __init__(self, points):
        if not isinstance(points, torch.Tensor) or not points.is_cuda:
            raise RuntimeError("PointGrid needs a CUDA tensor (no CPU fallback)")
        if points.dim() == 3 and points.shape[0] != 1:
            raise ValueError("PointGrid indexes one cloud (b = 1)")
        if points.dim() not in (2, 3) or points.shape[-1] != 3:
            raise ValueError(f"PointGrid: expected [n, 3] or [1, n, 3], got {tuple(points.shape)}")
        pts = points.detach().reshape(-1, 3).contiguous().float()
        if pts.shape[0] == 0:
            raise ValueError("PointGrid: empty point cloud")
        lib = _capi.load_library()
        self.points = pts
        self.n = pts.shape[0]
        self.nbytes = lib.l4d_nn_grid_bytes(self.n)
        self.grid = torch.empty(self.nbytes, dtype=torch.uint8, device=pts.device)
        nwork = lib.l4d_nn_grid_work_bytes(self.n)
        work = torch.empty(nwork, dtype=torch.uint8, device=pts.device)
        with torch.cuda.device(pts.device):
            rc = lib.l4d_nn_grid_build(pts.data_ptr(), self.n, self.grid.data_ptr(), self.nbytes, work.data_ptr(), nwork,
                                       _stream(pts))
        _capi.check(lib, rc, "l4d_nn_grid_build")

    def query(self, q, sum_parts=None, want_dist=True):
        """q [nq, 3] float32 contiguous -> (dist [nq] or None, idx [nq] int32): the nearest point of this cloud."""
        lib = _capi.load_library()
        nq = q.shape[0]
        dist = torch.empty(nq, device=q.device) if want_dist else None
        idx = torch.empty(nq, dtype=torch.int32, device=q.device)
        with torch.cuda.device(q.device):
            rc = lib.l4d_nn_grid_query(self.grid.data_ptr(), self.nbytes, self.n, q.data_ptr(), nq,
                                       dist.data_ptr() if want_dist else None, idx.data_ptr(),
                                       sum_parts.data_ptr() if sum_parts is not None else None, _stream(q))
        _capi.check(lib, rc, "l4d_nn_grid_query")
        return dist, idx


class _Chamfer3DGridFunction(Function):
    @staticmethod
    def forward(ctx, xyz1, xyz2, grid1, grid2):
        ctx.in_dtypes = (xyz1.dtype, xyz2.dtype)
        xyz1 = xyz1.contiguous().float()
        xyz2 = xyz2.contiguous().float()
        grid1 = grid1 if grid1 is not None else PointGrid(xyz1)
        grid2 = grid2 if grid2 is not None else PointGrid(xyz2)
        dist1, idx1 = grid2.query(xyz1[0])
        dist2, idx2 = grid1.query(xyz2[0])
        dist1, dist2, idx1, idx2 = dist1[None], dist2[None], idx1[None], idx2[None]
        ctx.save_for_backward(xyz1, xyz2, idx1, idx2)
        ctx.mark_non_differentiable(idx1, idx2)
        return dist1, dist2, idx1, idx2

    @staticmethod
    def backward(ctx, graddist1, graddist2, gradidx1, gradidx2):
        return chamfer_3DFunction.backward(ctx, graddist1, graddist2, gradidx1, gradidx2) + (None, None)


class chamfer_3DGrid(nn.Module):
    """``chamfer_3DDist`` with the search done through a uniform grid: same call, same four outputs, bit for bit, same
    backward (l4d_chamfer_backward on the returned indices).  Each argument is a [1, N, 3] tensor, indexed on the fly, or a
    prebuilt ``PointGrid`` (no gradient flows to a PointGrid)."""

    def forward(self, input1, input2):
        grids, clouds = [], []
        for name, x in (("xyz1", input1), ("xyz2", input2)):
            if isinstance(x, PointGrid):
                grids.append(x)
                clouds.append(x.points[None])
            else:
                _check_cloud(x, name)
                if x.shape[0] != 1:
                    raise ValueError("chamfer_3DGrid takes one cloud per side (b = 1); chamfer_3DDist handles batches")
                grids.append(None)
                clouds.append(x.contiguous())
        if clouds[0].device != clouds[1].device:
            raise ValueError("the two clouds are on different devices")
        return _Chamfer3DGridFunction.apply(clouds[0], clouds[1], grids[0], grids[1])
