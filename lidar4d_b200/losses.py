"""Main LiDAR loss of the reference's train_step (model/runner.py:179-213) as ONE CUDA launch that returns the summed
loss and, in the same pass, its gradient with respect to the render outputs (SURVEY.md 8(f) #2).

    loss = lidar_main_loss(out["depth_lidar"], out["image_lidar"], gt, alpha_d=opt.alpha_d, alpha_r=opt.alpha_r,
                           alpha_i=opt.alpha_i, smooth=opt.smooth_factor)

equals  (alpha_d*L1(depth*m, gt_d*m) + alpha_r*MSE(raydrop, clamp(m, s, 1-s)) + alpha_i*MSE(intensity*m, gt_i*m)).sum()
with m = gt[..., 0] (ray-drop mask), gt_i = gt[..., 1], gt_d = gt[..., 2] - the default criteria of main_lidar4d.py:63-66.

The rest of train_step (model/runner.py:255-369), each a CUDA op whose backward is one launch that reads the incoming
gradient from device memory (a GradScaler-scaled backward needs no host sync):

    loss = loss + line_of_sight_loss(out["weights"], out["z_vals"], gt, eps)        # --urf_loss
    loss = loss + lidar_patch_loss(out["depth_lidar"], gt, **vars(opt))             # patch batches

and the ray-drop refinement loop's BCE (model/runner.py:901; the loop itself is lidar4d_b200/refine.py):

    loss = raydrop_bce_loss(unet(masked_input), gt_raydrop)

Inputs are taken in fp32 whatever the surrounding autocast (the reference's Sobel conv2d runs in fp16 under its fp16
autocast; here it runs in fp32).  No CPU path."""
from __future__ import annotations

import torch

from . import _capi


class _MainLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, depth, image, gt, alpha_d, alpha_r, alpha_i, smooth):
        if not depth.is_cuda:
            raise RuntimeError("lidar_main_loss runs on CUDA only (no CPU fallback)")
        lib = _capi.load_library()
        n = depth.numel()
        d = depth.detach().contiguous().view(-1).float()
        im = image.detach().contiguous().view(-1, 2).float()
        g = gt.detach().contiguous().view(-1, 3).float()
        if im.shape[0] != n or g.shape[0] != n:
            raise ValueError("depth [.., N], image [.., N, 2] and gt [.., N, 3] must describe the same rays")
        loss = torch.zeros((), device=d.device)
        gd = torch.empty_like(d)
        gi = torch.empty_like(im)
        with torch.cuda.device(d.device):
            rc = lib.l4d_lidar_loss(d.data_ptr(), im.data_ptr(), g.data_ptr(), n, float(alpha_d), float(alpha_r), float(alpha_i),
                                    float(smooth), loss.data_ptr(), gd.data_ptr(), gi.data_ptr(),
                                    torch.cuda.current_stream(d.device).cuda_stream)
        _capi.check(lib, rc, "l4d_lidar_loss")
        ctx.save_for_backward(gd, gi)
        ctx.shapes = (depth.shape, image.shape)
        return loss

    @staticmethod
    def backward(ctx, g):
        gd, gi = ctx.saved_tensors
        return (gd * g).view(ctx.shapes[0]), (gi * g).view(ctx.shapes[1]), None, None, None, None, None


def lidar_main_loss(depth, image, gt, alpha_d=1.0, alpha_r=0.01, alpha_i=0.1, smooth=0.2):
    return _MainLoss.apply(depth, image, gt, alpha_d, alpha_r, alpha_i, smooth)


GRAD_CRITERIA = {"l1": 0, "mse": 1, "huber": 2, "bce": 3, "cos": 4}      # L4D_GRAD_* (main_lidar4d.py:183-188)
_SOBEL, _GRAD, _GRAD_NORM, _SPATIAL, _TV = 1, 2, 4, 8, 16                # L4D_PATCH_*


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


class _PatchLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, depth, gt, px, py, scale, crit, flags, a_grad, a_gn, a_sp, a_tv):
        lib = _capi.load_library()
        d = depth.detach().contiguous().view(-1).float()
        g = gt.detach().contiguous().view(-1, 3).float()
        n = d.numel()
        loss = torch.empty((), device=d.device)
        gd = torch.empty_like(d)
        with torch.cuda.device(d.device):
            rc = lib.l4d_patch_loss(d.data_ptr(), g.data_ptr(), n, px, py, float(scale), crit, flags, float(a_grad),
                                    float(a_gn), float(a_sp), float(a_tv), loss.data_ptr(), gd.data_ptr(), _stream(d))
        _capi.check(lib, rc, "l4d_patch_loss")
        ctx.save_for_backward(gd)
        ctx.shape = depth.shape
        return loss

    @staticmethod
    def backward(ctx, gl):
        (gd,) = ctx.saved_tensors
        lib = _capi.load_library()
        gl = gl.detach().float().contiguous()
        out = torch.empty_like(gd)
        with torch.cuda.device(gd.device):
            rc = lib.l4d_patch_loss_backward(gd.data_ptr(), gl.data_ptr(), gd.numel(), out.data_ptr(), _stream(gd))
        _capi.check(lib, rc, "l4d_patch_loss_backward")
        return (out.view(ctx.shape),) + (None,) * 10


_BCE_DTYPES = {torch.float32: _capi.DTYPE_F32, torch.float16: _capi.DTYPE_F16, torch.bfloat16: _capi.DTYPE_BF16}


class _RaydropBCE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target):
        lib = _capi.load_library()
        p = pred.detach().contiguous()
        t = target.detach().contiguous().float()
        loss = torch.empty((), device=p.device)
        work = torch.empty(lib.l4d_bce_loss_work_bytes(), dtype=torch.uint8, device=p.device)
        with torch.cuda.device(p.device):
            rc = lib.l4d_bce_loss(p.data_ptr(), _BCE_DTYPES[p.dtype], t.data_ptr(), p.numel(), loss.data_ptr(),
                                  work.data_ptr(), work.numel(), _stream(p))
        _capi.check(lib, rc, "l4d_bce_loss")
        ctx.save_for_backward(p, t)
        ctx.shape = pred.shape
        return loss

    @staticmethod
    def backward(ctx, gl):
        p, t = ctx.saved_tensors
        lib = _capi.load_library()
        gl = gl.detach().float().contiguous()
        out = torch.empty_like(p)
        with torch.cuda.device(p.device):
            rc = lib.l4d_bce_loss_backward(p.data_ptr(), _BCE_DTYPES[p.dtype], t.data_ptr(), p.numel(), gl.data_ptr(),
                                           out.data_ptr(), _stream(p))
        _capi.check(lib, rc, "l4d_bce_loss_backward")
        return out.view(ctx.shape), None


def raydrop_bce_loss(pred, target):
    """model/runner.py:901, ``torch.nn.BCELoss()(pred, target)`` (mean), as a device scalar with no host read, forward or
    backward.  pred is float32, float16 or bfloat16 (the U-Net's output under any autocast), target any float dtype, read
    as float32; the elements are computed in float32 and summed in double in a fixed order.  The gradient (pred's dtype)
    is torch's.  Unlike torch, which fires a device-side assert, a pred outside [0, 1] or NaN makes the loss NaN (and
    that element's gradient NaN).  No gradient flows to target."""
    if not (pred.is_cuda and target.is_cuda):
        raise RuntimeError("raydrop_bce_loss runs on CUDA only (no CPU fallback)")
    if pred.dtype not in _BCE_DTYPES:
        raise ValueError(f"pred must be float32, float16 or bfloat16, got {pred.dtype}")
    if target.shape != pred.shape:
        raise ValueError(f"target {tuple(target.shape)} and pred {tuple(pred.shape)} must have the same shape")
    if pred.numel() == 0:
        raise ValueError("raydrop_bce_loss of an empty tensor")
    return _RaydropBCE.apply(pred, target)


def lidar_patch_loss(depth, gt, patch_size, scale, depth_grad_loss="l1", sobel_grad=False, grad_loss=True, alpha_grad=0.1,
                     grad_norm_smooth=False, alpha_grad_norm=0.1, spatial_smooth=False, alpha_spatial=0.1, tv_loss=False,
                     alpha_tv=0.1, **_):
    """model/runner.py:278-369 as one launch: the depth-gradient loss of a patch batch and the optional smoothness terms,
    summed, with d loss / d depth.  depth [.., n] (the render's depth_lidar), gt [.., n, 3] = (raydrop, intensity,
    depth); the n rays are n / (px*py) patches of px rows x py columns, get_lidar_rays' order.  patch_size is an int,
    [p] or [px, py] (runner.py:279-284); px == 1 gives 0, as in the reference.  Keyword names are the reference's opt
    fields, so `**vars(opt)` can be passed (other keys are ignored)."""
    if isinstance(patch_size, int):
        px = py = patch_size
    elif len(patch_size) == 1:
        px = py = patch_size[0]
    else:
        px, py = patch_size
    px, py = int(px), int(py)
    if depth_grad_loss not in GRAD_CRITERIA:
        raise ValueError(f"depth_grad_loss must be one of {sorted(GRAD_CRITERIA)}, got {depth_grad_loss!r}")
    if not (depth.is_cuda and gt.is_cuda):
        raise RuntimeError("lidar_patch_loss runs on CUDA only (no CPU fallback)")
    n = depth.numel()
    if gt.numel() != 3 * n or gt.shape[-1] != 3:
        raise ValueError("depth [.., n] and gt [.., n, 3] must describe the same rays")
    if px < 1 or py < 1 or n % (px * py):
        raise ValueError(f"{n} rays are not a whole number of {px}x{py} patches")
    flags = ((_SOBEL if sobel_grad else 0) | (_GRAD if grad_loss else 0) | (_GRAD_NORM if grad_norm_smooth else 0)
             | (_SPATIAL if spatial_smooth else 0) | (_TV if tv_loss else 0))
    return _PatchLoss.apply(depth, gt, px, py, scale, GRAD_CRITERIA[depth_grad_loss], flags, alpha_grad, alpha_grad_norm,
                            alpha_spatial, alpha_tv)


class _LineOfSightLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, weights, z_vals, gt, eps):
        lib = _capi.load_library()
        n, S = weights.shape
        w = weights.detach().contiguous().float()
        z = z_vals.detach().contiguous().float()
        g = gt.detach().contiguous().view(-1, 3).float()
        loss = torch.empty((), device=w.device)
        work = torch.empty(lib.l4d_los_work_bytes(), dtype=torch.uint8, device=w.device)
        with torch.cuda.device(w.device):
            rc = lib.l4d_los_loss(w.data_ptr(), z.data_ptr(), g.data_ptr(), n, S, float(eps), loss.data_ptr(),
                                  work.data_ptr(), work.numel(), _stream(w))
        _capi.check(lib, rc, "l4d_los_loss")
        ctx.save_for_backward(w, z, g, work)
        ctx.eps = float(eps)
        return loss

    @staticmethod
    def backward(ctx, gl):
        w, z, g, work = ctx.saved_tensors
        lib = _capi.load_library()
        gl = gl.detach().float().contiguous()
        gw = torch.empty_like(w)
        with torch.cuda.device(w.device):
            rc = lib.l4d_los_loss_backward(w.data_ptr(), z.data_ptr(), g.data_ptr(), w.shape[0], w.shape[1], ctx.eps,
                                           work.data_ptr(), gl.data_ptr(), gw.data_ptr(), _stream(w))
        _capi.check(lib, rc, "l4d_los_loss_backward")
        return gw, None, None, None


def line_of_sight_loss(weights, z_vals, gt, eps):
    """model/runner.py:255-276 (URF's line-of-sight loss): 0.1 * loss_empty + 0.1 * loss_near over weights / z_vals
    [n, S] (the render's outputs) and gt [.., n, 3], with the caller's eps = 0.02 * 0.1 ** min(step / iters, 1).
    Differentiable in weights.  With no ray of gt depth > 0 the value is the reference's inf / nan."""
    if not (weights.is_cuda and z_vals.is_cuda and gt.is_cuda):
        raise RuntimeError("line_of_sight_loss runs on CUDA only (no CPU fallback)")
    if weights.dim() != 2 or z_vals.shape != weights.shape:
        raise ValueError("weights and z_vals must both be [n, S]")
    if gt.numel() != 3 * weights.shape[0] or gt.shape[-1] != 3:
        raise ValueError("gt must be [.., n, 3] for the n rays of weights")
    if weights.numel() == 0:
        raise ValueError("line_of_sight_loss of an empty batch (the reference's distr.max() raises too)")
    return _LineOfSightLoss.apply(weights, z_vals, gt, eps)


# ----------------------------------------------------------------------------------------------------------------------
# flow loss (model/runner.py:222-253)
# ----------------------------------------------------------------------------------------------------------------------
class FlowClouds:
    """Every frame's cloud and ground cloud on the device, uploaded once and converted as the reference converts them
    every step (float64 NumPy -> float32), each frame cloud with its nearest-neighbour index (chamfer.PointGrid).
    Build it once after ``process_pointcloud``; keys are the reference's (``f"{frame_idx}"``)."""

    def __init__(self, pc_list, pc_ground_list, device):
        from .chamfer import PointGrid
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("FlowClouds lives on a CUDA device (no CPU fallback)")

        def up(a):
            a = a if isinstance(a, torch.Tensor) else torch.from_numpy(a)
            return a.to(device).float().contiguous().view(-1, 3)

        self.device = device
        self.grids = {k: PointGrid(up(v)) for k, v in pc_list.items()}
        self.ground = {k: up(v) for k, v in pc_ground_list.items()}


class _FlowLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, flow, ground_flow, cur, terms):
        """flow [n, 6] of the current frame's cloud `cur` (a PointGrid), ground_flow [g, 6]; terms = [(dir, step, PointGrid
        of the neighbouring frame)].  Per term: warp + query of the static index, index of the warped cloud, query of it."""
        from .chamfer import PointGrid
        lib = _capi.load_library()
        P = _capi.FLOW_PARTS
        fl = flow.detach().contiguous().float()
        gf = ground_flow.detach().contiguous().float()
        dev, n = fl.device, cur.n
        if fl.shape != (n, 6) or gf.dim() != 2 or gf.shape[1] != 6:
            raise ValueError("flow must be [n, 6] for the n points of the frame's cloud, ground_flow [g, 6]")
        parts = torch.zeros((2 * len(terms) + 1) * P, dtype=torch.float64, device=dev)
        saved = []
        with torch.cuda.device(dev):
            for i, (d, step, tgt) in enumerate(terms):
                warped = torch.empty(n, 3, device=dev)
                idx1 = torch.empty(n, dtype=torch.int32, device=dev)
                rc = lib.l4d_flow_warp_query(cur.points.data_ptr(), fl.data_ptr(), n, d, float(step), tgt.grid.data_ptr(),
                                             tgt.nbytes, tgt.n, warped.data_ptr(), idx1.data_ptr(),
                                             parts[2 * i * P:].data_ptr(), _stream(fl))
                _capi.check(lib, rc, "l4d_flow_warp_query")
                _, idx2 = PointGrid(warped).query(tgt.points, sum_parts=parts[(2 * i + 1) * P:], want_dist=False)
                saved += [warped, idx1, idx2]
            if gf.shape[0]:
                rc = lib.l4d_flow_ground(gf.data_ptr(), gf.shape[0], parts[2 * len(terms) * P:].data_ptr(), _stream(fl))
                _capi.check(lib, rc, "l4d_flow_ground")
            loss = torch.empty((), device=dev)
            rc = lib.l4d_flow_loss_finish(parts.data_ptr(), 2 * len(terms) * P, P, loss.data_ptr(), _stream(fl))
            _capi.check(lib, rc, "l4d_flow_loss_finish")
        ctx.save_for_backward(gf, *saved)
        ctx.terms = terms
        ctx.in_dtypes = (flow.dtype, ground_flow.dtype)
        return loss

    @staticmethod
    def backward(ctx, gl):
        gf, *saved = ctx.saved_tensors
        lib = _capi.load_library()
        gl = gl.detach().float().contiguous()
        n = saved[0].shape[0] if saved else 0
        g_flow = torch.zeros(n, 6, device=gf.device) if saved else None
        g_ground = torch.empty_like(gf)
        with torch.cuda.device(gf.device):
            for i, (d, step, tgt) in enumerate(ctx.terms):
                warped, idx1, idx2 = saved[3 * i:3 * i + 3]
                rc = lib.l4d_flow_term_backward(warped.data_ptr(), n, tgt.points.data_ptr(), tgt.n, idx1.data_ptr(),
                                                idx2.data_ptr(), d, float(step), gl.data_ptr(), g_flow.data_ptr(), _stream(gf))
                _capi.check(lib, rc, "l4d_flow_term_backward")
            rc = lib.l4d_flow_ground_backward(gf.data_ptr(), gf.shape[0], gl.data_ptr(), g_ground.data_ptr(), _stream(gf))
            _capi.check(lib, rc, "l4d_flow_ground_backward")
        if g_flow is not None:
            g_flow = g_flow.to(ctx.in_dtypes[0])
        return g_flow, g_ground.to(ctx.in_dtypes[1]), None, None


def flow_loss_terms(clouds, frame_idx):
    """The chamfer terms of frame `frame_idx` in the reference's order: [(0 forward | 1 backward, step, PointGrid)] for
    step in (1, 2) and each direction whose frame exists."""
    terms = []
    for step in (1, 2):
        for d, sign in ((0, +1), (1, -1)):
            k = f"{frame_idx + sign * step}"
            if k in clouds.grids:
                terms.append((d, step, clouds.grids[k]))
    return terms


def flow_loss_from_flows(clouds, frame_idx, flow, ground_flow):
    """The flow loss given the two flow predictions as [n, 6] = (forward | backward) tensors: everything of
    model/runner.py:222-253 after the ``model.flow`` calls.  No device-to-host read, forward or backward."""
    cur = clouds.grids[f"{frame_idx}"]
    if flow.shape[0] != cur.n:
        raise ValueError("flow must be [n, 6] for the n points of the frame's cloud")
    return _FlowLoss.apply(flow, ground_flow, cur, flow_loss_terms(clouds, frame_idx))


def lidar_flow_loss(model, clouds, time, num_frames, ground_time=None):
    """model/runner.py:222-253: with pc the cloud of frame int(time * (num_frames - 1)) and flow = model.flow(pc, time),
    for step in (1, 2) and each direction whose frame exists, 0.5 * (sum dist1 + sum dist2) between pc + flow_dir * step and
    that frame's cloud, plus 0.001 * (sum |forward| + sum |backward|) of model.flow(ground, tau).  tau is drawn as the
    reference draws it (``torch.rand(1).to(time)``), so the CPU generator ends in the reference's state; `ground_time`
    overrides it.  A frame without a cloud raises KeyError.

        clouds = FlowClouds(trainer.pc_list, trainer.pc_ground_list, device)      # once, after process_pointcloud
        loss = loss + lidar_flow_loss(model, clouds, time_lidar, num_frames=opt.num_frames)
    """
    frame_idx = int(time * (num_frames - 1))
    cur = clouds.grids[f"{frame_idx}"]
    fl = model.flow(cur.points, time)
    ground = clouds.ground[f"{frame_idx}"]
    tau = torch.rand(1).to(time) if ground_time is None else ground_time
    zf = model.flow(ground, tau)
    return flow_loss_from_flows(clouds, frame_idx, torch.cat([fl["forward"], fl["backward"]], 1),
                                torch.cat([zf["forward"], zf["backward"]], 1))
