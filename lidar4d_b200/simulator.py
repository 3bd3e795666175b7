"""LiDAR sweeps from a trained model on the device: the reference's ``Simulator`` (model/simulator.py) and the image and
point-cloud outputs of ``Trainer.test`` and ``Trainer.evaluate_one_epoch`` (model/runner.py), backed by
``l4d_sweep_images`` of the C-ABI library and the existing unprojection.

  * ``sweep_images`` is one launch per frame: the ray-drop threshold, the masking, ``depth / scale`` and the 8-bit
    colour-mapped images, bit for bit as the reference's torch + NumPy + cv2 code computes them (see
    csrc/l4d_sweep.cuh for the rules).  The colour tables come from the caller (``colormap_luts`` builds them with cv2);
    the library holds no OpenCV data.
  * ``sweep_rays`` / ``sweep_times`` / ``shift_trajectory`` / ``kitti2nus`` are main_lidar4d_sim.py's ray set-up on
    caller-supplied poses; the KITTI-360 loader and the argument parser stay the caller's.
  * ``Simulator`` is the drop-in class.  Its frame loop never stops the GPU for a frame's host work: frame i+1 is
    enqueued before frame i's files are written, and frame i reaches the host through pinned buffers and an event.
  * ``test_outputs`` / ``validation_panel`` return what ``Trainer.test`` saves and the validation PNG array.
Inputs are CUDA tensors; there is no CPU path.
"""
import glob
import os
import time

import numpy as np
import torch

from . import _capi
from .convert import _unproject_device
from .rays import get_lidar_rays

_LAYOUTS = {"sim": _capi.SWEEP_SIM, "test": _capi.SWEEP_TEST, "eval": _capi.SWEEP_EVAL}
_PANEL_ROWS = {"sim": 9, "test": 7, "eval": 18}     # bytes per pixel of each layout's images (L4D_SWEEP_PANEL_BYTES)


def colormap_luts(device="cuda"):
    """(intensity, depth) colour tables, [256, 3] uint8 BGR on `device`: cv2.applyColorMap of 0..255 with colormap 1
    (BONE, the reference's intensity images) and 20 (TURBO, its depth images).  Needs cv2."""
    import cv2
    ramp = np.arange(256, dtype=np.uint8)[None]
    return tuple(torch.from_numpy(np.ascontiguousarray(cv2.applyColorMap(ramp, code)[0])).to(device) for code in (1, 20))


def _plane(x, name, H=None, W=None):
    if not torch.is_tensor(x) or not x.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (lidar4d_b200.simulator has no CPU path)")
    while x.dim() > 2 and x.shape[0] == 1:
        x = x[0]
    if x.dim() != 2 or (H is not None and tuple(x.shape) != (H, W)):
        raise ValueError(f"{name}: expected [H, W]{'' if H is None else f' = [{H}, {W}]'}, got {tuple(x.shape)}")
    return x.detach().contiguous()


def sweep_images(depth, image, raydrop=None, *, layout, scale=1.0, alpha_r=0.01, luts):
    """One rendered frame -> the reference's 8-bit images and point-cloud inputs, as device tensors, in one launch.

    depth [H, W] and image [H, W, 2] float32 (a leading 1 is accepted: the render's outputs reshaped as the reference
    does); raydrop, the U-Net's refined ray drop [H, W] in float32 or float16, replaces image channel 0 when given.
    layout names the reference caller:
      "sim"   Simulator.render: {"panel": [3H, W, 3] BGR, "pano": depth*mask / scale, "intensities": intensity*mask};
      "test"  Trainer.test_step + test (masking only when alpha_r > 0): {"raydrop": [H, W] 0 / 255, "intensity" and
              "depth": [H, W, 3] BGR, "pano": depth' / scale};
      "eval"  evaluate_one_epoch's validation PNG: {"panel": [6H, W, 3] BGR}.
    luts = (intensity, depth) [256, 3] uint8 device tables (``colormap_luts``).  bfloat16 is rejected, as the
    reference's ``.numpy()`` rejects it."""
    if layout not in _LAYOUTS:
        raise ValueError(f"layout must be one of {sorted(_LAYOUTS)}, got {layout!r}")
    img = image
    if not torch.is_tensor(img) or not img.is_cuda:
        raise RuntimeError("image must be a CUDA tensor (lidar4d_b200.simulator has no CPU path)")
    while img.dim() > 3 and img.shape[0] == 1:
        img = img[0]
    if img.dim() != 3 or img.shape[-1] != 2:
        raise ValueError(f"image: expected [H, W, 2], got {tuple(image.shape)}")
    H, W = int(img.shape[0]), int(img.shape[1])
    d = _plane(depth, "depth", H, W)
    for name, t in (("depth", d), ("image", img)):
        if t.dtype != torch.float32:
            raise TypeError(f"{name} must be float32, got {t.dtype}")
    img = img.detach().contiguous()
    dtype, r = _capi.SWEEP_F32, None
    if raydrop is not None:
        r = _plane(raydrop, "raydrop", H, W)
        if r.dtype == torch.float16:
            dtype = _capi.SWEEP_F16
        elif r.dtype != torch.float32:
            raise TypeError(f"raydrop must be float32 or float16, got {r.dtype}")
    lut_i, lut_d = luts
    for name, t in (("luts[0]", lut_i), ("luts[1]", lut_d)):
        if not torch.is_tensor(t) or not t.is_cuda or t.dtype != torch.uint8 or t.numel() != 768:
            raise ValueError(f"{name} must be a [256, 3] uint8 CUDA tensor")
    lut_i, lut_d = lut_i.contiguous(), lut_d.contiguous()
    dev = img.device
    panel = torch.empty(_PANEL_ROWS[layout] * H * W, dtype=torch.uint8, device=dev)
    pano = torch.empty(H, W, device=dev) if layout != "eval" else None
    inten = torch.empty(H, W, device=dev) if layout == "sim" else None
    lib = _capi.load_library()
    with torch.cuda.device(dev):
        rc = lib.l4d_sweep_images(d.data_ptr(), img.data_ptr(), r.data_ptr() if r is not None else None, dtype, H, W,
                                  _LAYOUTS[layout], float(np.float32(scale)), int(alpha_r > 0), lut_i.data_ptr(),
                                  lut_d.data_ptr(), panel.data_ptr(), pano.data_ptr() if pano is not None else None,
                                  inten.data_ptr() if inten is not None else None,
                                  torch.cuda.current_stream(dev).cuda_stream)
    _capi.check(lib, rc, "l4d_sweep_images")
    if layout == "sim":
        return {"panel": panel.view(3 * H, W, 3), "pano": pano, "intensities": inten}
    if layout == "test":
        return {"raydrop": panel[:H * W].view(H, W), "intensity": panel[H * W:4 * H * W].view(H, W, 3),
                "depth": panel[4 * H * W:].view(H, W, 3), "pano": pano}
    return {"panel": panel.view(6 * H, W, 3)}


def test_outputs(depth, image, raydrop=None, *, scale, alpha_r, lidar_K, luts):
    """What Trainer.test (runner.py:755-793) saves for one frame, from test_step's render outputs before its masking:
    {"raydrop": [H, W] uint8, "intensity", "depth": [H, W, 3] uint8 BGR (the applyColorMap images; the video frames are
    their [..., ::-1]), "points": [N, 3] float32 (the *_depth_lidar.npy cloud)}, as NumPy arrays.  One host read."""
    out = sweep_images(depth, image, raydrop, layout="test", scale=scale, alpha_r=alpha_r, luts=luts)
    cloud, count = _unproject_device(out["pano"], None, lidar_K)
    n = int(count.item())
    return {"raydrop": out["raydrop"].cpu().numpy(), "intensity": out["intensity"].cpu().numpy(),
            "depth": out["depth"].cpu().numpy(), "points": cloud[:n].cpu().numpy()}


def validation_panel(raydrop, intensity, depth, *, luts):
    """The [6H, W, 3] uint8 BGR array evaluate_one_epoch (runner.py:611-634) writes to validation/*.png, from
    eval_step's preds_raydrop (float32 or float16), preds_intensity and preds_depth ([1, H, W] or [H, W])."""
    i = _plane(intensity, "intensity")
    return sweep_images(depth, torch.stack((i, i), -1), raydrop, layout="eval", luts=luts)["panel"].cpu().numpy()


# ---- main_lidar4d_sim.py: rays, times and trajectories ---------------------------------------------------------------
def sweep_rays(lidar2world, offset, scale, H, W, fov_lidar, device="cuda"):
    """main_lidar4d_sim.py:132-164 on caller-supplied poses: lidar2world [B, 4, 4] (float64; the translation is offset
    and scaled in float64, then every pose is cast to float32) -> (rays_o, rays_d) [B, H*W, 3] float32 on `device`, all
    pixels in row-major order, through the library's ray kernel."""
    poses = torch.as_tensor(lidar2world, dtype=torch.float64).to(device).clone()
    if poses.dim() != 3 or tuple(poses.shape[1:]) != (4, 4):
        raise ValueError(f"lidar2world: expected [B, 4, 4], got {tuple(poses.shape)}")
    off = torch.as_tensor(np.asarray(offset, np.float64), device=poses.device)
    poses[:, :3, -1] = (poses[:, :3, -1] - off) * float(scale)
    r = get_lidar_rays(poses.float(), fov_lidar, int(H), int(W))
    return r["rays_o"], r["rays_d"]


def sweep_times(frame_ids, device="cuda"):
    """main_lidar4d_sim.py:166-170: (frame - first) / (last - first) per frame, float32 [N, 1] on `device`."""
    s, e = frame_ids[0], frame_ids[-1]
    t = np.asarray([np.asarray((f - s) / (e - s)) for f in frame_ids], dtype=np.float32)
    return torch.from_numpy(t).view(-1, 1).to(device).float()


def shift_trajectory(rays_o, shift_x, shift_y, shift_z, scale, align_axis=False):
    """main_lidar4d_sim.py:250-272, bit for bit: rays_o [B, N, 3] (one origin per frame) -> the shifted origins, same
    shape and device.  With align_axis the x / y shift follows the motion direction: forward = normalize(o[i+1] - o[i])
    of the unshifted origins (the last frame keeps the previous forward), left = (-f_y, f_x, f_z), z is not rotated;
    a Python-float shift is added as f32(shift * scale), a rotated (tensor) shift is multiplied by scale in float32.
    The per-frame arithmetic runs on the [B, 3] origins, on the host as the reference's CPU ops, and is then expanded."""
    import torch.nn.functional as F
    o = rays_o[:, 0, :].detach().to("cpu", torch.float32)
    shifted = o.clone()
    sx, sy, sz = shift_x, shift_y, shift_z
    forward = torch.tensor([[1, 0, 0]]).to(o)
    for i in range(o.shape[0]):
        if align_axis:
            if i < o.shape[0] - 1:
                forward = F.normalize((o[i + 1, :] - o[i, :]).unsqueeze(0), p=2)
            left = torch.tensor([-forward[:, 1], forward[:, 0], forward[:, 2]]).to(forward)
            sx = (shift_x * forward + shift_y * left)[:, 0]
            sy = (shift_x * forward + shift_y * left)[:, 1]
        shifted[i, 0:1] = shifted[i, 0:1] + sx * scale
        shifted[i, 1:2] = shifted[i, 1:2] + sy * scale
        shifted[i, 2:3] = shifted[i, 2:3] + sz * scale
    return shifted.to(rays_o.device)[:, None, :].expand_as(rays_o).contiguous()


def kitti2nus(opt):
    """main_lidar4d_sim.py:184-190: the KITTI-360 -> nuScenes sensor preset, applied to `opt` in place (and returned)."""
    opt.fov_lidar = [10.0, 40.0]
    opt.H_lidar = 32
    opt.W_lidar = 1024
    opt.far_lidar = 70
    opt.shift_z += 0.1 * opt.scale
    opt.use_refine = False
    return opt


# ---- the drop-in Simulator --------------------------------------------------------------------------------------------
class Simulator(object):
    """model/simulator.py's Simulator: same constructor, render / load_checkpoint / log, same files under the same names.
    render() keeps every frame on the device until its files are written and pipelines one frame deep."""

    def __init__(self, name, opt, model, device=None, mute=False, fp16=False, workspace="simulation",
                 use_checkpoint="latest_model", use_refine=True, H_lidar=66, W_lidar=1030):
        self.name = name
        self.opt = opt
        self.mute = mute
        self.fp16 = fp16
        self.workspace = workspace
        self.use_checkpoint = use_checkpoint
        self.use_refine = use_refine
        self.H_lidar, self.W_lidar = H_lidar, W_lidar
        self.time_stamp = time.strftime("%Y-%m-%d_%H-%M-%S")
        self.device = device if device is not None else torch.device("cuda:0")
        try:
            from rich.console import Console
            self.console = Console()
        except ImportError:
            self.console = None
        model.to(self.device)
        self.model = model
        self.luts = None                 # (intensity, depth) colour tables; built with cv2 at the first render if unset

        self.log_ptr = None
        if self.workspace is not None:
            os.makedirs(self.workspace, exist_ok=True)
            self.log_path = os.path.join(workspace, f"log_{self.name}.txt")
            self.log_ptr = open(self.log_path, "a+")
            self.ckpt_path = os.path.join(self.workspace, "checkpoints")
            self.best_path = f"{self.ckpt_path}/{self.name}.pth"

        self.log(f'[INFO] Simulator: {self.name} | {self.time_stamp} | {self.device} | {"fp16" if self.fp16 else "fp32"} | {self.workspace}')

        if self.workspace is not None:
            if self.use_checkpoint == "scratch":
                self.log("[INFO] Training from scratch ...")
            elif self.use_checkpoint == "latest":
                self.log("[INFO] Loading latest checkpoint ...")
                self.load_checkpoint()
            elif self.use_checkpoint == "latest_model":
                self.log("[INFO] Loading latest checkpoint (model only)...")
                self.load_checkpoint(model_only=True)
            elif self.use_checkpoint == "best":
                if os.path.exists(self.best_path):
                    self.log("[INFO] Loading best checkpoint ...")
                    self.load_checkpoint(self.best_path)
                else:
                    self.log(f"[INFO] {self.best_path} not found, loading latest ...")
                    self.load_checkpoint()
            else:
                self.log(f"[INFO] Loading {self.use_checkpoint} ...")
                self.load_checkpoint(self.use_checkpoint)

    def __del__(self):
        if getattr(self, "log_ptr", None):
            self.log_ptr.close()

    def log(self, *args, **kwargs):
        if not self.mute:
            if self.console is not None:
                self.console.print(*args, **kwargs)
            else:
                print(*args, **kwargs)
        if self.log_ptr:
            print(*args, file=self.log_ptr)
            self.log_ptr.flush()

    def _enqueue(self, rays_o, rays_d, t, host):
        """Render one frame and queue its images, cloud and row count into the pinned buffers `host`; returns the event
        recorded after those copies.  Nothing here waits for the device."""
        H, W = self.H_lidar, self.W_lidar
        with torch.autocast("cuda", enabled=self.fp16):
            out = self.model.render(rays_o, rays_d, t, staged=True, perturb=False, **vars(self.opt))
        image = out["image_lidar"].reshape(-1, H, W, 2)
        depth = out["depth_lidar"].reshape(-1, H, W)
        raydrop = None
        if self.use_refine:
            x = torch.cat([image[..., 0], image[..., 1], depth], dim=0).unsqueeze(0)
            raydrop = self.model.unet(x).squeeze(0)[0]
        s = sweep_images(depth[0], image[0], raydrop, layout="sim", scale=self.opt.scale, luts=self.luts)
        cloud, count = _unproject_device(s["pano"], s["intensities"], self.opt.fov_lidar)
        host["panel"].copy_(s["panel"], non_blocking=True)
        host["cloud"].copy_(cloud, non_blocking=True)
        host["count"].copy_(count, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        return ev

    def _write(self, i, ev, host, save_pc, save_img, frames):
        ev.synchronize()
        pred_lidar = host["cloud"][:int(host["count"][0])].numpy().copy()
        panel = host["panel"].numpy()
        if save_pc:
            path = os.path.join(self.workspace, "points", f"lidar4d_{i:04d}.npy")
            os.makedirs(os.path.dirname(path), exist_ok=True)
            np.save(path, pred_lidar)
        if save_img:
            import cv2
            path = os.path.join(self.workspace, "images", f"lidar4d_{i:04d}.png")
            os.makedirs(os.path.dirname(path), exist_ok=True)
            cv2.imwrite(path, panel)
        if frames is not None:
            frames.append(panel[..., ::-1].copy())          # cv2.COLOR_BGR2RGB
        return pred_lidar

    @torch.no_grad()
    def render(self, rays_o_lidar, rays_d_lidar, times_lidar, save_pc=True, save_img=True, save_video=True):
        """simulator.py:103-194: render every frame, write points/lidar4d_%04d.npy ([N, 4] float32 x, y, z, intensity),
        images/lidar4d_%04d.png (ray drop / intensity / depth, stacked) and video/lidar4d_sim.mp4 (5 fps); returns the
        last frame's cloud.  The times are read to the host once; frame i+1 is enqueued before frame i's files are
        written, so the host work overlaps the next render."""
        if save_video:
            import imageio                                   # fail before the first frame, not after the last
        if self.luts is None:
            self.luts = colormap_luts(self.device)
        B = rays_o_lidar.shape[0]
        H, W = self.H_lidar, self.W_lidar
        times = times_lidar.detach().reshape(B, -1)[:, :1].to("cpu", torch.float32)
        hosts = [{"panel": torch.empty(3 * H, W, 3, dtype=torch.uint8, pin_memory=True),
                  "cloud": torch.empty(H * W, 4, pin_memory=True),
                  "count": torch.empty(1, dtype=torch.int32, pin_memory=True)} for _ in range(min(B, 2))]
        frames = [] if save_video else None
        try:
            import tqdm
            bar = tqdm.tqdm(total=B)
        except ImportError:
            bar = None
        eng = self.model._engine
        was_static = eng.static_params
        self.model.static_params(True)
        pred_lidar, pending = None, None
        try:
            for i in range(B):
                ev = self._enqueue(rays_o_lidar[i].unsqueeze(0), rays_d_lidar[i].unsqueeze(0), times[i:i + 1], hosts[i % 2])
                if pending is not None:
                    pred_lidar = self._write(*pending, save_pc, save_img, frames)
                    if bar is not None:
                        bar.update(1)
                pending = (i, ev, hosts[i % 2])
            if pending is not None:
                pred_lidar = self._write(*pending, save_pc, save_img, frames)
                if bar is not None:
                    bar.update(1)
        finally:
            self.model.static_params(was_static)
            if bar is not None:
                bar.close()
        if save_video:
            path = os.path.join(self.workspace, "video", "lidar4d_sim.mp4")
            os.makedirs(os.path.dirname(path), exist_ok=True)
            imageio.mimwrite(path, np.stack(frames, axis=0), fps=5, quality=8, macro_block_size=1)
        return pred_lidar

    def load_checkpoint(self, checkpoint=None, model_only=True):
        if checkpoint is None:
            checkpoint_list = sorted(glob.glob(f"{self.ckpt_path}/{self.name}_ep*.pth"))
            if checkpoint_list:
                checkpoint = checkpoint_list[-1]
                self.log(f"[INFO] Latest checkpoint is {checkpoint}")
            else:
                self.log("[WARN] No checkpoint found, model randomly initialized.")
                return
        checkpoint_dict = torch.load(checkpoint, map_location=self.device)
        if "model" not in checkpoint_dict:
            self.model.load_state_dict(checkpoint_dict)
            self.log("[INFO] loaded model.")
            return
        missing_keys, unexpected_keys = self.model.load_state_dict(checkpoint_dict["model"], strict=False)
        self.log("[INFO] loaded model.")
        if len(missing_keys) > 0:
            self.log(f"[WARN] missing keys: {missing_keys}")
        if len(unexpected_keys) > 0:
            self.log(f"[WARN] unexpected keys: {unexpected_keys}")
        if model_only:
            return
        if "stats" in checkpoint_dict:
            self.stats = checkpoint_dict["stats"]
        if "epoch" in checkpoint_dict:
            self.epoch = checkpoint_dict["epoch"]
        if "global_step" in checkpoint_dict:
            self.global_step = checkpoint_dict["global_step"]
            self.log(f"[INFO] load at epoch {self.epoch}, global step {self.global_step}")
