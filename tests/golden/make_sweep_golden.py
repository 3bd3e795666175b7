"""Generate tests/golden/sweep_ref.npz: the files the reference's own, unmodified code writes from rendered frames -
Simulator.render driven by main_lidar4d_sim.main (with its _get_lidar_rays and trajectory loop), Trainer.test and
Trainer.evaluate_one_epoch's validation panel - on the frames of tests/sweep_cases.py, for tests/test_sweep_oracle.py
(CPU) and tests/test_gpu_sweep.py (the CUDA op against the reference).

Run where the reference checkout exists (CPU only, seconds; cv2 is the real one):
    python tests/golden/make_sweep_golden.py [OUT.npz]

Stand-ins (tests/ref_stubs.py and below): a model whose render() returns the case's frames in order, records the ray
origins, directions and times it is given, and whose unet() returns the case's refined ray drop (float16 where the
case says so, as the U-Net under fp16 autocast gives it); KITTI360Loader returns sweep_cases.poses; configargparse is
argparse; imageio records the frames it is asked to encode; Trainer is built without its constructor and
evaluate_one_epoch gets an eval_step returning the case's frames (no meters).  _get_frame_ids is replaced to give
short trajectories, and the one-frame trajectory keeps the first frame of a two-frame _get_lidar_rays.

Recorded, per case and frame i (full arrays for the 8x16 cases, SHA-256 digests of the others):
  <case>_sha256                 the rebuilt frames;
  sim_<case>_png<i> / _npy<i> / _video<i>   images/lidar4d_%04d.png (decoded), points/lidar4d_%04d.npy, video frame;
  sim_<case>_origins / _times   the shifted ray origins [B, 3] and times the render was given;
  sim_<case>_rays_d             every 61st ray direction of every frame, [B, n, 3];  sim_<case>_poses, _argv;
  test_<case>_raydrop<i> / _intensity<i> / _depth<i> / _points<i>     Trainer.test's PNGs / npy, or its video frames;
  eval_<case>_png<i>            the validation PNG;
  lut_intensity, lut_depth      cv2.applyColorMap of 0..255 with colormaps 1 and 20, [256, 3] BGR."""
import argparse
import os
import platform
import sys
import tempfile
import types
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
ROOT = os.path.dirname(TESTS)
sys.path.insert(0, ROOT)
sys.path.insert(0, TESTS)

import ref_stubs  # noqa: E402
import sweep_cases as SC  # noqa: E402

FULL = ("8x16", "8x16_f16")
RAY_STRIDE = 61
VIDEO = []


class StubModel(torch.nn.Module):
    def __init__(self, frames):
        super().__init__()
        self.frames, self.k, self.seen = frames, -1, []

    def render(self, rays_o, rays_d, time, staged=False, perturb=False, **kw):
        self.k += 1
        f = self.frames[self.k]
        self.seen.append((rays_o[0, 0].clone(), rays_d[0, ::RAY_STRIDE].clone(), float(time.reshape(-1)[0])))
        return {"depth_lidar": torch.from_numpy(f["depth"]).reshape(1, -1),
                "image_lidar": torch.from_numpy(f["image"]).reshape(1, -1, 2)}

    def unet(self, x):
        return torch.from_numpy(self.frames[self.k]["unet"])[None, None]


def _install(model_box, poses_box):
    class ArgumentParser(argparse.ArgumentParser):
        def add_argument(self, *a, is_config_file=False, **k):
            if is_config_file:
                return None
            return super().add_argument(*a, **k)

    class KITTI360Loader:
        def __init__(self, root):
            pass

        def load_lidars(self, sequence_name, frame_ids):
            return [poses_box[0][k] for k in range(len(frame_ids))]

    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m

    mod("imageio", mimwrite=lambda path, frames, **kw: VIDEO.append((os.path.basename(path), np.asarray(frames).copy())))
    mod("configargparse", ArgumentParser=ArgumentParser)
    mod("data")
    mod("data.preprocess")
    mod("data.preprocess.kitti360_loader", KITTI360Loader=KITTI360Loader)
    mod("model.lidar4d", LiDAR4D=lambda **kw: model_box[0])


def _store(fx, key, a, full):
    fx[key] = np.asarray(a) if full else np.array(SC.digest(np.asarray(a)))


def _png(path):
    import cv2
    return cv2.imread(path, cv2.IMREAD_UNCHANGED)


SIM_RUNS = {   # case -> (argv, frame ids, one-frame trajectory)
    "66x1030": (["--H_lidar", "66", "--W_lidar", "1030", "--shift_x", "3.0", "--shift_y", "1.5", "--shift_z", "0.5",
                 "--align_axis", "--offset", "1380", "3865", "115"], (100, 101), False),
    "32x1024": (["--kitti2nus", "--shift_x", "2.0", "--offset", "1380", "3865", "115"], (200, 201), True),
    "8x16": (["--H_lidar", "8", "--W_lidar", "16", "--shift_y", "-2.0", "--align_axis"],
             (300, 301), False),
}


def run_sim(fx, M, model_box, poses_box, case):
    argv, ids, one = SIM_RUNS[case]
    fr = SC.frames(None, case)
    fx[f"{case}_sha256"] = np.array(SC.frames_digest(fr))
    model_box[0] = model = StubModel(fr)
    poses_box[0] = poses = SC.poses(2, 7 + len(case))
    ws = tempfile.mkdtemp()
    M._get_frame_ids = lambda sequence_id: ids
    orig = M._get_lidar_rays
    if one:
        M._get_lidar_rays = lambda sid, opt, device: tuple(x[:1] for x in orig(sid, opt, device))
    VIDEO.clear()
    sys.argv = ["main_lidar4d_sim.py", "--workspace", ws, *argv]
    try:
        M.main()
    finally:
        M._get_lidar_rays = orig
    full = case in FULL
    B = len(model.seen)
    for i in range(B):
        _store(fx, f"sim_{case}_png{i}", _png(os.path.join(ws, "images", f"lidar4d_{i:04d}.png")), full)
        _store(fx, f"sim_{case}_npy{i}", np.load(os.path.join(ws, "points", f"lidar4d_{i:04d}.npy")), full)
        (name, video), = VIDEO
        assert name == "lidar4d_sim.mp4"
        _store(fx, f"sim_{case}_video{i}", video[i], full)
    fx[f"sim_{case}_origins"] = torch.stack([s[0] for s in model.seen]).numpy()
    fx[f"sim_{case}_rays_d"] = torch.stack([s[1] for s in model.seen]).numpy()
    fx[f"sim_{case}_times"] = np.array([s[2] for s in model.seen], np.float32)
    fx[f"sim_{case}_poses"] = poses
    fx[f"sim_{case}_argv"] = np.array(argv)
    print("sim", case, B, "frames")


TEST_RUNS = SC.TEST     # case -> (alpha_r, refine, write_video)


def _trainer(runner, model, ws, **opt):
    tr = runner.Trainer.__new__(runner.Trainer)
    tr.name, tr.epoch, tr.workspace, tr.mute, tr.log_ptr, tr.console, tr.fp16 = "lidar4d", 1, ws, True, None, None, False
    tr.opt = argparse.Namespace(**opt)
    tr.model = model
    tr.ema, tr.use_tensorboardX = None, False
    return tr


class _Loader:
    def __init__(self, H, W, n):
        self.batch_size, self.n = 1, n
        self._data = argparse.Namespace(H_lidar=H, W_lidar=W, intrinsics_lidar=(2.0, 26.9))

    def __len__(self):
        return self.n

    def __iter__(self):
        H, W = self._data.H_lidar, self._data.W_lidar
        for _ in range(self.n):
            yield {"rays_o_lidar": torch.zeros(1, H * W, 3), "rays_d_lidar": torch.zeros(1, H * W, 3),
                   "time": torch.zeros(1, 1), "H_lidar": H, "W_lidar": W}


def run_test(fx, runner, case):
    alpha_r, refine, write_video = TEST_RUNS[case]
    H, W, n, _, _ = SC.CASES[case]
    fr = SC.frames(None, case)
    fx[f"{case}_sha256"] = np.array(SC.frames_digest(fr))
    ws = tempfile.mkdtemp()
    tr = _trainer(runner, StubModel(fr), ws, scale=0.01, raydrop_loss="mse", alpha_r=alpha_r)
    VIDEO.clear()
    tr.test(_Loader(H, W, n), save_path=ws, name="t", write_video=write_video, refine=refine)
    full = case in FULL
    for i in range(n):
        _store(fx, f"test_{case}_points{i}", np.load(os.path.join(ws, f"test_t_{i + 1:04d}_depth_lidar.npy")), full)
        if write_video:
            (n1, v1), (n2, v2) = VIDEO
            assert (n1, n2) == ("t_lidar_rgb.mp4", "t_depth.mp4")
            _store(fx, f"test_{case}_intensity{i}", v1[i][..., ::-1], full)      # stored BGR, as the PNGs
            _store(fx, f"test_{case}_depth{i}", v2[i][..., ::-1], full)
        else:
            for kind in ("raydrop", "intensity", "depth"):
                _store(fx, f"test_{case}_{kind}{i}", _png(os.path.join(ws, f"test_t_{i + 1:04d}_{kind}.png")), full)
    print("test", case, n, "frames")


EVAL_RUNS = SC.EVAL


def run_eval(fx, runner, case):
    H, W, n, _, _ = SC.CASES[case]
    fr = SC.frames(None, case)
    fx[f"{case}_sha256"] = np.array(SC.frames_digest(fr))
    ws = tempfile.mkdtemp()
    tr = _trainer(runner, StubModel(fr), ws)
    tr.lidar_metrics, tr.stats, tr.best_mode = [], {"valid_loss": [], "results": []}, "min"
    it = iter(fr)

    def eval_step(data):
        f = next(it)
        r = torch.from_numpy(f["unet"])[None]
        return (torch.from_numpy(f["image"][..., 1].copy())[None], torch.from_numpy(f["depth"])[None], r, None, None, None,
                torch.zeros(()))

    tr.eval_step = eval_step
    tr.evaluate_one_epoch(_Loader(H, W, n), name="v")
    for i in range(n):
        _store(fx, f"eval_{case}_png{i}", _png(os.path.join(ws, "validation", f"v_{i + 1:04d}.png")), case in FULL)
    print("eval", case, n, "frames")


def main(out_path):
    import cv2
    warnings.simplefilter("ignore")
    model_box, poses_box = [None], [None]
    runner = ref_stubs.import_reference_runner()        # reference on sys.path, torch_ema / open3d / ... stand-ins
    _install(model_box, poses_box)
    runner.imageio = sys.modules["imageio"]             # the runner module was imported with tests/ref_stubs' module
    import main_lidar4d_sim as M
    cpu = platform.processor() or platform.machine()
    if os.path.exists("/proc/cpuinfo"):
        for line in open("/proc/cpuinfo"):
            if line.startswith("model name"):
                cpu = line.split(":", 1)[1].strip()
                break
    fx = {"numpy_version": np.array(np.__version__), "torch_version": np.array(torch.__version__),
          "cv2_version": np.array(cv2.__version__), "cpu": np.array(cpu)}
    ramp = np.arange(256, dtype=np.uint8)[None]
    fx["lut_intensity"] = cv2.applyColorMap(ramp, 1)[0]
    fx["lut_depth"] = cv2.applyColorMap(ramp, 20)[0]
    for case in SIM_RUNS:
        run_sim(fx, M, model_box, poses_box, case)
    for case in TEST_RUNS:
        run_test(fx, runner, case)
    for case in EVAL_RUNS:
        run_eval(fx, runner, case)
    np.savez_compressed(out_path, **fx)
    print(f"wrote {out_path} ({os.path.getsize(out_path)} bytes)")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 and not sys.argv[1].startswith("-") else os.path.join(HERE, "sweep_ref.npz"))
