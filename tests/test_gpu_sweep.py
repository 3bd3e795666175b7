"""GPU: the sweep images (l4d_sweep_images through lidar4d_b200.simulator) against the unmodified reference's outputs in
tests/golden/sweep_ref.npz and against oracle/sweep_oracle.py:
  - every panel, PNG and video frame bit-identical, on the golden frames and on random frames up to 128 x 2048;
  - the cloud inputs bit-identical, the clouds within the unprojection's tolerance;
  - sweep_rays to the reference's rays as get_lidar_rays is held to them, shift_trajectory bit-identical;
  - one launch per call, repeat calls identical, bfloat16 and bad arguments rejected;
  - Simulator.render end to end on the small test model with a RayDropUNet (needs cv2 for the PNGs)."""
import argparse
import os
import sys

import numpy as np
import pytest
import torch

import sweep_cases as SC
from oracle import sweep_oracle as SO

pytestmark = pytest.mark.gpu

FX = np.load(os.path.join(os.path.dirname(__file__), "golden", "sweep_ref.npz"), allow_pickle=False)
KITTI = (2.0, 26.9)


def _luts():
    return torch.from_numpy(FX["lut_intensity"]).cuda(), torch.from_numpy(FX["lut_depth"]).cuda()


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _bits_equal(a, b):
    """Bit-identical float32 arrays, NaNs compared by position only: the device writes the canonical NaN where the
    host keeps the input's payload."""
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    if a.shape != b.shape or not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    ok = ~np.isnan(a)
    return np.array_equal(a[ok].view(np.uint32), b[ok].view(np.uint32))


def _cloud_close(got, want):
    assert got.shape == want.shape
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    assert np.allclose(got[ok], want[ok], rtol=1e-6, atol=1e-6)


def _sim_images(f, refine, fov):
    from lidar4d_b200.simulator import sweep_images
    from lidar4d_b200.convert import _unproject_device
    r = _cuda(SC.raydrop_of(f, refine))
    out = sweep_images(_cuda(f["depth"]), _cuda(f["image"]), r, layout="sim", scale=SC.SCALE, luts=_luts())
    cloud, count = _unproject_device(out["pano"], out["intensities"], fov)
    return out, cloud[:int(count.item())].cpu().numpy()


@pytest.mark.parametrize("case", sorted(SC.SIM))
def test_sim_layout_matches_reference(case):
    refine, fov = SC.SIM[case]
    for i, f in enumerate(SC.frames(FX, case)[:FX[f"sim_{case}_times"].shape[0]]):
        out, cloud = _sim_images(f, refine, fov)
        panel = out["panel"].cpu().numpy()
        assert SC.same(FX, f"sim_{case}_png{i}", panel)
        assert SC.same(FX, f"sim_{case}_video{i}", panel[..., ::-1])
        _, opano, ointen, ocloud = SO.sim(SC.raydrop_of(f, refine), f["image"][..., 1], f["depth"], SC.SCALE, fov,
                                          FX["lut_intensity"], FX["lut_depth"])
        assert _bits_equal(out["pano"].cpu().numpy(), opano) and _bits_equal(out["intensities"].cpu().numpy(), ointen)
        _cloud_close(cloud, ocloud)


@pytest.mark.parametrize("case", sorted(SC.TEST))
def test_test_layout_matches_reference(case):
    from lidar4d_b200.simulator import test_outputs, sweep_images
    alpha_r, refine, _ = SC.TEST[case]
    for i, f in enumerate(SC.frames(FX, case)):
        r = SC.raydrop_of(f, refine)
        got = test_outputs(_cuda(f["depth"]), _cuda(f["image"]), _cuda(r), scale=SC.SCALE, alpha_r=alpha_r,
                           lidar_K=KITTI, luts=_luts())
        if f"test_{case}_raydrop{i}" in FX.files:
            assert SC.same(FX, f"test_{case}_raydrop{i}", got["raydrop"])
        assert SC.same(FX, f"test_{case}_intensity{i}", got["intensity"])
        assert SC.same(FX, f"test_{case}_depth{i}", got["depth"])
        _, _, _, opano, opoints = SO.test(r, f["image"][..., 1], f["depth"], SC.SCALE, alpha_r, KITTI,
                                          FX["lut_intensity"], FX["lut_depth"])
        pano = sweep_images(_cuda(f["depth"]), _cuda(f["image"]), _cuda(r), layout="test", scale=SC.SCALE,
                            alpha_r=alpha_r, luts=_luts())["pano"]
        assert _bits_equal(pano.cpu().numpy(), opano)
        _cloud_close(got["points"], opoints)


@pytest.mark.parametrize("case", SC.EVAL)
def test_eval_layout_matches_reference(case):
    from lidar4d_b200.simulator import validation_panel
    for i, f in enumerate(SC.frames(FX, case)):
        panel = validation_panel(_cuda(f["unet"])[None], _cuda(f["image"][..., 1])[None], _cuda(f["depth"])[None],
                                 luts=_luts())
        assert SC.same(FX, f"eval_{case}_png{i}", panel)


@pytest.mark.parametrize("H,W,seed", [(1, 1, 1), (3, 7, 2), (64, 2048, 3), (128, 2048, 4)])
@pytest.mark.parametrize("dtype", [np.float32, np.float16])
def test_random_frames_match_oracle(H, W, seed, dtype):
    from lidar4d_b200.simulator import sweep_images
    rng = np.random.default_rng(seed)
    f = SC._frame(rng, H, W, dtype) if H * W >= 8 else {
        "depth": rng.uniform(0, 2, (H, W)).astype(np.float32), "image": rng.uniform(0, 1, (H, W, 2)).astype(np.float32),
        "unet": rng.uniform(0, 1, (H, W)).astype(dtype)}
    L = (FX["lut_intensity"], FX["lut_depth"])
    r, I, D = f["unet"], f["image"][..., 1].copy(), f["depth"]
    args = (_cuda(D), _cuda(f["image"]), _cuda(r))
    s = sweep_images(*args, layout="sim", scale=0.37, luts=_luts())
    panel, opano, ointen, _ = SO.sim(r, I, D, 0.37, KITTI, *L)
    assert np.array_equal(s["panel"].cpu().numpy(), panel)
    assert _bits_equal(s["pano"].cpu().numpy(), opano) and _bits_equal(s["intensities"].cpu().numpy(), ointen)
    for alpha_r in (0.01, 0.0):
        t = sweep_images(*args, layout="test", scale=0.37, alpha_r=alpha_r, luts=_luts())
        rd, oi, od, opano, _ = SO.test(r, I, D, 0.37, alpha_r, KITTI, *L)
        assert np.array_equal(t["raydrop"].cpu().numpy(), rd)
        assert np.array_equal(t["intensity"].cpu().numpy(), oi) and np.array_equal(t["depth"].cpu().numpy(), od)
        assert _bits_equal(t["pano"].cpu().numpy(), opano)
    e = sweep_images(*args, layout="eval", luts=_luts())
    assert np.array_equal(e["panel"].cpu().numpy(), SO.evaluate(r, I, D, *L))


def test_one_launch_and_repeatable():
    from lidar4d_b200 import _capi
    from lidar4d_b200.simulator import sweep_images
    lib = _capi.load_library()
    f = SC.frames(FX, "66x1030_f16")[0]
    args = (_cuda(f["depth"]), _cuda(f["image"]), _cuda(f["unet"]))
    outs = []
    for layout in ("sim", "test", "eval"):
        for _ in range(2):
            n0 = lib.l4d_launch_count()
            o = sweep_images(*args, layout=layout, scale=SC.SCALE, luts=_luts())
            assert lib.l4d_launch_count() - n0 == 1
            outs.append({k: v.cpu().numpy() for k, v in o.items()})
        a, b = outs[-2:]
        assert all(a[k].tobytes() == b[k].tobytes() for k in a)


def test_rejects_bad_arguments():
    from lidar4d_b200.simulator import sweep_images
    f = SC.frames(FX, "8x16")[0]
    d, im, r = _cuda(f["depth"]), _cuda(f["image"]), _cuda(f["unet"])
    with pytest.raises(TypeError):
        sweep_images(d, im, r.bfloat16(), layout="sim", luts=_luts())
    with pytest.raises(TypeError):
        sweep_images(d.double(), im, r, layout="sim", luts=_luts())
    with pytest.raises(ValueError):
        sweep_images(d, im, r, layout="png", luts=_luts())
    with pytest.raises(ValueError):
        sweep_images(d[:4], im, r, layout="sim", luts=_luts())
    with pytest.raises(ValueError):
        sweep_images(d, im[..., :1], r, layout="sim", luts=_luts())
    with pytest.raises(ValueError):
        sweep_images(d, im, r, layout="sim", luts=(_luts()[0][:100], _luts()[1]))
    with pytest.raises(RuntimeError):
        sweep_images(d.cpu(), im, r, layout="sim", luts=_luts())


def _sim_opt(case):
    """The options main_lidar4d_sim.main ran case `case` with (its parser's defaults for the rest)."""
    from lidar4d_b200.simulator import kitti2nus
    p = argparse.ArgumentParser()
    for name, v in (("shift_x", 0.0), ("shift_y", 0.0), ("shift_z", 0.0), ("scale", 0.01)):
        p.add_argument(f"--{name}", type=float, default=v)
    p.add_argument("--offset", type=float, nargs="*", default=[0, 0, 0])
    p.add_argument("--H_lidar", type=int, default=66)
    p.add_argument("--W_lidar", type=int, default=1030)
    p.add_argument("--fov_lidar", type=float, nargs="*", default=[2.0, 26.9])
    p.add_argument("--far_lidar", type=float, default=81.0)
    p.add_argument("--use_refine", type=bool, default=True)
    p.add_argument("--align_axis", action="store_true")
    p.add_argument("--kitti2nus", action="store_true")
    opt = p.parse_args([str(a) for a in FX[f"sim_{case}_argv"]])
    return kitti2nus(opt) if opt.kitti2nus else opt


@pytest.mark.parametrize("case", sorted(SC.SIM))
def test_sweep_rays_and_trajectory(case):
    from lidar4d_b200.simulator import sweep_rays, shift_trajectory
    opt = _sim_opt(case)
    B = FX[f"sim_{case}_times"].shape[0]
    poses = FX[f"sim_{case}_poses"]                          # a one-frame case keeps frame 0 of two
    ro, rd = sweep_rays(poses, opt.offset, opt.scale, opt.H_lidar, opt.W_lidar, opt.fov_lidar)
    ro, rd = ro[:B], rd[:B]
    assert ro.shape == (B, opt.H_lidar * opt.W_lidar, 3)
    assert float((rd[:, ::61].cpu() - torch.from_numpy(FX[f"sim_{case}_rays_d"])).abs().max()) < 2e-6
    shifted = shift_trajectory(ro, opt.shift_x, opt.shift_y, opt.shift_z, opt.scale, opt.align_axis)
    assert shifted.shape == ro.shape and shifted.is_cuda
    assert _bits_equal(shifted[:, 0].cpu().numpy(), FX[f"sim_{case}_origins"])
    assert bool((shifted == shifted[:, :1]).all())


def _small_model():
    sys.path.insert(0, os.path.dirname(__file__))
    from parity_util import small_config, cuda_model_from_oracle
    from oracle import lidar4d_oracle as O
    from lidar4d_b200.raydrop_unet import RayDropUNet
    torch.manual_seed(0)
    model = cuda_model_from_oracle(O.build_seeded(small_config(), 5, flow_last_std=0.02))
    model.unet = RayDropUNet().cuda().eval()
    return model


def test_simulator_render_end_to_end(tmp_path):
    cv2 = pytest.importorskip("cv2")
    from lidar4d_b200.simulator import Simulator, sweep_images, sweep_rays, shift_trajectory, sweep_times
    from lidar4d_b200.convert import pano_to_lidar_with_intensities
    H, W = 16, 64
    model = _small_model()
    opt = argparse.Namespace(scale=0.01, fov_lidar=[2.0, 26.9], num_steps=48)
    poses = FX["sim_8x16_poses"]
    ro, rd = sweep_rays(poses, [1380, 3865, 115], opt.scale, H, W, opt.fov_lidar)
    ro = shift_trajectory(ro, 1.0, 0.5, 0.0, opt.scale, True)
    ro = ro - ro[:, :1].mean(0, keepdim=True)                 # keep the sensor inside the small model's box
    times = sweep_times([0, 1], device="cuda")
    sim = Simulator("lidar4d", opt, model, device=torch.device("cuda"), mute=True, workspace=str(tmp_path),
                    use_checkpoint="scratch", H_lidar=H, W_lidar=W)
    sim.luts = _luts()
    with torch.no_grad():                                     # stage the model once outside the checked loop
        model.render(ro[:1], rd[:1], times[:1].cpu(), staged=True, num_steps=48)
    torch.cuda.synchronize()
    frames = []

    class Recorder:
        @staticmethod
        def mimwrite(path, f, **kw):
            frames.append((path, np.asarray(f), kw))

    saved = sys.modules.get("imageio")
    sys.modules["imageio"] = Recorder
    times_host = times.cpu()
    torch.cuda.set_sync_debug_mode("error")                  # the frame loop: host times, no device read
    try:
        last = sim.render(ro, rd, times_host)
    finally:
        torch.cuda.set_sync_debug_mode("default")
        if saved is None:
            del sys.modules["imageio"]
        else:
            sys.modules["imageio"] = saved
    assert not model._engine.static_params
    with torch.no_grad():
        for i in range(2):
            out = model.render(ro[i:i + 1], rd[i:i + 1], times[i:i + 1].cpu(), staged=True, perturb=False, num_steps=48)
            image, depth = out["image_lidar"].reshape(1, H, W, 2), out["depth_lidar"].reshape(1, H, W)
            r = model.unet(torch.cat([image[..., 0], image[..., 1], depth], 0).unsqueeze(0)).squeeze(0)[0]
            s = sweep_images(depth[0], image[0], r, layout="sim", scale=opt.scale, luts=_luts())
            png = cv2.imread(str(tmp_path / "images" / f"lidar4d_{i:04d}.png"), cv2.IMREAD_UNCHANGED)
            assert png.dtype == np.uint8 and np.array_equal(png, s["panel"].cpu().numpy())
            npy = np.load(tmp_path / "points" / f"lidar4d_{i:04d}.npy")
            want = pano_to_lidar_with_intensities(s["pano"], s["intensities"], opt.fov_lidar).cpu().numpy()
            assert npy.dtype == np.float32 and npy.shape[1] == 4 and npy.tobytes() == want.tobytes()
            assert np.array_equal(frames[0][1][i], png[..., ::-1])
    assert last.tobytes() == npy.tobytes()
    (path, video, kw), = frames
    assert path == os.path.join(str(tmp_path), "video", "lidar4d_sim.mp4") and kw["fps"] == 5 and video.shape == (2, 3 * H, W, 3)

    n0 = model.gpu_launches
    sys.modules["imageio"] = None                             # not installed
    try:
        with pytest.raises(ImportError):
            sim.render(ro, rd, times, save_video=True)
    finally:
        if saved is None:
            del sys.modules["imageio"]
        else:
            sys.modules["imageio"] = saved
    assert model.gpu_launches == n0
