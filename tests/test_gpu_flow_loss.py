"""GPU: lidar_flow_loss (FlowClouds + the grid search + one autograd function over the flow) against the caller's
composition it replaces - model/runner.py:222-253 as tests/trainer_mirror.py restates it, copied here as a local function
with the brute-force chamfer op - on the clouds process_pointcloud builds from a synthetic loader."""
import os
import random
import sys

import numpy as np
import pytest
import torch

import ground_cases as GC

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
import make_ground_golden as MG  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
NUM_FRAMES = 6


def composition(model, cham_fn, pc_list, pc_ground_list, t, num_frames):
    """The flow-loss lines of trainer_mirror.MirrorTrainer.train_step, with their per-step uploads."""
    frame_idx = int(t * (num_frames - 1))
    dev = t.device
    loss = 0
    pc = torch.from_numpy(pc_list[f"{frame_idx}"]).to(dev).float().contiguous()
    fl = model.flow(pc, t)
    for step in (1, 2):
        for sign, key in ((+1, "forward"), (-1, "backward")):
            k = f"{frame_idx + sign * step}"
            if k in pc_list:
                pc_pred = pc + fl[key] * step
                other = torch.from_numpy(pc_list[k]).to(dev).float().contiguous()
                d1, d2, _, _ = cham_fn(pc_pred.unsqueeze(0), other.unsqueeze(0))
                loss = loss + (d1.sum() + d2.sum()) * 0.5
    ground = torch.from_numpy(pc_ground_list[f"{frame_idx}"]).to(dev).float().contiguous()
    zero_flow = model.flow(ground, torch.rand(1).to(t))
    return loss + 0.001 * (zero_flow["forward"].abs().sum() + zero_flow["backward"].abs().sum())


@pytest.fixture(scope="module")
def scene():
    from lidar4d_b200.losses import FlowClouds
    from lidar4d_b200.misc import process_pointcloud
    img, pose, _ = MG.chain_inputs()
    loader = [{"images_lidar": torch.from_numpy(img).to(torch.float16).cuda(), "poses_lidar": torch.from_numpy(pose).cuda(),
               "time": torch.tensor([[k / 5]], dtype=torch.float32, device="cuda")} for k in range(5)]
    random.seed(0)
    pcs, grounds = process_pointcloud(loader, 0.01, NUM_FRAMES, GC.K)
    assert sorted(pcs) == ["0", "1", "2", "3", "4"]
    return pcs, grounds, FlowClouds(pcs, grounds, DEV)


def _model(seed=3):
    from oracle import lidar4d_oracle as O
    from parity_util import small_config, cuda_model_from_oracle
    return cuda_model_from_oracle(O.build_seeded(small_config(), seed, flow_last_std=0.02))


def _flow_grads(model):
    return {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}


def _time(frame):
    return torch.tensor([[frame / (NUM_FRAMES - 1) + 1e-4]], dtype=torch.float32, device=DEV)


# frame 2: both neighbours at both steps; 0 and 4: the first and the last frame; 1 and 3: one side has step 1 only
@pytest.mark.parametrize("frame,scale", [(2, 1.0), (0, 1.0), (4, 1.0), (1, 1.0), (3, 65536.0)])
def test_matches_the_composition(scene, frame, scale):
    from lidar4d_b200.chamfer import chamfer_3DDist
    from lidar4d_b200.losses import flow_loss_terms, lidar_flow_loss
    pcs, grounds, clouds = scene
    assert len(flow_loss_terms(clouds, frame)) == {0: 2, 1: 3, 2: 4, 3: 3, 4: 2}[frame]
    model = _model()
    t = _time(frame)
    assert int(t * (NUM_FRAMES - 1)) == frame
    torch.manual_seed(7)
    want = composition(model, chamfer_3DDist(), pcs, grounds, t, NUM_FRAMES)
    state_ref = torch.get_rng_state()
    model.zero_grad()
    (want * scale).backward()
    g_ref = _flow_grads(model)
    torch.manual_seed(7)
    got = lidar_flow_loss(model, clouds, t, num_frames=NUM_FRAMES)
    assert torch.equal(torch.get_rng_state(), state_ref)
    model.zero_grad()
    (got * scale).backward()
    g_got = _flow_grads(model)
    assert got.shape == () and got.dtype == torch.float32
    assert abs(got.item() - want.item()) <= 1e-6 * abs(want.item()), (got.item(), want.item())
    assert sorted(g_got) == sorted(g_ref)
    assert sum(float(r.abs().max()) > 0 for r in g_ref.values()) >= 2        # the flow grid and the flow MLP at least
    for name, ref in g_ref.items():
        err = float((g_got[name] - ref).abs().max())
        assert err <= 1e-5 * float(ref.abs().max()), (name, err)
    # ground_time= overrides the draw and leaves the generator alone
    before = torch.get_rng_state()
    a = lidar_flow_loss(model, clouds, t, num_frames=NUM_FRAMES, ground_time=torch.tensor([0.3], device=DEV))
    b = lidar_flow_loss(model, clouds, t, num_frames=NUM_FRAMES, ground_time=torch.tensor([0.3], device=DEV))
    assert torch.equal(torch.get_rng_state(), before) and torch.equal(a, b)


def test_missing_frame_raises_key_error(scene):
    from lidar4d_b200.losses import lidar_flow_loss
    _, _, clouds = scene
    with pytest.raises(KeyError):
        lidar_flow_loss(_model(), clouds, torch.tensor([[1.0]], device=DEV), num_frames=NUM_FRAMES)      # frame 5


def test_no_host_sync_and_fixed_launch_count(scene):
    """The autograd function over given flows: no device-to-host read forward or backward, and a launch count that
    depends on the number of terms only (7 per term + ground + final sum forward; 1 per term + ground backward)."""
    from lidar4d_b200 import _capi
    from lidar4d_b200.losses import FlowClouds, flow_loss_from_flows
    _, _, clouds = scene
    lib = _capi.load_library()
    g = torch.Generator().manual_seed(5)
    small = {str(k): (torch.rand(200 + 10 * k, 3, generator=g) - 0.5).numpy().astype(np.float64) for k in range(5)}
    small_clouds = FlowClouds(small, {k: v[:50] for k, v in small.items()}, DEV)
    counts = []
    for cl in (clouds, small_clouds):
        n, ng = cl.grids["2"].n, cl.ground["2"].shape[0]
        flow = (torch.randn(n, 6, generator=g) * 1e-3).to(DEV).requires_grad_(True)
        gflow = (torch.randn(ng, 6, generator=g) * 1e-3).to(DEV).requires_grad_(True)
        scale = torch.tensor(65536.0, device=DEV)
        torch.cuda.synchronize()
        c0 = lib.l4d_launch_count()
        torch.cuda.set_sync_debug_mode("error")
        try:
            loss = flow_loss_from_flows(cl, 2, flow, gflow)
            c1 = lib.l4d_launch_count()
            (loss * scale).backward()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        counts.append((c1 - c0, lib.l4d_launch_count() - c1))
        assert bool(torch.isfinite(loss)) and float(flow.grad.abs().max()) > 0
        assert torch.equal(gflow.grad, 0.001 * 65536.0 * torch.sign(gflow.detach()))
    assert counts == [(4 * 7 + 2, 4 + 1)] * 2, counts


def test_training_iteration_with_autocast_and_grad_scaler(scene):
    """A MirrorTrainer whose flow loss is the new op, under fp16 autocast and GradScaler, against the unchanged mirror."""
    from lidar4d_b200.chamfer import chamfer_3DDist
    from lidar4d_b200.losses import lidar_flow_loss
    from lidar4d_b200.optim import Adam
    from trainer_mirror import MirrorTrainer, default_opt, synthetic_batch
    pcs, grounds, clouds = scene

    class FlowOpTrainer(MirrorTrainer):
        def train_step(self, data):
            self.opt.flow_loss = False
            try:
                *rest, loss = super().train_step(data)
            finally:
                self.opt.flow_loss = True
            return (*rest, loss + lidar_flow_loss(self.model, clouds, data["time"], num_frames=self.opt.num_frames))

    losses = []
    for cls in (MirrorTrainer, FlowOpTrainer):
        model = _model()
        opt = default_opt(num_frames=NUM_FRAMES, num_steps=48, near_lidar=0.0105, far_lidar=0.851, fp16=True)
        train, _, _, _ = synthetic_batch(64, frame=2, num_frames=NUM_FRAMES, seed=1, device=DEV)
        train["time"] = train["time"] + 1e-4
        tr = cls(opt, model, chamfer_3DDist(), pc_list=pcs, pc_ground_list=grounds, device=DEV, fp16=True,
                 optimizer=lambda m: Adam(m, m.get_params(1e-2), betas=(0.9, 0.99), eps=1e-15))
        torch.manual_seed(11)
        losses.append(tr.train_iteration(train))
    assert np.isfinite(losses[0]) and abs(losses[1] - losses[0]) <= 1e-5 * abs(losses[0]), losses
    assert float(tr.scaler.get_scale()) == 65536.0
