"""GPU: lidar4d_b200.misc (range filter, Open3D's statistical outlier removal, RANSAC ground removal, process_pointcloud)
against tests/golden/ground_ref.npz - the reference's own utils/misc.py and Trainer.process_pointcloud - and
oracle/ground_oracle.py.

Range-filter masks are bit-exact.  k-NN means are within 1e-13 relative of the oracle.  Outlier and RANSAC decisions
are identical except on points the oracle flags as within 4 ulps of a threshold (a parallel reduction or BLAS may decide
those either way); such points are counted, reported and must be at most 1e-4 of the cloud."""
import os
import random
import sys

import numpy as np
import pytest
import torch

from oracle import ground_oracle as GO
import ground_cases as GC

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
import make_ground_golden as MG  # noqa: E402

GOLD = os.path.join(os.path.dirname(__file__), "golden", "ground_ref.npz")
CASES = ["sweep_a", "sweep_b", "small70", "small200", "dup"]
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fx():
    return np.load(GOLD, allow_pickle=False)


def _cloud(fx, name):
    return GC.cloud(fx, name) if name.startswith("sweep") else fx[f"{name}_points"]


def _stages(fx, name):
    pc = _cloud(fx, name)
    rf = GC.unpack(fx[f"{name}_rf_keep"])
    pc1 = pc[rf].astype(np.float64)[GC.unpack(fx[f"{name}_sor1_keep"])]
    return pc, rf, pc1


def _allowed(got, want, near, n, what):
    diff = np.setxor1d(got, want)
    bad = np.setdiff1d(diff, near)
    print(f"[{what}] {len(diff)} decisions differ, all within 4 ulps of the threshold ({len(near)} flagged of {n})")
    assert len(bad) == 0, f"{what}: {len(bad)} decisions differ away from the threshold: {bad[:10]}"
    assert len(diff) <= 1e-4 * n


@pytest.mark.parametrize("name", CASES)
def test_range_filter_bit_exact(fx, name):
    from lidar4d_b200.misc import range_filter
    pc = _cloud(fx, name)
    tagged = torch.from_numpy(np.concatenate([pc, np.arange(len(pc), dtype=np.float32)[:, None]], 1)).cuda()
    out = range_filter(tagged).cpu().numpy()
    rf = GC.unpack(fx[f"{name}_rf_keep"])
    assert np.array_equal(out[:, 3].astype(np.int64), rf)
    assert np.array_equal(out[:, :3].view(np.uint32), pc[rf].view(np.uint32))


@pytest.mark.parametrize("name", CASES)
def test_outlier_removal_stage(fx, name):
    from lidar4d_b200.misc import knn_mean_dist, statistical_outlier_removal
    pc, rf, _ = _stages(fx, name)
    p = pc[rf].astype(np.float64)
    avg = knn_mean_dist(torch.from_numpy(p).cuda()).cpu().numpy()
    ref = GO.knn_mean_dist(p)
    assert np.all(np.abs(avg - ref) <= 1e-13 * np.abs(ref))
    pts, ind = statistical_outlier_removal(torch.from_numpy(p).cuda(), 64, 3.0)
    ind = ind.cpu().numpy()
    assert np.array_equal(pts.cpu().numpy(), p[ind])
    _, near, _, _ = GO.statistical_outlier_removal(p)
    _allowed(ind, GC.unpack(fx[f"{name}_sor1_keep"]), np.flatnonzero(near), len(p), f"{name} outliers")


@pytest.mark.parametrize("name", CASES)
def test_ransac_counts(fx, name):
    from lidar4d_b200 import misc
    _, _, pc1 = _stages(fx, name)
    pts = torch.from_numpy(pc1).cuda()
    mask = torch.zeros(len(pc1), dtype=torch.uint8, device="cuda")
    random.seed(int(fx[f"{name}_seed"]))
    got = [misc._ransac_into(pts, pc1, mask, 0.15)[1] for _ in range(6)]
    random.seed(int(fx[f"{name}_seed"]))
    nears = [GO.my_ransac(pc1, distance_threshold=0.15)[3] for _ in range(6)]
    for j in range(6):
        want = fx[f"{name}_ransac_counts_{j}"].tolist()
        assert len(got[j]) == len(want)
        slack = [abs(a - b) for a, b in zip(got[j], want)]
        assert all(s <= n for s, n in zip(slack, nears[j])), (j, got[j], want)


@pytest.mark.parametrize("name", CASES)
def test_point_removal_end_to_end(fx, name):
    from lidar4d_b200.misc import point_removal_stages, point_removal
    pc, _, pc1 = _stages(fx, name)
    random.seed(int(fx[f"{name}_seed"]))
    st = point_removal_stages(torch.from_numpy(pc).cuda())
    assert np.array_equal(random.getstate()[1], fx[f"{name}_rng_state"])
    for k, key in (("rf_keep", "rf_keep"), ("sor1_keep", "sor1_keep"), ("ground_index", "ground"), ("sor2_keep", "sor2_keep")):
        assert np.array_equal(st[k].cpu().numpy(), GC.unpack(fx[f"{name}_{key}"])), k
    for j in range(6):
        assert st["ransac_counts"][j] == fx[f"{name}_ransac_counts_{j}"].tolist()
    g = GC.unpack(fx[f"{name}_ground"])
    rest = np.delete(pc1, g, axis=0)
    assert np.array_equal(st["ground"].cpu().numpy(), pc1[g])
    assert np.array_equal(st["points"].cpu().numpy(), rest[GC.unpack(fx[f"{name}_sor2_keep"])])
    random.seed(int(fx[f"{name}_seed"]))
    a = point_removal(torch.from_numpy(pc).cuda())
    random.seed(int(fx[f"{name}_seed"]))
    b = point_removal(torch.from_numpy(pc).cuda())
    assert all(torch.equal(x, y) for x, y in zip(a, b))          # repeated calls are bit-identical


def _loader(dtype, times=(MG.CHAIN["time"],)):
    img, pose, _ = MG.chain_inputs()
    return [{"images_lidar": torch.from_numpy(img).to(dtype).cuda(), "poses_lidar": torch.from_numpy(pose).cuda(),
             "time": torch.tensor([[t]], dtype=torch.float32, device="cuda")} for t in times]


@pytest.mark.parametrize("tag,dtype", [("f32", torch.float32), ("f16", torch.float16)])
def test_process_pointcloud(fx, tag, dtype):
    """Given the cloud the reference unprojected, process_frame's float64 clouds are within 1e-12 relative of the
    reference's; end to end (with this project's unprojection, whose float32 trig may differ by an ulp from NumPy's)
    the same points come out, within a few float32 ulps."""
    from lidar4d_b200.misc import pano_depth, process_frame, process_pointcloud
    from lidar4d_b200.convert import pano_to_lidar
    img, pose, _ = MG.chain_inputs()
    pc_raw = fx[f"chain_{tag}_pc_raw"]
    got_raw = pano_to_lidar(pano_depth(torch.from_numpy(img).to(dtype).cuda(), MG.CHAIN["scale"]), GC.K).cpu().numpy()
    assert got_raw.shape == pc_raw.shape
    assert np.all(np.abs(got_raw - pc_raw) <= 2e-6 * np.linalg.norm(pc_raw, axis=1, keepdims=True))
    want = (fx[f"chain_{tag}_points"], fx[f"chain_{tag}_ground"])
    random.seed(MG.CHAIN["seed"])
    got = process_frame(torch.from_numpy(pc_raw).cuda(), torch.from_numpy(pose), MG.CHAIN["scale"])
    assert np.array_equal(random.getstate()[1], fx[f"chain_{tag}_rng_state"])
    for g, w in zip(got, want):
        assert g.dtype == np.float64 and g.shape == w.shape
        assert np.all(np.abs(g - w) <= 1e-12 * np.linalg.norm(w, axis=1, keepdims=True))
    random.seed(MG.CHAIN["seed"])
    pcs, grounds = process_pointcloud(_loader(dtype), MG.CHAIN["scale"], MG.CHAIN["num_frames"], GC.K)
    key = str(fx[f"chain_{tag}_key"])
    assert list(pcs) == [key] and list(grounds) == [key]
    for g, w in zip((pcs[key], grounds[key]), want):
        assert g.dtype == np.float64 and g.shape == w.shape
        assert np.all(np.abs(g - w) <= 1e-6 * np.linalg.norm(w, axis=1, keepdims=True))


@pytest.mark.parametrize("n", [3, 63, 64, 65, 67980])
def test_knn_sizes(n):
    from lidar4d_b200.misc import knn_mean_dist, statistical_outlier_removal
    g = np.random.default_rng(n)
    p = GC._q(g.uniform(-40, 40, (n, 3))).astype(np.float64)
    if n > 100:
        p[100:180] = p[5]                                       # a cluster of 81 duplicates: mean distance 0
    avg = knn_mean_dist(torch.from_numpy(p).cuda()).cpu().numpy()
    ref = GO.knn_mean_dist(p)
    assert np.all(np.abs(avg - ref) <= 1e-13 * np.abs(ref))
    if n > 100:
        assert np.all(avg[100:180] == 0)
    _, ind = statistical_outlier_removal(torch.from_numpy(p).cuda(), 64, 3.0)
    want, near, _, _ = GO.statistical_outlier_removal(p)
    _allowed(ind.cpu().numpy(), want, np.flatnonzero(near), n, f"n={n}")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_knn_grid_wraps():
    """n = 2 x (4 CTAs per SM x SMs) x 128 + 37 queries: every CTA of the k-NN grid (at most 3 per SM fit its 72 KB of
    shared memory) takes at least two query blocks."""
    from lidar4d_b200.misc import knn_mean_dist
    n = 2 * 4 * _sms() * 128 + 37
    g = np.random.default_rng(5)
    p = GC._q(g.normal(0, 15, (n, 3))).astype(np.float64)
    avg = knn_mean_dist(torch.from_numpy(p).cuda(), 64).cpu().numpy()
    ref = GO.knn_mean_dist(p)
    assert np.all(np.abs(avg - ref) <= 1e-13 * np.abs(ref))


def test_compaction_and_scoring_grids_wrap():
    """n = 2 x 16 x SMs x 1024 + 37 points: every CTA of the compaction and scoring grids (16 CTAs per SM) takes at
    least two tiles.  Range filter, outlier selection on given means, plane scores and mask, ground split, pose."""
    from lidar4d_b200 import misc
    n = 2 * 16 * _sms() * 1024 + 37
    g = np.random.default_rng(6)
    p32 = GC._q(g.uniform(-60, 60, (n, 3)) * [1, 1, 0.1])
    out = misc.range_filter(torch.from_numpy(p32).cuda()).cpu().numpy()
    assert np.array_equal(out, p32[GO.range_filter_mask(p32)[0]])
    p = p32.astype(np.float64)
    dp = torch.from_numpy(p).cuda()
    avg = g.uniform(0.0, 1.0, n)
    avg[::97] = 0.0
    stats = torch.empty(3, dtype=torch.float64, device="cuda")
    pts, ind = misc._select(dp, torch.from_numpy(avg).cuda(), 2.0, stats)
    thr, mean, std = GO.outlier_stats(avg, 2.0)
    s = stats.cpu().numpy()
    assert abs(s[1] - mean) <= 1e-12 * mean and abs(s[2] - std) <= 1e-12 * std
    want = np.flatnonzero((avg > 0) & (avg < thr))
    _allowed(ind.cpu().numpy(), want, np.flatnonzero(GO._near(avg, thr)), n, "select")
    assert np.array_equal(pts.cpu().numpy(), p[ind.cpu().numpy()])
    hyp = np.array([[0.01, -0.02, 1.0, 1.7], [1.0, 0.5, 0.0, -3.0], [0.0, 0.0, 2.0, -1.0]])
    hyp = np.concatenate([hyp, np.sqrt((hyp[:, :3] ** 2).sum(1))[:, None]], 1)
    counts = misc._plane_scorer(dp, 0.15)(hyp)
    mask = torch.zeros(n, dtype=torch.uint8, device="cuda")
    union = np.zeros(n, bool)
    for h, c in zip(hyp, counts):
        d = GO.plane_distances(p, h[:4], h[4])
        assert abs(int(c) - int((d < 0.15).sum())) <= int(GO._near(d, 0.15).sum())
        misc._mark_plane(dp, h[:4], h[4], 0.15, mask)
        union |= d < 0.15
    ground, gi, rest, ri = misc._split(dp, mask, -1.0)
    gm = union & (p[:, 2] < -1)
    assert np.array_equal(gi.cpu().numpy(), np.flatnonzero(gm)) and np.array_equal(ri.cpu().numpy(), np.flatnonzero(~gm))
    assert np.array_equal(ground.cpu().numpy(), p[gm]) and np.array_equal(rest.cpu().numpy(), p[~gm])
    pose = np.array([[0.6, -0.8, 0, 3.5], [0.8, 0.6, 0, -1.25], [0, 0, 1, 0.5], [0, 0, 0, 1]], np.float32)
    got = misc._transform(dp, pose, 0.01).cpu().numpy()
    X = p * 0.01
    P = pose.astype(np.float64)
    want = ((P[:3, 0] * X[:, :1] + P[:3, 1] * X[:, 1:2]) + P[:3, 2] * X[:, 2:3]) + P[:3, 3]
    assert np.array_equal(got, want)


def test_error_paths(monkeypatch):
    from lidar4d_b200 import misc
    with pytest.raises(ValueError):
        misc.my_ransac(torch.zeros(2, 3, dtype=torch.float64, device="cuda"))
    flat = np.zeros((50, 3))
    flat[:, 0] = np.arange(50)                                   # every draw fails |y0 - y1| >= 3
    monkeypatch.setattr(misc, "MAX_CONSECUTIVE_REJECTIONS", 2000)
    state = random.getstate()
    with pytest.raises(RuntimeError, match="rejected"):
        misc.my_ransac(torch.from_numpy(flat).cuda(), distance_threshold=0.15)
    random.setstate(state)


def test_flow_loss_iteration_on_processed_clouds():
    """The trainer's calling pattern (tests/trainer_mirror.py) runs a flow-loss training iteration on the pc_list /
    pc_ground_list process_pointcloud builds from a synthetic loader."""
    from lidar4d_b200.chamfer import chamfer_3DDist
    from lidar4d_b200.misc import process_pointcloud
    from lidar4d_b200.optim import Adam
    from oracle import lidar4d_oracle as O
    from parity_util import small_config, cuda_model_from_oracle
    from trainer_mirror import MirrorTrainer, default_opt, synthetic_batch
    dev = torch.device("cuda:0")
    random.seed(0)
    pcs, grounds = process_pointcloud(_loader(torch.float16, times=[k / 5 for k in range(5)]), 0.01, 6, GC.K)
    assert sorted(pcs) == ["0", "1", "2", "3", "4"]
    model = cuda_model_from_oracle(O.build_seeded(small_config(), 3, flow_last_std=0.02))
    opt = default_opt(num_frames=6, num_steps=48, near_lidar=0.0105, far_lidar=0.851, fp16=False)
    train, _, _, _ = synthetic_batch(64, frame=2, num_frames=6, seed=1, device=dev)
    tr = MirrorTrainer(opt, model, chamfer_3DDist(), pc_list=pcs, pc_ground_list=grounds, device=dev,
                       optimizer=lambda m: Adam(m, m.get_params(1e-2), betas=(0.9, 0.99), eps=1e-15))
    loss = tr.train_iteration(train)
    assert np.isfinite(loss)


def test_point_removal_takes_host_arrays(fx):
    """As runner.py:938-941 calls it (with lidar4d_b200.misc in place of utils.misc): a NumPy cloud in, float64 NumPy
    clouds out, the same as the CUDA path."""
    from lidar4d_b200.misc import point_removal
    pc = fx["small200_points"]
    random.seed(int(fx["small200_seed"]))
    pts, ground = point_removal(pc)
    assert isinstance(pts, np.ndarray) and pts.dtype == np.float64 and ground.dtype == np.float64
    assert np.array_equal(random.getstate()[1], fx["small200_rng_state"])
    random.seed(int(fx["small200_seed"]))
    d_pts, d_ground = point_removal(torch.from_numpy(pc).cuda())
    assert np.array_equal(pts, d_pts.cpu().numpy()) and np.array_equal(ground, d_ground.cpu().numpy())
