"""CPU: pins tests/gather_ref.py, the float64 reference that tests/test_gpu_gather_exact.py holds the split forward's
encoder stage to, and the bound of the fp16 hi + lo feature encoding.

  * the reference equals the float64 oracle's density(return_features=True) within its bound, at points where float32
    and float64 texel weights coincide (dyadic coordinates i / 256: every step of l4d_axis is exact there);
  * the host build's features lie within the bound: hs_density_forward (the sample-major gather through the pair records,
    l4d_encode2_time / l4d_plane_sample) at points on cell and texel edges, on the faces of the box and outside it, and
    the SoA features a contracted render saves (l4d_encode2_con / l4d_row_sample, what k_fwd_gather runs), with warped
    positions on both sides of [0, 1], at the first, an interior and the last frame and at an interior frame whose current
    query is a single slice;
  * l4d_tile_emit's split x -> (hi, lo), emulated in numpy, stays inside the tensor-core bound 2^-22 |x| + 2^-25 at
    magnitudes 1e-6 .. 1 and breaks a purely relative 2^-22 below 2^-3; its tiles pass the structural checks, which must
    allow exact ties (fp16_rn(hi + lo) != hi where |lo| is exactly half an ulp of hi)."""
import numpy as np
import pytest
import torch

import gather_ref as GR
import hostsim_util as HU
import scatter_ref as SR
from lidar4d_b200.geometry import make_frame
from oracle import lidar4d_oracle as O
from parity_util import small_config, test_rays as _rays
from test_scatter_ref import _edge_coords

FRAMES = ["first", "interior", "last", "single"]


def frame_time(cfg, which: str) -> float:
    return {"first": 0.0, "interior": 0.4, "last": 1.0}.get(which) if which != "single" else GR.special_times(cfg)[0]


def hold(hs, fr, x01, flow, feats, flow_in=None):
    """Every feature (and flow-MLP input) of the host build hs against the reference; returns the worst fractions of the
    bound."""
    nK = GR.feature_terms(hs.cfg, fr)
    tabs = GR.Tables(hs.cfg, hs.params, fr)
    worst = [0.0, 0.0]

    def on(p0, p1, o):
        r, A = o["features"]
        worst[0] = max(worst[0], float(GR.ratio(feats[p0:p1], r, GR.bound32(A, nK)).max()))
        if flow_in is not None:
            r, A = o["flow_in"]
            worst[1] = max(worst[1], float(GR.ratio(flow_in[p0:p1], r, GR.bound32(A, GR.FLOW_TERMS)).max()))
    GR.gather_reference(tabs, x01, flow, on)
    return worst


@pytest.mark.parametrize("which", ["first", "interior", "last"])
def test_reference_equals_oracle(which):
    cfg = small_config()
    t = frame_time(cfg, which)
    orc = O.build_seeded(cfg, 5, flow_last_std=0.05)
    with torch.no_grad():
        orc.P["flow_net/mlp/4/weight"].zero_()                        # flow 0: warped positions are the sample's
    params32 = {k: v.detach().clone().float() for k, v in orc.ref_state_dict().items()}
    orc.to_float64()
    fr = make_frame(t, cfg.num_frames, cfg.time_resolution)
    g = torch.Generator().manual_seed(7)
    x01 = torch.randint(1, 256, (8192, 3), generator=g).float() / 256
    with torch.no_grad():
        o = orc.density(x01.double() * 2 - 1, fr, return_features=True)
    assert float(o["flow"].abs().max()) == 0.0
    tabs = GR.Tables(cfg, params32, fr)
    nK = GR.feature_terms(cfg, fr)
    worst = [0.0, 0.0]

    def on(p0, p1, d):
        r, A = d["features"]
        worst[0] = max(worst[0], float(GR.ratio(o["features"][p0:p1], r, GR.bound32(A, nK)).max()))
        r, A = d["flow_in"]
        worst[1] = max(worst[1], float(GR.ratio(o["flow_in"][p0:p1], r, GR.bound32(A, GR.FLOW_TERMS)).max()))
    GR.gather_reference(tabs, x01, torch.zeros(6, x01.shape[0]), on)
    assert worst[0] <= 1.0 and worst[1] <= 1.0, worst
    assert float(o["features"].abs().min(0).values.max()) > 0
    print(f"[gather-ref] oracle t={t}: worst {worst[0]:.2e} (features), {worst[1]:.2e} (flow inputs) of the bound")


def edge_points(cfg, n: int, seed: int) -> np.ndarray:
    """x01 coordinates on and around texel edges of every plane resolution and the time axis, on hash-cell edges of the
    static grid ((k - 0.5) / scale, where fmaf(scale, x, 0.5) is an integer), 0, 1 and outside [0, 1]; mixed per axis."""
    pool = [_edge_coords(cfg.min_resolution * m) for m in cfg.plane_scales] + [_edge_coords(cfg.time_resolution)]
    gs = cfg.static_grid()
    for l in range(cfg.n_levels_hash):
        s = float(gs.scale[l])
        k = np.arange(0, int(s) + 2, max(1, int(s) // 64))
        pool.append(((k - 0.5) / s).astype(np.float32))
    pool = np.unique(np.concatenate(pool))
    rng = np.random.default_rng(seed)
    return rng.choice(pool, (n, 3)).astype(np.float32)


@pytest.mark.parametrize("which", FRAMES)
@pytest.mark.parametrize("flow", ["small", "large"])
def test_host_density_features(which, flow):
    """hs_density_forward: world x = 2 x01 - 1 (bound 1); the reference takes the x01 the host build computes from it."""
    cfg = small_config(n_levels_hash=5)
    orc = O.build_seeded(cfg, 9, flow_last_std={"small": 0.02, "large": 1.0}[flow])
    hs = HU.HostSim(orc)
    t = frame_time(cfg, which)
    fr = make_frame(t, cfg.num_frames, cfg.time_resolution)
    xw = torch.from_numpy(edge_points(cfg, 6000, 1)).double().mul(2).sub(1).float()
    out = hs.density(xw, t)
    b = torch.tensor(cfg.bound, dtype=torch.float32)
    x01 = (xw + b) / (b * 2.0)
    on_edge = int(((x01 == 0) | (x01 == 1)).sum())
    assert on_edge > 0 and bool(((x01 < 0) | (x01 > 1)).any())
    fl = out["flow"].t().contiguous()
    w = torch.cat([x01 + fl[:3].t(), x01 + fl[3:].t()])
    if flow == "large":
        assert bool((w < 0).any()) and bool((w > 1).any())
    worst = hold(hs, fr, x01, fl, out["features"])
    assert worst[0] <= 1.0, worst
    print(f"[gather-ref] host density {which} t={t} {flow} flow: worst {worst[0]:.3f} of the bound")


@pytest.mark.parametrize("which", FRAMES)
@pytest.mark.parametrize("flow", ["small", "large"])
def test_host_contracted_render_features(which, flow):
    """The SoA features and flow-MLP inputs a contracted training render saves (k_fwd_gather's per-sample code)."""
    cfg = small_config(n_levels_hash=3, bound=0.5)
    orc = O.build_seeded(cfg, 11, flow_last_std={"small": 0.02, "large": 1.0}[flow])
    hs = HU.HostSim(orc)
    t = frame_time(cfg, which)
    fr = make_frame(t, cfg.num_frames, cfg.time_resolution)
    ro, rd = _rays(4, 8)
    S = 45
    out = hs.render(ro, rd, t, S, perturb=True, seed=3, train=True, contracted=True)
    N = ro.shape[0]
    sv = SR.decode_saved(cfg, hs._saved, N, S)
    x01 = SR.sample_x01(torch.from_numpy(ro), torch.from_numpy(rd), out["z_vals"], cfg.bound)
    assert bool(((x01 == 0) | (x01 == 1)).any())                       # samples clamped to the box
    fl = sv["flow"].t()
    w = torch.cat([x01 + fl[:, :3], x01 + fl[:, 3:]])
    if flow == "large":
        assert bool((w < 0).any()) and bool((w > 1).any())
    worst = hold(hs, fr, x01, sv["flow"], sv["feat"].t(), sv["flow_in"].t())
    assert worst[0] <= 1.0 and worst[1] <= 1.0, worst
    print(f"[gather-ref] host contracted render {which} t={t} {flow} flow: worst {worst[0]:.3f} / {worst[1]:.3f}")


def test_tile_emit_encoding_bound():
    """hi + lo of l4d_tile_emit: |hi + lo - x| <= 2^-22 |x| + 2^-25 for host features scaled to 1e-6 .. 1; a purely
    relative 2^-22 holds from 2^-3 up and fails below it (fp16 subnormal residuals)."""
    cfg = small_config(n_levels_hash=3)
    orc = O.build_seeded(cfg, 2)
    hs = HU.HostSim(orc)
    xw = torch.rand(4096, 3, generator=torch.Generator().manual_seed(0)) * 1.8 - 0.9
    f = hs.density(xw, 0.4)["features"].numpy()
    f = f / np.abs(f).max(1, keepdims=True)
    worst_rel_small, worst_rel_large = 0.0, 0.0
    for e in range(-6, 1):
        x = (f * np.float32(10.0 ** e)).astype(np.float32)
        hi, lo = GR.emulate_tile_emit(x)
        got = hi.astype(np.float64) + lo.astype(np.float64)
        err = np.abs(got - x.astype(np.float64))
        assert bool((err <= GR.ENC_REL * np.abs(x) + GR.ENC_ABS).all()), e
        nz = np.abs(x) >= np.float32(10.0 ** (e - 1))            # this decade
        rel = err[nz] / np.abs(x[nz])
        small = np.abs(x[nz]) < 2.0 ** -3
        if small.any():
            worst_rel_small = max(worst_rel_small, float(rel[small].max()))
        if (~small).any():
            worst_rel_large = max(worst_rel_large, float(rel[~small].max()))
        print(f"[gather-ref] tile emit at 1e{e}: max |hi+lo-x|/|x| {float(rel.max()):.2e}")
    assert worst_rel_large <= GR.ENC_REL, worst_rel_large
    assert worst_rel_small > 100 * GR.ENC_REL, worst_rel_small


def test_tile_structure_allows_exact_ties():
    """Emulated tiles of values at every magnitude pass check_tile_structure; among them are exact ties, where the sum
    hi + lo rounds to fp16 away from hi (so `fp16_rn(hi + lo) == hi` alone is not an invariant of the encoding), and a
    padding row or a ones column written wrong is counted."""
    cfg = small_config(n_levels_hash=3)
    K, S, xc = cfg.sigma_in_dim, 200, (cfg.sigma_in_dim + 7) // 8
    assert K % 8 != 0
    g = np.random.default_rng(0)
    x = (g.uniform(-1, 1, (3, S, K)) * 10.0 ** g.integers(-6, 2, (3, S, K))).astype(np.float32)
    hi, lo = GR.emulate_tile_emit(x)
    rows = np.zeros((3, 256, 2, xc * 8), np.float16)
    rows[:, :S, 0, :K], rows[:, :S, 1, :K], rows[:, :S, 0, K:] = hi, lo, 1.0
    as_tiles = lambda r: torch.from_numpy(r).view(3, 2, 128, 2, xc, 8).permute(0, 1, 3, 4, 2, 5).contiguous()
    assert GR.check_tile_structure(cfg, as_tiles(rows), S) == dict(nonfinite=0, padding=0, ones=0, split=0)
    ties = (hi.astype(np.float32) + lo.astype(np.float32)).astype(np.float16) != hi
    assert int(ties.sum()) > 0
    bad = rows.copy()
    bad[0, S + 3, 1, 5] = 1e-7
    bad[1, 7, 0, K + 1] = 0.0
    bad[2, 9, 0, 0], bad[2, 9, 1, 0] = 1.0, 2.0 ** -10                # |lo| above half an ulp of hi
    got = GR.check_tile_structure(cfg, as_tiles(bad), S)
    assert got["padding"] == 1 and got["ones"] == 1 and got["split"] >= 1, got
