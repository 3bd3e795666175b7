"""CPU: pins tests/scatter_ref.py, the float64 reference that tests/test_gpu_scatter_exact.py holds the backward's
scatter stage to.  A wrong reference could let the GPU test pass for the wrong reason, so:

  * its saved-buffer layout is the one the library computes (l4d_saved_bytes, via the host build of l4d_host.h);
  * its float32 texel arithmetic is the kernels' l4d_bilerp bit for bit, at and around every place where it branches;
  * with random dL/dfeature it equals torch.autograd.grad of sum <dfeat, features> through the oracle's encoders in
    float64, at the first, an interior and the last frame, and its dL/dflow equals autograd w.r.t. the flow."""
import ctypes as C

import numpy as np
import pytest
import torch

import hostsim_util as HU
import scatter_ref as SR
from lidar4d_b200 import _capi
from lidar4d_b200.geometry import make_frame
from oracle import lidar4d_oracle as O
from parity_util import small_config, full_config


@pytest.mark.parametrize("cfg_name,n,S", [("small", 1, 2), ("small", 37, 333), ("L3", 5, 45), ("L5", 300, 129),
                                           ("full16", 4261, 768)])
def test_saved_layout_matches_library(cfg_name, n, S):
    cfg = {"small": small_config(), "L3": small_config(n_levels_hash=3), "L5": small_config(n_levels_hash=5),
           "full16": full_config(16)}[cfg_name]
    lib = HU.lib()
    want = lib.hs_saved_bytes(C.byref(_capi.make_config(cfg, True)), n, S)
    assert want > 0
    assert SR.saved_layout(cfg, n, S)["total"] == want


def _host_bilerp(cx, cy, W, H):
    lib = HU.lib()
    f = lib.hs_bilerp
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    f.restype = C.c_int
    cx, cy = np.ascontiguousarray(cx, np.float32), np.ascontiguousarray(cy, np.float32)
    n = cx.size
    idx, w = np.zeros((n, 4), np.int32), np.zeros((n, 6), np.float32)
    assert f(cx.ctypes.data, cy.ctypes.data, n, W, H, idx.ctypes.data, w.ctypes.data) == 0
    return idx, w


def _edge_coords(size: int) -> np.ndarray:
    """< 0, 0, every texel centre i/(size-1) and one ulp either side of it (where floor() of the pixel coordinate
    changes), the midpoints, 1 and > 1."""
    c = np.arange(size, dtype=np.float64) / (size - 1)
    e = c.astype(np.float32)
    pts = [np.float32([-0.5, -1e-7, -0.0, 0.0, 1.0, 1.0 + 1e-7, 1.5, np.float32(1) - np.float32(2 ** -24)]),
           e, np.nextafter(e, np.float32(-1)), np.nextafter(e, np.float32(2)),
           ((np.arange(size - 1) + 0.5) / (size - 1)).astype(np.float32)]
    return np.concatenate(pts).astype(np.float32)


@pytest.mark.parametrize("size", [2, 8, 9, 16, 32, 64, 100, 128, 256, 512])
def test_axis_matches_kernel_bilerp(size):
    cx = _edge_coords(size)
    cy = np.resize(np.random.default_rng(size).permutation(_edge_coords(8)), cx.size)
    idx, w = _host_bilerp(cx, cy, size, 8)
    for k, (c, s) in enumerate(((cx, size), (cy, 8))):
        i0, i1, w0, w1, gm = SR.axis(torch.from_numpy(c), s)
        assert np.array_equal(i0.numpy(), idx[:, 2 * k]), (size, k)
        assert np.array_equal(i1.numpy(), idx[:, 2 * k + 1]), (size, k)
        for got, col in ((w0, 2 * k), (w1, 2 * k + 1), (gm, 4 + k)):
            assert np.array_equal(got.numpy().view(np.uint32), w[:, col].view(np.uint32)), (size, k, col)


def test_sample_x01_matches_kernel_positions():
    """The sample positions the reference scatters at are the host build's z / x01 arithmetic, clamped samples included."""
    cfg = small_config(bound=0.5)
    hs = HU.HostSim(O.build_seeded(cfg, 2))
    rng = np.random.default_rng(0)
    ro = rng.uniform(-0.4, 0.4, (16, 3)).astype(np.float32)
    rd = rng.normal(size=(16, 3)).astype(np.float32)
    rd /= np.linalg.norm(rd, axis=1, keepdims=True)
    out = hs.render(ro, rd, 0.4, 64, perturb=True, seed=3)
    x01 = SR.sample_x01(torch.from_numpy(ro), torch.from_numpy(rd), out["z_vals"], cfg.bound)
    b = np.float32(cfg.bound)
    p = np.clip(ro[:, None, :] + rd[:, None, :] * out["z_vals"].numpy()[:, :, None], -b, b)
    want = ((p + b) / (b * np.float32(2))).reshape(-1, 3)
    assert np.array_equal(x01.numpy(), want)
    assert bool((x01 == 0).any()) and bool((x01 == 1).any())          # samples on the faces of the box


def _interior_points(cfg, x01: torch.Tensor, flow: torch.Tensor, margin: float = 0.02) -> torch.Tensor:
    """Points whose plane coordinates (current and warped) sit at least `margin` of a texel away from every texel
    edge at every scale, so that float32 and float64 texel selection and weights agree to ~1e-7 of a texel."""
    ok = torch.ones(x01.shape[0], dtype=torch.bool)
    coords = [x01, x01 + flow[:, :3], x01 + flow[:, 3:]]
    for s in range(cfg.n_levels_plane):
        R = cfg.min_resolution * cfg.plane_scales[s]
        for c in coords:
            ix = c.double() * (R - 1)
            fr = ix - torch.floor(ix)
            ok &= ((fr > margin) & (fr < 1 - margin) & (ix > 0) & (ix < R - 1)).all(1)
    return ok


@pytest.mark.parametrize("t", [0.0, 0.4, 1.0], ids=["first", "interior", "last"])
def test_reference_equals_autograd(t):
    cfg = small_config()
    orc = O.build_seeded(cfg, 5, flow_last_std=0.05)
    params32 = {k: v.detach().clone().float() for k, v in orc.ref_state_dict().items()}
    orc.to_float64()
    fr = make_frame(t, cfg.num_frames, cfg.time_resolution)
    assert (fr.has_fwd, fr.has_bwd) == {0.0: (True, False), 0.4: (True, True), 1.0: (False, True)}[t]
    g = torch.Generator().manual_seed(7)
    b = cfg.bound
    x = (torch.rand(16384, 3, generator=g) * 0.9 + 0.05) * 2 * b - b
    x01 = (x.float() + b) / (2 * b)                                     # the oracle's float32 x01 (density())
    with torch.no_grad():
        flow0 = orc.density(x, fr, return_features=True)["flow"]
    keep = _interior_points(cfg, x01, flow0.float())
    assert int(keep.sum()) > 2000
    x, x01 = x[keep], x01[keep]
    out = orc.density(x, fr, return_features=True)
    feats, flow, fin = out["features"], out["flow"], out["flow_in"]
    dfeat = torch.randn(feats.shape, generator=g, dtype=torch.float64).float()
    names = [k for k in params32 if k != "aabb" and ("hash" in k or "planes" in k or "grid_enc" in k)]
    targets = [orc.p(k) for k in names] + [flow, fin]
    grads = torch.autograd.grad((feats * dfeat.double()).sum(), targets, allow_unused=True)
    want = {k: (gk if gk is not None else torch.zeros_like(orc.p(k))) for k, gk in zip(names, grads)}
    dflow_want, dfin = grads[-2], grads[-1]

    ref = SR.scatter_reference(cfg, params32, fr, x01, dfeat, flow.detach().float().t().contiguous(),
                               dfin.float().t().contiguous())
    checked, worst = 0, 0.0
    for k in names:
        r = ref[k]
        err = (want[k].reshape(-1) - r[:, 0]).abs()
        bad = (err > 1e-3 * r[:, 1]) | ((r[:, 2] == 0) & (want[k].reshape(-1) != 0))
        assert not bool(bad.any()), (k, int(bad.sum()), float(err.max()))
        worst = max(worst, float((err / r[:, 1].clamp_min(1e-300)).max()))
        checked += int((r[:, 2] > 0).sum())
    assert float(want["flow_net.grid_enc.params"].abs().max()) > 0      # the flow grid got gradient through dL/dFin
    dw = dflow_want if dflow_want is not None else torch.zeros(x01.shape[0], 6, dtype=torch.float64)
    r = ref["dflow"]
    assert bool(((dw - r[..., 0]).abs() <= 1e-3 * r[..., 1]).all())
    live = [0, 1, 2] * fr.has_fwd + [3, 4, 5] * fr.has_bwd
    assert float(dw[:, live].abs().max()) > 0
    dead = [k for k in range(6) if k not in live]
    assert float(r[:, dead, 2].sum()) == 0 and float(dw[:, dead].abs().sum()) == 0
    assert checked > 10000
    print(f"[scatter-ref] t={t}: {int(keep.sum())} points, {checked} entries, worst |diff| / A {worst:.2e}")
