"""The image-metric kernels' arithmetic compiled for the CPU (tests/hostsim/imgmetricssim.cu over
lidar4d_b200/csrc/l4d_imgmetrics.cuh, contraction off) against SciPy and the oracle:
  - the column and row recurrences give the five filtered maps bit-identical to scipy.ndimage.uniform_filter;
  - the S-map function is bit-identical to the oracle's float32 expression given the same C1 / C2;
  - the clamp, |gt - pred|, the column sums and gt's NaN-propagating min / max are what NumPy computes."""
import ctypes as C
import os

import numpy as np
import pytest
from scipy.ndimage import uniform_filter

import image_metrics_cases as IC
from oracle import image_metrics_oracle as IO

SO = os.path.join(os.path.dirname(__file__), "hostsim", "_imgmetricssim.so")
FX = np.load(os.path.join(os.path.dirname(__file__), "golden", "image_metrics_ref.npz"), allow_pickle=False)


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(SO):
        pytest.fail(f"{SO} missing: run __graft_entry__.build()")
    h = C.CDLL(SO)
    P = C.c_void_p
    h.ims_maps.argtypes = [P, P, C.c_int, C.c_int, C.c_float, C.c_float, P, P, P, P, P, P, P]
    h.ims_line.argtypes = [P, C.c_int, P]
    h.ims_consts.argtypes = [C.c_float, C.c_float, P]
    h.ims_smap.argtypes = [P, C.c_size_t, C.c_float, C.c_float, P]
    return h


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def run_maps(lib, pred, gt, lo, hi):
    H, W = pred.shape
    pred, gt = np.ascontiguousarray(pred, np.float32), np.ascontiguousarray(gt, np.float32)
    cp, cg, ad = (np.empty((H, W), np.float32) for _ in range(3))
    maps = np.empty((5, H, W), np.float32)
    sq, mn, mx = np.empty(W), np.empty(W, np.float32), np.empty(W, np.float32)
    lib.ims_maps(_p(pred), _p(gt), H, W, lo, hi, _p(cp), _p(cg), _p(ad), _p(maps), _p(sq), _p(mn), _p(mx))
    return cp, cg, ad, maps, sq, mn, mx


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


@pytest.mark.parametrize("name", IC.IMAGE_CASES)
def test_maps_match_scipy_on_cases(lib, name):
    kind, p, g = IC.frame(FX, name)
    lo, hi, _ = IO.DEPTH if kind == "depth" else IO.INTENSITY
    lo, hi = np.float32(lo), np.float32(hi)
    cp, cg, ad, maps, sq, mn, mx = run_maps(lib, p[0], g[0], lo, hi)
    rp, rg = p[0].copy(), g[0].copy()
    for a in (rp, rg):
        a[a < lo] = lo
        a[a > hi] = hi
    assert _bits_equal(cp, rp) and _bits_equal(cg, rg)
    assert _bits_equal(ad, np.abs(rg - rp))
    for k, ref in enumerate(IO.filtered_maps(rp, rg)):
        assert _bits_equal(maps[k], ref), f"map {k}"
    d2 = ((rg - rp) ** 2).astype(np.float64)
    np.testing.assert_allclose(sq, d2.sum(0), rtol=1e-12)
    assert _bits_equal(mn, np.min(rg, 0)) and _bits_equal(mx, np.max(rg, 0))     # np.min / np.max propagate NaN


@pytest.mark.parametrize("mag", [1e-3, 1.0, 80.0])
@pytest.mark.parametrize("shape", [(66, 1030), (7, 7), (9, 8), (128, 257)])
def test_maps_match_scipy_random(lib, mag, shape):
    g = np.random.default_rng(7 + int(mag) + shape[1])
    x = (g.random(shape) * mag).astype(np.float32)
    y = (g.random(shape) * mag).astype(np.float32)
    maps = run_maps(lib, x, y, np.float32(-np.inf), np.float32(np.inf))[3]
    for k, ref in enumerate(IO.filtered_maps(x, y)):
        assert _bits_equal(maps[k], ref), f"map {k}"
    line = np.ascontiguousarray(x[0])
    out = np.empty_like(line)
    lib.ims_line(_p(line), len(line), _p(out))
    assert _bits_equal(out, uniform_filter(line, 7))


@pytest.mark.parametrize("name", IC.IMAGE_CASES)
def test_ssim_map_matches_oracle(lib, name):
    kind, p, g = IC.frame(FX, name)
    lo, hi, _ = IO.DEPTH if kind == "depth" else IO.INTENSITY
    cp, cg, _, maps, _, mn, mx = run_maps(lib, p[0], g[0], np.float32(lo), np.float32(hi))
    c = np.empty(2, np.float32)
    gmin, gmax = np.float32(np.min(cg)), np.float32(np.max(cg))
    lib.ims_consts(gmin, gmax, _p(c))
    with np.errstate(all="ignore"):
        C1, C2 = IO.ssim_constants(gmax - gmin, "mul")
        ref = IO.ssim_map(*IO.filtered_maps(cp, cg), C1, C2)
    assert _bits_equal(c, [C1, C2]) or (np.isnan(c).all() and np.isnan(C1))
    S = np.empty(maps[0].size, np.float32)
    lib.ims_smap(_p(maps), maps[0].size, C1, C2, _p(S))
    assert _bits_equal(S.reshape(ref.shape), ref)


def test_ssim_map_extremes(lib):
    """Random filtered maps with zero, tiny and large variances and every C1 / C2 regime."""
    g = np.random.default_rng(11)
    n = 200_000
    ux = g.choice([0.0, 1e-6, 0.5, 79.99], n).astype(np.float32) + g.random(n).astype(np.float32) * 1e-3
    uy = (ux + g.normal(0, 0.01, n)).astype(np.float32)
    uxx = (ux * ux + g.random(n) * 1e-3).astype(np.float32)
    uyy = (uy * uy + g.random(n) * 1e-3).astype(np.float32)
    uxy = (ux * uy + g.normal(0, 1e-4, n)).astype(np.float32)
    maps = np.ascontiguousarray(np.stack([ux, uy, uxx, uyy, uxy]))
    for R in (np.float32(0.0), np.float32(1.0), np.float32(79.999)):
        C1, C2 = IO.ssim_constants(R, "mul")
        with np.errstate(all="ignore"):
            ref = IO.ssim_map(ux, uy, uxx, uyy, uxy, C1, C2)
        S = np.empty(n, np.float32)
        lib.ims_smap(_p(maps), n, C1, C2, _p(S))
        assert _bits_equal(S, ref)
