"""CPU: the per-pixel rule of k_sweep_images compiled for the host (tests/hostsim/sweepsim.cu over
lidar4d_b200/csrc/l4d_sweep.cuh, contraction off) against NumPy, which is what the reference runs:
  - u8(r * 255) in float16 on all 65,536 half bit patterns;
  - u8(x * 255) in float32 on every float32 within 4 ulps of k/255, k = 0..256;
  - each dtype path (16 / 32 / 64) and the raw casts on 10^6 random values, out-of-range values, inf and NaN included;
  - the whole pixel function of every layout against oracle/sweep_oracle.py on the golden frames."""
import ctypes as C
import os

import numpy as np
import pytest

import sweep_cases as SC
from oracle import sweep_oracle as SO

SO_PATH = os.path.join(os.path.dirname(__file__), "hostsim", "_sweepsim.so")
FX = np.load(os.path.join(os.path.dirname(__file__), "golden", "sweep_ref.npz"), allow_pickle=False)
SIM, TEST, EVAL = 0, 1, 2


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(SO_PATH):
        pytest.fail(f"{SO_PATH} missing: run __graft_entry__.build()")
    h = C.CDLL(SO_PATH)
    P, N = C.c_void_p, C.c_size_t
    h.sws_r255_f16.argtypes = [P, N, P]
    h.sws_x255_f32.argtypes = [P, N, P]
    h.sws_x255_f64.argtypes = [P, P, N, P]
    h.sws_u8_f32.argtypes = [P, N, P]
    h.sws_u8_f64.argtypes = [P, N, P]
    h.sws_pixels.argtypes = [C.c_uint32, C.c_int, P, P, P, N, C.c_float, C.c_int, P, P, P]
    return h


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _call(fn, *arrays, out_n):
    out = np.empty(out_n, np.uint8)
    fn(*[_p(np.ascontiguousarray(a)) for a in arrays], out_n, _p(out))
    return out


def _wild(rng, n, dtype):
    """n values of `dtype`: mostly [-2, 3), then large, huge, +-inf and NaN."""
    x = rng.uniform(-2, 3, n)
    k = rng.integers(0, 6, n)
    x = np.where(k == 1, rng.uniform(-1e4, 1e4, n), x)
    x = np.where(k == 2, rng.uniform(-1e10, 1e10, n), x)
    x = np.where(k == 3, np.array([np.inf, -np.inf, np.nan, 2.0 ** 31, -(2.0 ** 31), 2.0 ** 31 - 1])[rng.integers(0, 6, n)], x)
    with np.errstate(over="ignore"):
        return x.astype(dtype)


def test_float16_all_bit_patterns(lib):
    h = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    r = h.view(np.float16)
    with np.errstate(all="ignore"):
        want = (r * 255).astype(np.uint8)
    got = _call(lib.sws_r255_f16, h, out_n=h.size)
    assert np.array_equal(got, want)
    with np.errstate(all="ignore"):
        finite = np.isfinite(r) & (r >= 0) & (r <= 1)
        diff = (r[finite] * 255).astype(np.uint8) != (r[finite].astype(np.float32) * 255).astype(np.uint8)
    assert diff.any()                              # the half product really differs from the float32 one


def test_float32_near_k_over_255(lib):
    base = (np.arange(257) / 255.0).astype(np.float32)
    xs = [base]
    up, down = base.copy(), base.copy()
    for _ in range(4):
        up, down = np.nextafter(up, np.float32(np.inf)), np.nextafter(down, np.float32(-np.inf))
        xs += [up, down]
    x = np.concatenate(xs)
    assert np.array_equal(_call(lib.sws_x255_f32, x, out_n=x.size), (x * 255).astype(np.uint8))


def test_random_values_every_dtype_path(lib):
    rng = np.random.default_rng(5)
    n = 10 ** 6
    with np.errstate(all="ignore"):
        x16 = _wild(rng, n, np.float16)
        assert np.array_equal(_call(lib.sws_r255_f16, x16.view(np.uint16), out_n=n), (x16 * 255).astype(np.uint8))
        x32 = _wild(rng, n, np.float32)
        assert np.array_equal(_call(lib.sws_x255_f32, x32, out_n=n), (x32 * 255).astype(np.uint8))
        m = rng.integers(0, 2, n)
        assert np.array_equal(_call(lib.sws_x255_f64, x32, m.astype(np.uint8), out_n=n), (x32 * m * 255).astype(np.uint8))
        assert np.array_equal(_call(lib.sws_u8_f32, x32, out_n=n), x32.astype(np.uint8))
        x64 = _wild(rng, n, np.float64)
        assert np.array_equal(_call(lib.sws_u8_f64, x64, out_n=n), x64.astype(np.uint8))
    assert np.array_equal(_call(lib.sws_u8_f32, np.array([300.7, -1, np.nan], np.float32), out_n=3), [44, 255, 0])


def _pixels(lib, layout, r, inten, depth, scale=SC.SCALE, test_mask=True):
    n = r.size
    codes = np.zeros((n, 6), np.uint8)
    pano, inten_out = np.zeros(n, np.float32), np.zeros(n, np.float32)
    is16 = r.dtype == np.float16
    rr = np.ascontiguousarray(r.reshape(-1).view(np.uint16) if is16 else r.reshape(-1))
    lib.sws_pixels(layout, int(is16), _p(rr), _p(np.ascontiguousarray(inten.reshape(-1))),
                   _p(np.ascontiguousarray(depth.reshape(-1))), n, float(np.float32(scale)), int(test_mask), _p(codes),
                   _p(pano), _p(inten_out))
    return codes, pano, inten_out


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("case", sorted(SC.CASES))
def test_pixel_function_matches_the_oracle(lib, case):
    L = (FX["lut_intensity"], FX["lut_depth"])
    for f in SC.frames(FX, case):
        H, W = f["depth"].shape
        I, D = f["image"][..., 1].copy(), f["depth"]
        for r in (f["unet"], f["image"][..., 0].copy()):
            c, pano, inten = _pixels(lib, SIM, r, I, D)
            panel, opano, ointen, _ = SO.sim(r, I, D, SC.SCALE, (2.0, 26.9), *L)
            assert np.array_equal(panel[:H].reshape(-1, 3)[:, 0], c[:, 0])
            assert np.array_equal(panel[H:2 * H].reshape(-1, 3), L[0][c[:, 1]])
            assert np.array_equal(panel[2 * H:].reshape(-1, 3), L[1][c[:, 2]])
            assert np.array_equal(_bits(pano), _bits(opano).reshape(-1)) and np.array_equal(_bits(inten), _bits(ointen).reshape(-1))
            for alpha_r in (0.01, 0.0):
                c, pano, _ = _pixels(lib, TEST, r, I, D, test_mask=alpha_r > 0)
                rd, oi, od, opano, _ = SO.test(r, I, D, SC.SCALE, alpha_r, (2.0, 26.9), *L)
                assert np.array_equal(rd.reshape(-1), c[:, 0])
                assert np.array_equal(oi.reshape(-1, 3), L[0][c[:, 1]]) and np.array_equal(od.reshape(-1, 3), L[1][c[:, 2]])
                assert np.array_equal(_bits(pano), _bits(opano).reshape(-1))
            c, _, _ = _pixels(lib, EVAL, r, I, D)
            panel = SO.evaluate(r, I, D, *L).reshape(6, H * W, 3)
            for row in range(6):
                want = panel[row]
                got = np.repeat(c[:, row:row + 1], 3, 1) if row % 3 == 0 else L[(row % 3) - 1][c[:, row]]
                assert np.array_equal(got, want), (case, row)
