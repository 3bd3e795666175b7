"""oracle/image_metrics_oracle.py against the reference (CPU).

tests/golden/image_metrics_ref.npz holds the rows the reference's own DepthMeter / IntensityMeter / RaydropMeter
returned (tests/golden/make_image_metrics_golden.py); the restatement must reproduce them: the order statistic and the
counts exactly, the float32 means within 1e-6 relative (NumPy's float32 sums may take another SIMD path on another
CPU).  The recurrence restatement of uniform_filter must equal SciPy's bit for bit."""
import os

import numpy as np
import pytest
from scipy.ndimage import uniform_filter

import image_metrics_cases as IC
from oracle import image_metrics_oracle as IO

FX = np.load(os.path.join(os.path.dirname(__file__), "golden", "image_metrics_ref.npz"), allow_pickle=False)


def _same_bits(a, b):
    a, b = np.float64(a), np.float64(b)
    return (np.isnan(a) and np.isnan(b)) or a.tobytes() == b.tobytes()


def _close(a, b, rel):
    a, b = np.float64(a), np.float64(b)
    if not np.isfinite(a) or not np.isfinite(b):
        return _same_bits(a, b) or (np.isnan(a) and np.isnan(b))
    return abs(a - b) <= rel * abs(b)


def _oracle_row(name):
    kind, p, g = IC.frame(FX, name)
    f = IO.depth_errors if kind == "depth" else IO.intensity_errors
    return kind, np.array(f(g, p, lpips_value=float(FX["lpips_sentinel"])), np.float64)


@pytest.mark.parametrize("name", IC.IMAGE_CASES)
def test_oracle_reproduces_reference_image_rows(name):
    _, row = _oracle_row(name)
    ref = FX[f"{name}_row"]
    assert _same_bits(row[1], ref[1]), "medae"
    assert row[2] == ref[2]
    for k in (0, 3, 4):
        assert _close(row[k], ref[k], 1e-6), (k, row[k], ref[k])


@pytest.mark.parametrize("name,ratio", [(n, r) for n, rs in IC.RAYDROP_CASES.items() for r in rs])
def test_oracle_reproduces_reference_raydrop_rows(name, ratio):
    _, p, g = IC.frame(FX, name)
    row = np.array(IO.raydrop_errors(p, g, ratio), np.float64)
    ref = FX[f"{name}_r{ratio:g}_row"]
    assert _close(row[0], ref[0], 1e-6)
    assert _same_bits(row[1], ref[1]) and _same_bits(row[2], ref[2])


def test_oracle_reproduces_reference_measure():
    for kind in ("depth", "intensity"):
        rows = np.stack([_oracle_row(n)[1] for n in IC.IMAGE_CASES if _oracle_row(n)[0] == kind])
        m, ref = rows.mean(0), FX[f"measure_{kind}"]
        assert all(_close(a, b, 1e-6) for a, b in zip(m, ref)), (m, ref)


def test_ssim_constant_switch():
    """powf and x*x squares of the SSIM constants agree to an ulp; "mul" is the kernels' choice."""
    for R in (np.float32(80.0), np.float32(1.0 - 1e-6), np.float32(37.4921875)):
        a, b = IO.ssim_constants(R, "powf"), IO.ssim_constants(R, "mul")
        for x, y in zip(a, b):
            assert x.dtype == np.float32 and abs(int(x.view(np.int32)) - int(y.view(np.int32))) <= 1


def _clamped(name):
    kind, p, g = IC.frame(FX, name)
    lo, hi, _ = IO.DEPTH if kind == "depth" else IO.INTENSITY
    p, g = np.clip(p[0], lo, hi), np.clip(g[0], lo, hi)    # NaN stays NaN, as the meters' masked assignment
    return p, g


@pytest.mark.parametrize("name", IC.IMAGE_CASES)
def test_recurrence_equals_scipy_on_cases(name):
    p, g = _clamped(name)
    for a, b in zip(IO.filtered_maps(p, g), IO.filtered_maps(p, g, IO.uniform_filter_rec)):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("mag", [1e-3, 1.0, 80.0])
@pytest.mark.parametrize("shape", [(66, 1030), (7, 7), (9, 8), (128, 257)])
def test_recurrence_equals_scipy_random(mag, shape):
    g = np.random.default_rng(int(mag * 1000) + shape[0])
    x = (g.random(shape) * mag).astype(np.float32)
    assert np.array_equal(uniform_filter(x, 7).view(np.uint32), IO.uniform_filter_rec(x).view(np.uint32))
    y = (g.normal(0, mag, shape)).astype(np.float32)             # signed values
    assert np.array_equal(uniform_filter(y, 7).view(np.uint32), IO.uniform_filter_rec(y).view(np.uint32))


def test_ssim_rejects_small_images():
    x = np.zeros((6, 9), np.float32)
    with pytest.raises(ValueError):
        IO.structural_similarity(x, x, data_range=1.0)
