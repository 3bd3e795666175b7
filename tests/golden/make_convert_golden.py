"""Generate tests/golden/convert_ref.npz: outputs of the reference's own utils/convert.py (lidar_to_pano_with_intensities,
pano_to_lidar_with_intensities) on synthetic LiDAR-like scans, for tests/test_convert_oracle.py (CPU, pins
oracle/convert_oracle.py bit for bit) and tests/test_gpu_convert.py (the CUDA ops against the reference).

Run where the reference checkout exists (CPU only, no GPU needed; the Python loop takes a few seconds per cloud):
    python tests/golden/make_convert_golden.py [OUT.npz]          # LIDAR4D_REFERENCE = checkout (default /root/reference)
NumPy's float32 arctan2 is platform code, so the NumPy version and its SIMD line are stored with the outputs.

Cases (all float32 [N, 4] clouds: x, y, z, intensity; lidar_K as the reference's Python floats):
  mixed  123,708 points, 66 x 1030, K = (2.0, 26.9): a full sensor sweep with ranges in [1, 90] (also the case
         `sweep` on its own), jittered directions (many pixels hit several times), exact duplicates (ties),
         zero-distance points at the start, middle and end (some on pixels that later points refill), points outside
         the field of view, points with beta just under 2 pi (c == W), and a few points within 2 ulps of a .5 rounding
         boundary of c or r.  Its coordinates are not stored: tests/convert_cases.py rebuilds the cloud from a seed and
         the few bit-built points stored here, and checks it against the stored SHA-256;
  half   1031 columns and an fov_up chosen so that every point with y = 0 and z = 0 (exact atan2 everywhere) has c and r
         within a few ulps of a .5 boundary;
  pixel  every point on one pixel: ranges with exact ties and zero-distance resets.
Unprojection: the reference's pano_to_lidar_with_intensities of the top 8 rows of the `sweep` range image with
negative, -0.0 and NaN pixels added (`unproj_*`)."""
import io
import os
import sys
from contextlib import redirect_stdout

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = os.environ.get("LIDAR4D_REFERENCE", "/root/reference")

from oracle import convert_oracle as CO  # noqa: E402
sys.path.insert(0, os.path.dirname(HERE))
import convert_cases  # noqa: E402

H, W, K = convert_cases.H, convert_cases.W, convert_cases.K


def reference_convert():
    sys.path.insert(0, REF)
    sys.dont_write_bytecode = True
    from utils import convert
    return convert


def _ulp(v):
    v = np.float32(v)
    return np.float64(np.nextafter(v, np.float32(np.inf)) - v)


def _near_half(rng, which, count, hh, ww, k):
    """`count` points whose float32 c (which = 0) or r (which = 1) before rounding is within 2 ulps of a .5 boundary."""
    out = []
    while len(out) < count:
        R = np.float32(rng.uniform(5, 60))
        if which == 0:
            tgt = rng.integers(200, ww - 30) + 0.5
            az = np.pi - tgt * (2 * np.pi / ww)
            el = np.deg2rad(rng.uniform(-20, 0))
        else:
            tgt = rng.integers(10, hh - 10) + 0.5
            el = (hh - tgt) * (k[1] / 180 * np.pi / hh) - (k[1] - k[0]) / 180 * np.pi
            az = rng.uniform(-3, 3)
        p = np.array([[np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el), 0.5]], np.float32) * np.float32([R, R, R, 1])
        j = 1 if which == 0 else 2                      # walk y (for c) or z (for r) one ulp at a time towards the boundary
        err = lambda q: abs(np.float64(CO.pre_round(q, hh, ww, k)[1 + which][0]) - tgt)
        for _ in range(4000):
            pre = CO.pre_round(p, hh, ww, k)[1 + which][0]
            if err(p) <= 2 * _ulp(pre):
                out.append(p[0].copy())
                break
            steps = []
            for to in (np.float32(np.inf), np.float32(-np.inf)):
                q = p.copy()
                q[0, j] = np.nextafter(q[0, j], to)
                steps.append((err(q), q))
            best = min(steps, key=lambda s: s[0])
            if best[0] >= err(p):
                break                                    # stuck between two float32 values: draw another point
            p = best[1]
    return np.array(out, np.float32)


def mixed_special(rng):
    """The points of the mixed cloud that are built bit by bit and stored (tests/convert_cases.py draws the rest):
    zero-distance groups - the exact origin, and coordinates whose squares underflow (dist == 0 with a real azimuth;
    z = 0 gives alpha = fov_down, row 5) on pixels that points after them refill - and 8 points within 2 ulps of a .5
    rounding boundary of c or r."""
    def zeros(m):
        a = rng.uniform(-np.pi, np.pi, m)
        z = np.stack([1e-30 * np.cos(a), 1e-30 * np.sin(a), np.zeros(m), rng.integers(0, 256, m) / 256], 1).astype(np.float32)
        z[: m // 4, :3] = 0
        return z
    halves = np.concatenate([_near_half(rng, 0, 4, H, W, K), _near_half(rng, 1, 4, H, W, K)])
    halves[:, 3] = (rng.integers(0, 256, len(halves)) / 256).astype(np.float32)
    return {"z0": zeros(40), "z1": zeros(40), "z2": zeros(40), "halves": halves}


def half_case(rng):
    """W = 1031 and an fov_up such that y = 0, z = 0 points (atan2 exactly 0 / pi) sit within 2 ulps of .5 in both c and
    r; the rounding there is the same on every platform."""
    hh, ww, fov = 66, 1031, 26.9
    fu0 = fov - (hh - 5.5) * (fov / hh)                # r = H - fov_down / (fov / H) = 5.5 exactly in real numbers
    for step in range(100000):
        fu = fu0 + (step // 2) * (1e-9 if step % 2 else -1e-9)
        r_pre = CO.pre_round(np.array([[1, 0, 0]], np.float32), hh, ww, (fu, fov))[2][0]
        if abs(np.float64(r_pre) - 5.5) <= 2 * _ulp(r_pre):
            break
    else:
        raise RuntimeError("no fov_up found")
    k = (fu, fov)
    c_pre = CO.pre_round(np.array([[1, 0, 0]], np.float32), hh, ww, k)[1][0]
    assert abs(np.float64(c_pre) - 515.5) <= 2 * _ulp(c_pre), c_pre
    m = 400
    rr = rng.uniform(1, 70, m).astype(np.float32)
    rr[100:140] = rr[60:100]                           # exact ties
    pts = np.zeros((m, 4), np.float32)
    pts[:, 0] = np.where(rng.random(m) < 0.5, rr, -rr)  # x < 0: beta = 0, c = 0
    pts[:, 3] = (rng.integers(0, 256, m) / 256).astype(np.float32)
    pts[200:260, 2] = (rr[200:260] * rng.uniform(-0.3, 0.03, 60)).astype(np.float32)    # other rows, same columns
    pts[300:305, :3] = 0                               # resets in the middle
    return pts, hh, ww, k


def pixel_case(rng):
    m = 2000
    base = np.array([0.6, -0.7, -0.05], np.float64)
    base /= np.linalg.norm(base)
    r = (rng.integers(1, 40, m) / 4).astype(np.float32)             # many exact ties
    pts = np.concatenate([(base[None] * r[:, None]).astype(np.float32), (rng.integers(0, 256, (m, 1)) / 256).astype(np.float32)], 1)
    pts[[0, 700, 1333, 1999], :3] = (base * 1e-30).astype(np.float32)   # zero distance on the same pixel
    return pts


def main(out_path):
    conv = reference_convert()
    rng = np.random.default_rng(2024)
    fx = {"numpy_version": np.array(np.__version__)}
    buf = io.StringIO()
    with redirect_stdout(buf):
        np.show_runtime()
    fx["numpy_simd"] = np.array(" ".join(buf.getvalue().split("'simd_extensions'")[1].split("}")[0].split()))
    special = mixed_special(rng)
    mixed, sw = convert_cases.build(special)
    sweep = mixed[sw]
    for k, v in special.items():
        fx[f"mixed_{k}"] = v
    fx["mixed_seed"] = np.array(convert_cases.SEED, np.int64)
    fx["mixed_sha256"] = np.array(convert_cases.digest(mixed))
    half, hh, hw, hk = half_case(rng)
    cases = {"mixed": (mixed, H, W, K), "sweep": (sweep, H, W, K), "half": (half, hh, hw, hk), "pixel": (pixel_case(rng), H, W, K)}
    for name, (pts, h, w, k) in cases.items():
        pano, inten = conv.lidar_to_pano_with_intensities(pts, h, w, list(k), max_depth=80)
        assert np.array_equal(pano.astype(np.float32).astype(np.float64), pano)     # every stored value is a float32
        pano, inten = pano.astype(np.float32), inten.astype(np.float32)
        fx[f"{name}_hw"] = np.array([h, w], np.int64)
        fx[f"{name}_K"] = np.array(k, np.float64)
        if name in ("mixed", "sweep"):                     # rebuilt from the seed; images stored compactly
            base = sw.start if name == "mixed" else 0
            code, k8 = convert_cases.encode_pano(pano, pts, base), convert_cases.encode_intensities(inten)
            assert np.array_equal(convert_cases.decode_pano(code, pts, base, pano.shape).view(np.uint32), pano.view(np.uint32))
            assert np.array_equal(convert_cases.decode_intensities(k8).view(np.uint32), inten.view(np.uint32))
            fx[f"{name}_pano_code"], fx[f"{name}_intensities_u8"] = code, k8
        else:
            fx[f"{name}_points"] = pts
            fx[f"{name}_pano"] = pano
            fx[f"{name}_intensities"] = inten
        print(f"{name}: {len(pts)} points, {int((pano != 0).sum())} pixels set")
    pano = convert_cases.decode_pano(fx["sweep_pano_code"], sweep, 0, (H, W))[:8].copy()   # the top 8 rows
    inten = convert_cases.decode_intensities(fx["sweep_intensities_u8"]).reshape(H, W)[:8].copy()
    flat = pano.reshape(-1)
    sel = rng.choice(np.flatnonzero(flat), 60, replace=False)
    flat[sel[:40]] = -flat[sel[:40]]
    flat[sel[40:50]] = -0.0
    flat[sel[50]] = np.nan
    fx["unproj_pano"] = pano
    fx["unproj_intensities"] = inten
    fx["unproj_points"] = conv.pano_to_lidar_with_intensities(pano, inten, list(K))
    assert fx["unproj_points"].dtype == np.float32
    np.savez_compressed(out_path, **fx)
    print(f"wrote {out_path} ({os.path.getsize(out_path)} bytes)")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "convert_ref.npz"))
