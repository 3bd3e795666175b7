"""GPU: range image <-> point cloud conversions (lidar4d_b200.convert) and the point-cloud metric (lidar4d_b200.metrics)
against the reference's own outputs (tests/golden/convert_ref.npz) and oracle/convert_oracle.py.

Rounding boundaries.  The device's atan2f is not NumPy's (neither is correctly rounded), so a point whose column or
row before rounding lies next to a .5 boundary may land one pixel over.  Such a point is a *boundary point* when the
reference's own float32 value v, taken to float64, lies within 8 float32 ulps of the boundary - ulps of v, or of the
atan2 result v is computed from, divided by the scale that turns that angle into pixels, whichever is larger (an angle
ulp is what the two atan2 implementations differ by; near c = 0 it spans many ulps of c).  Each boundary point is
projected on its own to see where the device puts it.  Boundary points that moved ("flips") are counted and printed,
must be at most 1e-4 of the cloud, and the whole device image must equal the reference's z-buffer fold with those
points moved to the device's pixels - bit for bit, depth and intensity.  Every pixel no flip touches therefore equals
the reference exactly.  No other difference is allowed."""
import numpy as np
import pytest
import torch

from oracle import convert_oracle as CO
from test_convert_oracle import GOLDEN, bits, load_case

pytestmark = pytest.mark.gpu

K = (2.0, 26.9)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def gpu_project(pts, h, w, k, max_depth=80):
    from lidar4d_b200.convert import lidar_to_pano_with_intensities
    t = torch.from_numpy(np.ascontiguousarray(pts, np.float32)).cuda()
    pano, inten = lidar_to_pano_with_intensities(t, h, w, k, max_depth=max_depth)
    return pano.cpu().numpy(), inten.cpu().numpy()


def gpu_unproject(pano, inten, k):
    from lidar4d_b200.convert import pano_to_lidar_with_intensities
    out = pano_to_lidar_with_intensities(torch.from_numpy(pano).cuda(), torch.from_numpy(inten).cuda(), k)
    return out.cpu().numpy()


def _ulp(v):
    v = np.abs(np.asarray(v, np.float32))
    return (np.nextafter(v, np.float32(np.inf)) - v).astype(np.float64)


def boundary_points(pts, h, w, k, max_depth=80):
    dist, c_pre, r_pre, a_xy, a_z = CO.pre_round(pts, h, w, k)
    fov_up, fov = k
    cs, rs = np.float32(2 * np.pi / w), np.float32(fov / 180 * np.pi / h)
    alpha = a_z + np.float32((fov - fov_up) / 180 * np.pi)
    with np.errstate(invalid="ignore"):
        win_c = 8 * np.maximum(_ulp(c_pre), _ulp(a_xy) / np.float64(cs))
        win_r = 8 * np.maximum(_ulp(r_pre), np.maximum(_ulp(a_z), _ulp(alpha)) / np.float64(rs))
        near = lambda v, win: np.abs(v.astype(np.float64) - (np.floor(v.astype(np.float64)) + 0.5)) <= win
        sel = (dist < np.float32(max_depth)) & (near(c_pre, win_c) | near(r_pre, win_r))
    return np.flatnonzero(sel)


def device_pixel(p, h, w, k, max_depth=80):
    """Where the device puts one point (-1: dropped); intensity 1 marks the pixel even at distance 0."""
    q = np.array([[p[0], p[1], p[2], 1.0]], np.float32)
    pano, inten = gpu_project(q, h, w, k, max_depth)
    hit = np.flatnonzero((pano.reshape(-1) != 0) | (inten.reshape(-1) != 0))
    assert len(hit) <= 1
    return int(hit[0]) if len(hit) else -1


def check_projection(pts, h, w, k, ref=None, max_depth=80, name=""):
    """Device projection of pts against the reference (ref = its (pano, intensities), else the oracle's), with the
    boundary bookkeeping of the module docstring.  Returns (boundary points, flips)."""
    pts = np.ascontiguousarray(pts, np.float32)
    pano, inten = gpu_project(pts, h, w, k, max_depth)
    o_pano, o_inten, pix = CO.project(pts, h, w, k, max_depth, return_pixels=True)
    if ref is not None:
        assert np.array_equal(bits(o_pano), bits(ref[0])) and np.array_equal(bits(o_inten), bits(ref[1]))
    cand = boundary_points(pts, h, w, k, max_depth)
    moved = pix.copy()
    flips = []
    for i in cand:
        d = device_pixel(pts[i], h, w, k, max_depth)
        if d != pix[i]:
            moved[i] = d
            flips.append(i)
    n = len(pts)
    print(f"[{name}] {n} points: {len(cand)} boundary points, {len(flips)} flipped")
    assert len(flips) <= 1e-4 * n
    inten_col = pts[:, 3] if pts.shape[1] > 3 else np.zeros(n, np.float32)
    dist = CO.pre_round(pts, h, w, k)[0]
    e_pano, e_inten = CO.zbuffer(moved, dist, inten_col, h, w)
    assert np.array_equal(bits(pano), bits(e_pano))
    assert np.array_equal(bits(inten), bits(e_inten))
    touched = np.zeros(h * w, bool)
    for i in flips:
        for q in (pix[i], moved[i]):
            if q >= 0:
                touched[q] = True
    keep = ~touched
    assert np.array_equal(bits(pano.reshape(-1)[keep]), bits(o_pano.reshape(-1)[keep]))
    assert np.array_equal(bits(inten.reshape(-1)[keep]), bits(o_inten.reshape(-1)[keep]))
    return cand, flips


def random_cloud(rng, n, k=K, r_max=90, spread=3.0):
    az = rng.uniform(-np.pi, np.pi, n)
    el = np.deg2rad(rng.uniform(k[0] - k[1] - spread, k[0] + spread, n))
    r = rng.uniform(0.5, r_max, n)
    return np.stack([np.cos(el) * np.cos(az) * r, np.cos(el) * np.sin(az) * r, np.sin(el) * r,
                     rng.integers(0, 1024, n) / 1024], 1).astype(np.float32)


# ------------------------------------------------------------------------------------------------ 4: projection
@pytest.mark.parametrize("name", ["mixed", "sweep", "half", "pixel"])
def test_projection_matches_reference_fixture(name):
    f = np.load(GOLDEN)
    pts, h, w, k, pano, inten = load_case(f, name)
    check_projection(pts, h, w, k, ref=(pano, inten), name=name)


def test_intensity_free_projection():
    """lidar_to_pano ([N, 3]) gives the depth image of lidar_to_pano_with_intensities (which the reference's own
    lidar_to_pano cannot: it raises TypeError)."""
    from lidar4d_b200.convert import lidar_to_pano
    f = np.load(GOLDEN)
    pts, h, w, k, pano, _ = load_case(f, "mixed")
    got = lidar_to_pano(torch.from_numpy(np.ascontiguousarray(pts[:, :3])).cuda(), h, w, list(k)).cpu().numpy()
    full, _ = gpu_project(pts, h, w, k)
    assert np.array_equal(bits(got), bits(full))


# ---------------------------------------------------------------------------------------------- 5: unprojection
def check_unprojection(pano, inten, k, ref=None):
    h, w = pano.shape
    keep = np.flatnonzero(pano.reshape(-1) != 0)            # NaN != 0: kept
    out = gpu_unproject(pano, inten, k)
    assert out.shape == (len(keep), 4)
    ids = gpu_unproject(pano, np.arange(h * w, dtype=np.float32).reshape(h, w), k)
    assert np.array_equal(ids[:, 3].astype(np.int64), keep)   # mask, count and order
    assert np.array_equal(bits(out[:, 3]), bits(inten.reshape(-1)[keep]))
    exp = CO.unproject(pano, inten, k) if ref is None else ref
    assert np.array_equal(bits(exp[:, 3]), bits(out[:, 3]))
    d = np.abs(pano.reshape(-1)[keep]).astype(np.float64)[:, None]
    nan = np.isnan(d[:, 0])
    assert np.array_equal(np.isnan(out[:, :3]).any(1), nan)
    err = np.abs(out[~nan, :3].astype(np.float64) - exp[~nan, :3])
    assert (err <= 2e-6 * d[~nan]).all(), float((err / np.maximum(d[~nan], 1e-30)).max())
    from lidar4d_b200.convert import pano_to_lidar
    xyz = pano_to_lidar(torch.from_numpy(pano).cuda(), k).cpu().numpy()
    assert np.array_equal(bits(xyz), bits(out[:, :3]))
    return out


def test_unprojection_matches_reference_fixture():
    f = np.load(GOLDEN)
    check_unprojection(f["unproj_pano"], f["unproj_intensities"], K, ref=f["unproj_points"])


@pytest.mark.parametrize("h,w", [(64, 2048), (66, 1030), (1, 1), (3, 1029)])
def test_unprojection_sizes(h, w):
    rng = np.random.default_rng(h * w)
    pano = rng.uniform(-5, 90, (h, w)).astype(np.float32)
    pano[rng.random((h, w)) < 0.4] = 0
    check_unprojection(pano, rng.random((h, w)).astype(np.float32), K)


def test_unprojection_of_empty_image():
    out = gpu_unproject(np.zeros((66, 1030), np.float32), np.ones((66, 1030), np.float32), K)
    assert out.shape == (0, 4)


# ------------------------------------------------------------------------------------------------- 6: round trip
@pytest.mark.parametrize("h,w", [(66, 1030), (64, 2048)])
def test_round_trip(h, w):
    """Unprojecting a range image and projecting the points again gives the image back: the same pixels and
    intensities, depths within float32 rounding of |direction| (the re-projected values sit on integers, far from
    any .5 boundary, so no pixel moves); the projection of the device's points also passes check_projection.
    Column 0 is the exception, in the reference too: its azimuth pi comes back through atan2 as just above -pi, so
    c rounds to W, which the reference drops rather than wraps (convert.py:54)."""
    rng = np.random.default_rng(7)
    pano, inten = CO.project(random_cloud(rng, 3 * h * w // 2), h, w, K)
    pts = gpu_unproject(pano, inten, K)
    cand, flips = check_projection(pts, h, w, K, name=f"round trip {h}x{w}")
    assert not flips
    back, back_i = gpu_project(pts, h, w, K)
    assert pano[:, 0].any() and not back[:, 0].any() and not back_i[:, 0].any()
    assert np.array_equal(back[:, 1:] != 0, pano[:, 1:] != 0)
    assert np.array_equal(bits(back_i[:, 1:]), bits(inten[:, 1:]))
    assert np.allclose(back[:, 1:], pano[:, 1:], rtol=1e-6, atol=0)


# ------------------------------------------------------------------------------------------------------ 8: sizes
def test_empty_cloud_gives_empty_image():
    pano, inten = gpu_project(np.zeros((0, 4), np.float32), 66, 1030, K)
    assert pano.shape == (66, 1030) and not pano.any() and not inten.any()


def test_single_point():
    p = np.array([[10.0, 3.0, -1.0, 0.25]], np.float32)
    check_projection(p, 66, 1030, K, name="n=1")
    assert np.count_nonzero(gpu_project(p, 66, 1030, K)[0]) == 1


def test_every_point_on_one_pixel():
    """Maximal atomic contention: 300 k points on one pixel, exact distance ties and zero-distance resets."""
    rng = np.random.default_rng(3)
    n = 300_000
    base = np.array([0.3, 0.9, -0.1])
    base /= np.linalg.norm(base)
    r = (rng.integers(1, 4000, n) / 64).astype(np.float32)
    pts = np.concatenate([(base[None] * r[:, None]).astype(np.float32), rng.random((n, 1)).astype(np.float32)], 1)
    pts[rng.choice(n, 50, replace=False), :3] = (base * 1e-30).astype(np.float32)
    pano, _ = gpu_project(pts, 66, 1030, K)
    assert np.count_nonzero(pano) <= 1
    check_projection(pts, 66, 1030, K, name="one pixel")


@pytest.mark.parametrize("h,w", [(64, 2048), (66, 1030)])
def test_random_clouds(h, w):
    rng = np.random.default_rng(h + w)
    pts = random_cloud(rng, 2 * h * w)
    pts[rng.choice(len(pts), 500, replace=False)] = pts[rng.choice(len(pts), 500, replace=False)]   # duplicates
    check_projection(pts, h, w, K, name=f"random {h}x{w}")
    check_projection(pts, h, w, K, max_depth=35.5, name=f"random {h}x{w} max_depth 35.5")


def test_launch_scale():
    """Every CTA of the grid-stride loops gets at least two units of work: 2 * 16 * SMs * 128 + 37 points (16 CTAs of
    128 threads fill an SM), and an image of more than 2 * 16 * SMs unprojection tiles of 1024 pixels."""
    n = 2 * 16 * sms() * 128 + 37
    rng = np.random.default_rng(11)
    check_projection(random_cloud(rng, n), 64, 2048, K, name="launch scale")
    h, w = 16 * sms() + 1, 2048
    assert (h * w + 1023) // 1024 >= 2 * 16 * sms()
    pano = rng.uniform(1, 90, (h, w)).astype(np.float32)
    pano[rng.random((h, w)) < 0.5] = 0
    check_unprojection(pano, rng.random((h, w)).astype(np.float32), K)


# ----------------------------------------------------------------------------------------------------- 7: metric
def restated_update(pred_pano, gt_pano, k, thr=0.05):
    """PointsMeter.update (utils/metrics.py:249-270) in torch with the project's chamfer_3DDist, on the clouds of
    lidar4d_b200.convert.pano_to_lidar.  Returns (cd, fscore, precision, recall, count1, n, count2, m)."""
    from lidar4d_b200.chamfer import chamfer_3DDist
    from lidar4d_b200.convert import pano_to_lidar
    a, b = pano_to_lidar(pred_pano, k), pano_to_lidar(gt_pano, k)
    dist1, dist2, _, _ = chamfer_3DDist()(a[None], b[None])
    cd = dist1.mean() + dist2.mean()
    p1 = torch.mean((dist1 < thr).float(), dim=1)
    p2 = torch.mean((dist2 < thr).float(), dim=1)
    f = 2 * p1 * p2 / (p1 + p2)
    f[torch.isnan(f)] = 0
    c1, c2 = int((dist1 < thr).sum()), int((dist2 < thr).sum())
    return float(cd), float(f[0]), float(p1[0]), float(p2[0]), c1, dist1.shape[1], c2, dist2.shape[1]


def metric_panos(seed, h=66, w=1030):
    rng = np.random.default_rng(seed)
    gt, _ = CO.project(random_cloud(rng, h * w), h, w, K)
    pred = gt + rng.normal(0, 0.2, gt.shape).astype(np.float32) * (gt != 0)
    pred[rng.random(gt.shape) < 0.05] = 0
    return torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda()


@pytest.mark.parametrize("seed", [0, 1])
def test_point_metrics_match_restated_update(seed):
    from lidar4d_b200.metrics import point_metrics
    pred, gt = metric_panos(seed)
    cd, f, p, r = (float(v) for v in point_metrics(pred, gt, K))
    rcd, rf, rp, rr, c1, n, c2, m = restated_update(pred, gt, K)
    assert p == np.float32(c1) / np.float32(n) and r == np.float32(c2) / np.float32(m)
    # torch.mean multiplies the exact float32 count by a float32 1/n, which can be 1 ulp off count / n
    assert abs(p - rp) <= np.spacing(np.float32(rp)) and abs(r - rr) <= np.spacing(np.float32(rr))
    assert abs(cd - rcd) <= 1e-6 * abs(rcd) and abs(f - rf) <= 1e-6 * abs(rf)
    print(f"[metric {seed}] cd {cd:.6g} (torch {rcd:.6g}), fscore {f:.6g}, precision {p:.6g}, recall {r:.6g}")
    again = [torch.stack(point_metrics(pred, gt, K)).cpu().numpy() for _ in range(3)]
    assert all(np.array_equal(bits(a), bits(again[0])) for a in again)


def test_point_metrics_threshold_and_zero_fscore():
    from lidar4d_b200.metrics import point_metrics
    pred, gt = metric_panos(5)
    cd, f, p, r = (float(v) for v in point_metrics(pred + 100 * (pred != 0), gt, K, threshold=1e-12))
    assert p == 0 and r == 0 and f == 0 and cd > 0


def test_empty_prediction_raises():
    from lidar4d_b200.metrics import PointsMeter, point_metrics
    _, gt = metric_panos(2)
    with pytest.raises(ValueError, match="empty"):
        point_metrics(torch.zeros_like(gt), gt, K)
    with pytest.raises(ValueError, match="empty"):
        PointsMeter(1.0, K).update(torch.zeros_like(gt)[None], gt[None])


def test_metric_reduction_at_launch_scale():
    """l4d_point_metrics on 2 * 16 * SMs * 128 + 37 distances against torch's reductions."""
    import ctypes as C
    from lidar4d_b200 import _capi
    lib = _capi.load_library()
    n = 2 * 16 * sms() * 128 + 37
    g = torch.Generator(device="cuda").manual_seed(0)
    d1 = torch.rand(n, device="cuda", generator=g) * 0.1
    d2 = torch.rand(n + 5, device="cuda", generator=g) * 0.2
    outs = []
    for _ in range(2):
        out = torch.empty(5, device="cuda")
        assert lib.l4d_point_metrics(d1.data_ptr(), n, d2.data_ptr(), n + 5, C.c_float(0.05), out.data_ptr(),
                                     torch.cuda.current_stream().cuda_stream) == 0
        outs.append(out.cpu().numpy())
    assert np.array_equal(bits(outs[0]), bits(outs[1]))
    cd, f, p, r, z = (float(v) for v in outs[0])
    exp_cd = float(d1.double().mean() + d2.double().mean())
    assert abs(cd - exp_cd) <= 1e-6 * exp_cd
    c1, c2 = int((d1 < 0.05).sum()), int((d2 < 0.05).sum())
    assert p == np.float32(c1) / np.float32(n) and r == np.float32(c2) / np.float32(n + 5) and z == 0
    assert f == np.float32(np.float32(np.float32(2 * np.float32(p)) * np.float32(r)) / np.float32(np.float32(p) + np.float32(r)))


def test_points_meter_drop_in():
    from lidar4d_b200.metrics import PointsMeter
    scale = 2.5
    meter = PointsMeter(scale, K)
    exp = []
    for seed in (3, 4, 6):
        pred, gt = metric_panos(seed)
        meter.update(pred[None] * scale, gt[None] * scale)
        exp.append(restated_update(pred * scale / scale, gt * scale / scale, K)[:2])
    assert meter.N == 3 and all(v.is_cuda for v in meter.V)
    got = meter.measure()
    assert got.shape == (2,)
    want = np.array(exp, np.float32).mean(0)
    assert np.allclose(got, want, rtol=1e-6, atol=0)
    assert meter.report().startswith("Point_error (CD, F-score) = ")

    class Writer:
        def add_scalar(self, tag, value, step):
            self.seen = (tag, float(value), step)
    w = Writer()
    meter.write(w, 7, prefix="evaluate")
    assert w.seen == ("evaluate/CD", float(got[0]), 7)
    meter.clear()
    assert meter.N == 0 and meter.V == []
