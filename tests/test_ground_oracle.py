"""CPU: oracle/ground_oracle.py against tests/golden/ground_ref.npz (the reference's own utils/misc.py point_removal),
the reference itself against the oracle where the checkout exists, the host RANSAC driver of lidar4d_b200.misc with a
NumPy scorer, and the argument checks of the ground-removal entry points (no launch, no GPU)."""
import os
import random
import sys

import numpy as np
import pytest

from oracle import ground_oracle as GO
import ground_cases as GC

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
import make_ground_golden as MG  # noqa: E402

GOLD = os.path.join(os.path.dirname(__file__), "golden", "ground_ref.npz")
CASES = ["sweep_a", "sweep_b", "small70", "small200", "dup"]
FAKE = 256              # a device pointer that is never dereferenced: the argument check returns first
BIG = 1 << 40


@pytest.fixture(scope="module")
def fx():
    return np.load(GOLD, allow_pickle=False)


def _cloud(fx, name):
    return GC.cloud(fx, name) if name.startswith("sweep") else fx[f"{name}_points"]


def _have_reference():
    return os.path.exists(os.path.join(MG.REF, "utils", "misc.py"))


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_fixture(fx, name):
    """Kept indices of every stage, every hypothesis count and the final RNG state equal the reference's."""
    random.seed(int(fx[f"{name}_seed"]))
    o = GO.point_removal(_cloud(fx, name))
    assert np.array_equal(random.getstate()[1], fx[f"{name}_rng_state"])
    for k in ("rf_keep", "sor1_keep", "ground", "sor2_keep"):
        assert np.array_equal(o[k], GC.unpack(fx[f"{name}_{k}"])), k
    for j in range(6):
        assert o["ransac_counts"][j] == fx[f"{name}_ransac_counts_{j}"].tolist()
    print(f"{name}: flagged near a threshold: range {len(o['rf_near'])}, outliers {len(o['sor1_near'])} + "
          f"{len(o['sor2_near'])}, RANSAC {sum(map(sum, o['ransac_near']))}")


@pytest.mark.skipif(not _have_reference(), reason="the reference checkout is not present")
@pytest.mark.parametrize("name", ["small70", "small200", "dup", "sweep_a"])
def test_stubbed_reference_matches_oracle(fx, name):
    misc = MG.reference_misc()
    pc = _cloud(fx, name)
    seed = int(fx[f"{name}_seed"])
    r = MG.run_reference(misc, pc, seed)
    random.seed(seed)
    o = GO.point_removal(pc)
    assert np.array_equal(r["rng_state"], np.array(random.getstate()[1], np.uint32))
    for k in ("rf_keep", "sor1_keep", "ground", "sor2_keep"):
        assert np.array_equal(np.asarray(r[k]), o[k]), k
    assert np.array_equal(r["points"], o["points"]) and np.array_equal(r["ground_points"], o["ground_points"])


def _numpy_scorer(pts, thr):
    return lambda hyp: [int((GO.plane_distances(pts, h[:4], h[4]) < thr).sum()) for h in hyp]


@pytest.mark.parametrize("batch", [1, 7, 256])
@pytest.mark.parametrize("name", ["small70", "small200", "dup", "sweep_b"])
def test_ransac_driver_rng_bookkeeping(fx, name, batch):
    """The draw-ahead driver of lidar4d_b200.misc, scored on the host, leaves random.getstate() where the oracle's
    sequential loop (equal to the reference's, test_oracle_matches_fixture) leaves it, with the same counts and plane."""
    from lidar4d_b200 import misc
    o_seed = int(fx[f"{name}_seed"])
    pc = _cloud(fx, name)
    pc1 = pc[GC.unpack(fx[f"{name}_rf_keep"])].astype(np.float64)[GC.unpack(fx[f"{name}_sor1_keep"])]
    random.seed(o_seed)
    for j in range(6):
        coeffs, r, counts = misc.ransac_drive(pc1, _numpy_scorer(pc1, 0.15), 0.15, batch=batch)
        assert counts == fx[f"{name}_ransac_counts_{j}"].tolist()
    assert np.array_equal(random.getstate()[1], fx[f"{name}_rng_state"])


@pytest.mark.skipif(not _have_reference(), reason="the reference checkout is not present")
def test_ransac_driver_against_reference_my_ransac():
    from lidar4d_b200 import misc
    ref = MG.reference_misc()
    g = np.random.default_rng(9)
    pc = np.concatenate([np.stack([g.uniform(-20, 20, 500), g.uniform(-15, 15, 500), -1.7 + g.normal(0, 0.05, 500)], 1),
                         g.uniform(-20, 20, (300, 3))])
    for thr in (0.15, 0.3):
        random.seed(4)
        idx, model = ref.my_ransac(pc, distance_threshold=thr)
        want = random.getstate()
        random.seed(4)
        coeffs, r, _ = misc.ransac_drive(pc, _numpy_scorer(pc, thr), thr, batch=5)
        assert random.getstate() == want
        assert np.array_equal(coeffs, model)
        assert np.array_equal(np.flatnonzero(GO.plane_distances(pc, coeffs, r) < thr), idx)


def test_ransac_driver_errors(monkeypatch):
    from lidar4d_b200 import misc
    with pytest.raises(ValueError):
        misc.ransac_drive(np.zeros((2, 3)), lambda h: [0] * len(h))
    flat = np.zeros((50, 3))
    flat[:, 0] = np.arange(50)
    monkeypatch.setattr(misc, "MAX_CONSECUTIVE_REJECTIONS", 500)
    with pytest.raises(RuntimeError, match="rejected"):
        misc.ransac_drive(flat, lambda h: [0] * len(h), 0.15)


def test_estimate_plane_matches_reference_expressions():
    from lidar4d_b200.misc import estimate_plane
    g = np.random.default_rng(3)
    for _ in range(200):
        xyz = g.normal(0, 10, (3, 3))
        for normalize in (True, False):
            a = estimate_plane(xyz, normalize)
            b = GO.estimate_plane(xyz)
            if not normalize:
                assert np.array_equal(a, b)
    assert estimate_plane(np.array([[0.0, 0, 0], [1, 0, 1], [2, 3, 4]])) is None          # zero component
    assert estimate_plane(np.array([[0.0, 0, 0], [1, 2, 3], [2, 4, 6]])) is None          # collinear


# --- C-ABI argument checks -------------------------------------------------------------------------------------------
def test_work_sizes():
    from lidar4d_b200 import _capi
    lib = _capi.load_library()
    assert lib.l4d_range_filter_work_bytes(67980) == (67980 + 1023) // 1024 * 4
    assert lib.l4d_ground_split_work_bytes(1) == 4
    assert lib.l4d_outlier_select_work_bytes(1024) == 32 + 4


def test_abi_errors():
    from lidar4d_b200 import _capi
    lib = _capi.load_library()
    F, B = FAKE, BIG
    rf = lambda pts=F, n=10, stride=3, out=F, count=F, work=F, nwork=B: lib.l4d_range_filter(
        pts, n, stride, 1.0, 50.0, -2.5, 4.0, out, count, work, nwork, None)
    assert rf(n=0) == -1 and rf(n=1 << 31) == -1 and rf(stride=2) == -1
    assert rf(pts=None) == -1 and rf(out=None) == -1 and rf(count=None) == -1
    assert rf(work=None) == -3 and rf(nwork=lib.l4d_range_filter_work_bytes(10) - 1) == -3
    assert b"work buffer too small" in lib.l4d_last_error()
    knn = lambda pts=F, n=10, k=64, avg=F: lib.l4d_knn_mean_dist(pts, n, k, avg, None)
    assert knn(n=0) == -1 and knn(n=1 << 31) == -1 and knn(k=0) == -1 and knn(k=65) == -1
    assert knn(pts=None) == -1 and knn(avg=None) == -1
    sel = lambda pts=F, n=10, avg=F, out=F, count=F, work=F, nwork=B: lib.l4d_outlier_select(
        pts, n, avg, 3.0, out, None, count, None, work, nwork, None)
    assert sel(n=0) == -1 and sel(pts=None) == -1 and sel(avg=None) == -1 and sel(out=None) == -1 and sel(count=None) == -1
    assert sel(work=None) == -3 and sel(nwork=lib.l4d_outlier_select_work_bytes(10) - 1) == -3
    sc = lambda pts=F, n=10, hyp=F, m=4, counts=F: lib.l4d_plane_scores(pts, n, hyp, m, 0.15, counts, None)
    assert sc(n=0) == -1 and sc(m=0) == -1 and sc(pts=None) == -1 and sc(hyp=None) == -1 and sc(counts=None) == -1
    pm = lambda pts=F, n=10, mask=F: lib.l4d_plane_mask(pts, n, 0.0, 0.0, 1.0, 1.7, 1.0, 0.15, mask, None)
    assert pm(n=0) == -1 and pm(pts=None) == -1 and pm(mask=None) == -1
    gs = lambda pts=F, n=10, mask=F, g=F, r=F, counts=F, work=F, nwork=B: lib.l4d_ground_split(
        pts, n, mask, -1.0, g, None, r, None, counts, work, nwork, None)
    assert gs(n=0) == -1 and gs(pts=None) == -1 and gs(mask=None) == -1 and gs(g=None) == -1 and gs(r=None) == -1
    assert gs(counts=None) == -1 and gs(work=None) == -3 and gs(nwork=lib.l4d_ground_split_work_bytes(10) - 1) == -3
    pt = lambda pts=F, n=10, pose=F, out=F: lib.l4d_pose_transform(pts, n, 0.01, pose, out, None)
    assert pt(n=0) == -1 and pt(pts=None) == -1 and pt(pose=None) == -1 and pt(out=None) == -1
    assert b"null pointer" in lib.l4d_last_error()
