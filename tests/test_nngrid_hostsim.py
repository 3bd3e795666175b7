"""CPU: the host build of the grid nearest-neighbour search (tests/hostsim/nngridsim.cu over
lidar4d_b200/csrc/l4d_nngrid.cuh) against oracle/chamfer_oracle.py, the brute-force fp32 restatement: dist and idx bit
for bit, whatever the order of the records inside a cell."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from oracle import chamfer_oracle as CO
import ground_cases as GC

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


@pytest.fixture(scope="module")
def sim():
    import __graft_entry__ as G
    lib = C.CDLL(G.build_nngridsim())
    lib.ns_query.restype = C.c_int
    lib.ns_query.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_int] + [C.c_void_p] * 4
    lib.ns_axis.restype = None
    lib.ns_axis.argtypes = [C.c_float, C.c_float, C.c_float, C.c_uint32, C.POINTER(C.c_float), C.POINTER(C.c_int32)]
    return lib


def grid_nn(lib, cloud, queries, reverse=0):
    cloud = np.ascontiguousarray(cloud, np.float32)
    queries = np.ascontiguousarray(queries, np.float32)
    nq = len(queries)
    dist, idx = np.empty(nq, np.float32), np.empty(nq, np.int32)
    cand, geo = np.empty(nq, np.uint32), np.zeros(10, np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = lib.ns_query(p(cloud), len(cloud), p(queries), nq, reverse, p(dist), p(idx), p(cand), p(geo))
    assert rc == 0, rc
    return dist, idx, cand, geo


def brute(queries, cloud):
    """The brute-force op's result.  For finite inputs that is the oracle's; with non-finite rows the kernel's strict '<'
    never lets a NaN or +inf distance win and (+inf, 0) stays (np.argmin would pick the NaN)."""
    q, c = np.asarray(queries, np.float32), np.asarray(cloud, np.float32)
    with np.errstate(all="ignore"):
        if np.isfinite(q).all() and np.isfinite(c).all():
            return CO.nn_distance(q, c)
        dx, dy, dz = ((c[None, :, a] - q[:, None, a]).astype(np.float32) for a in range(3))
        d = CO._fma32(dz, dz, CO._fma32(dx, dx, (dy * dy).astype(np.float32)))
    d = np.where(np.isnan(d), np.float32(np.inf), d)
    i = np.argmin(d, axis=1)
    dist = d[np.arange(len(q)), i]
    return dist, np.where(np.isinf(dist), 0, i).astype(np.int32)


def check(lib, cloud, queries, both_orders=True):
    """-> (cand, geo); asserts bit identity with the brute-force oracle for both fill orders of the cells."""
    rd, ri = brute(queries, cloud)
    for rev in ((0, 1) if both_orders else (0,)):
        d, i, cand, geo = grid_nn(lib, cloud, queries, rev)
        assert np.array_equal(d.view(np.uint32), rd.view(np.uint32)), "dist differs from the brute-force search"
        assert np.array_equal(i, ri), "idx differs from the brute-force search"
    return cand, geo


@pytest.mark.parametrize("n,m,seed", [(1, 1, 0), (1, 500, 1), (500, 1, 2), (37, 41, 3), (3000, 2000, 4), (20000, 700, 5)])
def test_uniform_clouds(sim, n, m, seed):
    g = np.random.default_rng(seed)
    cand, geo = check(sim, g.uniform(-1, 1, (n, 3)), g.uniform(-1, 1, (m, 3)))
    assert geo[3] <= geo[4] and geo[5] == n
    if n >= 3000:
        assert cand.mean() < 0.05 * n


def test_lattice_ties(sim):
    """Points and queries on a 1/256 lattice: thousands of exact ties, resolved to the smallest original index."""
    g = np.random.default_rng(7)
    cloud = g.integers(-12, 12, (6000, 3)).astype(np.float32) / 256
    q = g.integers(-14, 14, (3000, 3)).astype(np.float32) / 256
    d = ((cloud[None] - q[:300, None]) ** 2).sum(-1)
    assert ((d == d.min(1, keepdims=True)).sum(1) > 1).sum() > 100         # the fixture does contain ties
    check(sim, cloud, q)
    check(sim, np.repeat(cloud[:500], 5, 0), q)                            # and exact duplicates


@pytest.mark.parametrize("case", ["identical", "planar", "collinear", "two_points", "axis_pair"])
def test_degenerate_clouds(sim, case):
    g = np.random.default_rng(11)
    c = g.uniform(-1, 1, (800, 3)).astype(np.float32)
    if case == "identical":
        c[:] = c[0]
    elif case == "planar":
        c[:, 2] = 0.25
    elif case == "collinear":
        c[:, 1], c[:, 2] = -0.5, 0.125
    elif case == "two_points":
        c = c[:2]
    else:
        c = np.array([[0, 0, 0], [1e-3, 0, 0]], np.float32)
    q = np.concatenate([g.uniform(-1.5, 1.5, (600, 3)).astype(np.float32), c[:50]])
    _, geo = check(sim, c, q)
    if case == "identical":
        assert tuple(geo[:4]) == (1, 1, 1, 1)


def test_queries_far_outside_the_box(sim):
    g = np.random.default_rng(13)
    c = g.uniform(-1, 1, (5000, 3)).astype(np.float32)
    q = g.uniform(-1, 1, (300, 3)).astype(np.float32)
    q[:100] *= 50
    q[100:200, 0] += 1e6
    q[200:210] = [3e38, -3e38, 3e38]              # beyond every shell: the whole cloud is scanned
    q[210:220] = 1e30
    cand, _ = check(sim, c, q)
    assert cand[200:210].min() >= 5000
    far = c * np.float32(1e37) - np.float32(3e38)         # q - lo overflows for the queries on the other side
    check(sim, far, -far[:200])


def test_cell_faces_within_one_ulp(sim):
    """The attack on the stopping bound: points and queries a few ulps on either side of cell faces along each axis, where
    the rounding of the cell coordinate decides the cell."""
    g = np.random.default_rng(17)
    base = g.uniform(-1, 1, (4000, 3)).astype(np.float32) * np.array([1, 0.7, 0.2], np.float32) + np.float32(0.3)
    _, _, _, geo = grid_nn(sim, base, base[:1])
    lo = geo[6:9].view(np.float32)
    ih = geo[9:10].view(np.float32)[0]
    dims = geo[:3]
    pts, qs = [], []
    for a in range(3):
        for k in g.integers(1, max(2, dims[a]), 60):
            e = np.float32(lo[a] + np.float64(k) / np.float64(ih))
            ulp = np.float64(np.spacing(np.float32(max(abs(e), abs(e - lo[a])))))     # of the coarser of x and x - lo
            cells = set()
            for s in range(-8, 9):
                x = np.float32(np.float64(e) + s * 0.5 * ulp)
                u, c = C.c_float(), C.c_int32()
                sim.ns_axis(float(x), float(lo[a]), float(ih), int(dims[a]), C.byref(u), C.byref(c))
                cells.add(c.value)
                for dst in (pts, qs):
                    p = base[g.integers(0, len(base))].copy()
                    p[a] = x
                    dst.append(p)
            assert len(cells) >= 2 or k >= dims[a]          # the probes do straddle the face
    pts, qs = np.array(pts, np.float32), np.array(qs, np.float32)
    cloud = np.concatenate([base[:1500], pts])
    check(sim, cloud, np.concatenate([qs, base[1500:2500]]))
    check(sim, pts, qs)                                      # sparse: neighbours are whole cells away, bounds decide
    # the nearest point sits exactly across a face at a distance equal to the bound's neighbourhood
    for a in range(3):
        e = np.float32(lo[a] + np.float64(dims[a] // 2) / np.float64(ih))
        line = np.repeat(base[:1], 9, 0)
        line[:, a] = [np.nextafter(e, np.float32(s * np.inf), dtype=np.float32) if s else e for s in (-1, 0, 1)] * 3
        line[3:6, (a + 1) % 3] += np.float32(1) / np.float32(ih)
        line[6:9, (a + 2) % 3] -= np.float32(1) / np.float32(ih)
        check(sim, np.concatenate([base[:300], line]), line)


def test_non_finite_rows(sim):
    g = np.random.default_rng(19)
    c = g.uniform(-1, 1, (900, 3)).astype(np.float32)
    q = g.uniform(-1, 1, (400, 3)).astype(np.float32)
    c[0] = [np.nan, 0, 0]                     # index 0 must not be returned because of the (+inf, 0) start
    c[5, 1] = np.inf
    c[17, 2] = -np.inf
    c[100:110] = np.nan
    q[3, 0] = np.nan
    q[4, 1] = np.inf
    q[5] = -np.inf
    d, i, _, geo = grid_nn(sim, c, q)
    assert geo[5] == 900 - 13
    assert np.all(np.isinf(d[3:6])) and np.all(i[3:6] == 0)
    check(sim, c, q)
    check(sim, np.full((40, 3), np.nan, np.float32), q)              # no finite target: (+inf, 0) everywhere
    d, i, _, _ = grid_nn(sim, np.full((40, 3), np.inf, np.float32), q)
    assert np.all(np.isinf(d)) and np.all(i == 0)
    big = c.copy()
    big[1] = [3e38, 3e38, -3e38]              # finite, but the box's extent overflows: one cell
    big[2] = [-3e38, -3e38, 3e38]
    check(sim, big, q)


def _frame(seed, tilt):
    """A sweep through point_removal-like filtering (range, height, ego box), scaled as process_pointcloud scales it."""
    p = GC.sweep(seed, tilt=tilt)
    r = np.linalg.norm(p, axis=1)
    ego = (np.abs(p[:, 0]) < 2) & (np.abs(p[:, 1]) < 1) & (np.abs(p[:, 2]) < 2)
    keep = (r >= 2.75) & (r <= 50) & (p[:, 2] > -2.0) & (p[:, 2] < 4.0) & ~ego
    return (p[keep].astype(np.float64) * 0.01).astype(np.float32)


def test_sweeps_reduced(sim):
    a = _frame(*GC.SWEEPS["sweep_a"])[::9]
    b = _frame(*GC.SWEEPS["sweep_b"])[::7]
    check(sim, a, b)
    check(sim, b, a)


def test_sweeps_candidates_per_query(sim):
    """Neighbouring frames at full size with a 0.1 m synthetic flow: the search examines less than 5 % of the target
    cloud per query on average (the brute-force search examines all of it).  Bit identity on a strided sample."""
    a, b = _frame(*GC.SWEEPS["sweep_a"]), _frame(*GC.SWEEPS["sweep_b"])
    g = np.random.default_rng(23)
    f = g.normal(0, 1, a.shape)
    warped = (a + (f / np.linalg.norm(f, axis=1, keepdims=True) * 0.1 * 0.01).astype(np.float32)).astype(np.float32)
    for name, cloud, q in (("warped frame -> next frame", b, warped), ("next frame -> warped frame", warped, b)):
        d, i, cand, geo = grid_nn(sim, cloud, q)
        share = cand.mean() / len(cloud)
        print(f"[nngrid] {name}: {len(q)} queries, {len(cloud)} targets, grid {tuple(geo[:3])} = {geo[3]} cells of "
              f"{geo[4]}; {cand.mean():.1f} candidates per query on average ({100 * share:.2f} % of the cloud), "
              f"max {cand.max()}, {(cand >= len(cloud)).sum()} queries fell back to the full scan")
        assert share < 0.05
        s = slice(0, len(q), 29)
        rd, ri = CO.nn_distance(q[s], cloud)
        assert np.array_equal(d[s].view(np.uint32), rd.view(np.uint32)) and np.array_equal(i[s], ri)
