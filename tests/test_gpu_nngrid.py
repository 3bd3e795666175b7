"""GPU: chamfer_3DGrid (the grid nearest-neighbour search, l4d_nngrid.cuh) against chamfer_3DDist (the brute-force op, itself
pinned bit for bit to the reference's kernel by tests/test_chamfer.py) on the same tensors: dist1, dist2, idx1, idx2
bit-identical."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _uniform(n, m, seed, dup=False):
    g = np.random.default_rng(seed)
    x1 = g.uniform(-1, 1, (1, n, 3)).astype(np.float32)
    x2 = g.uniform(-1, 1, (1, m, 3)).astype(np.float32)
    if dup and m > 8:
        x2[:, m // 2:m // 2 + 4] = x2[:, 3:7]
        x1[:, :4] = x2[:, 3:7]
    return torch.from_numpy(x1).to(DEV), torch.from_numpy(x2).to(DEV)


def _same(a, b):
    for x, y, name in zip(a, b, ("dist1", "dist2", "idx1", "idx2")):
        assert x.shape == y.shape and x.dtype == y.dtype, name
        if x.dtype == torch.float32:
            assert torch.equal(x.view(torch.int32), y.view(torch.int32)), name
        else:
            assert torch.equal(x, y), name


def _check(x1, x2):
    from lidar4d_b200.chamfer import PointGrid, chamfer_3DDist, chamfer_3DGrid
    want = chamfer_3DDist()(x1, x2)
    f = chamfer_3DGrid()
    got = f(x1, x2)
    _same(got, want)
    _same(f(x1, x2), got)                                   # two calls are bit-identical
    g1, g2 = PointGrid(x1), PointGrid(x2[0])
    _same(f(g1, x2), want)
    _same(f(x1, g2), want)
    _same(f(g1, g2), want)
    return got


@pytest.mark.parametrize("n,m,seed,dup", [(1024, 1024, 3, False), (1, 513, 5, False), (700, 1, 6, False),
                                           (20000, 15000, 7, True), (4096, 4096, 11, True), (60000, 50000, 12, False),
                                           (1, 1, 13, False)])
def test_matches_brute_force(n, m, seed, dup):
    _check(*_uniform(n, m, seed, dup))


@pytest.mark.parametrize("case", ["lattice", "identical", "planar", "collinear", "outside", "nonfinite", "no_finite_target",
                                  "huge_extent"])
def test_special_clouds(case):
    g = np.random.default_rng(31)
    a = g.uniform(-1, 1, (3000, 3)).astype(np.float32)
    b = g.uniform(-1, 1, (2500, 3)).astype(np.float32)
    if case == "lattice":
        a = g.integers(-12, 12, (6000, 3)).astype(np.float32) / 256
        b = g.integers(-14, 14, (5000, 3)).astype(np.float32) / 256
    elif case == "identical":
        a[:] = a[0]
    elif case == "planar":
        a[:, 2] = 0.25
        b[:, 0] = -0.5
    elif case == "collinear":
        a[:, 1], a[:, 2] = -0.5, 0.125
    elif case == "outside":
        b[:500] *= 50
        b[500:600, 0] += 1e6
        b[600:610] = [3e38, -3e38, 3e38]
    elif case == "nonfinite":
        a[0] = [np.nan, 0, 0]
        a[5, 1] = np.inf
        a[100:110] = np.nan
        b[3, 0] = np.nan
        b[4] = -np.inf
    elif case == "no_finite_target":
        a[:] = np.nan
    else:
        a[1] = [3e38, 3e38, -3e38]
        a[2] = [-3e38, -3e38, 3e38]
    d1, d2, i1, i2 = _check(torch.from_numpy(a)[None].to(DEV), torch.from_numpy(b)[None].to(DEV))
    if case == "no_finite_target":
        assert bool(torch.isinf(d2).all()) and int(i2.abs().max()) == 0


def test_lidar_sweeps():
    """Neighbouring frames of the synthetic sensor (tests/ground_cases.py) through point_removal, at full size."""
    import random
    import ground_cases as GC
    from lidar4d_b200.misc import point_removal
    random.seed(0)
    clouds = []
    for seed, tilt in GC.SWEEPS.values():
        pts, _ = point_removal(torch.from_numpy(GC.sweep(seed, tilt=tilt)).to(DEV))
        clouds.append((pts * 0.01).float()[None].contiguous())
    assert min(c.shape[1] for c in clouds) > 20000
    _check(*clouds)


def test_gradients_match_brute_force():
    from lidar4d_b200.chamfer import chamfer_3DDist, chamfer_3DGrid
    x1, x2 = _uniform(5000, 4000, 41, dup=True)
    g = torch.Generator(device="cpu").manual_seed(1)
    w1, w2 = torch.randn(1, 5000, generator=g).to(DEV), torch.randn(1, 4000, generator=g).to(DEV)
    grads = []
    for f in (chamfer_3DDist(), chamfer_3DGrid()):
        a, b = x1.clone().requires_grad_(True), x2.clone().requires_grad_(True)
        d1, d2, _, _ = f(a, b)
        ((d1 * w1).sum() + (d2 * w2).sum()).backward()
        grads.append((a.grad, b.grad))
    for got, ref in zip(grads[1], grads[0]):
        assert float((got - ref).abs().max()) <= 1e-5 * float(ref.abs().max())      # fp32 atomics in another order


def test_invalid_arguments_leave_the_library_usable():
    from lidar4d_b200 import _capi
    from lidar4d_b200.chamfer import PointGrid, chamfer_3DGrid
    f = chamfer_3DGrid()
    x1, x2 = _uniform(300, 200, 51)
    with pytest.raises(ValueError):
        f(torch.cat([x1, x1]), torch.cat([x2, x2]))                     # b > 1
    with pytest.raises(ValueError):
        f(x1[:, :0], x2)                                                # empty cloud
    with pytest.raises(RuntimeError):
        f(x1.cpu(), x2.cpu())                                           # no CPU fallback
    with pytest.raises(ValueError):
        PointGrid(torch.zeros(0, 3, device=DEV))
    with pytest.raises(RuntimeError):
        PointGrid(torch.zeros(4, 3))
    lib = _capi.load_library()
    n = 300
    nb, nw = lib.l4d_nn_grid_bytes(n), lib.l4d_nn_grid_work_bytes(n)
    grid = torch.empty(nb, dtype=torch.uint8, device=DEV)
    work = torch.empty(nw, dtype=torch.uint8, device=DEV)
    pts = x1[0].contiguous()
    st = torch.cuda.current_stream().cuda_stream
    assert lib.l4d_nn_grid_build(pts.data_ptr(), n, grid.data_ptr(), nb - 1, work.data_ptr(), nw, st) != 0
    assert b"too small" in lib.l4d_last_error()
    assert lib.l4d_nn_grid_build(pts.data_ptr(), n, grid.data_ptr(), nb, work.data_ptr(), nw - 1, st) != 0
    assert b"too small" in lib.l4d_last_error()
    assert lib.l4d_nn_grid_build(pts.data_ptr(), 0, grid.data_ptr(), nb, work.data_ptr(), nw, st) != 0
    assert lib.l4d_nn_grid_build(None, n, grid.data_ptr(), nb, work.data_ptr(), nw, st) != 0
    assert lib.l4d_nn_grid_build(pts.data_ptr(), n, grid.data_ptr(), nb, work.data_ptr(), nw, st) == 0
    idx = torch.empty(200, dtype=torch.int32, device=DEV)
    dist = torch.empty(200, device=DEV)
    q = x2[0].contiguous()
    assert lib.l4d_nn_grid_query(grid.data_ptr(), nb - 1, n, q.data_ptr(), 200, dist.data_ptr(), idx.data_ptr(), None, st) != 0
    assert lib.l4d_nn_grid_query(grid.data_ptr(), nb, n, q.data_ptr(), 0, dist.data_ptr(), idx.data_ptr(), None, st) != 0
    assert lib.l4d_nn_grid_query(grid.data_ptr(), nb, n, q.data_ptr(), 200, None, idx.data_ptr(), None, st) != 0
    assert lib.l4d_nn_grid_query(grid.data_ptr(), nb, n, q.data_ptr(), 200, dist.data_ptr(), idx.data_ptr(), None, st) == 0
    torch.cuda.synchronize()
    _check(x1, x2)


def test_launches_do_not_depend_on_size():
    from lidar4d_b200 import _capi
    from lidar4d_b200.chamfer import PointGrid
    lib = _capi.load_library()
    counts = []
    for n in (10, 5000, 150000):
        x, q = _uniform(n, 2 * n, 61)
        c0 = lib.l4d_launch_count()
        grid = PointGrid(x)
        c1 = lib.l4d_launch_count()
        grid.query(q[0])
        counts.append((c1 - c0, lib.l4d_launch_count() - c1))
    assert counts == [(5, 1)] * 3
