"""Chamfer op (SURVEY.md 8(f) rank 1): oracle self-consistency on the CPU, parity through the C-ABI on the GPU."""
import os

import numpy as np
import pytest
import torch

from oracle import chamfer_oracle as CO


def _clouds(b, n, m, seed, dup=False):
    g = np.random.default_rng(seed)
    x1 = g.uniform(-1, 1, (b, n, 3)).astype(np.float32)
    x2 = g.uniform(-1, 1, (b, m, 3)).astype(np.float32)
    if dup and m > 8:          # exact duplicates in the target cloud: the smallest index has to win
        x2[:, m // 2:m // 2 + 4] = x2[:, 3:7]
        x1[:, :4] = x2[:, 3:7]
    return x1, x2


def test_oracle_matches_float64_cdist():
    x1, x2 = _clouds(2, 300, 411, 0, dup=True)
    d1, d2, i1, i2 = CO.chamfer_forward(x1, x2)
    for a, b, d, i in ((x1, x2, d1, i1), (x2, x1, d2, i2)):
        D = torch.cdist(torch.from_numpy(a).double(), torch.from_numpy(b).double()) ** 2
        dmin, _ = D.min(-1)
        assert np.allclose(d, dmin.numpy(), rtol=1e-5, atol=1e-9)
        picked = torch.gather(D, 2, torch.from_numpy(i.astype(np.int64))[..., None])[..., 0]
        assert np.allclose(picked.numpy(), dmin.numpy(), rtol=1e-5, atol=1e-9)
    assert (i1[:, :4] == np.arange(3, 7)).all()          # duplicates: first index wins (chamfer3D.cu:33,127)


def test_oracle_backward_matches_autograd():
    x1, x2 = _clouds(1, 64, 50, 1)
    d1, d2, i1, i2 = CO.chamfer_forward(x1, x2)
    g = np.random.default_rng(2)
    g1, g2 = g.normal(size=d1.shape).astype(np.float32), g.normal(size=d2.shape).astype(np.float32)
    gx1, gx2 = CO.chamfer_backward(x1, x2, g1, g2, i1, i2)
    t1 = torch.from_numpy(x1).double().requires_grad_(True)
    t2 = torch.from_numpy(x2).double().requires_grad_(True)
    D = torch.cdist(t1, t2) ** 2
    loss = (D.min(2)[0] * torch.from_numpy(g1).double()).sum() + (D.min(1)[0] * torch.from_numpy(g2).double()).sum()
    loss.backward()
    assert np.allclose(gx1, t1.grad.numpy(), rtol=1e-4, atol=1e-5)
    assert np.allclose(gx2, t2.grad.numpy(), rtol=1e-4, atol=1e-5)


def test_module_surface_and_argument_errors():
    from lidar4d_b200.chamfer import chamfer_3DDist, chamfer_3DFunction      # noqa: F401  (names of dist_chamfer_3D.py)
    f = chamfer_3DDist()
    with pytest.raises(ValueError):
        f(torch.zeros(1, 5, 2), torch.zeros(1, 5, 3))
    with pytest.raises(RuntimeError):
        f(torch.zeros(1, 5, 3), torch.zeros(1, 6, 3))       # CPU tensors: no fallback


CASES = [(1, 1024, 1024, 3, False), (2, 777, 1300, 4, True), (1, 1, 513, 5, False), (1, 700, 1, 6, False),
         (1, 20000, 15000, 7, True), (3, 50, 5000, 8, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,m,seed,dup", CASES)
def test_chamfer_forward_backward_gpu(b, n, m, seed, dup):
    from lidar4d_b200.chamfer import chamfer_3DDist
    dev = torch.device("cuda:0")
    x1, x2 = _clouds(b, n, m, seed, dup)
    rd1, rd2, ri1, ri2 = CO.chamfer_forward(x1, x2)
    t1 = torch.from_numpy(x1).to(dev).requires_grad_(True)
    t2 = torch.from_numpy(x2).to(dev).requires_grad_(True)
    d1, d2, i1, i2 = chamfer_3DDist()(t1, t2)
    assert i1.dtype == torch.int32 and d1.shape == (b, n) and d2.shape == (b, m)
    # distances: same fp32 expression as the reference kernel -> bit-exact against the fma-emulating oracle
    assert np.array_equal(d1.detach().cpu().numpy(), rd1) and np.array_equal(d2.detach().cpu().numpy(), rd2)
    assert np.array_equal(i1.cpu().numpy(), ri1) and np.array_equal(i2.cpu().numpy(), ri2)
    g = np.random.default_rng(seed + 100)
    g1, g2 = g.normal(size=rd1.shape).astype(np.float32), g.normal(size=rd2.shape).astype(np.float32)
    ((d1 * torch.from_numpy(g1).to(dev)).sum() + (d2 * torch.from_numpy(g2).to(dev)).sum()).backward()
    rg1, rg2 = CO.chamfer_backward(x1, x2, g1, g2, ri1, ri2)
    for got, ref in ((t1.grad, rg1), (t2.grad, rg2)):
        err = np.abs(got.cpu().numpy() - ref).max() / (np.abs(ref).max() + 1e-30)
        assert err < 1e-5, err


@pytest.mark.gpu
def test_chamfer_properties_full_size():
    """Size-independent properties at the flow-loss size (10^5 points): symmetry under swapping the clouds, zero
    distance and identity index for identical clouds, idempotence, gradient of sum(dist) sums to zero."""
    from lidar4d_b200.chamfer import chamfer_3DDist
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    a = (torch.rand(1, 100000, 3, generator=g) * 2 - 1).to(dev)
    bb = (torch.rand(1, 90000, 3, generator=g) * 2 - 1).to(dev)
    f = chamfer_3DDist()
    d1, d2, i1, i2 = f(a, bb)
    e2, e1, j2, j1 = f(bb, a)
    assert torch.equal(d1, e1) and torch.equal(d2, e2) and torch.equal(i1, j1) and torch.equal(i2, j2)
    s1, s2, k1, k2 = f(a, a.clone())
    assert float(s1.max()) == 0.0 and torch.equal(k1[0].long(), torch.arange(a.shape[1], device=dev))
    picked = ((a[0] - bb[0][i1[0].long()]) ** 2).sum(-1)
    assert torch.allclose(picked, d1[0], rtol=1e-5, atol=1e-9)
    a2 = a.clone().requires_grad_(True)
    b2 = bb.clone().requires_grad_(True)
    o1, o2, _, _ = f(a2, b2)
    (o1.sum() + o2.sum()).backward()
    tot = a2.grad.sum(1) + b2.grad.sum(1)
    assert float(tot.abs().max()) < 1e-2 * float(a2.grad.abs().sum())


# ---- the reference's OWN kernels (chamfer3D.cu NmDistanceKernel / NmDistanceGradKernel): their outputs on these cases, a
# fixed sample of query points per case, are stored in tests/golden/chamfer_ref.npz (tests/golden/make_chamfer_golden.py) -------
GOLD = os.path.join(os.path.dirname(__file__), "golden", "chamfer_ref.npz")
REF_CASES = CASES + [(1, 4096, 4096, 11, True), (1, 60000, 50000, 12, False), (2, 1, 1, 13, False)]


def golden_sample(count, seed, k=2048):
    """Flat indices of the stored query points: all of them up to k, else a seeded sample (sorted)."""
    if count <= k:
        return np.arange(count, dtype=np.int64)
    return np.sort(np.random.default_rng(seed).choice(count, k, replace=False)).astype(np.int64)


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,m,seed,dup", REF_CASES)
def test_chamfer_bit_exact_against_reference_kernel(b, n, m, seed, dup):
    """Distances AND indices of l4d_chamfer_forward equal NmDistanceKernel's (chamfer3D.cu:11-133) bit for bit - also on
    exact duplicates (ties -> smallest index) - and the gradients equal NmDistanceGradKernel's (:154-174) to fp32
    atomics re-ordering.  This pins oracle/chamfer_oracle.py's assumed fma contraction as well."""
    from lidar4d_b200.chamfer import chamfer_3DDist
    fx = np.load(GOLD)
    key = f"{b}_{n}_{m}_{seed}_{int(dup)}"
    dev = torch.device("cuda:0")
    x1, x2 = _clouds(b, n, m, seed, dup)
    t1 = torch.from_numpy(x1).to(dev).requires_grad_(True)
    t2 = torch.from_numpy(x2).to(dev).requires_grad_(True)
    d1, d2, i1, i2 = chamfer_3DDist()(t1, t2)
    o1, o2, oi1, oi2 = CO.chamfer_forward(x1, x2)                            # the numpy oracle agrees with the real kernel
    g = torch.Generator().manual_seed(seed)
    g1, g2 = torch.randn(b, n, generator=g).to(dev), torch.randn(b, m, generator=g).to(dev)
    ((d1 * g1).sum() + (d2 * g2).sum()).backward()
    for side, (d, i, o, oi, grad) in enumerate(((d1, i1, o1, oi1, t1.grad), (d2, i2, o2, oi2, t2.grad))):
        sel = fx[f"{key}_sel{side}"]
        assert np.array_equal(sel, golden_sample(d.numel(), seed + side))
        rd, ri, rg = fx[f"{key}_d{side}"], fx[f"{key}_i{side}"], fx[f"{key}_g{side}"]
        assert np.array_equal(d.detach().reshape(-1).cpu().numpy()[sel], rd)
        assert np.array_equal(i.reshape(-1).cpu().numpy()[sel], ri)
        assert np.array_equal(o.reshape(-1)[sel], rd) and np.array_equal(oi.reshape(-1)[sel], ri)
        got = grad.reshape(-1, 3).cpu().numpy()[sel]
        assert float(np.abs(got - rg).max()) <= 1e-5 * float(np.abs(rg).max()) + 1e-12
