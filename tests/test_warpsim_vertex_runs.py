"""The vertex-run reduction of lidar4d_b200/csrc/l4d_bwd.cuh (l4d_vertex_runs + l4d_vertex_sum: one gradient update per
distinct grid vertex of a warp) executed on the CPU by tests/hostsim/vertexsim.cu (on warpsim.cu's lockstep warp emulator),
against a brute-force per-vertex reference: every issued slot must hold the sum over all lanes of its ray that touch that
vertex, and the issue count must equal the number of distinct (ray, vertex) pairs of the warp's active lanes."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def ws(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("vertexsim") / "_vertexsim.so")
    subprocess.run(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC,-ffp-contract=off",
                    "-gencode", "arch=compute_90a,code=sm_90a", "-o", so, os.path.join(HERE, "hostsim", "vertexsim.cu"),
                    "-lpthread"], check=True)
    lib = C.CDLL(so)
    ip, fp, up = C.POINTER(C.c_int), C.POINTER(C.c_float), C.POINTER(C.c_uint)
    lib.vs_vertex_runs.argtypes = [C.c_int, ip, ip, ip, fp, up]
    lib.vs_static_level.argtypes = [C.c_float, C.c_uint32, C.c_uint32, C.c_int, fp, fp, ip, fp, fp]
    return lib


def _p(a, t=C.c_float):
    return a.ctypes.data_as(C.POINTER(t))


def _run(ws, cells, seg, active, rng):
    D = cells.shape[1]
    K, F = 1 << D, (1 if D == 2 else 4)
    v = rng.normal(size=(32, K, F)).astype(np.float32)
    v[~active] = 0.0
    out = v.copy()
    issue = np.zeros(32, np.uint32)
    c = np.ascontiguousarray(cells, np.int32)
    s = np.ascontiguousarray(seg, np.int32)
    a = np.ascontiguousarray(active, np.int32)
    assert ws.vs_vertex_runs(D, _p(c, C.c_int), _p(s, C.c_int), _p(a, C.c_int), _p(out), _p(issue, C.c_uint)) == 0
    return v, out, issue


def _check(ws, cells, seg, active, seed=0):
    rng = np.random.default_rng(seed)
    D = cells.shape[1]
    K = 1 << D
    v, out, issue = _run(ws, cells, seg, active, rng)
    offs = [np.array([(s >> a) & 1 for a in range(D)]) for s in range(K)]
    ref = {}
    for i in range(32):
        if not active[i]:
            continue
        for s in range(K):
            key = (int(seg[i]),) + tuple(int(t) for t in cells[i] + offs[s])
            ref[key] = ref.get(key, 0.0) + v[i, s].astype(np.float64)
    got = {}
    for i in range(32):
        assert active[i] or issue[i] == 0
        for s in range(K):
            if (int(issue[i]) >> s) & 1:
                key = (int(seg[i]),) + tuple(int(t) for t in cells[i] + offs[s])
                assert key not in got, f"vertex {key} issued twice"
                got[key] = out[i, s]
    assert sorted(got) == sorted(ref)                       # one update per distinct vertex, none lost
    for key, want in ref.items():
        np.testing.assert_allclose(got[key], want, rtol=2e-6, atol=2e-6 * max(1.0, float(np.abs(want).max())))
    return len(got)


def _ray_cells(D, start, step, n=32, res=None):
    t = np.arange(n)[:, None]
    c = np.floor(np.asarray(start, np.float64)[None, :] + t * np.asarray(step, np.float64)[None, :]).astype(np.int64)
    return c if res is None else np.clip(c, 0, res - 1)


@pytest.mark.parametrize("D", [2, 3])
@pytest.mark.parametrize("signs", [(1, 1, 1), (-1, 1, 1), (1, -1, 1), (1, 1, -1), (-1, -1, -1)])
@pytest.mark.parametrize("speed", [0.05, 0.3, 0.7, 1.6, 2.5])
def test_rays_increasing_and_decreasing_along_each_axis(ws, D, signs, speed):
    step = np.array([0.9, 0.6, 0.35])[:D] * speed * np.array(signs[:D])     # speed >= 1.6: jumps of |delta| >= 2
    cells = _ray_cells(D, [100.3, 200.7, 50.1][:D], step)
    n = _check(ws, cells, np.zeros(32, np.int32), np.ones(32, bool), seed=int(speed * 10))
    assert n <= 32 * (1 << D)


@pytest.mark.parametrize("D", [2, 3])
@pytest.mark.parametrize("split", [1, 7, 16, 31])
def test_a_warp_that_straddles_two_rays(ws, D, split):
    a = _ray_cells(D, [10.2, 10.2, 10.2][:D], [0.1, 0.05, 0.02][:D])
    b = a.copy()                                # the second ray passes through the same cells: its lanes must not join
    cells = np.concatenate([a[:split], b[split:]])
    seg = np.array([5] * split + [6] * (32 - split), np.int32)
    _check(ws, cells, seg, np.ones(32, bool), seed=split)


@pytest.mark.parametrize("D", [2, 3])
@pytest.mark.parametrize("n_active", [1, 9, 25, 31])
def test_inactive_tail_lanes(ws, D, n_active):
    cells = _ray_cells(D, [3.5, 4.5, 5.5][:D], [0.2, 0.1, 0.3][:D])
    cells[n_active:] = cells[n_active - 1]      # the lanes past the end shadow the last sample
    active = np.arange(32) < n_active
    _check(ws, cells, np.zeros(32, np.int32), active, seed=n_active)


@pytest.mark.parametrize("D", [2, 3])
def test_still_ray_reduces_once_per_vertex(ws, D):
    cells = np.full((32, D), 7, np.int64)
    assert _check(ws, cells, np.zeros(32, np.int32), np.ones(32, bool)) == 1 << D


@pytest.mark.parametrize("D", [2, 3])
def test_random_walks(ws, D):
    rng = np.random.default_rng(D)
    for trial in range(20):
        steps = rng.integers(-1, 2, size=(32, D)) * (rng.uniform(size=(32, 1)) < 0.5)
        steps[rng.uniform(size=32) < 0.1] *= 3                # occasional jumps
        cells = 50 + np.cumsum(steps, 0)                     # not monotone: a vertex may be left and re-entered
        seg = np.cumsum(rng.uniform(size=32) < 0.05).astype(np.int32)
        active = rng.uniform(size=32) < 0.9
        if not active.any():
            continue
        # runs that are not contiguous get one update each: compare per contiguous run, via the summed table instead
        v, out, issue = _run(ws, cells, seg, active, np.random.default_rng(trial))
        K = 1 << D
        offs = [tuple((s >> a) & 1 for a in range(D)) for s in range(K)]
        ref, got = {}, {}
        for i in range(32):
            for s in range(K):
                key = (int(seg[i]),) + tuple(int(c + o) for c, o in zip(cells[i], offs[s]))
                if active[i]:
                    ref[key] = ref.get(key, 0.0) + v[i, s].astype(np.float64)
                if (int(issue[i]) >> s) & 1:
                    got[key] = got.get(key, 0.0) + out[i, s].astype(np.float64)
        assert sorted(got) == sorted(ref)
        for key in ref:
            np.testing.assert_allclose(got[key], ref[key], rtol=1e-5, atol=1e-5)


def _rays3(n, rng, step, per_ray):
    x = np.zeros((n, 3), np.float32)
    seg = np.zeros(n, np.int32)
    for s in range(0, n, per_ray):
        o = rng.uniform(0.2, 0.8, 3)
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        x[s:s + per_ray] = np.clip(o + d * np.arange(min(per_ray, n - s))[:, None] * step, 0.0, 1.0)
        seg[s:s + per_ray] = s // per_ray
    return x, seg


@pytest.mark.parametrize("res,entries,step,per_ray", [(512, 1 << 19, 0.00055, 96), (1176, 1 << 19, 0.00055, 45),
                                                      (2703, 1 << 19, 0.0003, 77), (16, 4096, 0.004, 96),
                                                      (96, 64, 0.004, 96), (96, 64, 0.004, 45)])
def test_static_level_matches_the_per_lane_scatter(ws, res, entries, step, per_ray):
    """The static-hash sink of k_bwd_scatter_static against the plain per-lane scatter, with rays that straddle warps
    (per_ray not a multiple of 32) and with a hashed level whose tiny table (96^3 vertices into 64 entries) makes many
    distinct vertices share one entry: the sink keys on vertices, so collisions are summed, never merged."""
    rng = np.random.default_rng(res + per_ray)
    n = 32 * 12
    x, seg = _rays3(n, rng, step, per_ray)
    dd = rng.normal(size=(n, 4)).astype(np.float32)
    Ga, Gr = np.zeros((entries, 4), np.float32), np.zeros((entries, 4), np.float32)
    assert ws.vs_static_level(float(res - 1), res, entries, n, _p(np.ascontiguousarray(x)), _p(dd), _p(seg, C.c_int),
                              _p(Ga), _p(Gr)) == 0
    assert np.abs(Gr).max() > 0
    np.testing.assert_allclose(Ga, Gr, rtol=1e-5, atol=1e-5 * float(np.abs(Gr).max()))
