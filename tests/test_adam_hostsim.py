"""CPU: k_adam_flat's per-element update (l4d_adam_elem, compiled for the host by tests/hostsim/adamsim.cu) is bit for bit
torch 2.11's fused Adam (fused_adam_utils.cuh adam_math) in every value regime, stays within a recorded bound of a float64
Adam on the same fp32 inputs, and l4d_adam_step rejects every malformed argument before it launches anything."""
import ctypes as C

import numpy as np
import pytest

import __graft_entry__
from lidar4d_b200 import _capi
from lidar4d_b200.geometry import FieldConfig

B1, B2, EPS = np.float32(0.9), np.float32(0.99), np.float32(1e-15)     # main_lidar4d.py:298-300
STEPS = (1, 2, 3, 4, 11, 14, 100, 10_000, 1_000_000)
LRS = (np.float32(1e-2), np.float32(1e-3), np.float32(3.7e-4))
N = 1 << 20
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(__graft_entry__.build_adamsim())
        P, F = C.c_void_p, C.c_float
        L.as_kernel.argtypes = L.as_torch.argtypes = [C.c_int64, P, P, P, P] + [F] * 7
        L.as_former.argtypes = [C.c_int64, P, P, P, P] + [F] * 5 + [C.c_uint32]
        L.as_kernel.restype = L.as_torch.restype = L.as_former.restype = None
        _LIB = L
    return _LIB


def bias(step):
    """fp32 bias corrections (any fp32 values serve: both sides receive the same ones)."""
    bc1 = np.float32(1) - B1 ** np.float32(step)
    bc2s = np.sqrt(np.float32(1) - B2 ** np.float32(step))
    return np.float32(bc1), np.float32(bc2s)


def _ptr(a):
    return a.ctypes.data


def run(fn, p, m, v, g, step, lr, scale=np.float32(1)):
    """One step of `fn` ('kernel', 'torch' or 'former') on copies; scale = inv_scale (torch gets 1 / scale)."""
    p, m, v, g = (np.ascontiguousarray(x, dtype=np.float32).copy() for x in (p, m, v, g))
    bc1, bc2s = bias(step)
    L = lib()
    if fn == "kernel":
        L.as_kernel(p.size, _ptr(p), _ptr(m), _ptr(v), _ptr(g), scale, B1, B2, EPS, lr, bc1, bc2s)
    elif fn == "torch":
        L.as_torch(p.size, _ptr(p), _ptr(m), _ptr(v), _ptr(g), np.float32(1) / scale, B1, B2, EPS, lr, bc1, bc2s)
    else:
        L.as_former(p.size, _ptr(p), _ptr(m), _ptr(v), _ptr(g), scale, B1, B2, EPS, lr, step)
    return p, m, v


def logu(rng, lo, hi, n, signed=True):
    x = (10.0 ** rng.uniform(lo, hi, n)).astype(np.float32)
    return x * rng.choice(np.float32([-1, 1]), n) if signed else x


def regime(name, rng, n=N):
    """(p, m, v, g, inv_scale per element) of one value regime"""
    p, m, g = logu(rng, -8, 3, n), logu(rng, -8, 3, n), logu(rng, -8, 3, n)
    v = logu(rng, -16, 6, n, signed=False)
    s = np.ones(n, np.float32)
    if name == "g_zero":
        g = np.where(rng.random(n) < 0.5, np.float32(0), np.float32(-0.0)).astype(np.float32)
    elif name == "g_tiny":                                 # g^2 subnormal or 0, g itself down to subnormal
        g = logu(rng, -45, -19, n)
        m, v = logu(rng, -30, -10, n), logu(rng, -44, -20, n, signed=False)
    elif name == "update_subnormal":                       # a / den subnormal, p subnormal or tiny
        p, m = logu(rng, -45, -30, n), logu(rng, -40, -25, n)
        v, g = logu(rng, -8, 2, n, signed=False), np.zeros(n, np.float32)
    elif name == "v_large":                                # v >= 2^64
        v = (2.0 ** rng.uniform(64, 127.9, n)).astype(np.float32)
        m = logu(rng, -8, 30, n)
    elif name == "g_huge":                                 # g^2 = inf
        g = logu(rng, np.log10(1.9e19), 38.5, n)
    elif name == "nonfinite":
        g = rng.choice(np.float32([np.inf, -np.inf, np.nan, 1.0, -0.5]), n)
    elif name == "inv_scale":
        k = rng.integers(-16, 17, n)
        s = (2.0 ** k).astype(np.float32)
        g = (g * (2.0 ** -k)).astype(np.float32)          # the scaled gradient GradScaler would hand in
    return p, m, v, g, s


REGIMES = ("magnitudes", "g_zero", "g_tiny", "update_subnormal", "v_large", "g_huge", "nonfinite", "inv_scale")


def step_slices(n):
    """the regime's elements are split over every (step, lr) case"""
    edges = np.linspace(0, n, len(STEPS) + 1).astype(int)
    return [(STEPS[j], LRS[j % len(LRS)], slice(edges[j], edges[j + 1])) for j in range(len(STEPS))]


def apply(fn, p, m, v, g, s):
    P, M, V = p.copy(), m.copy(), v.copy()
    for step, lr, sl in step_slices(p.size):
        for sc in np.unique(s[sl]):
            idx = np.arange(sl.start, sl.stop)[s[sl] == sc]
            P[idx], M[idx], V[idx] = run(fn, p[idx], m[idx], v[idx], g[idx], step, lr, sc)
    return P, M, V


def bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.int32)


def mismatches(a, b):
    return int((bits(a) != bits(b)).sum())


@pytest.mark.parametrize("name", REGIMES)
def test_kernel_update_is_torch_fused_adam_bit_for_bit(name):
    """p, m and v compared as int32: signed zeros and NaN payload-free patterns must match too."""
    p, m, v, g, s = regime(name, np.random.default_rng(REGIMES.index(name)))
    kern, ref = apply("kernel", p, m, v, g, s), apply("torch", p, m, v, g, s)
    for what, a, b in zip("pmv", kern, ref):
        assert mismatches(a, b) == 0, (name, what, mismatches(a, b))


def test_subnormal_moments_over_2000_zero_gradient_steps():
    """m and v decay through the subnormal range to 0 while p keeps moving; every step bit-equal to torch."""
    rng = np.random.default_rng(11)
    n = 1 << 16
    p = logu(rng, -8, 3, n)
    m, v = logu(rng, -38, -10, n), logu(rng, -44, -20, n, signed=False)
    g = np.where(rng.random(n) < 0.25, logu(rng, -45, -20, n), np.float32(0)).astype(np.float32)
    k = (p, m, v)
    t = (p, m, v)
    seen_sub = 0
    for step in range(1, 2001):
        gs = g if step == 1 else np.zeros_like(g)
        k = run("kernel", *k, gs, step, LRS[1])
        t = run("torch", *t, gs, step, LRS[1])
        if step % 50 == 0 or step < 5:
            for what, a, b in zip("pmv", k, t):
                assert mismatches(a, b) == 0, (step, what)
            seen_sub += int(((np.abs(t[2]) < 2.0 ** -126) & (t[2] != 0)).sum())
    for what, a, b in zip("pmv", k, t):
        assert mismatches(a, b) == 0, what
    assert seen_sub > 0


def test_former_update_fails_both_checks():
    """The former arithmetic (lerp first moment, unfused second moment, double-precision bias corrections, unconditional
    2^64 scaling) is caught by the bit-equality check on ordinary values, and it freezes parameters with v >= 2^64."""
    rng = np.random.default_rng(5)
    p, m, v, g, s = regime("magnitudes", rng, 1 << 17)
    for step in (1, 2, 3):
        old, ref = run("former", p, m, v, g, step, LRS[0]), run("torch", p, m, v, g, step, LRS[0])
        assert mismatches(old[1], ref[1]) > 0.05 * p.size       # lerp form of exp_avg: ~18 % of entries
        if step > 1:                                            # bias correction rounded differently at steps 2, 3
            assert mismatches(old[0], ref[0]) > 0.05 * p.size
    p, m, v, g, s = regime("v_large", rng, 1 << 16)
    old, ref = run("former", p, m, v, g, 1, LRS[0]), run("torch", p, m, v, g, 1, LRS[0])
    frozen = bits(old[0]) == bits(p)
    moved = bits(ref[0]) != bits(p)
    assert (frozen & moved).sum() > 0.25 * p.size          # the rest move by less than half an ulp of p in torch too
    # one parameter, g = 5e10 at step 1: the former update leaves p = 1, torch moves it by lr
    one = [np.float32([x]) for x in (1.0, 0.0, 0.0, 5e10)]
    assert run("former", *one, 1, np.float32(0.01))[0][0] == 1.0
    assert run("torch", *one, 1, np.float32(0.01))[0][0] == np.float32(0.99)
    assert run("kernel", *one, 1, np.float32(0.01))[0][0] == np.float32(0.99)


# ---- float64 Adam on the same fp32 inputs -----------------------------------------------------------------------
# |fp32 - float64| <= k * 2^-24 * A (+ absolute terms of the subnormal range), A = the sum of the magnitudes of the terms.
# k counts the roundings each result goes through: m two (inner and outer fma), v three (g*g and the two fmas), p four
# before m's and v's errors propagate.  Measured worst over the regimes below: m 1.89, v 2.56, p 2.62.
ULP_BOUND = dict(m=2.0, v=3.0, p=4.0)
TINY = 2.0 ** -149


@pytest.mark.parametrize("name", ["magnitudes", "g_zero", "g_tiny", "update_subnormal", "v_large", "inv_scale"])
def test_kernel_update_within_bound_of_float64_adam(name):
    p, m, v, g, s = regime(name, np.random.default_rng(100 + REGIMES.index(name)), 1 << 18)
    P, M, V = apply("kernel", p, m, v, g, s)
    b1, b2, eps = float(B1), float(B2), float(EPS)
    gd, md, vd, pd = (x.astype(np.float64) for x in (g * s, m, v, p))
    m64 = b1 * md + (1 - b1) * gd
    v64 = b2 * vd + (1 - b2) * gd * gd
    a_m = b1 * np.abs(md) + (1 - b1) * np.abs(gd)
    a_v = b2 * vd + (1 - b2) * gd * gd
    step_size = np.empty_like(pd)
    bc2s = np.empty_like(pd)
    for step, lr, sl in step_slices(p.size):
        b_1, b_2 = bias(step)
        step_size[sl], bc2s[sl] = float(lr) / float(b_1), float(b_2)
    den = np.sqrt(v64) / bc2s + eps
    u64 = step_size * m64 / den
    p64 = pd - u64
    # the update inherits m's error (relative to A_m, or absolute for a subnormal m) scaled by step_size / den, and
    # torch's order rounds step_size * m before the division, which is absolute 2^-149 / den when that product is subnormal
    a_p = np.abs(pd) + np.abs(u64) + step_size * a_m / den
    worst = {}
    for k, got, ref, a, tiny in (("m", M, m64, a_m, TINY), ("v", V, v64, a_v, TINY),
                                 ("p", P, p64, a_p, TINY * (2 + (step_size + 1) / den))):
        err = np.abs(got.astype(np.float64) - ref) - tiny
        units = np.max(np.where(err > 0, err / (a * 2.0 ** -24 + 1e-300), 0.0))
        worst[k] = units
        assert units <= ULP_BOUND[k], (name, k, units)
    print(name, {k: round(float(x), 3) for k, x in worst.items()})


# ---- l4d_adam_step argument validation (no GPU: every branch returns before the launch) ---------------------------
FAKE = 1 << 20                                        # 16-byte aligned, never dereferenced


def _groups(*ranges, lr=1e-3):
    arr = (_capi.L4DAdamGroup * max(1, len(ranges)))()
    for i, (b, e) in enumerate(ranges):
        arr[i].begin, arr[i].end, arr[i].lr = b, e, lr
    return arr


CASES = [
    # (label, overrides, expected code, message fragment)
    ("null params", dict(params=None), -1, b"null pointer"),
    ("null grads", dict(grads=None), -1, b"null pointer"),
    ("null exp_avg", dict(exp_avg=None), -1, b"null pointer"),
    ("null exp_avg_sq", dict(exp_avg_sq=None), -1, b"null pointer"),
    ("null groups", dict(groups=None), -1, b"null pointer"),
    ("0 groups", dict(n_groups=0), -1, b"1..64 Adam groups"),
    ("65 groups", dict(n_groups=65), -1, b"1..64 Adam groups"),
    ("arena not whole chunks", dict(n_floats=8192 + 4), -1, b"multiple of 1024 floats"),
    ("step 0", dict(step=0), -1, b"step >= 1"),
    ("params misaligned", dict(params=FAKE + 4), -1, b"16-byte aligned"),
    ("exp_avg_sq misaligned", dict(exp_avg_sq=FAKE + 4), -1, b"16-byte aligned"),
    ("unsorted groups", dict(groups=[(4096, 8192), (0, 1024)]), -1, b"sorted, disjoint"),
    ("overlapping groups", dict(groups=[(0, 2048), (1024, 4096)]), -1, b"sorted, disjoint"),
    ("begin not chunk-aligned", dict(groups=[(512, 1024)]), -1, b"sorted, disjoint"),
    ("end not a multiple of 4", dict(groups=[(0, 1026)]), -1, b"sorted, disjoint"),
    ("end beyond the arena", dict(groups=[(0, 8192 + 4)]), -1, b"sorted, disjoint"),
    ("empty group", dict(groups=[(1024, 1024)]), -1, b"sorted, disjoint"),
    ("master without staged", dict(master=True, staged=None), -1, b"without a staged buffer"),
    ("staged too small", dict(master=True, staged=FAKE, staged_bytes=1024), -3, b"staged buffer too small"),
]


@pytest.mark.parametrize("label,over,code,msg", CASES, ids=[c[0].replace(" ", "-") for c in CASES])
def test_adam_step_rejects_bad_arguments_without_launching(label, over, code, msg):
    L = _capi.load_library()
    cfg = _capi.make_config(FieldConfig())
    a = dict(params=FAKE, grads=FAKE, exp_avg=FAKE, exp_avg_sq=FAKE, n_floats=8192, groups=[(0, 4096)], n_groups=None,
             step=1, master=None, staged=None, staged_bytes=0)
    a.update(over)
    groups = None if a["groups"] is None else _groups(*a["groups"])
    n_groups = a["n_groups"] if a["n_groups"] is not None else len(a["groups"] or [None])
    master = _capi.L4DMasterParams() if a["master"] else None
    before = L.l4d_launch_count()
    L.l4d_last_error()
    rc = L.l4d_adam_step(C.byref(cfg), a["params"], a["grads"], a["exp_avg"], a["exp_avg_sq"], a["n_floats"], groups,
                         n_groups, 0.9, 0.99, 1e-15, a["step"], 1.0, 0,
                         C.byref(master) if master is not None else None, a["staged"], a["staged_bytes"], None)
    assert rc == code, (label, rc, L.l4d_last_error())
    assert msg in L.l4d_last_error(), label
    assert L.l4d_launch_count() == before
