"""GPU: the split forward's encoder stage, value by value, against a float64 evaluation of its own inputs.

k_contract_dynamic (DevModel::hd_con), k_contract_planes (DevModel::pl_con), the flow-grid gather of k_fwd_flow_tc /
k_fwd_gather (the flow-MLP inputs) and k_fwd_gather with its level-major l4d_static_sweep (the features, as fp16 hi + lo
operand tiles in tensor-core mode or fp32 SoA planes in fp32 mode) make no decisions once the sample positions and the
flow are given.  tests/gather_ref.py evaluates what they should write in float64; every feature of every sample, every
flow-MLP input, every live hd_con entry and every live pl_con entry is held to

    |got - ref| <= (n + 16) * 2^-24 * A              (fp32 values; A = sum of the magnitudes of the n terms)
    ... + 2^-22 * |ref| + 2^-25                      (features carried as fp16 hi + lo)

and the operand tiles are checked structurally (gather_ref.check_tile_structure: finite, zero padding rows, ones-padding
columns, hi a nearest fp16 value of hi + lo with |lo| <= ulp(hi) / 2).  The buffer is read after a grad-mode forward
(the autograd node of the render keeps it); no backward runs, so nothing has been written over the flow-MLP inputs.

Cases, in both split modes:
  a. the benchmark configuration (L = 16, S = 768, jitter) at N = 2 * 16 * SMs + 37 rays of a synthetic sweep, with
     white-noise and with initialisation-scale tables; every CTA of k_fwd_gather, l4d_static_sweep and k_fwd_flow_tc
     gets >= 2 units of work at any grid the hardware allows (<= 16 CTAs of 128 threads per SM);
  b. L = 3, 4, 5, 9 with S = 2, 45, 129, 333 (odd-level sweep tail; ones-padding columns at K = 85, 99, 127; 4- and
     1-wide stores of unaligned dynamic-hash rows; one-row tiles; partial last tiles), and one-ray launches;
  c. frames at t = 0, an interior t, t = 1 (last slice read through pair T - 2), an interior t whose current query is
     `single`, and a t whose time coordinate lies on a time-texel row (wy1 = 0);
  d. rays leaving the box through a face, an edge and a corner, bound = 0.5, a flow that takes many warped positions
     outside [0, 1] on both sides, and a zero flow;
  e. band-limited tables, tables at tiny-cuda-nn's +-1e-4 with planes at the reference's initialisation, and planes
     scaled so that features reach ~1e3.
Each case prints the worst fraction of the bound and the number of values checked per output kind; tensor-core cases
also print the share of features below 2^-3, where the 2^-25 floor rather than the relative term bounds the encoding,
and the largest |hi + lo - ref| / |ref|."""
import ctypes
import time

import numpy as np
import pytest
import torch

import gather_ref as GR
import scatter_ref as SR
import test_gpu_scatter_exact as SX
from lidar4d_b200.geometry import make_frame
from oracle import lidar4d_oracle as O
from parity_util import small_config, cuda_model_from_oracle, test_rays as _rays
from saved_util import saved_features

pytestmark = pytest.mark.gpu
MODES = ("tc", "fp32")
MAX_CTAS_128 = 16                 # 2048 threads per SM / 128-thread CTAs


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def forward_saved(m, ro, rd, t, S):
    """Grad-mode render; returns (outputs, saved buffer of the forward)."""
    dev = torch.device("cuda:0")
    m._jitter_calls = 0
    out = m.render(ro[None].to(dev), rd[None].to(dev), torch.tensor([[t]]), num_steps=S, perturb=True)
    saved = out["weights_sum_lidar"].grad_fn.saved
    assert saved is not None, "the render saved nothing (no parameter requires grad?)"
    torch.cuda.synchronize()
    return {k: v.detach() for k, v in out.items()}, saved


def assert_gather_exact(m, ro, rd, t, S, mode, what):
    """Grad-mode forward, then every value the encoder stage wrote against tests/gather_ref.py."""
    dev = torch.device("cuda:0")
    cfg = m.cfg
    N = ro.shape[0]
    tc = mode == "tc"
    t0 = time.perf_counter()
    out, saved = forward_saved(m, ro, rd, t, S)
    eng = m._engine
    assert SR.saved_layout(cfg, N, S)["total"] == eng._lib().l4d_saved_bytes(ctypes.byref(eng.ccfg), N, S)
    sv = SR.decode_saved(cfg, saved, N, S)
    x01 = SR.sample_x01(ro.to(dev), rd.to(dev), out["z_vals"], cfg.bound)
    fr = make_frame(t, cfg.num_frames, cfg.time_resolution)
    tabs = GR.Tables(cfg, {k: p.detach() for k, p in m.named_parameters()}, fr)
    stats, bad = {}, {}

    def hold(name, r, count):
        w, n = stats.get(name, (0.0, 0))
        stats[name] = (max(w, float(r.max()) if r.numel() else 0.0), n + count)
        nb = int((r > 1).sum())
        if nb:
            i = int(torch.argmax(r))
            bad[name] = bad.get(name, "") + f" {nb} over the bound (worst {float(r.reshape(-1)[i]):.2f} at flat {i});"

    for qi, _, _ in GR.queries(fr):
        for p in range(3):
            r = GR.ratio(sv["hd_con"][qi][p], *_table_bound(tabs.hd_con[qi, p], 8))
            hold("hd_con", r, r.numel())
        for s in range(cfg.n_levels_plane):
            for tt in range(3):
                r = GR.ratio(sv["pl_con"][qi][s][tt], *_table_bound(tabs.pl_con[qi, s, tt], 2))
                hold("pl_con", r, r.numel())

    feats = saved_features(cfg, saved, N, S, "tc") if tc else sv["feat"].t()
    nK = GR.feature_terms(cfg, fr).to(dev)
    floor, rel = [0, 0], 0.0

    def on_chunk(p0, p1, o):
        nonlocal rel
        ref, A = o["features"]
        got = feats[p0:p1]
        b = GR.tile_bound(ref, A, nK) if tc else GR.bound32(A, nK)
        hold("features", GR.ratio(got, ref, b), ref.numel())
        ref_f, A_f = o["flow_in"]
        hold("flow_in", GR.ratio(sv["flow_in"][:, p0:p1].t(), ref_f, GR.bound32(A_f, GR.FLOW_TERMS)), ref_f.numel())
        if tc:
            floor[0] += int((ref.abs() < 2.0 ** -3).sum())
            floor[1] += ref.numel()
            nz = ref != 0
            if bool(nz.any()):
                rel = max(rel, float(((got.double() - ref).abs()[nz] / ref.abs()[nz]).max()))
    GR.gather_reference(tabs, x01, sv["flow"], on_chunk)
    if tc:
        tiles = GR.check_tile_structure(cfg, sv["feat_tiles"], S)
        bad.update({f"tiles/{k}": f" {v} values" for k, v in tiles.items() if v})
    assert not bad, f"{what}: {bad}"
    msg = ", ".join(f"{k} {w:.3f} of the bound over {n}" for k, (w, n) in stats.items())
    if tc:
        msg += f"; features in the 2^-25 floor {floor[0] / max(floor[1], 1):.3f}, max |hi+lo-ref|/|ref| {rel:.2e}"
    print(f"[gather-exact] {what}: {msg}; {time.perf_counter() - t0:.1f} s")
    return out, sv, x01, feats


def _table_bound(ref_a, n):
    ref, A = ref_a
    return ref, GR.bound32(A, n)


# ---- a. the benchmark configuration ---------------------------------------------------------------------------------------
def full_model(mode, tables, seed=0):
    """The benchmark's model: white-noise tables as in the scatter test ("noise"), or tiny-cuda-nn's +-1e-4 hash tables with
    the reference's plane initialisation, spatial planes uniform(0.1, 0.5) and time planes 1 ("init")."""
    from lidar4d_b200 import LiDAR4D
    torch.manual_seed(seed)
    m = LiDAR4D(num_frames=51, near_lidar=0.0105, far_lidar=0.851, n_levels_hash=16).cuda()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for k, p in m.named_parameters():
            if "hash" in k or "grid_enc" in k:
                u = torch.rand(p.shape, generator=g) - 0.5
                p.copy_((u if tables == "noise" else u * 2e-4).cuda())
            elif k.endswith("mlp.4.weight"):
                p.copy_((torch.randn(p.shape, generator=g) * 0.02).cuda())
            elif "planes" in k:
                if tables == "noise":
                    p.add_((torch.randn(p.shape, generator=g) * 0.1).cuda())
                elif int(k.split(".")[-1]) in SR.TIME_PLANES:
                    p.fill_(1.0)
                else:
                    p.copy_((torch.rand(p.shape, generator=g) * 0.4 + 0.1).cuda())
    m.set_mlp_fp16(mode == "tc")
    m.jitter_seed = 5
    return m


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("tables", ["noise", "init"])
def test_benchmark_config(dev, mode, tables):
    from lidar4d_b200.rays import synthetic_sweep
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    N, S = 2 * MAX_CTAS_128 * sms + 37, 768
    units = {"k_fwd_gather": N * ((S + 127) // 128) if mode == "tc" else (N * S + 127) // 128,
             "l4d_static_sweep": (N * S + 127) // 128, "k_fwd_flow_tc": (N * S + 127) // 128}
    assert all(u >= 2 * MAX_CTAS_128 * sms for u in units.values()), units
    ro, rd, _ = synthetic_sweep(25)
    sel = np.linspace(0, ro.shape[0] - 1, N).astype(np.int64)
    ro, rd = torch.from_numpy(ro[sel]).contiguous(), torch.from_numpy(rd[sel]).contiguous()
    m = full_model(mode, tables)
    assert_gather_exact(m, ro, rd, 0.5, S, mode, f"L16 S768 N{N} {mode} {tables}")


# ---- b. level counts, sample counts, one-ray launches ---------------------------------------------------------------------
def small_oracle(seed, tables="noise", **over):
    orc = SX.small_oracle(seed, **over)
    if tables == "band":
        O.band_limit_tables(orc)
    elif tables == "init":
        init = O.OracleLiDAR4D(orc.cfg)                       # the reference's initialisation, +-1e-4 hash tables
        with torch.no_grad():
            for k, v in orc.P.items():
                if "hash" in k or "grid_enc" in k or "planes" in k:
                    v.copy_(init.P[k])
    elif tables == "large":
        with torch.no_grad():
            for k, v in orc.P.items():
                if "planes" in k:
                    v.mul_(20.0)
    return orc


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("S", [2, 45, 129, 333])
@pytest.mark.parametrize("L", [3, 4, 5, 9])
def test_levels_and_samples(dev, mode, L, S):
    orc = small_oracle(3, n_levels_hash=L)
    m = cuda_model_from_oracle(orc).set_mlp_fp16(mode == "tc")
    m.jitter_seed = 3
    ro, rd = _rays(8, 5)
    assert_gather_exact(m, torch.from_numpy(ro), torch.from_numpy(rd), 0.4, S, mode, f"L{L} S{S} {mode}")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("L,S", [(3, 2), (5, 333), (9, 129)])
def test_one_ray(dev, mode, L, S):
    orc = small_oracle(4, n_levels_hash=L)
    m = cuda_model_from_oracle(orc).set_mlp_fp16(mode == "tc")
    m.jitter_seed = 4
    ro, rd = _rays(1, 1)
    assert_gather_exact(m, torch.from_numpy(ro), torch.from_numpy(rd), 0.4, S, mode, f"one ray L{L} S{S} {mode}")


# ---- c. frames --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("which", ["first", "interior", "last", "single", "on-row"])
def test_frames(dev, mode, which):
    orc = small_oracle(5)
    cfg = orc.cfg
    single, row = GR.special_times(cfg)
    t = {"first": 0.0, "interior": 0.4, "last": 1.0, "single": single, "on-row": row}[which]
    fr = make_frame(t, cfg.num_frames, cfg.time_resolution)
    if which == "last":
        assert fr.cur.single and fr.cur.slice_lo == cfg.time_resolution - 1 and not fr.has_fwd
    if which == "first":
        assert not fr.has_bwd
    m = cuda_model_from_oracle(orc).set_mlp_fp16(mode == "tc")
    m.jitter_seed = 5
    ro, rd = _rays(8, 5)
    assert_gather_exact(m, torch.from_numpy(ro), torch.from_numpy(rd), t, 129, mode, f"t={t!r} ({which}) {mode}")


# ---- d. rays that leave the box, warped positions outside it ----------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ["exits", "bound0.5", "large-flow", "zero-flow"])
def test_clamped_and_warped_samples(dev, mode, name):
    S, t = 256, 0.4
    orc, ro, rd = SX.case_setup(name, 3)
    m = cuda_model_from_oracle(orc).set_mlp_fp16(mode == "tc")
    m.jitter_seed = 3
    _, sv, x01, _ = assert_gather_exact(m, ro, rd, t, S, mode, f"{name} {mode}")
    counts, _ = SX.clamp_counts(x01, S)
    assert min(counts) > 0, counts
    fl = sv["flow"].t()
    warped = torch.cat([x01 + fl[:, :3], x01 + fl[:, 3:]], 0)
    if name == "large-flow":
        assert float((warped < 0).any(1).double().mean()) > 0.01 and float((warped > 1).any(1).double().mean()) > 0.01
    if name == "zero-flow":
        assert float(fl.abs().max()) == 0.0


# ---- e. tables ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("tables", ["band", "init", "large"])
def test_tables(dev, mode, tables):
    orc = small_oracle(6, tables)
    m = cuda_model_from_oracle(orc).set_mlp_fp16(mode == "tc")
    m.jitter_seed = 6
    ro, rd = _rays(8, 5)
    _, _, _, feats = assert_gather_exact(m, torch.from_numpy(ro), torch.from_numpy(rd), 0.4, 129, mode,
                                         f"{tables} tables {mode}")
    fmax = float(feats.abs().max())
    if tables == "large":
        assert 500.0 < fmax < 65504.0 / 4, fmax
    if tables == "init":
        hs = slice(2 * orc.cfg.plane_dim, orc.cfg.sigma_in_dim)
        assert float(feats[:, hs].abs().max()) < 1e-3
