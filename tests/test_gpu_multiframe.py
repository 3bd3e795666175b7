"""GPU: rays of several frames in one render launch (L4DFrameTable through the split and fused pipelines).

A render over rows [B, N, 3] at B different times is one launch per table of up to L4D_MAX_FRAMES rows.  Ray (b, j) keeps
the jitter index ray_offset + b * N + j of the flattened launch, so the launch must equal B single-frame launches with
ray_offset = b * N: forwards bit for bit, gradients at the run-to-run noise floor of the multi-frame launch.  The row times
of the small config (num_frames = 6, 8 time slices) hit the first frame (no backward neighbour), the last (no forward
neighbour), interior frames, a time on a slice (`single`), two equal rows and rows whose slice pairs differ."""
import numpy as np
import pytest
import torch

from lidar4d_b200 import _capi
from test_gpu_launch_scale import (MODES, MODE_IDS, CAP, n_wrap, rays_for, small_oracle, model_for, upstream, render,
                                   backward, grads_of, assert_grads_additive, assert_oracle_parity, upstream_pattern)

pytestmark = pytest.mark.gpu
TIMES = [0.0, 1.0, 0.5, 0.5, 0.3, 0.62, 2.0 / 7.0]
OUT_KEYS = ("depth_lidar", "image_lidar", "weights_sum_lidar", "weights", "z_vals")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def wrap_rows(B: int) -> int:
    """Rays per row so that B rows exceed N_WRAP, and not a multiple of the SM count."""
    N = n_wrap() // B + 1
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return N + 1 if N % sms == 0 else N


def multi_render(m, ro, rd, times, S, perturb, dev):
    """One call over B rows of N rays at the B row times."""
    B = len(times)
    N = ro.shape[0] // B
    m._jitter_calls = 0
    return m.render(ro.view(B, N, 3).to(dev), rd.view(B, N, 3).to(dev), torch.tensor(times, dtype=torch.float32).view(B, 1),
                    num_steps=S, perturb=perturb)


def flat(out):
    return {k: (out[k].reshape(-1) if k == "depth_lidar" else out[k].reshape(-1, 2) if k == "image_lidar" else out[k])
            for k in OUT_KEYS}


def multi_step(m, ro, rd, times, S, perturb, U, dev):
    m.zero_grad(set_to_none=True)
    out = flat(multi_render(m, ro, rd, times, S, perturb, dev))
    if U is not None:
        ks = list(U)
        torch.autograd.backward([out[k] for k in ks], [U[k] for k in ks])
    return {k: v.detach() for k, v in out.items()}, (grads_of(m) if U is not None else None)


def row_steps(m, ro, rd, times, S, perturb, U, dev):
    """Each row as its own single-frame launch (ray_offset = b * N), gradients accumulated without zero_grad."""
    N = ro.shape[0] // len(times)
    m.zero_grad(set_to_none=True)
    outs = []
    for b, t in enumerate(times):
        out = render(m, ro, rd, t, S, perturb, b * N, N, dev)
        if U is not None:
            backward(out, U, b * N, N)
        outs.append(flat({k: v.detach() for k, v in out.items()}))
    return {k: torch.cat([o[k] for o in outs], 0) for k in OUT_KEYS}, (grads_of(m) if U is not None else None)


def assert_equal_outputs(a, b, what):
    for k in OUT_KEYS:
        assert a[k].shape == b[k].shape, (what, k, a[k].shape, b[k].shape)
        assert torch.equal(a[k], b[k]), (what, k, float((a[k] - b[k]).abs().max()))


def work_is_zero(m):
    torch.cuda.synchronize()
    return all(int(w.count_nonzero()) == 0 for w in m._engine._works.values())


def check_multi_vs_rows(m, ro, rd, times, S, dev, pipeline, what, seed=11):
    """1. forwards bit for bit with and without jitter; 2. gradients under upstream gradients on all four outputs, at the
    additivity bar of the multi-frame launch's own noise floor, identical touched sets, the work buffer zero after."""
    for perturb in (False, True):
        one, _ = multi_step(m, ro, rd, times, S, perturb, None, dev)
        rows, _ = row_steps(m, ro, rd, times, S, perturb, None, dev)
        assert_equal_outputs(one, rows, f"{what} perturb={perturb}")
    U = upstream(ro.shape[0], S, seed, dev)
    one1, G1 = multi_step(m, ro, rd, times, S, True, U, dev)
    assert work_is_zero(m), what
    one2, G2 = multi_step(m, ro, rd, times, S, True, U, dev)
    assert_equal_outputs(one1, one2, what + " rerun")
    noise = max(float((G1[k] - G2[k]).abs().max()) / max(float(G1[k].abs().max()), 1e-30) for k in G1)
    _, G_rows = row_steps(m, ro, rd, times, S, True, U, dev)
    assert work_is_zero(m), what
    assert_grads_additive(G1, G_rows, noise, what, CAP[pipeline])


@pytest.mark.parametrize("mode,pipeline", MODES, ids=MODE_IDS)
def test_multiframe_equals_rows_wrapping(dev, mode, pipeline):
    """Rows x N beyond N_WRAP, N not a multiple of the SM count: every persistent grid wraps across frame boundaries."""
    S, seed = 200, 3
    B = len(TIMES)
    N = wrap_rows(B)
    assert B * N > n_wrap()
    m = model_for(small_oracle(seed), mode, pipeline, seed)
    ro, rd = rays_for(B * N)
    check_multi_vs_rows(m, ro, rd, TIMES, S, dev, pipeline, f"multi-frame {mode}/{pipeline} B={B} N={N} S={S}")


def test_multiframe_benchmarked_config(dev):
    """L = 16, S = 768 (the benchmark's configuration), tensor-core split pipeline, wrapping."""
    from lidar4d_b200 import LiDAR4D
    from lidar4d_b200.rays import synthetic_sweep
    S = 768
    B = len(TIMES)
    N = wrap_rows(B)
    torch.manual_seed(0)
    m = LiDAR4D(num_frames=6, near_lidar=0.0105, far_lidar=0.851, n_levels_hash=16).to(dev)
    g = torch.Generator().manual_seed(0)
    with torch.no_grad():
        for k, p in m.named_parameters():
            if "hash" in k or "grid_enc" in k:
                p.copy_((torch.rand(p.shape, generator=g) - 0.5).to(dev))
            elif k.endswith("mlp.4.weight"):
                p.copy_((torch.randn(p.shape, generator=g) * 0.02).to(dev))
            elif "planes" in k:
                p.add_((torch.randn(p.shape, generator=g) * 0.1).to(dev))
    m.set_mlp_fp16(True)
    m.jitter_seed = 5
    ro, rd, _ = synthetic_sweep(7)
    sel = np.arange(0, 65536, 13)[:B * N]
    ro, rd = torch.from_numpy(ro[sel]).contiguous(), torch.from_numpy(rd[sel]).contiguous()
    check_multi_vs_rows(m, ro, rd, TIMES, S, dev, "split", f"multi-frame L16 tc/split B={B} N={N} S={S}", seed=12)


@pytest.mark.parametrize("mode,pipeline", MODES, ids=MODE_IDS)
def test_multiframe_inference_chunking(dev, mode, pipeline):
    """No-grad multi-frame renders in chunks that cut rows (each chunk's launch gets the frames it covers) equal the
    grad-mode forward bit for bit."""
    S, seed, N = 200, 3, 97
    B = len(TIMES)
    m = model_for(small_oracle(seed), mode, pipeline, seed)
    ro, rd = rays_for(B * N)
    ref, _ = multi_step(m, ro, rd, TIMES, S, True, None, dev)
    for c in (1, 7, N - 1, 2048):
        m.infer_ray_chunk = c
        with torch.no_grad():
            got = flat(multi_render(m, ro, rd, TIMES, S, True, dev))
        assert_equal_outputs(got, ref, f"{mode}/{pipeline} infer_ray_chunk={c}")


@pytest.mark.parametrize("mode,pipeline", MODES, ids=MODE_IDS)
def test_row_grouping(dev, mode, pipeline):
    """L4D_MAX_FRAMES + 3 rows: two launches (16 rows, then 3), still the per-row renders bit for bit."""
    S, seed, N = 160, 3, 41
    times = [abs(TIMES[i % len(TIMES)] - 0.01 * (i // len(TIMES))) for i in range(_capi.MAX_FRAMES + 3)]   # in [0, 1]
    m = model_for(small_oracle(seed), mode, pipeline, seed)
    ro, rd = rays_for(len(times) * N)
    n0 = m.gpu_launches
    one, _ = multi_step(m, ro, rd, times, S, True, None, dev)
    n_multi = m.gpu_launches - n0
    rows, _ = row_steps(m, ro, rd, times, S, True, None, dev)
    assert_equal_outputs(one, rows, f"{mode}/{pipeline} {len(times)} rows")
    assert n_multi > 0


@pytest.mark.parametrize("mode,pipeline", MODES, ids=MODE_IDS)
def test_multiframe_oracle(dev, mode, pipeline):
    """One multi-frame launch against the oracle run per row (band-limited tables, float32 and float64 oracles, the
    DESIGN 2(5) criteria of assert_oracle_parity)."""
    S, seed, N = 200, 3, 64
    B = len(TIMES)
    m = model_for(small_oracle(seed, smooth=True), mode, pipeline, seed)
    ro, rd = rays_for(B * N)
    U = upstream_pattern("all", B * N, S, dev)
    out, G = multi_step(m, ro, rd, TIMES, S, True, U, dev)
    mask = out["weights"].cpu() > 1e-4
    res = []
    for f64 in (False, True):
        orc = small_oracle(seed, smooth=True)
        if f64:
            orc.to_float64()
        Uc = {k: v.cpu() for k, v in U.items()}
        refs = []
        for b, t in enumerate(TIMES):
            sl = slice(b * N, (b + 1) * N)
            ref = orc.render(ro[sl], rd[sl], t, num_steps=S, perturb=True, seed=seed, ray_offset=b * N,
                             mask_override=mask[sl])
            torch.autograd.backward([ref[k] for k in Uc], [Uc[k][sl].to(ref[k].dtype) for k in Uc])
            refs.append({k: v.detach() for k, v in ref.items()})
        res += [{k: torch.cat([r[k] for r in refs], 0) for k in refs[0]}, orc.ref_named_grads()]
    out = {k: v.cpu() for k, v in out.items()}
    G = {k: v.cpu() for k, v in G.items()}
    assert_oracle_parity(out, G, tuple(res), f"multi-frame oracle {mode}/{pipeline} B={B} N={N} S={S}")


def test_api_time_shapes_launches_and_restaging(dev):
    """A bad time shape raises ValueError; B equal row times issue exactly the launches of the flattened one-frame call;
    re-staging between a multi-frame forward and its backward raises."""
    S, seed, N, B = 64, 3, 32, 4
    m = model_for(small_oracle(seed), "tc", "split", seed)
    ro, rd = rays_for(B * N)
    ro3, rd3 = ro.view(B, N, 3).to(dev), rd.view(B, N, 3).to(dev)
    for bad in (torch.zeros(B, 2), torch.zeros(B + 1, 1), torch.zeros(1, B)):
        with pytest.raises(ValueError):
            m.render(ro3, rd3, bad, num_steps=S)
    for train in (False, True):
        with torch.set_grad_enabled(train):
            m.render(ro3, rd3, torch.tensor([[0.4]]), num_steps=S)           # warm-up (staging, workspaces)
            torch.cuda.synchronize()
            n0 = m.gpu_launches
            a = m.render(ro3, rd3, torch.tensor([[0.4]]), num_steps=S)
            n1 = m.gpu_launches
            b = m.render(ro3, rd3, torch.full((B, 1), 0.4), num_steps=S)
            n2 = m.gpu_launches
        assert n2 - n1 == n1 - n0, (train, n1 - n0, n2 - n1)
        for k in OUT_KEYS:
            assert torch.equal(a[k], b[k]), (train, k)
    m.zero_grad(set_to_none=True)
    out = m.render(ro3, rd3, torch.tensor(TIMES[:B]).view(B, 1), num_steps=S)
    m.invalidate_staged()
    m.render(ro3[:1], rd3[:1], torch.tensor([[0.4]]), num_steps=S)            # re-stages the working set
    with pytest.raises(RuntimeError, match="changed between this forward and its backward"):
        out["depth_lidar"].sum().backward()
    m._engine.reset_work()
