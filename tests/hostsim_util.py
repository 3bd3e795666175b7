"""Test helper: drive tests/hostsim/_hostsim.so (the kernels' per-sample code
compiled for the CPU) with parameters taken from an oracle model.  Test
infrastructure only."""
import ctypes as C
import os
import subprocess

import numpy as np
import torch

from lidar4d_b200 import _capi
from lidar4d_b200.geometry import make_frame

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostsim", "hostsim.cu")
SO = os.path.join(HERE, "hostsim", "_hostsim.so")
_LIB = None


def build(force=False):
    deps = [SRC] + [os.path.join(HERE, "..", "lidar4d_b200", "csrc", f)
                    for f in ("l4d_core.cuh", "l4d_bwd.cuh", "l4d_host.h")]
    if not force and os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in deps):
        return SO
    cmd = ["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC,-ffp-contract=off",
           "-gencode", "arch=compute_90a,code=sm_90a", "-o", SO, SRC]
    subprocess.run(cmd, check=True)
    return SO


WS_SRC = os.path.join(HERE, "hostsim", "warpsim.cu")
WS_SO = os.path.join(HERE, "hostsim", "_warpsim.so")


def build_warpsim(force=False):
    """tests/hostsim/warpsim.cu: the warp-collective gradient sinks compiled for the CPU on a 32-thread lockstep emulator."""
    deps = [WS_SRC] + [os.path.join(HERE, "..", "lidar4d_b200", "csrc", f) for f in ("l4d_core.cuh", "l4d_bwd.cuh")]
    if not force and os.path.exists(WS_SO) and all(os.path.getmtime(WS_SO) >= os.path.getmtime(d) for d in deps):
        return WS_SO
    cmd = ["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC,-ffp-contract=off",
           "-gencode", "arch=compute_90a,code=sm_90a", "-o", WS_SO, WS_SRC, "-lpthread"]
    subprocess.run(cmd, check=True)
    return WS_SO


def lib():
    global _LIB
    if _LIB is None:
        build()
        _LIB = _capi.declare(C.CDLL(SO), prefix="hs_", host_sim=True)
    return _LIB


class HostSim:
    """Holds staged params (host memory) for one oracle model."""

    def __init__(self, oracle, mlp_fp16=False):
        self.L = lib()
        self.cfg = oracle.cfg
        self.ccfg = _capi.make_config(self.cfg, mlp_fp16=mlp_fp16)
        self.params = {k: v.detach().contiguous().float() for k, v in oracle.ref_state_dict().items() if k != "aabb"}
        tab = _capi.L4DMasterParams()
        _capi.fill_pointer_table(tab, self.cfg, lambda n: self.params[n].data_ptr())
        nb = self.L.hs_staged_bytes(C.byref(self.ccfg))
        assert nb > 0, self.L.hs_last_error()
        self.staged = torch.zeros(nb, dtype=torch.uint8)
        rc = self.L.hs_stage_params(C.byref(self.ccfg), C.byref(tab), self.staged.data_ptr())
        assert rc == 0

    def frame(self, time):
        return _capi.make_frame_struct(make_frame(time, self.cfg.num_frames, self.cfg.time_resolution))

    def _rays(self, ro, rd, S, perturb, seed, ray_offset):
        r = _capi.L4DRays()
        self._ro = torch.as_tensor(ro, dtype=torch.float32).contiguous()
        self._rd = torch.as_tensor(rd, dtype=torch.float32).contiguous()
        r.rays_o, r.rays_d = self._ro.data_ptr(), self._rd.data_ptr()
        r.n_rays, r.n_steps, r.perturb = self._ro.shape[0], S, int(perturb)
        r.seed, r.ray_offset = seed, ray_offset
        return r

    def render(self, ro, rd, time, S, perturb=False, seed=0, ray_offset=0, train=False, contracted=False):
        """contracted=True: dynamic hash gathered from the per-launch contracted tables (k_contract_dynamic's mirror)"""
        fr = self.frame(time)
        rays = self._rays(ro, rd, S, perturb, seed, ray_offset)
        rays.reserved = 4 if contracted else 0
        N = rays.n_rays
        out = {k: torch.zeros(s) for k, s in [("depth", N), ("image", (N, 2)), ("wsum", N),
                                               ("weights", (N, S)), ("z_vals", (N, S))]}
        saved = None
        if train:
            saved = torch.zeros(self.L.hs_saved_bytes(C.byref(self.ccfg), N, S), dtype=torch.uint8)
        rc = self.L.hs_render_forward(C.byref(self.ccfg), self.staged.data_ptr(), C.byref(fr), C.byref(rays),
                                      out["depth"].data_ptr(), out["image"].data_ptr(), out["wsum"].data_ptr(),
                                      out["weights"].data_ptr(), out["z_vals"].data_ptr(),
                                      saved.data_ptr() if train else None)
        assert rc == 0, self.L.hs_last_error()
        self._saved, self._fr, self._rays_s = saved, fr, rays
        return out

    def saved_compositing_inputs(self):
        """σ [N, S] and the attribute heads' outputs [2, N, S] (0 outside the attribute mask) that the last
        render(train=True) saved, as the backward reads them."""
        from scatter_ref import saved_layout
        N, S = self._rays_s.n_rays, self._rays_s.n_steps
        L = saved_layout(self.cfg, N, S)
        f32 = lambda name, n: self._saved[L[name]:L[name] + 4 * n].view(torch.float32)
        return dict(sigma=f32("sigma", N * S).view(N, S).clone(), attr=f32("attr", 2 * N * S).view(2, N, S).clone())

    def _grad_tables(self):
        grads = {k: torch.zeros_like(v) for k, v in self.params.items()}
        tab = _capi.L4DMasterGrads()
        _capi.fill_pointer_table(tab, self.cfg, lambda n: grads[n].data_ptr())
        work = torch.zeros(self.L.hs_grad_work_bytes(C.byref(self.ccfg)), dtype=torch.uint8)
        return grads, tab, work

    def backward(self, g_depth, g_image, g_wsum=None, g_weights=None, comb=False):
        """comb=True: dynamic-hash gradients go through the slice-independent accumulators + fold of the split pipeline"""
        self._rays_s.reserved = 2 if comb else 0
        grads, tab, work = self._grad_tables()
        gd = torch.as_tensor(g_depth, dtype=torch.float32).contiguous()
        gi = torch.as_tensor(g_image, dtype=torch.float32).contiguous()
        gw = None if g_wsum is None else torch.as_tensor(g_wsum, dtype=torch.float32).contiguous()
        gww = None if g_weights is None else torch.as_tensor(g_weights, dtype=torch.float32).contiguous()
        rc = self.L.hs_render_backward(C.byref(self.ccfg), self.staged.data_ptr(), C.byref(self._fr),
                                       C.byref(self._rays_s), self._saved.data_ptr(), gd.data_ptr(), gi.data_ptr(),
                                       gw.data_ptr() if gw is not None else None,
                                       gww.data_ptr() if gww is not None else None, C.byref(tab), work.data_ptr())
        assert rc == 0, self.L.hs_last_error()
        rc = self.L.hs_unstage_grads(C.byref(self.ccfg), work.data_ptr(), C.byref(tab))
        assert rc == 0
        return grads

    def flow(self, x, time, g_flow=None):
        fr = self.frame(time)
        x = torch.as_tensor(x, dtype=torch.float32).contiguous()
        n = x.shape[0]
        out = torch.zeros(n, 6)
        saved = torch.zeros(16, n)
        rc = self.L.hs_flow_forward(C.byref(self.ccfg), self.staged.data_ptr(), C.byref(fr), x.data_ptr(), n,
                                    out.data_ptr(), saved.data_ptr())
        assert rc == 0
        if g_flow is None:
            return out
        grads, tab, work = self._grad_tables()
        g = torch.as_tensor(g_flow, dtype=torch.float32).contiguous()
        rc = self.L.hs_flow_backward(C.byref(self.ccfg), self.staged.data_ptr(), C.byref(fr), x.data_ptr(), n,
                                     saved.data_ptr(), g.data_ptr(), C.byref(tab), work.data_ptr())
        assert rc == 0
        rc = self.L.hs_unstage_grads(C.byref(self.ccfg), work.data_ptr(), C.byref(tab))
        assert rc == 0
        return out, grads

    def hash_indices(self, grid_id, level, x):
        x = torch.as_tensor(x, dtype=torch.float32).contiguous()
        n, D = x.shape
        idx = torch.zeros(n, 1 << D, dtype=torch.int32)
        w = torch.zeros(n, 1 << D)
        rc = self.L.hs_hash_indices(C.byref(self.ccfg), grid_id, level, x.data_ptr(), n, idx.data_ptr(), w.data_ptr())
        assert rc == 0
        return idx.numpy().view(np.uint32), w.numpy()

    def density(self, x, time):
        fr = self.frame(time)
        x = torch.as_tensor(x, dtype=torch.float32).contiguous()
        n = x.shape[0]
        sigma, geo = torch.zeros(n), torch.zeros(n, 15)
        feats, flow = torch.zeros(n, self.cfg.sigma_in_dim), torch.zeros(n, 6)
        rc = self.L.hs_density_forward(C.byref(self.ccfg), self.staged.data_ptr(), C.byref(fr), x.data_ptr(), n,
                                       sigma.data_ptr(), geo.data_ptr(), feats.data_ptr(), flow.data_ptr())
        assert rc == 0
        return dict(sigma=sigma, geo_feat=geo, features=feats, flow=flow)
