"""Drop-in `LiDAR4D` / `LiDAR_Renderer` nn.Modules backed by liblidar4d_b200.so.

API mirrored from the reference (paths relative to the reference checkout):
  LiDAR4D.__init__ kwargs           model/lidar4d.py:23-45, main_lidar4d.py:155-179
  render(rays_o, rays_d, time, staged, max_ray_batch, **kw) -> dict   model/renderer.py:142-186
  run(rays_o, rays_d, time, num_steps, perturb, **kw) -> dict         model/renderer.py:44-140
  flow(x, t) -> {"forward","backward"}                                model/lidar4d.py:124-137
  density(x, t) -> {"sigma","geo_feat"}                               model/lidar4d.py:139-188
  get_params(lr)                                                      model/lidar4d.py:226-237
  state_dict keys / shapes                                            SURVEY.md 8(b)

There is no PyTorch/CPU implementation of the math in this file: every call
lands in the CUDA library through ctypes and raises if that is impossible.
"""
from __future__ import annotations

import ctypes as C
import itertools
import math
import weakref
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn as nn

from . import _capi
from .geometry import FieldConfig, make_frame, make_time_query


# =============================================================================
# parameter containers with the reference's module / parameter names
# =============================================================================
class _Submodule(nn.Module):
    """A submodule of LiDAR4D that runs its own CUDA op: it reaches the owner's engine through a weak link that
    LiDAR4D sets after construction (a registered back-reference would make the module tree cyclic)."""

    _owner_ref = None

    def _owner(self) -> "LiDAR4D":
        owner = self._owner_ref() if self._owner_ref is not None else None
        if owner is None:
            raise RuntimeError(f"{type(self).__name__} runs through the LiDAR4D that owns it; build it inside a LiDAR4D")
        return owner


class _TcnnParams(_Submodule):
    """Stands where a tcnn.Encoding / tcnn.Network stood: a flat fp32 `params` vector and `n_output_dims`
    (hash_field.py:137-139, lidar4d.py:84,96,108).  `kind` says which encoding or network it is, and thereby what its
    forward runs: "hash_static", ("hash_slice", plane, slice), "flow_grid", "freq", "sigma", "raydrop", "intensity"."""

    def __init__(self, n_params: int, n_output_dims: int, init: str, kind=None, **kw):
        super().__init__()
        self.n_output_dims = n_output_dims
        self.kind = kind
        p = torch.empty(n_params)
        if init == "hash":
            p.uniform_(-1e-4, 1e-4)                      # tcnn grid init [tcnn-ext]
        elif init == "mlp":
            o = 0
            dims = kw["dims"]
            for i in range(len(dims) - 1):               # xavier-uniform per [out,in] matrix [tcnn-ext]
                n = dims[i] * dims[i + 1]
                s = math.sqrt(6.0 / (dims[i] + dims[i + 1]))
                p[o:o + n].uniform_(-s, s)
                o += n
        elif init == "empty":
            pass
        self.params = nn.Parameter(p)

    def forward(self, x):
        """tcnn semantics on x [N, in] (encodings: coordinates in [0, 1]) -> [N, n_output_dims] float32.  Networks pad
        their input with ones to the network width and give dL/dx; encodings give no input gradient."""
        owner = self._owner()
        c = owner.cfg
        k = self.kind
        if k == "hash_static":
            return _run_module(owner, "enc", _capi.MOD_HASH_STATIC, x, 3, 4 * c.n_levels_hash,
                               ["hash_encoder.hash_static.params"], "hash_encoder.hash_static")
        if isinstance(k, tuple) and k[0] == "hash_slice":
            _, p, t = k
            return _run_module(owner, "enc", _capi.MOD_HASH_SLICE0 + p, x, 2, 4 * c.n_levels_hash,
                               [f"hash_encoder.hash_dynamic.{p}.hash_t.{t}.params"],
                               f"hash_encoder.hash_dynamic[{p}].hash_t[{t}]", slice_=t)
        if k == "flow_grid":
            return _run_module(owner, "enc", _capi.MOD_FLOW_GRID, x, 3, 8 * c.flow_n_levels,
                               ["flow_net.grid_enc.params"], "flow_net.grid_enc")
        if k == "freq":
            return _run_module(owner, "enc", _capi.MOD_FREQ, x, 3, c.view_dim, [], "view_encoder")
        if k == "sigma":
            return _run_module(owner, "mlp", _capi.NET_SIGMA, x, c.sigma_in_dim, 1 + c.geo_feat_dim,
                               ["sigma_net.params"], "sigma_net", input_grad=True)
        if k in ("raydrop", "intensity"):
            net = _capi.NET_RAYDROP if k == "raydrop" else _capi.NET_INTENSITY
            return _run_module(owner, "mlp", net, x, c.attr_in_dim, 1, [f"{k}_net.params"], f"{k}_net",
                               input_grad=True)
        raise RuntimeError(f"this _TcnnParams ({k!r}) has no forward")


class _HashGridT(_Submodule):
    def __init__(self, n_params, time_resolution, n_output_dims, plane: int):
        super().__init__()
        self.hash_t = nn.ModuleList([_TcnnParams(n_params, n_output_dims * 4, "hash", kind=("hash_slice", plane, s))
                                     for s in range(time_resolution)])
        self.n_output_dims = n_output_dims
        self.plane = plane

    def forward(self, x, t):
        """HashGridT.forward (hash_field.py:76-88): x [N,2] in [0,1], t a float or a one-element tensor -> [N, L]."""
        owner = self._owner()
        c = owner.cfg
        return _run_module(owner, "enc", _capi.MOD_HASH_T0 + self.plane, x, 2, c.n_levels_hash,
                           [f"hash_encoder.hash_dynamic.{self.plane}.hash_t.{s}.params" for s in range(c.time_resolution)],
                           f"hash_encoder.hash_dynamic[{self.plane}]", t=t)


class _HashGrid4D(_Submodule):
    def __init__(self, cfg: FieldConfig):
        super().__init__()
        gs = cfg.static_grid()
        self.hash_static = _TcnnParams(gs.n_params, gs.n_output_dims, "hash", kind="hash_static")
        self.hash_dynamic = nn.ModuleList([
            _HashGridT(cfg.dynamic_grid(p).n_params, cfg.time_resolution, cfg.hash_dynamic_dim // 3, p) for p in range(3)])
        self.n_output_dims = cfg.hash_static_dim + cfg.hash_dynamic_dim

    def forward_static(self, x):
        return self.hash_static(x)

    def forward_dynamic(self, x, t):
        """hash_field.py:146-158: x [N,3] in [0,1] -> cat(xy, xz, yz planes at t) [N, 3L]."""
        owner = self._owner()
        c = owner.cfg
        names = [f"hash_encoder.hash_dynamic.{p}.hash_t.{s}.params" for p in range(3) for s in range(c.time_resolution)]
        return _run_module(owner, "enc", _capi.MOD_HASH_DYNAMIC, x, 3, 3 * c.n_levels_hash, names,
                           "hash_encoder.forward_dynamic", t=t)

    def forward(self, x, t):
        return [self.forward_static(x), self.forward_dynamic(x, t)]


_STATIC_PLANES, _DYNAMIC_PLANES = (0, 1, 3), (2, 4, 5)


class _Planes4D(_Submodule):
    """planes_field.py:144-190: ModuleList over scales of ParameterList over the 6 planes."""

    def __init__(self, cfg: FieldConfig):
        super().__init__()
        self.planes = nn.ModuleList()
        combs = list(itertools.combinations(range(4), 2))
        for mult in cfg.plane_scales:
            reso = [cfg.min_resolution * mult] * 3 + [cfg.time_resolution]
            pl = nn.ParameterList()
            for comb in combs:
                t = torch.empty([1, cfg.n_features_per_level_plane] + [reso[cc] for cc in comb[::-1]])
                if 3 in comb:
                    nn.init.ones_(t)
                else:
                    nn.init.uniform_(t, a=0.1, b=0.5)
                pl.append(nn.Parameter(t))
            self.planes.append(pl)
        self.n_output_dims = 2 * cfg.plane_dim

    def _sample(self, xt, dynamic: bool):
        owner = self._owner()
        c = owner.cfg
        names = [f"planes_encoder.planes.{s}.{ci}" for s in range(c.n_levels_plane)
                 for ci in (_DYNAMIC_PLANES if dynamic else _STATIC_PLANES)]
        return _run_module(owner, "enc", _capi.MOD_PLANES_DYNAMIC if dynamic else _capi.MOD_PLANES_STATIC, xt, 4,
                           c.plane_dim, names, "planes_encoder", input_grad=True)

    def forward_static(self, xt):
        """planes_field.py:198-209: xt [N,4] in [0,1] -> [N, 8S]; differentiable w.r.t. the planes and xt."""
        return self._sample(xt, False)

    def forward_dynamic(self, xt):
        """planes_field.py:211-222: time planes at each row's own xt[:, 3]."""
        return self._sample(xt, True)

    def forward(self, xt):
        return [self.forward_static(xt), self.forward_dynamic(xt)]


class _FlowField(_Submodule):
    def __init__(self, cfg: FieldConfig):
        super().__init__()
        gf = cfg.flow_grid()
        self.grid_enc = _TcnnParams(gf.n_params, gf.n_output_dims, "hash", kind="flow_grid")
        h = cfg.hidden_dim_flow
        self.mlp = nn.Sequential(nn.Linear(gf.n_output_dims // 4, h, bias=False), nn.ReLU(),
                                 nn.Linear(h, h, bias=False), nn.ReLU(), nn.Linear(h, 6, bias=False))
        torch.nn.init.normal_(self.mlp[-1].weight.data, 0, 0.001)     # flow_field.py:100

    def forward(self, xt):
        """flow_field.py:113-130: xt [N,4] in [0,1] -> flow [N,6].  The time of every row is xt[0,3] (as there), read
        on the device.  Differentiable w.r.t. the grid and the three Linear weights, not w.r.t. xt."""
        owner = self._owner()
        return _run_module(owner, "enc", _capi.MOD_FLOW, xt, 4, 6,
                           ["flow_net.grid_enc.params", "flow_net.mlp.0.weight", "flow_net.mlp.2.weight",
                            "flow_net.mlp.4.weight"], "flow_net")


# =============================================================================
# engine: flat arenas, staging, pointer tables, launches
# =============================================================================
ARENA_ALIGN = 1024          # floats; = L4D_ADAM_CHUNK of include/lidar4d_b200.h


class _Engine:
    """Owns what the kernels need besides the caller's tensors:

    * ONE flat fp32 parameter arena - every hot-path parameter's ``.data`` is a view into it (state_dict keys, shapes
      and ``load_state_dict`` are unchanged; after ``model.to(device)`` the views are rebuilt lazily) - and ONE flat
      fp32 gradient arena that every ``.grad`` views: the backward kernels accumulate straight into it (no per-launch
      allocation, no autograd accumulation pass), ``RayShardedDP`` all-reduces it in place, ``lidar4d_b200.optim.Adam``
      updates both arenas in one launch;
    * the staged working set (fp16 tables, channels-last planes, MLP operand copies), refreshed when a master changed;
    * the persistent gradient work buffer (zero between launches: the fold kernels clear what they consume).
    """

    def __init__(self, owner: "LiDAR4D", cfg=None):
        self.owner = owner
        self.cfg = cfg if cfg is not None else owner.cfg
        # default = what the reference does: tiny-cuda-nn's FullyFusedMLP consumes fp16 copies of its fp32 parameters;
        # this is also the mode that runs the dense kernels on the wgmma tensor cores
        self.mlp_fp16 = True
        self.ccfg = _capi.make_config(self.cfg, True)
        self.names = _capi.param_names(self.cfg)
        self.lib = None
        self.staged = None
        self._stamp = None
        self._staged_grad_mode = None
        self._chk = None
        self._chk_grad = None      # device checksum of the masters at grad-mode submodule calls (note_grad_content)
        self.stage_gen = 0         # bumped by every re-staging; forward records it, backward checks it
        self.static_params = False # True: skip the content check of no-grad calls (tight inference loops)
        self.flat_p = None
        self.flat_g = None
        self._works = {}
        self._tensors = None
        self._mtab = None
        self.offsets = None        # name -> (offset, numel) in floats
        self.total = 0
        self._gtab = None
        self.hash_grads_hook = None  # (torch.cuda.Event, callable): see parallel.RayShardedDP.final_backward
        self.timing = None         # {'fwd': [(ev0, ev1)], 'bwd': [...]}: CUDA events around the fused kernels

    def __deepcopy__(self, memo):
        """copy.deepcopy(model) (some EMA / checkpoint helpers do this): the copy gets a FRESH engine - ctypes pointer
        tables cannot be copied and its arenas are rebuilt lazily around the copied parameters on first use."""
        owner = memo.get(id(self.owner), self.owner)
        new = _Engine.__new__(_Engine)
        memo[id(self)] = new
        _Engine.__init__(new, owner, cfg=self.cfg)       # (the owner's own attributes are still being copied at this point)
        new.set_mlp_fp16(self.mlp_fp16)
        new.static_params = self.static_params
        return new

    def set_mlp_fp16(self, on: bool):
        if bool(on) != self.mlp_fp16:
            self.mlp_fp16 = bool(on)
            self.ccfg = _capi.make_config(self.cfg, self.mlp_fp16)
            self._stamp = None            # force re-staging

    def _lib(self):
        if self.lib is None:
            self.lib = _capi.load_library()
        return self.lib

    def tensors(self) -> Dict[str, torch.Tensor]:
        """name -> Parameter of every tensor the hot path reads (cached: walking named_parameters() costs ~0.1 ms and
        this is called several times per step; LiDAR4D._apply / load_state_dict drop the cache)."""
        ts = self._tensors
        if ts is None:
            sd = dict(self.owner.named_parameters())
            ts = self._tensors = {n: sd[n] for n in self.names}
        return ts

    def drop_caches(self):
        self._tensors, self._mtab = None, None

    def device(self) -> torch.device:
        return self.owner.aabb.device

    def _require_cuda(self, *ts):
        dev = self.device()
        if dev.type != "cuda":
            raise RuntimeError("lidar4d_b200 runs on CUDA (sm_90a) only; move the model with .cuda() "
                               "(there is no CPU fallback)")
        for t in ts:
            if t is not None and t.device != dev:
                raise RuntimeError(f"tensor on {t.device}, model on {dev}")

    def stream(self) -> int:
        return torch.cuda.current_stream(self.device()).cuda_stream

    def _events(self, kind):
        if self.timing is None:
            return None
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        self.timing[kind].append(ev)
        return ev

    @property
    def n_launches(self) -> int:
        """Kernels this library launched (counted inside the library, l4d_launch_count)."""
        return int(self._lib().l4d_launch_count())

    # ---- flat arenas ------------------------------------------------------------
    def _layout(self, ts):
        if self.offsets is None:
            o, offs = 0, {}
            for n in self.names:
                offs[n] = (o, ts[n].numel())
                o += (ts[n].numel() + ARENA_ALIGN - 1) // ARENA_ALIGN * ARENA_ALIGN
            self.offsets, self.total = offs, o
        return self.offsets

    def ensure_flat(self, ts=None) -> bool:
        """Make every hot-path parameter a view into the flat arena.  Returns True if the arena was (re)built."""
        ts = ts or self.tensors()
        offs = self._layout(ts)
        dev = self.device()
        if self.flat_p is not None and self.flat_p.device == dev:
            base = self.flat_p.data_ptr()
            if all(t.data_ptr() == base + 4 * offs[n][0] for n, t in ts.items()):
                return False
        for n, t in ts.items():
            if t.dtype != torch.float32 or t.device != dev:
                raise RuntimeError(f"parameter {n} must be fp32 on {dev} (got {t.dtype} on {t.device})")
        flat = torch.zeros(self.total, dtype=torch.float32, device=dev)
        with torch.no_grad():
            for n, t in ts.items():
                o, k = offs[n]
                v = flat[o:o + k].view(t.shape)
                v.copy_(t)
                t.data = v
        self.flat_p, self.flat_g, self._gtab, self._stamp, self._mtab = flat, None, None, None, None
        return True

    def attach_grads(self):
        """Point every trainable parameter's .grad at its slice of the flat gradient arena (zeroing slices whose
        .grad was None / copying foreign gradients in) and return the pointer table the kernels accumulate into."""
        ts = self.tensors()
        self.ensure_flat(ts)
        fresh = False
        if self.flat_g is None or self.flat_g.device != self.flat_p.device:
            self.flat_g = torch.zeros(self.total, dtype=torch.float32, device=self.flat_p.device)
            self._gtab, fresh = None, True
        base = self.flat_g.data_ptr()
        stale, n_train = [], 0
        for n, t in ts.items():
            if not t.requires_grad:
                continue
            n_train += 1
            g = t.grad
            if g is None or g.data_ptr() != base + 4 * self.offsets[n][0] or g.dtype != torch.float32 or g.shape != t.shape:
                stale.append((n, t, g))
        if stale:
            all_none = len(stale) == n_train and all(g is None for _, _, g in stale)
            with torch.no_grad():
                if all_none and not fresh:
                    self.flat_g.zero_()                     # the usual case: optimizer.zero_grad(set_to_none=True)
                for n, t, g in stale:
                    o, k = self.offsets[n]
                    v = self.flat_g[o:o + k].view(t.shape)
                    if not all_none:
                        if g is None:
                            v.zero_()
                        else:
                            v.copy_(g)
                    t.grad = v
        if self._gtab is None:
            self._gtab = _capi.L4DMasterGrads()
            _capi.fill_pointer_table(self._gtab, self.cfg, lambda n: base + 4 * self.offsets[n][0])
        return self._gtab

    def work(self, n_frames: int = 1):
        """Persistent zero-initialised gradient work buffer (plane / MLP grads in working layout, slice-independent
        hash accumulators, once per frame of a multi-frame launch) of the CURRENT stream: every kernel that consumes a
        region clears it again, so launches that overlap on different streams need their own (a fold kernel of one must
        not clear what the scatter of the other is still adding).  Grows on demand to the size of n_frames frames."""
        key = (self.device(), self.stream())
        w = self._works.get(key)
        n = self._lib().l4d_grad_work_bytes_frames(C.byref(self.ccfg), n_frames)
        if n == 0:
            raise RuntimeError("l4d_grad_work_bytes_frames: " + self._lib().l4d_last_error().decode())
        if w is None or w.numel() < n:
            w = self._works[key] = torch.zeros(n, dtype=torch.uint8, device=self.device())
        return w

    def reset_work(self):
        """Call after an exception inside a backward left a work buffer half-consumed."""
        for w in self._works.values():
            w.zero_()

    def infer_workspace(self, n_rays: int, S: int, n_frames: int = 1):
        """Persistent exchange workspace of no-grad renders through the split pipeline (grown on demand)."""
        n = self._lib().l4d_saved_bytes_frames(C.byref(self.ccfg), n_rays, S, n_frames)
        ws = getattr(self, "_infer_ws", None)
        if ws is None or ws.device != self.device() or ws.numel() < n:
            self._infer_ws = ws = torch.empty(n, dtype=torch.uint8, device=self.device())
        return ws, n

    # ---- staging ----------------------------------------------------------------
    def invalidate_staged(self):
        """Force the next call to refresh the kernels' working set.  Needed after in-place writes that bypass
        autograd's version counter in GRAD mode (``p.data.copy_()``); no-grad calls check the content themselves."""
        self._stamp = None

    def _checksum(self) -> int:
        return int(self.flat_p.view(torch.int32).sum(dtype=torch.int64))

    def master_table(self):
        base = self.flat_p.data_ptr()
        if self._mtab is None or self._mtab[0] != base:
            tab = _capi.L4DMasterParams()
            _capi.fill_pointer_table(tab, self.cfg, lambda n: base + 4 * self.offsets[n][0])
            self._mtab = (base, tab)
        return self._mtab[1]

    def ensure_staged(self, across_grad_mode: bool = False):
        """Refresh the fp16 / channels-last / transposed working set when a master parameter changed.
        Change detection: autograd version counters (optimizer.step, load_state_dict) in grad mode; in no-grad mode
        additionally the CONTENT (one reduction + one 8-byte read), because torch_ema's copy_to()/restore()
        (runner.py:565-567,680,820) write through ``.data`` and leave the counters alone; and always when the grad mode
        flipped since the last staging (eval -> train after ema.restore()).
        across_grad_mode (submodule calls): a grad-mode forward written with the submodules makes some of its calls under
        torch.no_grad() (lidar4d.py:160-161,169-170), and re-staging there would invalidate that forward's backward.  A
        grad -> no-grad flip therefore keeps the working set when the masters' content equals what the grad-mode
        submodule calls since the staging recorded (note_grad_content); without such a record, or with other content
        (an EMA swap), it re-stages as above."""
        lib = self._lib()
        ts = self.tensors()
        reflat = self.ensure_flat(ts)
        grad_mode = torch.is_grad_enabled()
        stamp = tuple(t._version for t in ts.values())
        need = (self.staged is None or reflat or stamp != self._stamp or self.staged.device != self.device())
        flip = grad_mode != self._staged_grad_mode
        if (across_grad_mode and flip and not need and not grad_mode and self._chk_grad is not None
                and self._checksum() == int(self._chk_grad)):
            return
        need = need or flip
        chk = None
        if not need and not grad_mode and not self.static_params:
            chk = self._checksum()
            need = chk != self._chk
        if not need:
            return
        nbytes = lib.l4d_staged_bytes(C.byref(self.ccfg))
        if nbytes == 0:
            raise RuntimeError("unsupported configuration: " + lib.l4d_last_error().decode())
        if self.staged is None or self.staged.device != self.device() or self.staged.numel() != nbytes:
            self.staged = torch.zeros(nbytes, dtype=torch.uint8, device=self.device())
        self.stage(_capi.STAGE_TABLES | _capi.STAGE_SMALL)
        self._stamp, self._staged_grad_mode = stamp, grad_mode
        if not grad_mode and not self.static_params:
            self._chk = chk if chk is not None else self._checksum()

    def stage(self, what: int):
        lib = self._lib()
        tab = self.master_table()
        with torch.cuda.device(self.device()):
            rc = lib.l4d_stage_params_ex(C.byref(self.ccfg), C.byref(tab), self.staged.data_ptr(), self.staged.numel(),
                                         what, self.stream())
        _capi.check(lib, rc, "l4d_stage_params_ex")
        self.stage_gen += 1
        self._chk_grad = None

    def note_grad_content(self):
        """Record (on the device, no host read) the masters' content of a grad-mode submodule call, once per staging:
        ensure_staged(across_grad_mode=True) compares a later no-grad call against it."""
        if self._chk_grad is None and self._staged_grad_mode:
            self._chk_grad = self.flat_p.view(torch.int32).sum(dtype=torch.int64)

    def params_updated_by_optimizer(self, tables_staged: bool):
        """lidar4d_b200.optim.Adam wrote the parameter arena (and, fused, the fp16 tables): finish the refresh."""
        if self.staged is None:
            self._stamp = None
            return
        self.stage(_capi.STAGE_SMALL if tables_staged else (_capi.STAGE_TABLES | _capi.STAGE_SMALL))
        self._chk = None
        self._staged_grad_mode = True

    def check_generation(self, ctx_gen: int, what: str):
        if ctx_gen != self.stage_gen:
            raise RuntimeError(
                f"{what}: the model's parameters (or its MLP precision mode) changed between this forward and its "
                "backward; the kernels' working set was re-staged in between.  Run backward before optimizer.step() / "
                "set_mlp_fp16() / load_state_dict().")

    def frame(self, time) -> _capi.L4DFrame:
        if torch.is_tensor(time):
            time = float(time.reshape(-1)[0])          # same host sync as lidar4d.py:143
        return _capi.make_frame_struct(make_frame(time, self.cfg.num_frames, self.cfg.time_resolution))

    def render_frames(self, time, rays_shape):
        """The frames of a render call as [(first row, rows, L4DFrame or L4DFrameTable)]: one L4DFrame for a single time
        (a float or a one-element tensor) or for B equal row times; otherwise one frame per row of rays [B, N, 3], in
        tables of at most MAX_FRAMES rows.  One device->host read of the times, as for one frame."""
        if not torch.is_tensor(time) or time.numel() == 1:
            return [(0, None, self.frame(time))]
        B = rays_shape[0] if len(rays_shape) == 3 else None
        if B is None or time.numel() != B or tuple(time.shape) not in ((B,), (B, 1)):
            raise ValueError(f"time must be one value or one per row of rays [B, N, 3] (shape [B] or [B, 1]); got time "
                             f"{tuple(time.shape)} for rays {tuple(rays_shape)}")
        times = time.detach().reshape(-1).tolist()
        if all(t == times[0] for t in times):
            return [(0, None, _capi.make_frame_struct(make_frame(times[0], self.cfg.num_frames, self.cfg.time_resolution)))]
        return [(b0, len(rows), _capi.make_frame_table(rows, rays_shape[1]))
                for b0, rows in row_frame_groups(self.cfg, times)]


def row_frame_groups(cfg, times):
    """[(first row, [L4DFrame of each row])] in groups of at most MAX_FRAMES rows: make_frame of every row's time."""
    frames = [_capi.make_frame_struct(make_frame(t, cfg.num_frames, cfg.time_resolution)) for t in times]
    return [(b0, frames[b0:b0 + _capi.MAX_FRAMES]) for b0 in range(0, len(frames), _capi.MAX_FRAMES)]


def _sub_table(tab: _capi.L4DFrameTable, h: int, n: int) -> _capi.L4DFrameTable:
    """The frames of rays [h, h + n) of a launch over `tab`."""
    rpf, ph = tab.rays_per_frame, tab.first_ray_phase + h
    first, last = ph // rpf, (ph + n - 1) // rpf
    return _capi.make_frame_table([tab.frames[i] for i in range(first, last + 1)], rpf, ph % rpf)


class _RenderFn(torch.autograd.Function):
    """Fused render forward / backward.  Parameters are passed as inputs so that autograd schedules the backward;
    their gradients are accumulated by the kernels straight into the flat gradient arena that every ``.grad`` views
    (model.grad_mode == "arena", the default), or returned to autograd as fresh tensors ("autograd": works with
    torch.autograd.grad, costs one arena allocation + one accumulation pass per backward)."""

    @staticmethod
    def forward(ctx, eng: _Engine, rays_o, rays_d, frame, S, perturb, seed, ray_offset, want_weights, train, *params):
        """frame: one L4DFrame for every ray, or an L4DFrameTable (several frames in one launch)."""
        lib = eng._lib()
        multi = isinstance(frame, _capi.L4DFrameTable)
        n_frames = frame.n_frames if multi else 1
        N = rays_o.shape[0]
        dev = rays_o.device
        depth = torch.empty(N, device=dev)
        image = torch.empty(N, 2, device=dev)
        wsum = torch.empty(N, device=dev)
        weights = torch.empty(N, S, device=dev) if want_weights else None
        zvals = torch.empty(N, S, device=dev) if want_weights else None
        rays = _capi.L4DRays()
        rays.rays_o, rays.rays_d = rays_o.data_ptr(), rays_d.data_ptr()
        rays.n_rays, rays.n_steps, rays.perturb = N, S, int(bool(perturb))
        rays.seed, rays.ray_offset = int(seed), int(ray_offset)
        fused = eng.owner.pipeline == "fused"
        rays.reserved = 1 if fused else 0
        saved, nsaved = None, 0
        chunk = N
        if train:
            nsaved = lib.l4d_saved_bytes_frames(C.byref(eng.ccfg), N, S, n_frames)
            saved = torch.empty(nsaved, dtype=torch.uint8, device=dev)
        elif not fused:
            # inference through the split pipeline: the kernels exchange feature tiles through a workspace; walk the rays
            # in chunks over ONE persistent workspace (config 4: 131,072 rays per frame would otherwise need 160 GB)
            chunk = min(N, int(eng.owner.infer_ray_chunk))
            saved, nsaved = eng.infer_workspace(chunk, S, n_frames)
        ev = eng._events("fwd")
        with torch.cuda.device(dev):
            if ev: ev[0].record()
            for h in range(0, N, chunk):
                n = min(chunk, N - h)
                rays.rays_o, rays.rays_d, rays.n_rays = rays_o.data_ptr() + 12 * h, rays_d.data_ptr() + 12 * h, n
                rays.ray_offset = int(ray_offset) + h
                fwd = lib.l4d_render_forward_frames if multi else lib.l4d_render_forward
                fr = _sub_table(frame, h, n) if multi and n < N else frame
                rc = fwd(
                    C.byref(eng.ccfg), eng.staged.data_ptr(), C.byref(fr), C.byref(rays),
                    depth.data_ptr() + 4 * h, image.data_ptr() + 8 * h, wsum.data_ptr() + 4 * h,
                    weights.data_ptr() + 4 * h * S if want_weights else None, zvals.data_ptr() + 4 * h * S if want_weights else None,
                    saved.data_ptr() if saved is not None else None, nsaved, eng.stream())
                _capi.check(lib, rc, "l4d_render_forward")
            if ev: ev[1].record()
        ctx.eng, ctx.frame, ctx.rays_args = eng, frame, (N, S, int(bool(perturb)), int(seed), int(ray_offset))
        ctx.saved, ctx.nsaved = (saved, nsaved) if train else (None, 0)
        ctx.fused = fused
        ctx.rays_o, ctx.rays_d = rays_o, rays_d
        ctx.stage_gen = eng.stage_gen
        ctx.want_weights = want_weights
        if want_weights:
            ctx.mark_non_differentiable(zvals)
            return depth, image, wsum, weights, zvals
        return depth, image, wsum

    @staticmethod
    def backward(ctx, g_depth, g_image, g_wsum, *rest):
        eng = ctx.eng
        lib = eng._lib()
        if ctx.saved is None:
            raise RuntimeError("render was run without saving activations (no_grad / eval)")
        eng.check_generation(ctx.stage_gen, "render backward")
        N, S, perturb, seed, ray_offset = ctx.rays_args
        dev = ctx.rays_o.device
        g_weights = rest[0] if (ctx.want_weights and len(rest) > 0) else None
        z = lambda t, shape: (torch.zeros(shape, device=dev) if t is None else t.contiguous().float())
        g_depth, g_image = z(g_depth, (N,)), z(g_image, (N, 2))
        g_wsum = None if g_wsum is None else g_wsum.contiguous().float()
        g_weights = None if g_weights is None else g_weights.contiguous().float()
        arena = eng.owner.grad_mode == "arena"
        tab, views = (eng.attach_grads(), None) if arena else _scratch_grads(eng)
        multi = isinstance(ctx.frame, _capi.L4DFrameTable)
        work = eng.work(ctx.frame.n_frames if multi else 1)
        rays = _capi.L4DRays()
        rays.rays_o, rays.rays_d = ctx.rays_o.data_ptr(), ctx.rays_d.data_ptr()
        rays.n_rays, rays.n_steps, rays.perturb, rays.seed, rays.ray_offset = N, S, perturb, seed, ray_offset
        rays.reserved = 1 if ctx.fused else 0
        ev = eng._events("bwd")
        with torch.cuda.device(dev):
            if ev: ev[0].record()
            hook = eng.hash_grads_hook if arena else None      # (event, callback) armed by RayShardedDP for the step's last backward
            bwd = lib.l4d_render_backward_frames if multi else lib.l4d_render_backward_ex
            rc = bwd(
                C.byref(eng.ccfg), eng.staged.data_ptr(), C.byref(ctx.frame), C.byref(rays),
                ctx.saved.data_ptr(), ctx.nsaved, g_depth.data_ptr(), g_image.data_ptr(),
                g_wsum.data_ptr() if g_wsum is not None else None,
                g_weights.data_ptr() if g_weights is not None else None,
                C.byref(tab), work.data_ptr(), work.numel(), hook[0].cuda_event if hook else None, eng.stream())
            if ev: ev[1].record()
            _capi.check(lib, rc, "l4d_render_backward")
            if hook:
                eng.hash_grads_hook = None
                hook[1]()
            rc = lib.l4d_unstage_grads(C.byref(eng.ccfg), work.data_ptr(), work.numel(), C.byref(tab), eng.stream())
            _capi.check(lib, rc, "l4d_unstage_grads")
        ctx.saved = None
        if arena:
            return (None,) * (10 + len(eng.names))
        return (None,) * 10 + tuple(views[n] for n in eng.names)


def _scratch_grads(eng: _Engine):
    """grad_mode == "autograd": a fresh zeroed arena whose views are handed to autograd."""
    ts = eng.tensors()
    eng.ensure_flat(ts)
    flat = torch.zeros(eng.total, dtype=torch.float32, device=eng.device())
    views = {n: flat[o:o + k].view(ts[n].shape) for n, (o, k) in eng.offsets.items()}
    tab = _capi.L4DMasterGrads()
    _capi.fill_pointer_table(tab, eng.cfg, lambda n: views[n].data_ptr())
    return tab, views


class _FlowFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, eng: _Engine, x, frame, train, *params):
        lib = eng._lib()
        n = x.shape[0]
        flow = torch.empty(n, 6, device=x.device)
        saved = torch.empty(16, n, device=x.device) if train else None
        with torch.cuda.device(x.device):
            rc = lib.l4d_flow_forward(C.byref(eng.ccfg), eng.staged.data_ptr(), C.byref(frame), x.data_ptr(), n,
                                      flow.data_ptr(), saved.data_ptr() if train else None, eng.stream())
        _capi.check(lib, rc, "l4d_flow_forward")
        ctx.eng, ctx.frame, ctx.x, ctx.saved, ctx.stage_gen = eng, frame, x, saved, eng.stage_gen
        return flow

    @staticmethod
    def backward(ctx, g_flow):
        eng = ctx.eng
        lib = eng._lib()
        if ctx.saved is None:
            raise RuntimeError("flow was run without saving activations")
        eng.check_generation(ctx.stage_gen, "flow backward")
        x = ctx.x
        n = x.shape[0]
        g_flow = g_flow.contiguous().float()
        arena = eng.owner.grad_mode == "arena"
        tab, views = (eng.attach_grads(), None) if arena else _scratch_grads(eng)
        work = eng.work()
        with torch.cuda.device(x.device):
            rc = lib.l4d_flow_backward(C.byref(eng.ccfg), eng.staged.data_ptr(), C.byref(ctx.frame), x.data_ptr(), n,
                                       ctx.saved.data_ptr(), g_flow.data_ptr(), C.byref(tab), work.data_ptr(), work.numel(),
                                       eng.stream())
            _capi.check(lib, rc, "l4d_flow_backward")
            rc = lib.l4d_unstage_grads(C.byref(eng.ccfg), work.data_ptr(), work.numel(), C.byref(tab), eng.stream())
            _capi.check(lib, rc, "l4d_unstage_grads")
        if arena:
            return (None,) * (4 + len(eng.names))
        flow_names = {"flow_net.grid_enc.params", "flow_net.mlp.0.weight", "flow_net.mlp.2.weight", "flow_net.mlp.4.weight"}
        return (None,) * 4 + tuple(views[n] if n in flow_names else None for n in eng.names)


_HEAD_NAMES = ("intensity_net.params", "raydrop_net.params")


class _DensityFn(torch.autograd.Function):
    """LiDAR4D.density with a backward (l4d_density_forward_ex / l4d_density_backward).  Parameters are inputs as in
    _RenderFn, with the same two grad modes; the points get no gradient.  Outputs: sigma, geo_feat and, when asked for,
    the features and the flow (non-differentiable)."""

    @staticmethod
    def forward(ctx, eng: _Engine, x, frame, want_feats, *params):
        lib = eng._lib()
        n = x.shape[0]
        dev = x.device
        sigma = torch.empty(n, device=dev)
        geo = torch.empty(n, 15, device=dev)
        feats = torch.empty(n, eng.cfg.sigma_in_dim, device=dev) if want_feats else None
        flow = torch.empty(n, 6, device=dev) if want_feats else None
        nsaved = lib.l4d_density_saved_bytes(C.byref(eng.ccfg), n)
        saved = torch.empty(nsaved, dtype=torch.uint8, device=dev)
        if n:
            with torch.cuda.device(dev):
                rc = lib.l4d_density_forward_ex(C.byref(eng.ccfg), eng.staged.data_ptr(), C.byref(frame), x.data_ptr(), n,
                                                sigma.data_ptr(), geo.data_ptr(), feats.data_ptr() if want_feats else None,
                                                flow.data_ptr() if want_feats else None, saved.data_ptr(), nsaved,
                                                eng.stream())
            _capi.check(lib, rc, "l4d_density_forward_ex")
        ctx.eng, ctx.frame, ctx.x, ctx.saved, ctx.nsaved, ctx.stage_gen = eng, frame, x, saved, nsaved, eng.stage_gen
        ctx.set_materialize_grads(False)        # an unused output passes NULL to the kernel instead of zeros
        if want_feats:
            ctx.mark_non_differentiable(feats, flow)
            return sigma, geo, feats, flow
        return sigma, geo

    @staticmethod
    def backward(ctx, g_sigma, g_geo, *rest):
        eng = ctx.eng
        lib = eng._lib()
        if ctx.saved is None:
            raise RuntimeError("density backward: the saved activations were already consumed by an earlier backward")
        eng.check_generation(ctx.stage_gen, "density backward")
        x = ctx.x
        n = x.shape[0]
        arena = eng.owner.grad_mode == "arena"
        tab, views = (eng.attach_grads(), None) if arena else _scratch_grads(eng)
        if n and (g_sigma is not None or g_geo is not None):
            g_sigma = None if g_sigma is None else g_sigma.contiguous().float()
            g_geo = None if g_geo is None else g_geo.contiguous().float()
            work = eng.work()
            with torch.cuda.device(x.device):
                rc = lib.l4d_density_backward(C.byref(eng.ccfg), eng.staged.data_ptr(), C.byref(ctx.frame), x.data_ptr(), n,
                                              ctx.saved.data_ptr(), ctx.nsaved,
                                              g_sigma.data_ptr() if g_sigma is not None else None,
                                              g_geo.data_ptr() if g_geo is not None else None,
                                              C.byref(tab), work.data_ptr(), work.numel(), eng.stream())
                _capi.check(lib, rc, "l4d_density_backward")
                rc = lib.l4d_unstage_grads(C.byref(eng.ccfg), work.data_ptr(), work.numel(), C.byref(tab), eng.stream())
                _capi.check(lib, rc, "l4d_unstage_grads")
        ctx.saved = None
        if arena:
            return (None,) * (4 + len(eng.names))
        return (None,) * 4 + tuple(None if k in _HEAD_NAMES else views[k] for k in eng.names)


def _head_grads(eng: _Engine):
    """Zeroed gradient buffers of the two attribute heads and a pointer table holding only them (the attribute backward
    writes no other sink, and l4d_unstage_grads skips null ones)."""
    ts = eng.tensors()
    bufs = {k: torch.zeros_like(ts[k]) for k in _HEAD_NAMES}
    tab = _capi.L4DMasterGrads()
    tab.intensity_net = bufs["intensity_net.params"].data_ptr()
    tab.raydrop_net = bufs["raydrop_net.params"].data_ptr()
    return tab, bufs


class _AttributeFn(torch.autograd.Function):
    """LiDAR4D.attribute with a backward (l4d_attribute_forward / l4d_attribute_backward).  Differentiable w.r.t.
    geo_feat and the two head nets (inputs w_int, w_drop); d and the mask get no gradient.  Nothing is saved on the GPU:
    the backward recomputes the heads from d, geo_feat and the mask."""

    @staticmethod
    def forward(ctx, eng: _Engine, d, geo, m8, w_int, w_drop):
        lib = eng._lib()
        n = d.shape[0]
        ctx.empty = n == 0 or (m8 is not None and not bool(m8.any()))     # host sync, as lidar4d.py:201
        if ctx.empty:
            out = torch.zeros(n, 2, device=d.device)
        else:
            out = torch.empty(n, 2, device=d.device)
            with torch.cuda.device(d.device):
                rc = lib.l4d_attribute_forward(C.byref(eng.ccfg), eng.staged.data_ptr(), d.data_ptr(), geo.data_ptr(),
                                               m8.data_ptr() if m8 is not None else None, n, out.data_ptr(), eng.stream())
            _capi.check(lib, rc, "l4d_attribute_forward")
        ctx.eng, ctx.stage_gen = eng, eng.stage_gen
        ctx.save_for_backward(d, geo, m8)
        return out

    @staticmethod
    def backward(ctx, g_out):
        eng = ctx.eng
        lib = eng._lib()
        eng.check_generation(ctx.stage_gen, "attribute backward")
        d, geo, m8 = ctx.saved_tensors
        need_geo = ctx.needs_input_grad[2]
        need_w = ctx.needs_input_grad[4] or ctx.needs_input_grad[5]
        if ctx.empty:
            return None, None, (torch.zeros_like(geo) if need_geo else None), None, None, None
        n = d.shape[0]
        g_out = g_out.contiguous().float()
        g_geo = torch.empty(n, 15, device=d.device) if need_geo else None
        arena = eng.owner.grad_mode == "arena"
        tab, bufs = (eng.attach_grads(), None) if (arena and need_w) else _head_grads(eng)
        work = eng.work()
        with torch.cuda.device(d.device):
            rc = lib.l4d_attribute_backward(C.byref(eng.ccfg), eng.staged.data_ptr(), d.data_ptr(), geo.data_ptr(),
                                            m8.data_ptr() if m8 is not None else None, n, g_out.data_ptr(),
                                            g_geo.data_ptr() if g_geo is not None else None, C.byref(tab),
                                            work.data_ptr(), work.numel(), eng.stream())
            _capi.check(lib, rc, "l4d_attribute_backward")
            rc = lib.l4d_unstage_grads(C.byref(eng.ccfg), work.data_ptr(), work.numel(), C.byref(tab), eng.stream())
            _capi.check(lib, rc, "l4d_unstage_grads")
        gw = (None, None) if (arena or not need_w) else (bufs["intensity_net.params"], bufs["raydrop_net.params"])
        return (None, None, g_geo, None) + gw


def _module_launch(eng: _Engine, kind: str, ident: int, q, slice_: int, x: torch.Tensor, out_dim: int):
    lib = eng._lib()
    n = x.shape[0]
    out = torch.empty(n, out_dim, device=x.device)
    if n:
        with torch.cuda.device(x.device):
            if kind == "enc":
                rc = lib.l4d_encoder_forward(C.byref(eng.ccfg), eng.staged.data_ptr(), ident, C.byref(q), slice_,
                                             x.data_ptr(), n, out.data_ptr(), eng.stream())
            else:
                rc = lib.l4d_mlp_forward(C.byref(eng.ccfg), eng.staged.data_ptr(), ident, x.data_ptr(), n, out.data_ptr(),
                                         eng.stream())
        _capi.check(lib, rc, f"l4d_{'encoder' if kind == 'enc' else 'mlp'}_forward")
    return out


# encoder modules whose backward accumulates into grad_work (planes, flow MLP), folded by l4d_unstage_grads
_WORK_MODULES = (_capi.MOD_PLANES_STATIC, _capi.MOD_PLANES_DYNAMIC, _capi.MOD_FLOW)


class _ModuleFn(torch.autograd.Function):
    """One submodule call with a backward (l4d_encoder_backward / l4d_mlp_backward).  `params` are the module's own
    parameters (named by `names`), with the two grad modes of _RenderFn; x gets dL/dx where the op gives one (planes,
    networks).  Nothing is saved on the GPU: the backward recomputes from x."""

    @staticmethod
    def forward(ctx, eng: _Engine, kind, ident, q, slice_, out_dim, names, x, *params):
        out = _module_launch(eng, kind, ident, q, slice_, x, out_dim)
        ctx.eng, ctx.kind, ctx.ident, ctx.q, ctx.slice_, ctx.names = eng, kind, ident, q, slice_, names
        ctx.stage_gen = eng.stage_gen
        ctx.save_for_backward(x)
        return out

    @staticmethod
    def backward(ctx, g_out):
        eng = ctx.eng
        lib = eng._lib()
        eng.check_generation(ctx.stage_gen, "submodule backward")
        (x,) = ctx.saved_tensors
        n = x.shape[0]
        g_out = g_out.contiguous().float()
        want_x = ctx.needs_input_grad[7]
        g_x = torch.zeros_like(x) if want_x else None
        arena = eng.owner.grad_mode == "arena"
        tab, views = (eng.attach_grads(), None) if arena else _scratch_grads(eng)
        if n:
            work = eng.work()
            with torch.cuda.device(x.device):
                if ctx.kind == "enc":
                    rc = lib.l4d_encoder_backward(C.byref(eng.ccfg), eng.staged.data_ptr(), ctx.ident, C.byref(ctx.q),
                                                  ctx.slice_, x.data_ptr(), n, g_out.data_ptr(),
                                                  g_x.data_ptr() if want_x else None, C.byref(tab), work.data_ptr(),
                                                  work.numel(), eng.stream())
                else:
                    rc = lib.l4d_mlp_backward(C.byref(eng.ccfg), eng.staged.data_ptr(), ctx.ident, x.data_ptr(), n,
                                              g_out.data_ptr(), g_x.data_ptr() if want_x else None, C.byref(tab),
                                              work.data_ptr(), work.numel(), eng.stream())
                _capi.check(lib, rc, f"l4d_{'encoder' if ctx.kind == 'enc' else 'mlp'}_backward")
                if ctx.kind == "mlp" or ctx.ident in _WORK_MODULES:     # the hash encodings write master gradients only
                    rc = lib.l4d_unstage_grads(C.byref(eng.ccfg), work.data_ptr(), work.numel(), C.byref(tab),
                                               eng.stream())
                    _capi.check(lib, rc, "l4d_unstage_grads")
        pg = (None,) * len(ctx.names) if arena else tuple(views[k] for k in ctx.names)
        return (None,) * 7 + (g_x,) + pg


def _run_module(owner: "LiDAR4D", kind: str, ident: int, x, in_dim: int, out_dim: int, names, label: str,
                input_grad: bool = False, t=None, slice_: int = 0):
    """Run one submodule op on x [..., in_dim] -> [N, out_dim].  In grad mode, with a parameter of `names` requiring grad
    (or x, for ops with an input gradient), through _ModuleFn; otherwise one launch."""
    eng = owner._engine
    if not torch.is_tensor(x) or x.shape[-1] != in_dim:
        raise ValueError(f"{label}: expected a tensor [N, {in_dim}], got {tuple(getattr(x, 'shape', ()))}")
    eng._require_cuda(x)
    grad = torch.is_grad_enabled()
    if grad and x.requires_grad and not input_grad:
        raise NotImplementedError(f"{label}: no gradient with respect to its input is implemented; detach the input "
                                  "(the reference's own composition never needs it)")
    q = _capi.L4DTimeQuery()
    if t is not None:
        if torch.is_tensor(t):
            if t.numel() != 1:
                raise ValueError(f"{label}: t must be a float or a one-element tensor")
            t = float(t.reshape(-1)[0])     # one device->host read, the host branch of HashGridT.forward (hash_field.py:82)
        q = _capi.make_time_query(make_time_query(t, owner.cfg.time_resolution))
    eng.ensure_staged(across_grad_mode=True)
    if grad:
        eng.note_grad_content()
    ts = eng.tensors()
    params = [ts[k] for k in names]
    x2 = x.reshape(-1, in_dim)
    if grad and (any(p.requires_grad for p in params) or (input_grad and x.requires_grad)):
        xin = x2.contiguous().float() if input_grad else x2.detach().contiguous().float()
        return _ModuleFn.apply(eng, kind, ident, q, slice_, out_dim, tuple(names), xin, *params)
    return _module_launch(eng, kind, ident, q, slice_, x2.detach().contiguous().float(), out_dim)


# =============================================================================
# public modules
# =============================================================================
class LiDAR_Renderer(nn.Module):
    """model/renderer.py:13-186 API."""

    def __init__(self, bound=1, near_lidar=0.01, far_lidar=0.81, density_scale=1, active_sensor=False):
        super().__init__()
        self.bound = bound
        self.near_lidar = near_lidar
        self.far_lidar = far_lidar
        self.density_scale = density_scale
        self.active_sensor = active_sensor
        aabb = torch.FloatTensor([-bound, -bound, -bound, bound, bound, bound])
        self.register_buffer("aabb", aabb)

    def forward(self, x, d):
        raise NotImplementedError()

    def run(self, rays_o, rays_d, time, num_steps=768, perturb=False, **kwargs):
        raise NotImplementedError()

    def render(self, rays_o, rays_d, time, staged=False, max_ray_batch=4096, **kwargs):
        """renderer.py:142-186.  `staged` keeps the reference's chunked contract
        (only depth/image returned); chunks may be larger here because nothing of
        size [N*S, C] is materialised."""
        B, N = rays_o.shape[:2]
        device = rays_o.device
        if staged:
            depth = torch.empty((B, N), device=device)
            image = torch.empty((B, N, self.out_lidar_dim), device=device)
            for b in range(B):
                head = 0
                while head < N:
                    tail = min(head + max_ray_batch, N)
                    r = self.run(rays_o[b:b + 1, head:tail], rays_d[b:b + 1, head:tail], time[b:b + 1], **kwargs)
                    depth[b:b + 1, head:tail] = r["depth_lidar"]
                    image[b:b + 1, head:tail] = r["image_lidar"]
                    head += max_ray_batch
            return {"depth_lidar": depth, "image_lidar": image}
        return self.run(rays_o, rays_d, time, **kwargs)


class LiDAR4D(LiDAR_Renderer):
    def __init__(self, min_resolution=32, base_resolution=512, max_resolution=32768, time_resolution=8,
                 n_levels_plane=4, n_features_per_level_plane=8, n_levels_hash=8, n_features_per_level_hash=4,
                 log2_hashmap_size=19, num_layers_flow=3, hidden_dim_flow=64, num_layers_sigma=2,
                 hidden_dim_sigma=64, geo_feat_dim=15, num_layers_lidar=3, hidden_dim_lidar=64, out_lidar_dim=2,
                 num_frames=51, bound=1, unet: Optional[nn.Module] = None, **kwargs):
        renderer_kw = {k: kwargs[k] for k in ("near_lidar", "far_lidar", "density_scale", "active_sensor") if k in kwargs}
        super().__init__(bound, **renderer_kw)
        self.cfg = FieldConfig(
            min_resolution=min_resolution, base_resolution=base_resolution, max_resolution=max_resolution,
            time_resolution=time_resolution, n_levels_plane=n_levels_plane,
            n_features_per_level_plane=n_features_per_level_plane, n_levels_hash=n_levels_hash,
            n_features_per_level_hash=n_features_per_level_hash, log2_hashmap_size=log2_hashmap_size,
            hash_size_dynamic=tuple(kwargs.get("hash_size_dynamic", (15, 13, 13))),
            num_layers_flow=num_layers_flow, hidden_dim_flow=hidden_dim_flow, num_layers_sigma=num_layers_sigma,
            hidden_dim_sigma=hidden_dim_sigma, geo_feat_dim=geo_feat_dim, num_layers_lidar=num_layers_lidar,
            hidden_dim_lidar=hidden_dim_lidar, out_lidar_dim=out_lidar_dim, num_frames=num_frames, bound=float(bound),
            near_lidar=float(self.near_lidar), far_lidar=float(self.far_lidar), density_scale=float(self.density_scale),
            active_sensor=bool(self.active_sensor),
            **{k: kwargs[k] for k in ("flow_base_resolution", "flow_max_resolution", "flow_log2_hashmap_size") if k in kwargs})
        c = self.cfg
        c.validate()
        self.out_lidar_dim = out_lidar_dim
        self.num_frames = num_frames

        self.planes_encoder = _Planes4D(c)
        self.hash_encoder = _HashGrid4D(c)
        self.view_encoder = _TcnnParams(0, c.view_dim, "empty", kind="freq")
        self.flow_net = _FlowField(c)
        self.sigma_net = _TcnnParams(c.mlp_param_count(c.sigma_in_pad, 64, 1), 1 + geo_feat_dim, "mlp", kind="sigma",
                                     dims=[c.sigma_in_pad, 64, 16])
        self.intensity_net = _TcnnParams(c.mlp_param_count(c.attr_in_pad, 64, 2), 1, "mlp", kind="intensity",
                                         dims=[c.attr_in_pad, 64, 64, 16])
        self.raydrop_net = _TcnnParams(c.mlp_param_count(c.attr_in_pad, 64, 2), 1, "mlp", kind="raydrop",
                                       dims=[c.attr_in_pad, 64, 64, 16])
        # U-Net ray-drop refinement is a per-image post-process outside the hot path (SURVEY.md 8(f) #3);
        # callers that need it pass the reference's module in (model/unet.py), its state_dict keys stay `unet.*`.
        self.unet = unet if unet is not None else nn.Identity()

        self.materialize_weights = True    # return `weights` / `z_vals` like renderer.py:134-140
        # "split": gather / dense / scatter kernels exchanging SoA planes (default, faster);
        # "fused": the single-kernel forward and backward (csrc/l4d_kernels.cu)
        self.pipeline = "split"
        # "arena": the backward kernels accumulate into the flat gradient arena that every .grad views (default);
        # "autograd": gradients are returned to autograd as tensors (torch.autograd.grad, hooks), slower
        self.grad_mode = "arena"
        self.infer_ray_chunk = 2048        # rays per launch of a no-grad render (bounds the exchange workspace: 2.5 GB at L=16)
        self.jitter_seed = 0
        self._jitter_calls = 0
        self._engine = _Engine(self)
        self._link_submodules()

    def _link_submodules(self):
        ref = weakref.ref(self)
        for m in self.modules():
            if isinstance(m, _Submodule):
                m._owner_ref = ref

    def __setstate__(self, state):            # copy.deepcopy / unpickling: the copies' submodules run through the copy
        super().__setstate__(state)
        self._link_submodules()

    # ---- precision / pipeline switches ------------------------------------------------------
    def set_mlp_fp16(self, on: bool = True):
        """True: MLP weights are consumed as fp16-rounded working copies of the fp32 masters (exactly how
        tiny-cuda-nn's FullyFusedMLP holds them) and the dense kernels of the split pipeline run on the
        wgmma tensor cores with hi/lo-split fp16 activations (fp32-class accuracy) -- the default.
        False: fp32 weights on the fp32-FMA kernels (bit-for-bit the fp32 oracle's arithmetic, ~2x slower)."""
        self._engine.set_mlp_fp16(on)
        return self

    def invalidate_staged(self):
        """Refresh the kernels' working set at the next call.  Only needed after in-place parameter writes that bypass
        autograd's version counter WHILE GRADIENTS ARE ENABLED (``p.data.copy_(...)``); optimizer steps,
        ``load_state_dict`` and anything done before a ``torch.no_grad()`` render (torch_ema ``copy_to``/``restore``
        around evaluation, runner.py:565-567,680) are detected automatically."""
        self._engine.invalidate_staged()
        return self

    def prepare_grads(self):
        """Attach every parameter's .grad to the flat gradient arena (clearing it if the grads were None) on the current
        stream.  Call once after ``zero_grad`` when the backward passes of one optimiser step are spread over several
        CUDA streams, before those streams fork: otherwise the first backward to run would clear the arena on ITS stream."""
        self._engine._require_cuda()
        self._engine.ensure_staged()          # a pending re-staging must not happen on one of the forked streams either
        self._engine.attach_grads()
        return self

    def static_params(self, on: bool = True):
        """Promise that parameters do not change between no-grad calls (skips the per-call content check, one
        reduction + an 8-byte device->host read): for tight inference loops such as a trajectory render."""
        self._engine.static_params = bool(on)
        return self

    # ---- nn.Module plumbing -----------------------------------------------------------------
    def forward(self, x, d, t):
        pass

    def _apply(self, fn, *a, **k):          # .to() / .cuda() / .float(): parameters may be re-created
        r = super()._apply(fn, *a, **k)
        if hasattr(self, "_engine"):
            self._engine.drop_caches()
        return r

    def _params_list(self) -> List[torch.Tensor]:
        ts = self._engine.tensors()
        return [ts[n] for n in self._engine.names]

    # ---- LiDAR_Renderer.run (renderer.py:44-140) -----------------------------------------------
    def run(self, rays_o, rays_d, time, num_steps=768, perturb=False, ray_offset=0, **kwargs):
        if not 2 <= int(num_steps) <= 8192:
            # at num_steps = 1 the reference's deltas z[..., 1:] - z[..., :-1] are empty: its weights come out [N, 0] and
            # depth / image / weights_sum 0, an artefact of broadcasting an empty tensor rather than a render
            raise ValueError(f"num_steps must be in [2, 8192], got {num_steps} (the reference renders nothing below 2 samples)")
        eng = self._engine
        prefix = rays_o.shape[:-1]
        ro = rays_o.detach().contiguous().view(-1, 3).float()
        rd = rays_d.detach().contiguous().view(-1, 3).float()
        eng._require_cuda(ro, rd)
        eng.ensure_staged()
        groups = eng.render_frames(time, tuple(rays_o.shape))
        params = self._params_list()
        train = torch.is_grad_enabled() and any(p.requires_grad for p in params)
        seed = 0
        if perturb:
            seed = self.jitter_seed + self._jitter_calls
            self._jitter_calls += 1
        want_w = bool(self.materialize_weights)
        if len(groups) == 1 and groups[0][1] is None:
            out = _RenderFn.apply(eng, ro, rd, groups[0][2], int(num_steps), bool(perturb), seed, int(ray_offset), want_w,
                                  train, *params)
        else:
            # one launch per table of rows; ray (b, j) keeps the jitter index ray_offset + b * N + j of the flattened launch
            N = rays_o.shape[1]
            outs = [_RenderFn.apply(eng, ro[b0 * N:(b0 + k) * N], rd[b0 * N:(b0 + k) * N], tab, int(num_steps),
                                    bool(perturb), seed, int(ray_offset) + b0 * N, want_w, train, *params)
                    for b0, k, tab in groups]
            out = outs[0] if len(outs) == 1 else tuple(torch.cat(parts) for parts in zip(*outs))
        res = {"depth_lidar": out[0].view(*prefix), "image_lidar": out[1].view(*prefix, self.out_lidar_dim),
               "weights_sum_lidar": out[2]}
        if want_w:
            res["weights"], res["z_vals"] = out[3], out[4]
        return res

    # ---- LiDAR4D.flow (lidar4d.py:124-137) -------------------------------------------------------
    def flow(self, x, t):
        eng = self._engine
        x = x.detach().contiguous().view(-1, 3).float()
        eng._require_cuda(x)
        eng.ensure_staged()
        frame = eng.frame(t)
        params = self._params_list()
        train = torch.is_grad_enabled() and any(p.requires_grad for p in params)
        fl = _FlowFn.apply(eng, x, frame, train, *params)
        return {"forward": fl[:, :3], "backward": fl[:, 3:]}

    # ---- LiDAR4D.density (lidar4d.py:139-188) -----------------------------------------------------
    def density(self, x, t=None, return_features: bool = False):
        """x [N,3] in [-bound, bound] -> {"sigma" [N], "geo_feat" [N,15]} (+ "features", "flow" with return_features).
        In grad mode, when a parameter requires grad, sigma and geo_feat are differentiable w.r.t. every parameter the
        reference's density reaches: planes, static hash, the current time's dynamic-hash slices (the warped queries are
        no_grad there too), flow grid and flow MLP, sigma net.  No gradient flows to x (as render() treats its rays);
        features and flow are non-differentiable.  Otherwise this is an inference call with no saved state."""
        if torch.is_grad_enabled() and any(p.requires_grad for p in self._params_list()):
            eng = self._engine
            x = x.detach().contiguous().view(-1, 3).float()
            eng._require_cuda(x)
            eng.ensure_staged()
            frame = eng.frame(t)
            out = _DensityFn.apply(eng, x, frame, bool(return_features), *self._params_list())
            res = {"sigma": out[0], "geo_feat": out[1]}
            if return_features:
                res.update(features=out[2], flow=out[3])
            return res
        return self._density_inference(x, t, return_features)

    @torch.no_grad()
    def _density_inference(self, x, t=None, return_features: bool = False):
        eng = self._engine
        lib = eng._lib()
        x = x.detach().contiguous().view(-1, 3).float()
        eng._require_cuda(x)
        eng.ensure_staged()
        frame = eng.frame(t)
        n = x.shape[0]
        sigma = torch.empty(n, device=x.device)
        geo = torch.empty(n, 15, device=x.device)
        feats = torch.empty(n, self.cfg.sigma_in_dim, device=x.device) if return_features else None
        flow = torch.empty(n, 6, device=x.device) if return_features else None
        with torch.cuda.device(x.device):
            rc = lib.l4d_density_forward(C.byref(eng.ccfg), eng.staged.data_ptr(), C.byref(frame), x.data_ptr(), n,
                                         sigma.data_ptr(), geo.data_ptr(),
                                         feats.data_ptr() if return_features else None,
                                         flow.data_ptr() if return_features else None, eng.stream())
        _capi.check(lib, rc, "l4d_density_forward")
        out = {"sigma": sigma, "geo_feat": geo}
        if return_features:
            out.update(features=feats, flow=flow)
        return out

    # ---- LiDAR4D.attribute (lidar4d.py:191-223); render() has the heads fused in -------------------------------------
    def attribute(self, x, d, mask=None, geo_feat=None, **kwargs):
        """x is unused (as in the reference); d [N,3] unit directions, geo_feat [N,15], mask [N] bool or None.
        Returns [N,2] = (raydrop, intensity); rows outside the mask are zero.
        In grad mode the result is differentiable w.r.t. geo_feat and both head nets (whichever require grad); no
        gradient flows to d.  An empty mask returns zeros and back-propagates zeros without a launch."""
        heads = [self._engine.tensors()[k] for k in _HEAD_NAMES]
        if torch.is_grad_enabled() and (geo_feat.requires_grad or any(p.requires_grad for p in heads)):
            eng = self._engine
            d = d.detach().contiguous().view(-1, 3).float()
            n = d.shape[0]
            geo = geo_feat.contiguous().view(n, 15).float()
            eng._require_cuda(d, geo)
            eng.ensure_staged()
            m8 = None if mask is None else mask.detach().contiguous().view(n).to(torch.uint8)
            ts = eng.tensors()
            return _AttributeFn.apply(eng, d, geo, m8, ts[_HEAD_NAMES[0]], ts[_HEAD_NAMES[1]])
        return self._attribute_inference(x, d, mask, geo_feat, **kwargs)

    @torch.no_grad()
    def _attribute_inference(self, x, d, mask=None, geo_feat=None, **kwargs):
        eng = self._engine
        lib = eng._lib()
        d = d.detach().contiguous().view(-1, 3).float()
        eng._require_cuda(d)
        eng.ensure_staged()
        n = d.shape[0]
        geo = geo_feat.detach().contiguous().view(n, 15).float()
        m8 = None if mask is None else mask.detach().contiguous().view(n).to(torch.uint8)
        out = torch.empty(n, self.out_lidar_dim, device=d.device)
        with torch.cuda.device(d.device):
            rc = lib.l4d_attribute_forward(C.byref(eng.ccfg), eng.staged.data_ptr(), d.data_ptr(), geo.data_ptr(),
                                           m8.data_ptr() if m8 is not None else None, n, out.data_ptr(), eng.stream())
        _capi.check(lib, rc, "l4d_attribute_forward")
        return out

    @torch.no_grad()
    def hash_indices(self, grid_id: int, level: int, x: torch.Tensor):
        """Parity hook: uint32 corner indices + weights of one level (grid_id 0 static, 1-3 dynamic, 4 flow)."""
        eng = self._engine
        lib = eng._lib()
        x = x.detach().contiguous().float()
        eng._require_cuda(x)
        n, D = x.shape
        idx = torch.empty(n, 1 << D, dtype=torch.int32, device=x.device)
        w = torch.empty(n, 1 << D, device=x.device)
        with torch.cuda.device(x.device):
            rc = lib.l4d_hash_indices(C.byref(eng.ccfg), grid_id, level, x.data_ptr(), n, idx.data_ptr(), w.data_ptr(),
                                      eng.stream())
        _capi.check(lib, rc, "l4d_hash_indices")
        return idx, w

    # ---- optimizer utils (lidar4d.py:226-237) ----------------------------------------------------
    def get_params(self, lr):
        return [
            {"params": self.planes_encoder.parameters(), "lr": lr},
            {"params": self.hash_encoder.parameters(), "lr": lr},
            {"params": self.view_encoder.parameters(), "lr": lr},
            {"params": self.flow_net.parameters(), "lr": 0.1 * lr},
            {"params": self.sigma_net.parameters(), "lr": 0.1 * lr},
            {"params": self.intensity_net.parameters(), "lr": 0.1 * lr},
            {"params": self.raydrop_net.parameters(), "lr": 0.1 * lr},
        ]

    @property
    def gpu_launches(self) -> int:
        return self._engine.n_launches
