"""Adam for the LiDAR4D hot path: one CUDA launch over the model's flat parameter / gradient arenas, fused with the
refresh of the fp16 hash tables the render kernels read (SURVEY.md 8(f) #4).

Drop-in for the optimiser the reference builds in main_lidar4d.py:298-300
    optimizer = lambda model: torch.optim.Adam(model.get_params(opt.lr), betas=(0.9, 0.99), eps=1e-15)
->  optimizer = lambda model: lidar4d_b200.optim.Adam(model, model.get_params(opt.lr), betas=(0.9, 0.99), eps=1e-15)
It is a torch.optim.Optimizer (param_groups / state_dict / LambdaLR / GradScaler.step work as usual).  After every step
the parameters and both moments are bit-identical to torch.optim.Adam(..., fused=True) of torch 2.11 (no weight decay, no
amsgrad) on the same gradients, and the fp16 hash tables it refreshes are byte-identical to a from-scratch staging
(tests/test_gpu_adam_exact.py).  The default, non-fused torch.optim.Adam rounds differently.  There is no CPU path.
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable

import torch

from . import _capi


class Adam(torch.optim.Optimizer):
    def __init__(self, model, params: Iterable, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8):
        if not hasattr(model, "_engine"):
            raise TypeError("lidar4d_b200.optim.Adam(model, params, ...): model must be a lidar4d_b200.LiDAR4D")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps))
        self._eng = model._engine
        b, e = self.param_groups[0]["betas"], self.param_groups[0]["eps"]
        for g in self.param_groups:
            if tuple(g["betas"]) != tuple(b) or g["eps"] != e:
                raise ValueError("all groups must share betas and eps (only lr is per group, as in lidar4d.py:226-237)")
        self._exp_avg = None
        self._exp_avg_sq = None
        self._step = 0
        self._arena_id = None
        self._seg_cache = None

    # ---- arena bookkeeping ---------------------------------------------------------------------------------------
    def _segments(self):
        """One Adam segment per hash table (they emit their fp16 copies), the other tensors merged per lr.  The segment
        STRUCTURE is cached per (arena, equality pattern of the group learning rates); a scheduler that rescales the
        rates only rewrites the lr fields."""
        eng = self._eng
        ts = eng.tensors()
        eng.ensure_flat(ts)
        lrs = [float(g["lr"]) for g in self.param_groups]
        key = (id(eng.flat_p), tuple(lrs.index(l) for l in lrs))
        if self._seg_cache is not None and self._seg_cache[0] == key:
            _, arr, n, owner = self._seg_cache
            for i in range(n):
                arr[i].lr = lrs[owner[i]]
            return arr, n
        by_ptr = {t.data_ptr(): nme for nme, t in ts.items()}
        group_of = {}
        for gi, g in enumerate(self.param_groups):
            for p in g["params"]:
                if p.numel() == 0:
                    continue
                nme = by_ptr.get(p.data_ptr())
                if nme is None:
                    raise ValueError("lidar4d_b200.optim.Adam only updates the hot-path parameters of its model "
                                     "(use torch.optim.Adam for the others, e.g. the U-Net)")
                group_of[nme] = gi
        segs = []                                             # [begin, end, group index, is_table]
        for nme in eng.names:                                 # arena order
            if nme not in group_of:
                continue
            o, k = eng.offsets[nme]
            table = ("hash" in nme) or nme.endswith("grid_enc.params")
            end = o + (k + 3) // 4 * 4
            gi = group_of[nme]
            if segs and not table and not segs[-1][3] and lrs[segs[-1][2]] == lrs[gi]:
                segs[-1][1] = end
            else:
                segs.append([o, end, gi, table])
        if len(segs) > _capi.ADAM_MAX_SEGMENTS:
            raise ValueError("too many Adam segments")
        arr = (_capi.L4DAdamGroup * len(segs))()
        for i, (b, e, gi, _) in enumerate(segs):
            arr[i].begin, arr[i].end, arr[i].lr = b, e, lrs[gi]
        self._seg_cache = (key, arr, len(segs), [sg[2] for sg in segs])
        return arr, len(segs)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        eng = self._eng
        lib = eng._lib()
        eng._require_cuda()
        arr, n = self._segments()
        tab_g = eng.attach_grads()              # parameters that never got a gradient take part with zeros, like torch
        if self._arena_id != id(eng.flat_p):
            if self._exp_avg is not None and self._exp_avg.numel() == eng.total:
                self._exp_avg, self._exp_avg_sq = self._exp_avg.to(eng.flat_p.device), self._exp_avg_sq.to(eng.flat_p.device)
            else:
                self._exp_avg = torch.zeros_like(eng.flat_p)
                self._exp_avg_sq = torch.zeros_like(eng.flat_p)
            self._arena_id = id(eng.flat_p)
        self._step += 1
        b1, b2 = self.param_groups[0]["betas"]
        fuse = eng.staged is not None
        master = eng.master_table() if fuse else None
        with torch.cuda.device(eng.device()):
            rc = lib.l4d_adam_step(C.byref(eng.ccfg), eng.flat_p.data_ptr(), eng.flat_g.data_ptr(),
                                   self._exp_avg.data_ptr(), self._exp_avg_sq.data_ptr(), eng.total, arr, n,
                                   float(b1), float(b2), float(self.param_groups[0]["eps"]), self._step, 1.0, 0,
                                   C.byref(master) if fuse else None, eng.staged.data_ptr() if fuse else None,
                                   eng.staged.numel() if fuse else 0, eng.stream())
        _capi.check(lib, rc, "l4d_adam_step")
        eng.params_updated_by_optimizer(tables_staged=fuse)
        return loss

    # ---- checkpointing (runner.py:955-1073 saves optimizer.state_dict()) ---------------------------------------------
    def state_dict(self):
        sd = super().state_dict()
        sd["l4d_flat"] = {"step": self._step,
                          "exp_avg": None if self._exp_avg is None else self._exp_avg.detach().clone(),
                          "exp_avg_sq": None if self._exp_avg_sq is None else self._exp_avg_sq.detach().clone()}
        return sd

    def load_state_dict(self, sd):
        sd = dict(sd)
        flat = sd.pop("l4d_flat", None)
        super().load_state_dict(sd)
        if flat is not None:
            self._step = int(flat["step"])
            self._exp_avg, self._exp_avg_sq = flat["exp_avg"], flat["exp_avg_sq"]
            self._arena_id = None
