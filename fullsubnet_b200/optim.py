"""``clip_grad_norm_`` + ``torch.optim.Adam.step`` (fullsubnet/trainer.py:65-68, train.py:55-59) as three kernel
launches without a host synchronisation (fsn_clip_adam_steps).  State keys (``step``, ``exp_avg``, ``exp_avg_sq``) and
``param_groups`` follow torch.optim.Adam, so checkpoints written by either optimiser load into the other.  Like
torch.optim.Adam, each parameter counts its own steps: one whose grad is None is skipped and its count stays."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib


class FusedClipAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, max_norm=None):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=0, amsgrad=False))
        self.max_norm = max_norm
        self.last_norm = None  # device tensor [2]: total gradient norm, applied coefficient
        self._scratch = None

    def _merged_groups(self):
        """clip_grad_norm_(model.parameters()) clips by the GLOBAL norm over every parameter (trainer.py:65-67), and
        one fsn_clip_adam call computes one norm: groups that share their hyper-parameters are merged into one call;
        groups that differ cannot share a launch."""
        groups = [g for g in self.param_groups if any(p.grad is not None for p in g["params"])]
        if len(groups) <= 1:
            return groups
        keys = {(g["lr"], tuple(g["betas"]), g["eps"]) for g in groups}
        if len(keys) > 1 and self.max_norm:
            raise NotImplementedError("FusedClipAdam: param groups with different lr/betas/eps cannot share the global "
                                      "gradient norm of one fsn_clip_adam call; use one group or max_norm=None")
        if len(keys) > 1:
            return groups
        merged = dict(groups[0])
        merged["params"] = [p for g in groups for p in g["params"]]
        return [merged]

    @torch.no_grad()
    def step(self, closure=None, grad_scale: float = 1.0):
        assert closure is None
        lib = _lib.load()
        for group in self._merged_groups():
            ps = [p for p in group["params"] if p.grad is not None]
            if not ps:
                continue
            if len(ps) > _lib.MAX_PARAM_TENSORS:
                raise NotImplementedError(f"FusedClipAdam handles <= {_lib.MAX_PARAM_TENSORS} tensors per group")
            L = _lib.ParamList()
            L.n = len(ps)
            steps = (C.c_int * len(ps))()
            for i, p in enumerate(ps):
                _lib.require_cuda(p, "parameter")
                st = self.state[p]
                if not st:
                    st["step"] = torch.tensor(0.0)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["step"] += 1
                steps[i] = int(st["step"])
                g = p.grad
                if not g.is_contiguous() or g.dtype != torch.float32:
                    raise RuntimeError("FusedClipAdam needs contiguous fp32 gradients")
                L.param[i], L.grad[i] = p.data_ptr(), g.data_ptr()
                L.exp_avg[i], L.exp_avg_sq[i] = st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr()
                L.numel[i] = p.numel()
            device = ps[0].device
            with torch.cuda.device(device):
                if self._scratch is None or self._scratch.device != device:
                    self._scratch = torch.empty(lib.fsn_clip_adam_scratch_bytes(), dtype=torch.uint8, device=device)
                self.last_norm = torch.empty(2, dtype=torch.float32, device=device)
                b1, b2 = group["betas"]
                _lib.check(lib.fsn_clip_adam_steps(C.byref(L), float(self.max_norm or 0.0), float(grad_scale),
                                                   group["lr"], b1, b2, group["eps"], steps, self.last_norm.data_ptr(),
                                                   self._scratch.data_ptr(), self._scratch.numel(),
                                                   _lib.stream_ptr(device)))
            # the kernel wrote through raw pointers: tell autograd / the packed-weight caches (keyed on
            # (data_ptr, _version), fullsubnet/model.py:_packed_sb) that the parameters changed
            torch._C._increment_version(ps)
        return None
