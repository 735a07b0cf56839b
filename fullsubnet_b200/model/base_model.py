"""Host-side pieces of audio_zen/model/base_model.py that the drop-in Model needs:
norm_wrapper (:356-372) name checking and weight_init (:374-439, CPU-side initialisation); plus the flat-gradient
buffers the training steps of fullsubnet and fast_fullsubnet share."""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.init as init


class BaseModel(nn.Module):
    NORM_TYPES = {"offline_laplace_norm": 0, "cumulative_laplace_norm": 1}
    _UPSTREAM_NORMS = ("offline_laplace_norm", "cumulative_laplace_norm", "offline_gaussian_norm",
                       "cumulative_layer_norm", "forgetting_norm")

    def __init__(self):
        super().__init__()

    def norm_wrapper(self, norm_type: str) -> int:
        if norm_type in self.NORM_TYPES:
            return self.NORM_TYPES[norm_type]
        if norm_type in self._UPSTREAM_NORMS:
            raise NotImplementedError(f"norm_type {norm_type!r} is not built into libfsn_b200 yet (SURVEY 8f)")
        raise NotImplementedError(
            "You must set up a type of Norm. e.g. offline_laplace_norm, cumulative_laplace_norm, forgetting_norm, etc.")

    def weight_init(self, m):
        """base_model.py:374-439 restricted to the module types this model contains."""
        if isinstance(m, nn.Linear):
            init.xavier_normal_(m.weight.data)
            init.normal_(m.bias.data)
        elif isinstance(m, (nn.LSTM, nn.GRU)):
            for param in m.parameters():
                if len(param.shape) >= 2:
                    init.orthogonal_(param.data)
                else:
                    init.normal_(param.data)

    def flat_grad(self):
        """Makes every ``p.grad`` a view into one persistent flat fp32 buffer (keeping current values) and returns
        the buffer: one ``all_reduce`` then moves every gradient of the model (SURVEY 8e)."""
        params = list(self.parameters())
        flat = getattr(self, "_flat", None)
        ok = flat is not None and flat.device == params[0].device and all(
            p.grad is not None and p.grad.data_ptr() == flat.data_ptr() + 4 * off
            for p, off in zip(params, self._flat_offsets))
        if not ok:
            flat = torch.zeros(sum(p.numel() for p in params), dtype=torch.float32, device=params[0].device)
            offs, off = [], 0
            for p in params:
                view = flat[off:off + p.numel()].view_as(p)
                if p.grad is not None:
                    view.copy_(p.grad)
                p.grad = view
                offs.append(off)
                off += p.numel()
            self._flat, self._flat_offsets = flat, offs
        return flat

    def _new_flat_grads(self, device):
        """One flat fp32 buffer holding every gradient in parameter order (what the single all-reduce of
        base_trainer.py:32 / SURVEY 8e moves) and the per-parameter views into it."""
        params = list(self.named_parameters())
        flat = torch.empty(sum(p.numel() for _, p in params), dtype=torch.float32, device=device)
        views, off = {}, 0
        for k, p in params:
            views[k] = flat[off:off + p.numel()].view_as(p)
            off += p.numel()
        return flat, views
