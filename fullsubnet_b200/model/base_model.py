"""Host-side pieces of audio_zen/model/base_model.py that the drop-in Model needs:
norm_wrapper (:356-372) name checking and weight_init (:374-439, CPU-side initialisation); plus the training step
that fullsubnet, fast_fullsubnet and fullband_baseline share (autograd Function, precision choice, flat gradients),
and the fused wav -> wav call of the models that have one."""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn
import torch.nn.init as init

from .. import _lib


class TrainStep(torch.autograd.Function):
    """Model.forward with back-propagation through time in libfsn_b200.  The parameters are passed as inputs so
    autograd (and DDP's hooks) route the gradients to them exactly as for the reference's nn.LSTM / nn.Linear modules.
    The model names its library entry points and supplies the descriptor, the weight / gradient arguments and the
    output shape (BaseModel's training-step hooks)."""

    @staticmethod
    def forward(ctx, model, x, *params):
        device = x.device
        lib = _lib.load()
        query, fwd, _ = (getattr(lib, name) for name in model.TRAIN_ENTRY_POINTS)
        with torch.cuda.device(device):
            desc = model._train_desc()
            weights = model._train_weights()
            dims, out_shape = model._train_io(x, desc)
            n = _lib.check_workspace(query(C.byref(desc), *dims))
            ws = torch.empty(n, dtype=torch.uint8, device=device)
            out = torch.empty(out_shape, dtype=torch.float32, device=device)
            _lib.check(fwd(C.byref(desc), *weights, x.data_ptr(), *dims, out.data_ptr(), ws.data_ptr(), n,
                           _lib.stream_ptr(device)))
        ctx.model, ctx.ws, ctx.dims, ctx.desc = model, ws, dims, desc
        ctx.versions = model._version_key()
        return out

    @staticmethod
    def backward(ctx, dy):
        model = ctx.model
        if ctx.versions != model._version_key():
            raise RuntimeError("fullsubnet_b200: a parameter was modified in place between forward and backward")
        if ctx.ws is None:
            raise RuntimeError("fullsubnet_b200: backward through the same forward twice (activations were released)")
        dy = dy.contiguous().float()
        device = dy.device
        bwd = getattr(_lib.load(), model.TRAIN_ENTRY_POINTS[2])
        names = [k for k, _ in model.named_parameters()]
        _, grads = model._new_flat_grads(device)
        with torch.cuda.device(device):
            weights = model._train_weights()
            g = model._train_grads(grads)
            _lib.check(bwd(C.byref(ctx.desc), *weights, dy.data_ptr(), *ctx.dims, *g, ctx.ws.data_ptr(), ctx.ws.numel(),
                           _lib.stream_ptr(device)))
        ctx.ws = None
        return (None, None) + tuple(grads[k] for k in names)


class BaseModel(nn.Module):
    NORM_TYPES = {"offline_laplace_norm": 0, "cumulative_laplace_norm": 1, "forgetting_norm": 4}
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

    # ---------------------------------------------------------------- training step (TrainStep)
    # Each trainable model sets TRAIN_ENTRY_POINTS (library workspace query, forward, backward), TRAIN_TF32_STACKS (the
    # SequenceModel attributes whose hidden sizes decide train_precision="auto") and implements _train_desc(),
    # _train_weights() and _train_grads(grads): the descriptor and the ctypes arguments of the weights / gradients.
    # _train_io / _train_out_shape give the size arguments of the entry points and the output shape.
    TRAIN_ENTRY_POINTS: tuple = ()
    TRAIN_TF32_STACKS: tuple = ()

    def _resolve_train_precision(self) -> str:
        """"fp32" (FMA) or "tf32_tc" (wgmma tf32); "auto" = tf32_tc when the TRAIN_TF32_STACKS hidden sizes are
        multiples of 4."""
        if self.train_precision == "auto":
            ok = all(getattr(self, s).hidden_size % 4 == 0 for s in self.TRAIN_TF32_STACKS)
            return "tf32_tc" if ok else "fp32"
        if self.train_precision not in ("fp32", "tf32_tc"):
            raise ValueError("train_precision must be 'fp32', 'tf32_tc' or 'auto'")
        return self.train_precision

    def _records_grad(self) -> bool:
        """True when this forward is a training step: gradients are enabled and the parameters require them.  A
        partially frozen model raises."""
        if not (torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())):
            return False
        if not all(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("fullsubnet_b200: partially frozen models are not built")
        return True

    def _train_io(self, x, desc):
        """(the size arguments of the training entry points, the output shape) for the input x: (B, T) and
        _train_out_shape for a spectrogram [B,1,F,T]."""
        B, _, F, T = x.shape
        return (B, T), self._train_out_shape(desc, B, F, T)

    def _train_out_shape(self, desc, B, F, T):
        return (B, 2, F, T)

    # ---------------------------------------------------------------- fused wav -> wav call (_enhance_call)
    # Each model with one sets ENHANCE_ENTRY_POINTS (library workspace query, call) and implements _enhance_args(device):
    # the descriptor and the ctypes arguments of the weights.
    ENHANCE_ENTRY_POINTS: tuple = ()

    def _enhance_call(self, noisy, *args):
        """One fused library call: noisy [B,L] -> (enhanced [B,L], crm [B,2,F,T] or None, pcm int16 [B,L] or None).
        ``args`` = (*stft, lengths, return_crm, gain): ``stft`` is (n_fft, hop_length, win_length) for the models that
        take the Inferencer's STFT geometry and empty for one whose descriptor holds its own; clip b is row b's first
        lengths[b] samples (all L when lengths is None), its outputs 0 past them; ``gain`` None: no int16 output."""
        *stft, lengths, return_crm, gain = args
        B, L = noisy.shape
        lens = None if lengths is None else _lib.lengths_table(lengths, B, L)
        x = _lib.require_cuda(noisy, "noisy")
        n_fft, hop = stft[:2] if stft else (self.n_fft, self.hop_length)
        F, T = n_fft // 2 + 1, 1 + L // hop
        device = x.device
        lib = _lib.load()
        query, call = (getattr(lib, name) for name in self.ENHANCE_ENTRY_POINTS)
        with torch.cuda.device(device):
            desc, weights = self._enhance_args(device)
            n = _lib.check_workspace(query(C.byref(desc), B, L, *stft[:2]))
            crm = torch.empty(B, 2, F, T, dtype=torch.float32, device=device) if return_crm else None
            pcm = None if gain is None else torch.empty(B, L, dtype=torch.int16, device=device)
            ws = torch.empty(n, dtype=torch.uint8, device=device)
            out = torch.empty(B, L, dtype=torch.float32, device=device)
            _lib.check(call(C.byref(desc), *weights, x.data_ptr(), None if lens is None else lens.ctypes.data, B, L,
                            *stft, out.data_ptr(), _lib.ptr(crm), _lib.ptr(pcm), 0.0 if gain is None else float(gain),
                            ws.data_ptr(), n, _lib.stream_ptr(device)))
        return out, crm, pcm

    def _version_key(self):
        return tuple((p.data_ptr(), p._version) for p in self.parameters())

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


class SpectrogramEnhance:
    """enhance / enhance_pcm of the models that take the Inferencer's STFT geometry (fullsubnet, fullband_baseline)."""

    @torch.no_grad()
    def enhance(self, noisy, n_fft=512, hop_length=256, win_length=512, return_crm=False, lengths=None):
        """Fused wav -> wav path of Inferencer.full_band_crm_mask (recipes/.../inferencer.py:130-145), batched over
        independent clips in one library call: noisy [B,L] -> enhanced [B,L].

        ``lengths`` (B ints, or a CPU integer tensor; max must be L; power-of-two n_fft): clips of different lengths in
        one call.  Clip b is ``noisy[b, :lengths[b]]``; the rest of the row is never read.  Its outputs equal the call on
        that clip alone, bit for bit; ``enhanced[b, lengths[b]:]`` and the cRM frames ``t >= 1 + lengths[b] //
        hop_length`` are 0.  ``return_crm`` additionally returns the [B,2,F,T_max] model output."""
        assert noisy.dim() == 2, "noisy must be [B, L]"
        out, crm, _ = self._enhance_call(noisy, n_fft, hop_length, win_length, lengths, return_crm, None)
        return (out, crm) if return_crm else out

    @torch.no_grad()
    def enhance_pcm(self, noisy, n_fft=512, hop_length=256, win_length=512, gain=0.8 * 32767.0, lengths=None):
        """``enhance`` plus the int16 scaling of the reference host loop (audio_zen/inferencer/base_inferencer.py:
        181-182) in the same call, the per-clip max|y| reduced in the iSTFT epilogue: noisy [B,L] -> (enhanced float32
        [B,L], pcm int16 [B,L]).  ``lengths``: as in ``enhance``; each clip is scaled by the peak of its own samples and
        its pcm row is 0 past them."""
        assert noisy.dim() == 2, "noisy must be [B, L]"
        out, _, pcm = self._enhance_call(noisy, n_fft, hop_length, win_length, lengths, False, gain)
        return out, pcm
