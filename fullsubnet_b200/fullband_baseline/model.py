"""Drop-in for recipes/dns_interspeech_2020/fullband_baseline/model.py:8-68 (class Model; SURVEY 8f rank 3).

Same constructor kwargs and ``state_dict`` keys (``fullband_model.sequence_model.weight_ih_l{0,1,2}`` ...,
``fullband_model.fc_output_layer.*``); ``forward(noisy_mag [B,1,F,T]) -> [B,2,F,T]`` is one call into libfsn_b200
(``fsn_fullband_forward``).  With gradients enabled the forward keeps its activations (``fsn_fullband_train_forward``)
and ``loss.backward()`` runs back-propagation through time in the library (``fsn_fullband_train_backward``), the
training step of fullband_baseline/trainer.py:32-71."""
from __future__ import annotations

import ctypes as C
import os

import torch

from .. import _lib
from ..model.base_model import BaseModel
from ..model.module.sequence_model import SequenceModel


def _grad_struct(grads: dict, num_layers: int) -> "_lib.FullbandGrads":
    g = _lib.FullbandGrads()
    for l in range(num_layers):
        g.layer[l] = _lib.LstmGrads(*(grads[f"fullband_model.sequence_model.{n}_l{l}"].data_ptr()
                                      for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")))
    g.fc_w = grads["fullband_model.fc_output_layer.weight"].data_ptr()
    g.fc_b = grads["fullband_model.fc_output_layer.bias"].data_ptr()
    return g


class _TrainForward(torch.autograd.Function):
    """Model.forward with back-propagation through time in libfsn_b200 (fsn_fullband_train_forward /
    fsn_fullband_train_backward).  The parameters are passed as inputs so autograd (and DDP's hooks) route the gradients
    to them exactly as for the reference's nn.LSTM / nn.Linear modules."""

    @staticmethod
    def forward(ctx, model, x, *params):
        B, _, F, T = x.shape
        device = x.device
        lib = _lib.load()
        with torch.cuda.device(device):
            d = model._desc(_lib.PREC[model._resolve_train_precision()])
            layers, fc_w, fc_b = model._weight_ptrs()
            n = lib.fsn_fullband_train_workspace_bytes(C.byref(d), B, T)
            if n == 0:
                _lib.check_workspace(n)
            ws = torch.empty(n, dtype=torch.uint8, device=device)
            out = torch.empty(B, 2, F, T, dtype=torch.float32, device=device)
            _lib.check(lib.fsn_fullband_train_forward(C.byref(d), layers, fc_w, fc_b, x.data_ptr(), B, T, out.data_ptr(),
                                                      ws.data_ptr(), n, _lib.stream_ptr(device)))
        ctx.model, ctx.ws, ctx.dims, ctx.desc = model, ws, (B, T), d
        ctx.versions = model.fullband_model.version_key()
        return out

    @staticmethod
    def backward(ctx, dout):
        model, (B, T) = ctx.model, ctx.dims
        if ctx.versions != model.fullband_model.version_key():
            raise RuntimeError("fullsubnet_b200: a parameter was modified in place between forward and backward")
        if ctx.ws is None:
            raise RuntimeError("fullsubnet_b200: backward through the same forward twice (activations were released)")
        dout = dout.contiguous().float()
        device = dout.device
        lib = _lib.load()
        names = [k for k, _ in model.named_parameters()]
        _, grads = model._new_flat_grads(device)
        with torch.cuda.device(device):
            layers, fc_w, fc_b = model._weight_ptrs()
            g = _grad_struct(grads, model.fullband_model.num_layers)
            _lib.check(lib.fsn_fullband_train_backward(C.byref(ctx.desc), layers, fc_w, fc_b, dout.data_ptr(), B, T,
                                                       C.byref(g), ctx.ws.data_ptr(), ctx.ws.numel(),
                                                       _lib.stream_ptr(device)))
        ctx.ws = None
        return (None, None) + tuple(grads[k] for k in names)


class Model(BaseModel):
    def __init__(self, num_freqs, hidden_size, sequence_model, output_activate_function, look_ahead,
                 norm_type="offline_laplace_norm", weight_init=True):
        super().__init__()
        self.fullband_model = SequenceModel(input_size=num_freqs, output_size=num_freqs * 2, hidden_size=hidden_size,
                                            num_layers=3, bidirectional=False, sequence_model=sequence_model,
                                            output_activate_function=output_activate_function)
        self.num_freqs = num_freqs
        self.look_ahead = look_ahead
        self.norm = self.norm_wrapper(norm_type)
        # arithmetic of the training step's GEMMs: "fp32" (FMA) | "tf32_tc" (wgmma tf32 for the LSTM layers) | "auto" =
        # tf32_tc when hidden_size is a multiple of 4
        self.train_precision = os.environ.get("FSN_TRAIN_PRECISION", "auto")
        if weight_init:
            self.apply(self.weight_init)

    def _resolve_train_precision(self) -> str:
        if self.train_precision == "auto":
            return "tf32_tc" if self.fullband_model.hidden_size % 4 == 0 else "fp32"
        if self.train_precision not in ("fp32", "tf32_tc"):
            raise ValueError("train_precision must be 'fp32', 'tf32_tc' or 'auto'")
        return self.train_precision

    def _desc(self, prec: int = 0):
        seq = self.fullband_model
        return _lib.FullbandDesc(num_freqs=self.num_freqs, hidden=seq.hidden_size, num_layers=seq.num_layers,
                                 look_ahead=self.look_ahead, activation=_lib.ACT[seq.output_activate_function],
                                 norm_type=self.norm, precision=prec, cell_type=_lib.CELL[seq.cell])

    def _weight_ptrs(self):
        seq = self.fullband_model
        layers = (_lib.LstmLayer * seq.num_layers)(*(seq.layer_struct(l) for l in range(seq.num_layers)))
        return (layers, *seq.fc_ptrs())

    def forward(self, noisy_mag):
        """noisy_mag [B,1,F,T] -> [B,2,F,T]  (fullband_baseline/model.py:46-68)."""
        assert noisy_mag.dim() == 4
        batch_size, num_channels, num_freqs, num_frames = noisy_mag.size()
        assert num_channels == 1, f"{self.__class__.__name__} takes the mag feature as inputs."
        assert num_freqs == self.num_freqs, f"num_freqs {num_freqs} != {self.num_freqs}"
        x = _lib.require_cuda(noisy_mag, "noisy_mag")
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            # training step (fullband_baseline/trainer.py:32-71): kernels that keep the activations for BPTT
            if not all(p.requires_grad for p in self.parameters()):
                raise NotImplementedError("fullsubnet_b200: partially frozen models are not built")
            if self.fullband_model.cell != "LSTM":
                raise NotImplementedError("fullsubnet_b200: fullband_baseline training is built for LSTM only")
            return _TrainForward.apply(self, x, *self.parameters())
        lib = _lib.load()
        with torch.cuda.device(x.device):
            d = self._desc()
            layers, fc_w, fc_b = self._weight_ptrs()
            n = _lib.check_workspace(lib.fsn_fullband_workspace_bytes(C.byref(d), batch_size, num_frames))
            ws = torch.empty(n, dtype=torch.uint8, device=x.device)
            out = torch.empty(batch_size, 2, num_freqs, num_frames, dtype=torch.float32, device=x.device)
            _lib.check(lib.fsn_fullband_forward(C.byref(d), layers, fc_w, fc_b, x.data_ptr(), batch_size, num_frames,
                                                out.data_ptr(), ws.data_ptr(), n, _lib.stream_ptr(x.device)))
        return out
