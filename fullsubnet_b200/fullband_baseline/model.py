"""Drop-in for recipes/dns_interspeech_2020/fullband_baseline/model.py:8-68 (class Model; SURVEY 8f rank 3).

Same constructor kwargs and ``state_dict`` keys (``fullband_model.sequence_model.weight_ih_l{0,1,2}`` ...,
``fullband_model.fc_output_layer.*``); ``forward(noisy_mag [B,1,F,T]) -> [B,2,F,T]`` is one call into libfsn_b200
(``fsn_fullband_forward``).  ``enhance`` / ``enhance_pcm`` run the wav -> wav path of ``Inferencer.full_band_crm_mask``
for a batch of clips, of equal or different lengths, in one call (``fsn_fullband_enhance``).  With gradients enabled the forward keeps its activations (``fsn_fullband_train_forward``)
and ``loss.backward()`` runs back-propagation through time in the library (``fsn_fullband_train_backward``), the
training step of fullband_baseline/trainer.py:32-71."""
from __future__ import annotations

import ctypes as C
import os

import torch

from .. import _lib
from ..model.base_model import BaseModel, SpectrogramEnhance, TrainStep
from ..model.module.sequence_model import SequenceModel


class Model(SpectrogramEnhance, BaseModel):
    # fused wav -> wav call (enhance / enhance_pcm): stft -> model -> mask + istft [-> int16] in one library call
    ENHANCE_ENTRY_POINTS = ("fsn_fullband_enhance_workspace_bytes", "fsn_fullband_enhance")
    # training step (fullband_baseline/trainer.py:32-71): fsn_fullband_train_forward keeps the activations,
    # fsn_fullband_train_backward runs BPTT
    TRAIN_ENTRY_POINTS = ("fsn_fullband_train_workspace_bytes", "fsn_fullband_train_forward", "fsn_fullband_train_backward")
    TRAIN_TF32_STACKS = ("fullband_model",)
    # chunked streaming (fullsubnet_b200.stream.Streamer): state / workspace queries, delay, step
    STREAM_ENTRY_POINTS = ("fsn_fullband_stream_state_bytes", "fsn_fullband_stream_workspace_bytes",
                           "fsn_fullband_stream_delay", "fsn_fullband_stream_step")

    def __init__(self, num_freqs, hidden_size, sequence_model, output_activate_function, look_ahead,
                 norm_type="offline_laplace_norm", weight_init=True, precision=None):
        super().__init__()
        self.fullband_model = SequenceModel(input_size=num_freqs, output_size=num_freqs * 2, hidden_size=hidden_size,
                                            num_layers=3, bidirectional=False, sequence_model=sequence_model,
                                            output_activate_function=output_activate_function)
        self.num_freqs = num_freqs
        self.look_ahead = look_ahead
        self.norm = self.norm_wrapper(norm_type)
        # inference arithmetic: "fp32" (= "auto") only.  The tensor-core stack misses the reference gates on this model
        # (f16x3_tc: 1.8e-4 waveform max-abs on the clipping weight set; f16_tc: 1.6e-3 relative cRM), so it is not
        # built, and the process-wide FSN_PRECISION of the other models is not read here.
        self.precision = precision or "auto"
        # arithmetic of the training step's GEMMs: "fp32" (FMA) | "tf32_tc" (wgmma tf32 for the LSTM layers) | "auto" =
        # tf32_tc when hidden_size is a multiple of 4
        self.train_precision = os.environ.get("FSN_TRAIN_PRECISION", "auto")
        if weight_init:
            self.apply(self.weight_init)

    def _resolve_precision(self) -> str:
        if self.precision not in ("fp32", "auto"):
            raise ValueError("fullband_baseline precision must be 'fp32' or 'auto': the tensor-core precisions are not "
                             "built for this model")
        return "fp32"

    def _infer_desc(self):
        return self._desc(_lib.PREC[self._resolve_precision()])

    def _enhance_args(self, device):
        return self._infer_desc(), self._weight_ptrs()

    def _stream_desc(self):
        return self._infer_desc()

    def _stream_weights(self):
        return self._weight_ptrs()

    def _train_desc(self):
        return self._desc(_lib.PREC[self._resolve_train_precision()])

    def _train_weights(self):
        return self._weight_ptrs()

    def _train_grads(self, grads):
        g = _lib.FullbandGrads()
        for l in range(self.fullband_model.num_layers):
            g.layer[l] = SequenceModel.grads_struct(grads, "fullband_model.", l)
        g.fc_w = grads["fullband_model.fc_output_layer.weight"].data_ptr()
        g.fc_b = grads["fullband_model.fc_output_layer.bias"].data_ptr()
        return (C.byref(g),)

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
        if self._records_grad():
            if self.fullband_model.cell != "LSTM":
                raise NotImplementedError("fullsubnet_b200: fullband_baseline training is built for LSTM only")
            return TrainStep.apply(self, x, *self.parameters())
        lib = _lib.load()
        with torch.cuda.device(x.device):
            d = self._infer_desc()
            layers, fc_w, fc_b = self._weight_ptrs()
            n = _lib.check_workspace(lib.fsn_fullband_workspace_bytes(C.byref(d), batch_size, num_frames))
            ws = torch.empty(n, dtype=torch.uint8, device=x.device)
            out = torch.empty(batch_size, 2, num_freqs, num_frames, dtype=torch.float32, device=x.device)
            _lib.check(lib.fsn_fullband_forward(C.byref(d), layers, fc_w, fc_b, x.data_ptr(), batch_size, num_frames,
                                                out.data_ptr(), ws.data_ptr(), n, _lib.stream_ptr(x.device)))
        return out
