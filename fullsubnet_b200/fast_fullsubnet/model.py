"""Drop-in for recipes/dns_interspeech_2020/fast_fullsubnet/model.py:11-202 (class Model, BASELINE config 4).

Same constructor kwargs and the same 31 ``state_dict`` entries (incl. the ``mel_scale.fb`` buffer that
torchaudio's MelScale registers); ``forward(mix_mag [B,1,F,T]) -> [B,2,F,T]`` is one call into libfsn_b200
(``fsn_fast_model_forward``).  In train mode with gradients enabled the forward keeps its activations
(``fsn_fast_train_forward``) and ``loss.backward()`` runs back-propagation through time in the library
(``fsn_fast_train_backward``), the training step of fast_fullsubnet/trainer.py:45-56."""
from __future__ import annotations

import ctypes as C
import math
import os

import torch
import torch.nn as nn

from .. import _lib
from ..model.base_model import BaseModel, TrainStep
from ..model.module.sequence_model import SequenceModel


def melscale_fbanks(n_freqs: int, n_mels: int, sample_rate: int = 16000, f_min: float = 0.0, f_max: float = 8000.0):
    """HTK mel filterbank [n_freqs, n_mels] = torchaudio.functional.melscale_fbanks(norm=None, mel_scale='htk'),
    the buffer behind torchaudio.transforms.MelScale (fast_fullsubnet/model.py:57-63)."""
    all_freqs = torch.linspace(0, sample_rate // 2, n_freqs)
    m_min = 2595.0 * math.log10(1.0 + f_min / 700.0)
    m_max = 2595.0 * math.log10(1.0 + f_max / 700.0)
    f_pts = 700.0 * (10 ** (torch.linspace(m_min, m_max, n_mels + 2) / 2595.0) - 1.0)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts.unsqueeze(0) - all_freqs.unsqueeze(1)
    return torch.max(torch.zeros(1), torch.min((-1.0 * slopes[:, :-2]) / f_diff[:-1], slopes[:, 2:] / f_diff[1:]))


_LAYERS = (("enc1", "encoder.0.", 0), ("enc2", "encoder.1.", 0), ("dec1", "decoder_lstm.0.", 0),
           ("dec2", "decoder_lstm.1.", 0))
_LINEARS = (("enc_fc", "encoder.1."), ("bn_fc", "bottleneck."), ("dec_fc", "decoder_lstm.1."))


def _grad_struct(grads: dict) -> "_lib.FastGrads":
    g = _lib.FastGrads()
    for field, prefix, l in _LAYERS:
        setattr(g, field, SequenceModel.grads_struct(grads, prefix, l))
    for l in range(2):
        g.bn[l] = SequenceModel.grads_struct(grads, "bottleneck.", l)
    for field, prefix in _LINEARS:
        setattr(g, field + "_w", grads[f"{prefix}fc_output_layer.weight"].data_ptr())
        setattr(g, field + "_b", grads[f"{prefix}fc_output_layer.bias"].data_ptr())
    return g


class _MelScale(nn.Module):
    """Owns the ``fb`` buffer under the reference's key ``mel_scale.fb``."""

    def __init__(self, n_mels, n_stft):
        super().__init__()
        self.register_buffer("fb", melscale_fbanks(n_stft, n_mels))


class Model(BaseModel):
    # forgetting_norm is built for fullsubnet and fullband_baseline only: it stays an unbuilt upstream norm here
    NORM_TYPES = {"offline_laplace_norm": 0, "cumulative_laplace_norm": 1}
    # training step (fast_fullsubnet/trainer.py:45-56): fsn_fast_train_forward keeps the activations,
    # fsn_fast_train_backward runs BPTT
    TRAIN_ENTRY_POINTS = ("fsn_fast_train_workspace_bytes", "fsn_fast_train_forward", "fsn_fast_train_backward")
    TRAIN_TF32_STACKS = ("bottleneck",)
    # chunked streaming (fullsubnet_b200.stream.Streamer, precision="fp32" with cumulative_laplace_norm): state /
    # workspace queries, delay, step
    STREAM_ENTRY_POINTS = ("fsn_fast_stream_state_bytes", "fsn_fast_stream_workspace_bytes", "fsn_fast_stream_delay",
                           "fsn_fast_stream_step")
    # the same on the fp16 tensor cores (Streamer(tensor_cores=True), the model's f16x3_tc / f16_tc precision)
    STREAM_TC_ENTRY_POINTS = ("fsn_fast_stream_tc_state_bytes", "fsn_fast_stream_tc_workspace_bytes",
                              "fsn_fast_stream_tc_delay", "fsn_fast_stream_tc_step")

    def __init__(self, look_ahead, shrink_size, sequence_model, num_mels, encoder_input_size, bottleneck_hidden_size,
                 bottleneck_num_layers, noisy_input_num_neighbors, encoder_output_num_neighbors,
                 norm_type="offline_laplace_norm", weight_init=False, precision=None):
        super().__init__()
        assert sequence_model in ("GRU", "LSTM"), f"{self.__class__.__name__} only support GRU and LSTM."
        self.encoder = nn.Sequential(
            SequenceModel(input_size=64, hidden_size=384, output_size=0, num_layers=1, bidirectional=False,
                          sequence_model=sequence_model, output_activate_function=None),
            SequenceModel(input_size=384, hidden_size=257, output_size=64, num_layers=1, bidirectional=False,
                          sequence_model=sequence_model, output_activate_function="ReLU"))
        self.mel_scale = _MelScale(n_mels=num_mels, n_stft=encoder_input_size)
        self.bottleneck = SequenceModel(
            input_size=(noisy_input_num_neighbors * 2 + 1) + (encoder_output_num_neighbors * 2 + 1), output_size=1,
            hidden_size=bottleneck_hidden_size, num_layers=bottleneck_num_layers, bidirectional=False,
            sequence_model=sequence_model, output_activate_function="ReLU")
        self.decoder_lstm = nn.Sequential(
            SequenceModel(input_size=64 + 64, hidden_size=512, output_size=0, num_layers=1, bidirectional=False,
                          sequence_model=sequence_model, output_activate_function=None),
            SequenceModel(input_size=512, hidden_size=512, output_size=257 * 2, num_layers=1, bidirectional=False,
                          sequence_model=sequence_model, output_activate_function=None))
        self.shrink_size = shrink_size
        self.look_ahead = look_ahead
        self.num_mels = num_mels
        self.encoder_input_size = encoder_input_size
        self.noisy_input_num_neighbors = noisy_input_num_neighbors
        self.enc_output_num_neighbors = encoder_output_num_neighbors
        # offline_laplace_norm or cumulative_laplace_norm (both norms, every precision, inference and training); the
        # other upstream norms raise NotImplementedError
        self.norm = self.norm_wrapper(norm_type)
        # arithmetic: 'fp32' (FMA kernels) | 'f16x3_tc' (tensor cores, hi+lo split operands, the fp32 error class) |
        # 'f16_tc' (tensor cores, single pass, ~1e-4) | 'auto' = f16x3_tc when the shape allows, else fp32.  The
        # tensor-core modes run the bottleneck on the wgmma sub-band kernel and the encoder / decoder LSTMs + Linears
        # on the hoisted-GEMM + persistent-recurrence kernels (fsn_lstm_rec_tc.cu)
        self.precision = precision or os.environ.get("FSN_PRECISION", "auto")
        # arithmetic of the training step's GEMMs: "fp32" (FMA) | "tf32_tc" (wgmma tf32 for every LSTM layer whose hidden
        # size is a multiple of 4; enc2 with 257 units stays fp32) | "auto" = tf32_tc when the bottleneck allows it
        self.train_precision = os.environ.get("FSN_TRAIN_PRECISION", "auto")
        self.sequence_model_type = sequence_model
        self._packed = None
        self._packed_key = None
        if num_mels != 64 or encoder_input_size != 257:
            raise NotImplementedError("the reference hard-codes 64 mel bins / 257 frequencies in its layer sizes")
        if weight_init:
            self.apply(self.weight_init)

    def _resolve_precision(self) -> str:
        d = self._desc(_lib.PREC["f16_tc"])
        ok = _lib.load().fsn_fast_packed_bytes(C.byref(d)) > 0
        if self.precision == "auto":
            return "f16x3_tc" if ok else "fp32"
        if self.precision not in ("fp32", "f16_tc", "f16x3_tc"):
            raise ValueError("precision must be 'fp32', 'f16x3_tc', 'f16_tc' or 'auto'")
        if self.precision != "fp32" and not ok:
            raise NotImplementedError("the tensor-core precisions need bottleneck_hidden_size = 384, 2 layers and input width <= 32")
        return self.precision

    def _stream_desc(self):
        """Descriptor of the streaming calls: the fp32 kernels only, so an explicit precision="fp32" (under "auto" the
        whole-clip call runs the tensor cores, which a stream could not match)."""
        if self.precision != "fp32":
            raise NotImplementedError(f"fullsubnet_b200: fast_fullsubnet streaming is built for precision=\"fp32\" "
                                      f"(this model has precision={self.precision!r})")
        return self._desc(_lib.PREC["fp32"])

    def _stream_weights(self):
        return (C.byref(self._weight_struct()),)

    def _stream_tc_desc(self):
        """Descriptor of the tensor-core streaming calls: the model's resolved precision, which must be f16x3_tc or
        f16_tc (so "auto" streams the bits of the whole-clip call wherever that call runs the tensor cores)."""
        prec = self._resolve_precision()
        if prec == "fp32":
            raise NotImplementedError("fullsubnet_b200: this model resolves to precision=\"fp32\", and tensor-core "
                                      "streaming (tensor_cores=True) needs f16x3_tc or f16_tc; stream it with the default "
                                      "Streamer(model, slots) (tensor_cores=False)")
        return self._desc(_lib.PREC[prec])

    def _stream_tc_weights(self):
        self._stream_tc_desc()
        _, w = self._structs(next(self.parameters()).device)  # with the cached packed bottleneck image
        return (C.byref(w),)

    def _train_desc(self):
        return self._desc(_lib.PREC[self._resolve_train_precision()])

    def _train_weights(self):
        return (C.byref(self._weight_struct()),)

    def _train_grads(self, grads):
        return (C.byref(_grad_struct(grads)),)

    def _desc(self, prec: int):
        return _lib.FastDesc(num_freqs=self.encoder_input_size, look_ahead=self.look_ahead, shrink_size=self.shrink_size,
                          num_mels=self.num_mels, enc1_hidden=384, enc2_hidden=257,
                          bn_hidden=self.bottleneck.hidden_size, bn_layers=self.bottleneck.num_layers, dec_hidden=512,
                          noisy_num_neighbors=self.noisy_input_num_neighbors,
                          enc_num_neighbors=self.enc_output_num_neighbors, precision=prec,
                          cell_type=_lib.CELL[self.sequence_model_type], norm_type=self.norm)

    def _weight_struct(self):
        """Raw device pointers of every parameter (fsn_fast_weights, no packed bottleneck image)."""
        w = _lib.FastWeights()
        fb = self.mel_scale.fb
        if not fb.is_cuda:
            raise RuntimeError("fullsubnet_b200: call model.cuda() first - there is no CPU path.")
        w.mel_fb = fb.contiguous().data_ptr()
        w.enc1, w.enc2 = self.encoder[0].layer_struct(0), self.encoder[1].layer_struct(0)
        w.enc_fc_w, w.enc_fc_b = self.encoder[1].fc_ptrs()
        for l in range(self.bottleneck.num_layers):
            w.bn[l] = self.bottleneck.layer_struct(l)
        w.bn_fc_w, w.bn_fc_b = self.bottleneck.fc_ptrs()
        w.dec1, w.dec2 = self.decoder_lstm[0].layer_struct(0), self.decoder_lstm[1].layer_struct(0)
        w.dec_fc_w, w.dec_fc_b = self.decoder_lstm[1].fc_ptrs()
        w.bn_packed = None
        return w

    def _structs(self, device):
        prec = self._resolve_precision()
        d = self._desc(_lib.PREC[prec])
        w = self._weight_struct()
        if prec != "fp32":  # tile-ordered fp16 image of the bottleneck weights, rebuilt when a parameter changes
            key = (self.bottleneck.version_key(), str(device), prec)
            if self._packed is None or self._packed_key != key:
                lib = _lib.load()
                buf = torch.empty(lib.fsn_fast_packed_bytes(C.byref(d)), dtype=torch.uint8, device=device)
                _lib.check(lib.fsn_fast_pack_bn_weights(C.byref(d), C.byref(w), buf.data_ptr(), _lib.stream_ptr(device)))
                self._packed, self._packed_key = buf, key
            w.bn_packed = self._packed.data_ptr()
        return d, w

    def forward(self, mix_mag):
        """mix_mag [B,1,F,T] -> [B,2,F,T]  (fast_fullsubnet/model.py:143-202)."""
        assert mix_mag.dim() == 4
        batch_size, num_channels, num_freqs, num_frames = mix_mag.size()
        assert num_channels == 1, f"{self.__class__.__name__} takes a magnitude feature as the input."
        assert num_freqs == self.encoder_input_size
        x = _lib.require_cuda(mix_mag, "mix_mag")
        if self.training and self._records_grad():
            return TrainStep.apply(self, x, *self.parameters())
        lib = _lib.load()
        with torch.cuda.device(x.device):
            d, w = self._structs(x.device)
            n = _lib.check_workspace(lib.fsn_fast_workspace_bytes(C.byref(d), batch_size, num_frames))
            ws = torch.empty(n, dtype=torch.uint8, device=x.device)
            out = torch.empty(batch_size, 2, num_freqs, num_frames, dtype=torch.float32, device=x.device)
            _lib.check(lib.fsn_fast_model_forward(C.byref(d), C.byref(w), x.data_ptr(), batch_size, num_frames,
                                                  out.data_ptr(), ws.data_ptr(), n, _lib.stream_ptr(x.device)))
        return out
