"""Drop-in for recipes/dns_interspeech_2020/improved_fullsubnet/model.py:452-591 (class Model, BASELINE config 5).

Same constructor kwargs and ``state_dict`` keys (``fb_model.*``, ``sb_model.sb_models.{s}.*``);
``forward(y [B,L] | [B,1,L]) -> [B,1,L]`` (waveform in, enhanced waveform out) is one call into libfsn_b200
(``fsn_improved_forward``: STFT -> |X|^fdrc -> full band -> per-section sub bands -> element-wise mask -> iSTFT).  With
gradients enabled the output is differentiable like the reference module's: the forward keeps its activations
(``fsn_improved_train_forward``) and ``loss.backward()`` runs the iSTFT adjoint and back-propagation through time in the
library (``fsn_improved_train_backward``), so any loss on the enhanced waveform trains the model."""
from __future__ import annotations

import ctypes as C
import os

import torch
import torch.nn as nn

from .. import _lib
from ..model.base_model import BaseModel, TrainStep
from ..model.module.sequence_model import SequenceModel


class SubbandModel(nn.Module):
    """Parameter container with the reference's layout (model.py:250-318): one 2-layer stack per section."""

    def __init__(self, freq_cutoffs, sb_num_center_freqs, sb_num_neighbor_freqs, fb_num_center_freqs,
                 fb_num_neighbor_freqs, hidden_size, sequence_model, activate_function):
        super().__init__()
        assert len(freq_cutoffs) + 1 == len(sb_num_center_freqs) == len(sb_num_neighbor_freqs) \
            == len(fb_num_center_freqs) == len(fb_num_neighbor_freqs)
        self.hidden_size = hidden_size
        self.sb_models = nn.ModuleList([
            SequenceModel(input_size=(sb_num_center_freqs[s] + sb_num_neighbor_freqs[s] * 2)
                          + (fb_num_center_freqs[s] + fb_num_neighbor_freqs[s] * 2),
                          output_size=sb_num_center_freqs[s] * 2, hidden_size=hidden_size, num_layers=2,
                          bidirectional=False, sequence_model=sequence_model, output_activate_function=activate_function)
            for s in range(len(sb_num_center_freqs))])
        self.freq_cutoffs = list(freq_cutoffs)
        self.sb_num_center_freqs = list(sb_num_center_freqs)
        self.sb_num_neighbor_freqs = list(sb_num_neighbor_freqs)
        self.fb_num_center_freqs = list(fb_num_center_freqs)
        self.fb_num_neighbor_freqs = list(fb_num_neighbor_freqs)


class Model(BaseModel):
    # training step (wav in, wav out; upstream ships no trainer): fsn_improved_train_forward keeps the activations,
    # fsn_improved_train_backward runs the iSTFT adjoint and BPTT
    TRAIN_ENTRY_POINTS = ("fsn_improved_train_workspace_bytes", "fsn_improved_train_forward", "fsn_improved_train_backward")
    TRAIN_TF32_STACKS = ("fb_model", "sb_model")
    # waveform in, waveform out with the model's own STFT: the Inferencer calls enhance / enhance_pcm instead of computing
    # a magnitude spectrogram for it
    WAVEFORM_INPUT = True
    # fused wav -> wav call (enhance / enhance_pcm); its STFT geometry is in the descriptor
    ENHANCE_ENTRY_POINTS = ("fsn_improved_enhance_workspace_bytes", "fsn_improved_enhance")

    def __init__(self, n_fft=512, hop_length=128, win_length=512, fdrc=0.5, num_freqs=257, freq_cutoffs=[20, 80],
                 sb_num_center_freqs=[1, 4, 8], sb_num_neighbor_freqs=[15, 15, 15], fb_num_center_freqs=[1, 4, 8],
                 fb_num_neighbor_freqs=[15, 15, 15], fb_hidden_size=512, sb_hidden_size=384, sequence_model="LSTM",
                 fb_output_activate_function=False, sb_output_activate_function=False,
                 norm_type="offline_laplace_norm"):
        super().__init__()
        self.n_fft, self.hop_length, self.win_length, self.fdrc = n_fft, hop_length, win_length, fdrc
        self.num_freqs = num_freqs
        self.fb_model = SequenceModel(input_size=num_freqs - 1, output_size=num_freqs - 1, hidden_size=fb_hidden_size,
                                      num_layers=2, bidirectional=False, sequence_model=sequence_model,
                                      output_activate_function=fb_output_activate_function)
        self.sb_model = SubbandModel(freq_cutoffs, sb_num_center_freqs, sb_num_neighbor_freqs, fb_num_center_freqs,
                                     fb_num_neighbor_freqs, sb_hidden_size, sequence_model, sb_output_activate_function)
        if len(sb_num_center_freqs) > _lib.IMP_MAX_SECTIONS:
            raise NotImplementedError(f"libfsn_b200 builds at most {_lib.IMP_MAX_SECTIONS} sub-band sections")
        if norm_type != "offline_laplace_norm":
            # model.py:226-236 also offers cumulative_laplace_norm / offline_gaussian_norm
            raise NotImplementedError("libfsn_b200 builds offline_laplace_norm for improved_fullsubnet")
        self.norm_type = norm_type
        # arithmetic of the sub-band sections (98 % of the FLOPs):
        #   "fp32"     FMA kernels
        #   "tf32_tc"  wgmma tf32 GEMMs, fp32 accumulate, one launch per layer and step (waveform within 1e-4)
        #   "f16x3_tc" each section in one persistent wgmma launch, fp16 hi+lo split of weights and state: the fp32
        #              error class (sb_hidden in {128, 256, 384}); the full band on the compensated tensor-core layers
        #   "f16_tc"   the same with single fp16 / tf32 passes
        #   "auto"     tf32_tc when sb_hidden % 4 == 0, else fp32
        self.precision = os.environ.get("FSN_IMPROVED_PRECISION", "auto")
        self._packed = {}  # section -> (key, fsn_improved_pack_sb_weights image)
        # arithmetic of the training step's GEMMs: "fp32" (FMA) | "tf32_tc" (wgmma tf32 for the LSTM layers) | "auto" =
        # tf32_tc when fb_hidden_size and sb_hidden_size are multiples of 4
        self.train_precision = os.environ.get("FSN_TRAIN_PRECISION", "auto")

    def _resolve_precision(self) -> str:
        ok = self.sb_model.sb_models[0].hidden_size % 4 == 0
        if self.precision == "auto":
            return "tf32_tc" if ok else "fp32"
        if self.precision not in ("fp32", "tf32_tc", "f16x3_tc", "f16_tc"):
            raise ValueError("precision must be 'fp32', 'tf32_tc', 'f16x3_tc', 'f16_tc' or 'auto'")
        return self.precision

    def _structs(self, device=None):
        d, w = self._desc(self._resolve_precision()), self._weights()
        if d.precision in (_lib.PREC["f16x3_tc"], _lib.PREC["f16_tc"]):
            for s in range(d.num_sections):
                w.sb_packed[s] = self._packed_section(d, w, s, device)
        return d, w

    def _packed_section(self, desc, w, s, device):
        """fp16 image of section s's recurrent weights (fsn_improved_pack_sb_weights), rebuilt when any of its parameters
        changes."""
        key = (self.sb_model.sb_models[s].version_key(), str(device), int(desc.precision), int(desc.sb_hidden))
        hit = self._packed.get(s)
        if hit is None or hit[0] != key:
            lib = _lib.load()
            n = _lib.check_workspace(lib.fsn_improved_packed_bytes(C.byref(desc), s))
            buf = torch.empty(n, dtype=torch.uint8, device=device)
            _lib.check(lib.fsn_improved_pack_sb_weights(C.byref(desc), C.byref(w), s, buf.data_ptr(),
                                                        _lib.stream_ptr(device)))
            hit = self._packed[s] = (key, buf)
        return hit[1].data_ptr()

    def _enhance_args(self, device):
        self._check_sections()
        d, w = self._structs(device)
        return d, (C.byref(w),)

    def _desc(self, precision: str) -> "_lib.ImprovedDesc":
        sb = self.sb_model
        d = _lib.ImprovedDesc(n_fft=self.n_fft, hop_length=self.hop_length, win_length=self.win_length,
                              num_freqs=self.num_freqs, fdrc=float(self.fdrc), num_sections=len(sb.sb_models),
                              fb_hidden=self.fb_model.hidden_size, sb_hidden=sb.sb_models[0].hidden_size,
                              fb_activation=_lib.ACT[self.fb_model.output_activate_function],
                              sb_activation=_lib.ACT[sb.sb_models[0].output_activate_function],
                              precision=_lib.PREC[precision],
                              cell_type=_lib.CELL[self.fb_model.cell])
        for s in range(len(sb.sb_models)):
            if s < len(sb.freq_cutoffs):
                d.freq_cutoffs[s] = sb.freq_cutoffs[s]
            d.sb_num_center[s], d.sb_num_neighbor[s] = sb.sb_num_center_freqs[s], sb.sb_num_neighbor_freqs[s]
            d.fb_num_center[s], d.fb_num_neighbor[s] = sb.fb_num_center_freqs[s], sb.fb_num_neighbor_freqs[s]
        return d

    def _weights(self) -> "_lib.ImprovedWeights":
        sb = self.sb_model
        w = _lib.ImprovedWeights()
        w.fb = self.fb_model.weight_struct()
        for s, m in enumerate(sb.sb_models):
            w.sb[s] = m.weight_struct()
        return w

    def _train_desc(self):
        return self._desc(self._resolve_train_precision())

    def _train_weights(self):
        return (C.byref(self._weights()),)

    def _train_grads(self, grads):
        g = _lib.ImprovedGrads()
        g.fb = SequenceModel.seq_grads_struct(grads, "fb_model.")
        for s in range(len(self.sb_model.sb_models)):
            g.sb[s] = SequenceModel.seq_grads_struct(grads, f"sb_model.sb_models.{s}.")
        return (C.byref(g),)

    def _train_io(self, x, desc):
        B, L = x.shape
        return (B, L), (B, 1, L)

    def _check_sections(self):
        sb = self.sb_model
        bounds = [0] + sb.freq_cutoffs + [self.num_freqs - 1]
        for s in range(len(sb.sb_models)):  # model.py:341-345 (both the noisy and the full-band unfold)
            if (bounds[s + 1] - bounds[s]) % sb.sb_num_center_freqs[s] or \
                    (bounds[s + 1] - bounds[s]) % sb.fb_num_center_freqs[s]:
                raise ValueError(
                    "The number of center frequencies should be divisible by the subband freqency interval. "
                    f"Got {sb.sb_num_center_freqs[s]} and {bounds[s + 1] - bounds[s]}.")

    def forward(self, y, return_crm: bool = False):
        """y [B,L] or [B,1,L] -> enhanced [B,1,L]  (model.py:541-591).  ``return_crm`` additionally returns the
        [B,2,F,T] mask (Nyquist row zero) - an extension used by the parity tests."""
        ndim = y.dim()
        assert ndim in (2, 3), "Input must be 2D (B, T) or 3D tensor (B, 1, T)"
        if ndim == 3:
            assert y.size(1) == 1, "Input must be 2D (B, T) or 3D tensor (B, 1, T)"
            y = y.squeeze(1)
        x = _lib.require_cuda(y, "y")
        B, L = x.shape
        self._check_sections()
        if self._records_grad():
            if return_crm:
                raise NotImplementedError("fullsubnet_b200: return_crm is built for inference only (use torch.no_grad())")
            if y.requires_grad:  # the library computes no input gradient; returning None would silently zero it
                raise NotImplementedError("fullsubnet_b200: improved_fullsubnet training computes no gradient for the input")
            if self.fb_model.cell != "LSTM":
                raise NotImplementedError("fullsubnet_b200: improved_fullsubnet training is built for LSTM only")
            return TrainStep.apply(self, x, *self.parameters())
        lib = _lib.load()
        with torch.cuda.device(x.device):
            d, w = self._structs(x.device)
            n = _lib.check_workspace(lib.fsn_improved_workspace_bytes(C.byref(d), B, L))
            ws = torch.empty(n, dtype=torch.uint8, device=x.device)
            out = torch.empty(B, 1, L, dtype=torch.float32, device=x.device)
            crm = torch.empty(B, 2, self.num_freqs, 1 + L // self.hop_length, dtype=torch.float32,
                              device=x.device) if return_crm else None
            _lib.check(lib.fsn_improved_forward(C.byref(d), C.byref(w), x.data_ptr(), B, L, out.data_ptr(),
                                                _lib.ptr(crm), ws.data_ptr(), n, _lib.stream_ptr(x.device)))
        return (out, crm) if return_crm else out

    @torch.no_grad()
    def enhance(self, y, lengths=None, return_crm: bool = False):
        """y [B,L] -> enhanced [B,L] in one library call (fsn_improved_enhance); with ``lengths=None`` the bits of
        ``forward``.  ``lengths`` (B ints, or a CPU integer tensor; max must be L): clips of different lengths in one
        call.  Clip b is ``y[b, :lengths[b]]``; the rest of the row is never read.  Its outputs equal the call on that
        clip alone, bit for bit; ``enhanced[b, lengths[b]:]`` and the cRM frames ``t >= 1 + lengths[b] // hop_length``
        are 0.  ``return_crm`` additionally returns the [B,2,F,T_max] mask."""
        assert y.dim() == 2, "y must be [B, L]"
        out, crm, _ = self._enhance_call(y, lengths, return_crm, None)
        return (out, crm) if return_crm else out

    @torch.no_grad()
    def enhance_pcm(self, y, gain=0.8 * 32767.0, lengths=None):
        """``enhance`` plus the int16 scaling of the reference host loop (audio_zen/inferencer/base_inferencer.py:
        181-182) in the same call, the per-clip max|y| reduced in the iSTFT epilogue: y [B,L] -> (enhanced float32
        [B,L], pcm int16 [B,L]).  ``lengths``: as in ``enhance``; each clip is scaled by the peak of its own samples
        and its pcm row is 0 past them."""
        assert y.dim() == 2, "y must be [B, L]"
        out, _, pcm = self._enhance_call(y, lengths, False, gain)
        return out, pcm
