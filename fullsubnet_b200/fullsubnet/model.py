"""Drop-in for recipes/dns_interspeech_2020/fullsubnet/model.py:9-136 (class Model).

Same constructor kwargs, same 20 ``state_dict`` entries, same ``forward`` contract
(``noisy_mag [B,1,F,T] -> cRM [B,2,F',T]``, incl. drop_band when B > 1), but the whole forward
is one call into libfsn_b200 (``fsn_model_forward``): look-ahead pad, both laplace norms (second
in closed form), full-band 2xLSTM + Linear + ReLU, sub-band unfold (never materialised),
sub-band 2xLSTM + Linear, output re-layout."""
from __future__ import annotations

import ctypes as C
import os

import torch

from .. import _lib
from ..model.base_model import BaseModel, TrainStep
from ..model.module.sequence_model import SequenceModel


class Model(BaseModel):
    # training step (trainer.py:56-63): fsn_train_forward keeps the activations, fsn_train_backward runs BPTT
    TRAIN_ENTRY_POINTS = ("fsn_train_workspace_bytes", "fsn_train_forward", "fsn_train_backward")
    TRAIN_TF32_STACKS = ("fb_model", "sb_model")

    def __init__(self, num_freqs, look_ahead, sequence_model, fb_num_neighbors, sb_num_neighbors,
                 fb_output_activate_function, sb_output_activate_function, fb_model_hidden_size,
                 sb_model_hidden_size, norm_type="offline_laplace_norm", num_groups_in_drop_band=2,
                 weight_init=True, precision=None):
        super().__init__()
        assert sequence_model in ("GRU", "LSTM"), f"{self.__class__.__name__} only support GRU and LSTM."
        self.fb_model = SequenceModel(
            input_size=num_freqs, output_size=num_freqs, hidden_size=fb_model_hidden_size, num_layers=2,
            bidirectional=False, sequence_model=sequence_model, output_activate_function=fb_output_activate_function)
        self.sb_model = SequenceModel(
            input_size=(sb_num_neighbors * 2 + 1) + (fb_num_neighbors * 2 + 1), output_size=2,
            hidden_size=sb_model_hidden_size, num_layers=2, bidirectional=False, sequence_model=sequence_model,
            output_activate_function=sb_output_activate_function)
        self.sequence_model_type = sequence_model  # "LSTM" (every shipped recipe) | "GRU" (fp32 inference kernels)
        self.num_freqs = num_freqs
        self.sb_num_neighbors = sb_num_neighbors
        self.fb_num_neighbors = fb_num_neighbors
        self.look_ahead = look_ahead
        self.norm_type = norm_type
        self.norm = self.norm_wrapper(norm_type)
        self.num_groups_in_drop_band = num_groups_in_drop_band
        # arithmetic of the sub-band stack (99 % of the FLOPs):
        #   "fp32"     fp32 FMA kernels
        #   "f16x3_tc" wgmma, fp16 hi+lo split of weights and state, 3 MMAs per product: the fp32 error class
        #              (cRM ~1e-6 rel, waveform <= 1e-4 abs even where decompress_cIRM amplifies x100)
        #   "f16_tc"   wgmma, single fp16 pass: about 2x faster, cRM within 1e-3 rel; opt-in
        #   "auto"     f16x3_tc when the shape allows, else fp32 -- the default never trades the reference's accuracy
        self.precision = precision or os.environ.get("FSN_PRECISION", "auto")
        # arithmetic of the training step's GEMMs: "fp32" (FMA) or "tf32_tc" (wgmma tf32); the reference
        # trains under fp16 autocast (trainer.py:56), so both are at least its precision
        self.train_precision = os.environ.get("FSN_TRAIN_PRECISION", "auto")
        self._packed = None
        self._packed_key = None
        if weight_init:
            self.apply(self.weight_init)

    # ---------------------------------------------------------------- C-ABI plumbing
    def _resolve_precision(self) -> str:
        if self.precision != "auto":
            if self.precision not in ("fp32", "f16_tc", "f16x3_tc"):
                raise ValueError("precision must be 'fp32', 'f16x3_tc', 'f16_tc' or 'auto'")
            return self.precision
        if self.sequence_model_type != "LSTM":
            return "fp32"
        d = self._desc("f16x3_tc", 1)
        return "f16x3_tc" if _lib.load().fsn_sb_packed_bytes(C.byref(d)) > 0 else "fp32"

    def _train_desc(self):
        return self._desc(self._resolve_train_precision(), int(self.num_groups_in_drop_band))

    def _train_weights(self):
        return C.byref(self.fb_model.weight_struct()), C.byref(self.sb_model.weight_struct())

    def _train_grads(self, grads):
        return (C.byref(SequenceModel.seq_grads_struct(grads, "fb_model.")),
                C.byref(SequenceModel.seq_grads_struct(grads, "sb_model.")))

    def _train_out_shape(self, desc, B, F, T):
        G = desc.num_groups_in_drop_band if B > 1 and desc.num_groups_in_drop_band > 1 else 1
        return (B, 2, F // G, T)

    def _desc(self, precision: str, num_groups: int) -> "_lib.ModelDesc":
        return _lib.ModelDesc(
            num_freqs=self.num_freqs, look_ahead=self.look_ahead, fb_num_neighbors=self.fb_num_neighbors,
            sb_num_neighbors=self.sb_num_neighbors, fb_hidden=self.fb_model.hidden_size,
            sb_hidden=self.sb_model.hidden_size, fb_activation=_lib.ACT[self.fb_model.output_activate_function],
            sb_activation=_lib.ACT[self.sb_model.output_activate_function], norm_type=self.norm,
            num_groups_in_drop_band=num_groups, precision=_lib.PREC[precision], cell_type=_lib.CELL[self.sequence_model_type])

    def _packed_sb(self, desc, sb_w, device):
        """Tile-ordered fp16 image of the sub-band weights, rebuilt when any parameter changes."""
        key = (self.sb_model.version_key(), str(device), int(desc.precision))
        if self._packed is None or self._packed_key != key:
            lib = _lib.load()
            n = lib.fsn_sb_packed_bytes(C.byref(desc))
            buf = torch.empty(n, dtype=torch.uint8, device=device)
            _lib.check(lib.fsn_pack_sb_weights(C.byref(desc), C.byref(sb_w), buf.data_ptr(), _lib.stream_ptr(device)))
            self._packed, self._packed_key = buf, key
        return self._packed

    def _prepare(self, device, num_groups):
        prec = self._resolve_precision()
        desc = self._desc(prec, num_groups)
        fb_w, sb_w = self.fb_model.weight_struct(), self.sb_model.weight_struct()
        packed = self._packed_sb(desc, sb_w, device) if prec in ("f16_tc", "f16x3_tc") else None
        return desc, fb_w, sb_w, packed

    # ---------------------------------------------------------------- reference API
    def forward(self, noisy_mag):
        """noisy_mag [B,1,F,T] -> [B,2,F,T]  (or [B,2,F//G,T], batch order 0,2,4,..,1,3,5,.. when B>1, G>1)."""
        assert noisy_mag.dim() == 4
        batch_size, num_channels, num_freqs, num_frames = noisy_mag.size()
        assert num_channels == 1, f"{self.__class__.__name__} takes the mag feature as inputs."
        assert num_freqs == self.num_freqs, f"num_freqs {num_freqs} != {self.num_freqs}"
        x = _lib.require_cuda(noisy_mag, "noisy_mag")
        if self._records_grad():
            return TrainStep.apply(self, x, *self.parameters())
        device = x.device
        lib = _lib.load()
        with torch.cuda.device(device):
            desc, fb_w, sb_w, packed = self._prepare(device, int(self.num_groups_in_drop_band))
            G = desc.num_groups_in_drop_band if batch_size > 1 and desc.num_groups_in_drop_band > 1 else 1
            f_out = num_freqs // G if G > 1 else num_freqs
            ws_bytes = lib.fsn_model_workspace_bytes(C.byref(desc), batch_size, num_frames)
            if ws_bytes == 0:
                _lib.check_workspace(ws_bytes)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
            out = torch.empty(batch_size, 2, f_out, num_frames, dtype=torch.float32, device=device)
            _lib.check(lib.fsn_model_forward(C.byref(desc), C.byref(fb_w), C.byref(sb_w), _lib.ptr(packed),
                                             x.data_ptr(), batch_size, num_frames, out.data_ptr(), ws.data_ptr(),
                                             ws_bytes, _lib.stream_ptr(device)))
        return out

    @staticmethod
    def _lengths_table(lengths, B, L):
        """Per-clip lengths (sequence of B ints or a CPU integer tensor) -> contiguous int32 host array."""
        return _lib.lengths_table(lengths, B, L)

    def _enhance_varlen(self, x, lens, n_fft, hop_length, win_length, crm, pcm, gain):
        """One fsn_enhance_varlen call: clip b is row b's first lens[b] samples; out [B,L] is 0 past them."""
        B, L = x.shape
        device = x.device
        lib = _lib.load()
        with torch.cuda.device(device):
            desc, fb_w, sb_w, packed = self._prepare(device, 1)
            ws_bytes = _lib.check_workspace(lib.fsn_enhance_varlen_workspace_bytes(C.byref(desc), B, L, n_fft, hop_length))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
            out = torch.empty(B, L, dtype=torch.float32, device=device)
            _lib.check(lib.fsn_enhance_varlen(C.byref(desc), C.byref(fb_w), C.byref(sb_w), _lib.ptr(packed), x.data_ptr(),
                                              lens.ctypes.data, B, L, n_fft, hop_length, win_length, out.data_ptr(),
                                              _lib.ptr(crm), _lib.ptr(pcm), float(gain), ws.data_ptr(), ws_bytes,
                                              _lib.stream_ptr(device)))
        return out

    @torch.no_grad()
    def enhance(self, noisy, n_fft=512, hop_length=256, win_length=512, return_crm=False, lengths=None):
        """Fused wav -> wav path of Inferencer.full_band_crm_mask (recipes/.../inferencer.py:130-145),
        batched over independent clips: noisy [B,L] -> enhanced [B,L].

        ``lengths`` (B ints, or a CPU integer tensor; max must be L): clips of different lengths in one call
        (fsn_enhance_varlen).  Clip b is ``noisy[b, :lengths[b]]``; the rest of the row is never read.  Its outputs
        equal the call on that clip alone, bit for bit; ``enhanced[b, lengths[b]:]`` and the cRM frames
        ``t >= 1 + lengths[b] // hop_length`` are 0."""
        assert noisy.dim() == 2, "noisy must be [B, L]"
        lens = None if lengths is None else self._lengths_table(lengths, *noisy.shape)
        x = _lib.require_cuda(noisy, "noisy")
        B, L = x.shape
        device = x.device
        if lens is not None:
            crm = torch.empty(B, 2, n_fft // 2 + 1, 1 + L // hop_length, dtype=torch.float32,
                              device=device) if return_crm else None
            out = self._enhance_varlen(x, lens, n_fft, hop_length, win_length, crm, None, 0.0)
            return (out, crm) if return_crm else out
        lib = _lib.load()
        with torch.cuda.device(device):
            desc, fb_w, sb_w, packed = self._prepare(device, 1)
            ws_bytes = lib.fsn_enhance_workspace_bytes(C.byref(desc), B, L, n_fft, hop_length)
            if ws_bytes == 0:
                _lib.check_workspace(ws_bytes)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
            out = torch.empty(B, L, dtype=torch.float32, device=device)
            crm = torch.empty(B, 2, n_fft // 2 + 1, 1 + L // hop_length, dtype=torch.float32,
                              device=device) if return_crm else None
            _lib.check(lib.fsn_enhance(C.byref(desc), C.byref(fb_w), C.byref(sb_w), _lib.ptr(packed), x.data_ptr(),
                                       B, L, n_fft, hop_length, win_length, out.data_ptr(), _lib.ptr(crm),
                                       ws.data_ptr(), ws_bytes, _lib.stream_ptr(device)))
        return (out, crm) if return_crm else out

    @torch.no_grad()
    def enhance_pcm(self, noisy, n_fft=512, hop_length=256, win_length=512, gain=0.8 * 32767.0, lengths=None):
        """``enhance`` plus the int16 scaling of the reference host loop (audio_zen/inferencer/base_inferencer.py:
        181-182) in the same library call (fsn_enhance_pcm: per-clip max|y| reduced in the iSTFT epilogue):
        noisy [B,L] -> (enhanced float32 [B,L], pcm int16 [B,L]).  ``lengths``: as in ``enhance``; each clip is
        scaled by the peak of its own samples and its pcm row is 0 past them."""
        assert noisy.dim() == 2, "noisy must be [B, L]"
        lens = None if lengths is None else self._lengths_table(lengths, *noisy.shape)
        x = _lib.require_cuda(noisy, "noisy")
        B, L = x.shape
        device = x.device
        if lens is not None:
            pcm = torch.empty(B, L, dtype=torch.int16, device=device)
            return self._enhance_varlen(x, lens, n_fft, hop_length, win_length, None, pcm, gain), pcm
        lib = _lib.load()
        with torch.cuda.device(device):
            desc, fb_w, sb_w, packed = self._prepare(device, 1)
            ws_bytes = lib.fsn_enhance_workspace_bytes(C.byref(desc), B, L, n_fft, hop_length)
            if ws_bytes == 0:
                _lib.check_workspace(ws_bytes)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
            out = torch.empty(B, L, dtype=torch.float32, device=device)
            pcm = torch.empty(B, L, dtype=torch.int16, device=device)
            _lib.check(lib.fsn_enhance_pcm(C.byref(desc), C.byref(fb_w), C.byref(sb_w), _lib.ptr(packed), x.data_ptr(),
                                           B, L, n_fft, hop_length, win_length, out.data_ptr(), pcm.data_ptr(),
                                           float(gain), ws.data_ptr(), ws_bytes, _lib.stream_ptr(device)))
        return out, pcm
