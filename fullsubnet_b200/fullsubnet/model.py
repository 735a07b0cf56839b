"""Drop-in for recipes/dns_interspeech_2020/fullsubnet/model.py:9-136 (class Model).

Same constructor kwargs, same 20 ``state_dict`` entries, same ``forward`` contract
(``noisy_mag [B,1,F,T] -> cRM [B,2,F',T]``, incl. drop_band when B > 1), but the whole forward
is one call into libfsn_b200 (``fsn_model_forward``): look-ahead pad, both laplace norms (second
in closed form), full-band 2xLSTM + Linear + ReLU, sub-band unfold (never materialised),
sub-band 2xLSTM + Linear, output re-layout.  ``enhance`` / ``enhance_pcm`` run the wav -> wav path of
``Inferencer.full_band_crm_mask`` for a batch of clips, of equal or different lengths, in one call (``fsn_enhance``)."""
from __future__ import annotations

import ctypes as C
import os

import torch

from .. import _lib
from ..model.base_model import BaseModel, SpectrogramEnhance, TrainStep
from ..model.module.sequence_model import SequenceModel


class Model(SpectrogramEnhance, BaseModel):
    # fused wav -> wav call (enhance / enhance_pcm): stft -> model -> mask + istft [-> int16] in one library call
    ENHANCE_ENTRY_POINTS = ("fsn_enhance_workspace_bytes", "fsn_enhance")
    # training step (trainer.py:56-63): fsn_train_forward keeps the activations, fsn_train_backward runs BPTT
    TRAIN_ENTRY_POINTS = ("fsn_train_workspace_bytes", "fsn_train_forward", "fsn_train_backward")
    TRAIN_TF32_STACKS = ("fb_model", "sb_model")
    # chunked streaming (fullsubnet_b200.stream.Streamer, precision="fp32" with cumulative_laplace_norm or
    # forgetting_norm): state / workspace queries, delay, step
    STREAM_ENTRY_POINTS = ("fsn_stream_state_bytes", "fsn_stream_workspace_bytes", "fsn_stream_delay", "fsn_stream_step")
    # the same on the fp16 tensor cores (Streamer(tensor_cores=True), the model's f16x3_tc / f16_tc precision)
    STREAM_TC_ENTRY_POINTS = ("fsn_stream_tc_state_bytes", "fsn_stream_tc_workspace_bytes", "fsn_stream_tc_delay",
                              "fsn_stream_tc_step")

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

    def _stream_desc(self):
        """Descriptor of the streaming calls: the fp32 kernels only, so an explicit precision="fp32" (under "auto" the
        whole-clip call runs the sub band on the tensor cores, which a stream could not match)."""
        if self.precision != "fp32":
            raise NotImplementedError(f"fullsubnet_b200: fullsubnet streaming is built for precision=\"fp32\" "
                                      f"(this model has precision={self.precision!r})")
        return self._desc("fp32", int(self.num_groups_in_drop_band))

    def _stream_weights(self):
        return C.byref(self.fb_model.weight_struct()), C.byref(self.sb_model.weight_struct())

    def _stream_tc_desc(self):
        """Descriptor of the tensor-core streaming calls: the model's resolved precision, which must be f16x3_tc or
        f16_tc (so "auto" streams the bits of the whole-clip call wherever that call runs the tensor cores)."""
        prec = self._resolve_precision()
        if prec == "fp32":
            raise NotImplementedError("fullsubnet_b200: this model resolves to precision=\"fp32\"; stream it with the "
                                      "default Streamer(model, slots) (tensor_cores=False)")
        return self._desc(prec, 1)

    def _stream_tc_weights(self):
        desc = self._stream_tc_desc()
        device = next(self.parameters()).device
        fb_w, sb_w = self.fb_model.weight_struct(), self.sb_model.weight_struct()
        packed = self._packed_sb(desc, sb_w, device)
        return C.byref(fb_w), C.byref(sb_w), _lib.ptr(packed)

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

    def _enhance_args(self, device):
        desc, fb_w, sb_w, packed = self._prepare(device, 1)
        return desc, (C.byref(fb_w), C.byref(sb_w), _lib.ptr(packed))

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
            ws_bytes = _lib.check_workspace(lib.fsn_model_workspace_bytes(C.byref(desc), batch_size, num_frames))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
            out = torch.empty(batch_size, 2, f_out, num_frames, dtype=torch.float32, device=device)
            _lib.check(lib.fsn_model_forward(C.byref(desc), C.byref(fb_w), C.byref(sb_w), _lib.ptr(packed),
                                             x.data_ptr(), batch_size, num_frames, out.data_ptr(), ws.data_ptr(),
                                             ws_bytes, _lib.stream_ptr(device)))
        return out
