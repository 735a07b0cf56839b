"""Drop-in for the hot-path mode of recipes/dns_interspeech_2020/inferencer.py
(``Inferencer.full_band_crm_mask`` :130-145) and the parts of
audio_zen/inferencer/base_inferencer.py it relies on (attribute names ``model``, ``device``,
``torch_stft``, ``torch_istft``; ``_load_model`` :144-161).  Dataset / wav-file handling
(librosa, soundfile) is outside the hot path (SURVEY section 2) and not rebuilt here: construct
with a model, or with the reference's (config, checkpoint_path) pair.  The host loop around the path (SURVEY 8f
rank 2) is here in batched form: ``enhance_files`` (wav load -> grouped batches -> fused enhance + int16 -> wav write)."""
from __future__ import annotations

from functools import partial
from typing import Optional

import numpy as np
import torch

from .acoustics.feature import istft, stft
from .acoustics.mask import decompress_cIRM
from .utils import initialize_module, prepare_device, read_wav


def plan_batches(lengths, batch_size: int, max_padding: float = 0.0):
    """Batches of clip indices for the file loop.  ``max_padding == 0``: clips of exactly equal length, at most
    ``batch_size`` per batch (shortest length first, file order within a length).  ``max_padding > 0``: the clips sorted
    by length are cut into consecutive runs of at most ``batch_size`` clips whose padding -- B * L_max minus the samples
    of the B clips -- stays within ``max_padding * B * L_max``; one such batch is one library call with per-clip
    lengths."""
    if batch_size < 1:
        raise ValueError("batch_size must be >= 1")
    if not 0.0 <= max_padding < 1.0:
        raise ValueError("max_padding must be in [0, 1)")
    lens = [int(v) for v in lengths]
    order = sorted(range(len(lens)), key=lambda i: (lens[i], i))
    batches, cur, total = [], [], 0
    for i in order:
        L = lens[i]  # the longest of cur + [i]: ascending order
        n = len(cur) + 1
        fits = len(cur) < batch_size and (n * L - (total + L) <= max_padding * n * L if max_padding > 0 else
                                          (not cur or lens[cur[0]] == L))
        if cur and not fits:
            batches.append(cur)
            cur, total = [], 0
        cur.append(i)
        total += L
    if cur:
        batches.append(cur)
    return batches


def takes_waveform(model) -> bool:
    """Whether ``model`` maps waveforms to waveforms with its own STFT (improved_fullsubnet) instead of taking the
    Inferencer's magnitude spectrogram."""
    return bool(getattr(type(model), "WAVEFORM_INPUT", False))


def has_fused_call(model) -> bool:
    """Whether ``model`` runs wav -> wav (STFT, model, mask + iSTFT, int16) in one library call with per-clip lengths
    (``enhance`` / ``enhance_pcm``): the models that set ENHANCE_ENTRY_POINTS."""
    return bool(getattr(type(model), "ENHANCE_ENTRY_POINTS", ()))


class Inferencer:
    def __init__(self, config: Optional[dict] = None, checkpoint_path=None, output_dir=None, model=None,
                 device=None):
        self.device = torch.device(device) if device is not None else prepare_device(torch.cuda.device_count())
        if model is not None:
            self.model = model.to(self.device).eval()
        else:
            self.model, self.epoch = self._load_model(config["model"], checkpoint_path, self.device)
        acoustics = (config or {}).get("acoustics")
        if takes_waveform(self.model):
            # the model computes its own STFT: n_fft / hop / window come from it, and a config must agree with it
            own = {"n_fft": self.model.n_fft, "hop_length": self.model.hop_length, "win_length": self.model.win_length}
            bad = {k: acoustics[k] for k in own if acoustics is not None and k in acoustics and acoustics[k] != own[k]}
            if bad:
                raise ValueError(f"acoustics {bad} disagree with the model's own STFT {own}")
            acoustics = dict(acoustics or {"sr": 16000}, **own)
        elif acoustics is None:
            acoustics = {"n_fft": 512, "hop_length": 256, "win_length": 512, "sr": 16000}
        self.acoustic_config = acoustics
        self.n_fft, self.hop_length = acoustics["n_fft"], acoustics["hop_length"]
        self.win_length, self.sr = acoustics["win_length"], acoustics.get("sr", 16000)
        self.torch_stft = partial(stft, n_fft=self.n_fft, hop_length=self.hop_length, win_length=self.win_length)
        self.torch_istft = partial(istft, n_fft=self.n_fft, hop_length=self.hop_length, win_length=self.win_length)
        self.inference_config = (config or {}).get("inferencer", {"type": "full_band_crm_mask", "args": {}})
        self.config = config

    @staticmethod
    def _load_model(model_config, checkpoint_path, device):
        """base_inferencer.py:144-161 (strict load, DDP 'module.' prefix stripped)."""
        model = initialize_module(model_config["path"], args=model_config["args"], initialize=True)
        ckpt = torch.load(checkpoint_path, map_location="cpu")
        sd = {k.replace("module.", ""): v for k, v in ckpt["model"].items()}
        model.load_state_dict(sd)
        model.to(device)
        model.eval()
        return model, ckpt["epoch"]

    @torch.no_grad()
    def full_band_crm_mask(self, noisy, inference_args=None):
        """inferencer.py:130-145, op by op through the drop-in functions: noisy [1,L] -> np.float32 [L].  A model that
        takes waveforms (improved_fullsubnet) is the whole path: its enhanced waveform."""
        if takes_waveform(self.model):
            return self.model(noisy.reshape(1, -1)).detach().reshape(-1).cpu().numpy()
        noisy_mag, _, noisy_real, noisy_imag = self.torch_stft(noisy)
        noisy_mag = noisy_mag.unsqueeze(1)
        pred_crm = self.model(noisy_mag)
        pred_crm = pred_crm.permute(0, 2, 3, 1)
        pred_crm = decompress_cIRM(pred_crm)
        enhanced_real = pred_crm[..., 0] * noisy_real - pred_crm[..., 1] * noisy_imag
        enhanced_imag = pred_crm[..., 1] * noisy_real + pred_crm[..., 0] * noisy_imag
        enhanced = self.torch_istft((enhanced_real, enhanced_imag), length=noisy.size(-1), input_type="real_imag")
        enhanced = enhanced.detach().squeeze(0).cpu().numpy()
        return enhanced

    def supports_lengths(self) -> bool:
        """Whether clips of different lengths can share one call: improved_fullsubnet (every n_fft it accepts), and
        fullsubnet and fullband_baseline with a power-of-two n_fft."""
        if takes_waveform(self.model):
            return True
        return has_fused_call(self.model) and self.n_fft & (self.n_fft - 1) == 0

    def _stft_args(self) -> tuple:
        """The STFT geometry a fused call takes: none for a model with its own (improved_fullsubnet)."""
        return () if takes_waveform(self.model) else (self.n_fft, self.hop_length, self.win_length)

    def _check_lengths(self, lengths) -> None:
        if lengths is not None and not has_fused_call(self.model):
            raise NotImplementedError(f"{type(self.model).__module__}: per-clip lengths are built for fullsubnet, "
                                      "improved_fullsubnet and fullband_baseline only")

    @torch.no_grad()
    def enhance_batch(self, noisy: torch.Tensor, lengths=None, return_crm: bool = False):
        """The same path for B independent clips in ONE library call (the model's fused call): pinned/host or device
        ``noisy`` [B,L] -> device tensor [B,L].  Equivalent to looping full_band_crm_mask over the clips.
        ``lengths`` (models with a fused call): clip b is ``noisy[b, :lengths[b]]``, its row 0 past it.
        ``return_crm``: (enhanced, the model output [B,2,F,T] the mask was built from)."""
        self._check_lengths(lengths)
        x = noisy.to(self.device, non_blocking=True)
        if has_fused_call(self.model):
            return self.model.enhance(x, *self._stft_args(), lengths=lengths, return_crm=return_crm)
        # other models (fast_fullsubnet): same flow, three library calls (stft -> model -> mask + istft)
        import ctypes as C  # noqa: F401
        from . import _lib
        B, L = x.shape
        F, T = self.n_fft // 2 + 1, 1 + L // self.hop_length
        buf = torch.empty(3, B, F, T, dtype=torch.float32, device=x.device)
        out = torch.empty(B, L, dtype=torch.float32, device=x.device)
        lib = _lib.load()
        with torch.cuda.device(x.device):
            st = _lib.stream_ptr(x.device)
            x = _lib.require_cuda(x, "noisy")
            _lib.check(lib.fsn_stft(x.data_ptr(), B, L, self.n_fft, self.hop_length, self.win_length, buf[0].data_ptr(),
                                    None, buf[1].data_ptr(), buf[2].data_ptr(), None, 0, st))
            crm = self.model(buf[0].unsqueeze(1)).contiguous()
            _lib.check(lib.fsn_istft(buf[1].data_ptr(), buf[2].data_ptr(), 1, crm.data_ptr(), B, T, self.n_fft,
                                     self.hop_length, self.win_length, L, out.data_ptr(), st))
        return (out, crm) if return_crm else out

    @torch.no_grad()
    def enhance_to_pcm(self, noisy: torch.Tensor, lengths=None) -> torch.Tensor:
        """enhance_batch + the int16 scaling of base_inferencer.py:181-182 on the device: noisy [B,L] -> int16 [B,L]
        (what the reference hands to ``sf.write``); only B*L*2 bytes come back to the host.  ``lengths``: as in
        ``enhance_batch``; each clip is scaled by its own peak."""
        from . import _lib
        self._check_lengths(lengths)
        if has_fused_call(self.model):  # peak in the iSTFT epilogue, one scaling pass
            x = noisy.to(self.device, non_blocking=True)
            return self.model.enhance_pcm(x, *self._stft_args(), gain=0.8 * float(np.iinfo(np.int16).max),
                                          lengths=lengths)[1]
        # models without a fused call (fast_fullsubnet): enhance_batch, then the two-pass int16 kernel
        enhanced = self.enhance_batch(noisy)
        B, L = enhanced.shape
        pcm = torch.empty(B, L, dtype=torch.int16, device=enhanced.device)
        with torch.cuda.device(enhanced.device):
            _lib.check(_lib.load().fsn_peak_normalize_int16(enhanced.data_ptr(), B, L, 0.8 * float(np.iinfo(np.int16).max),
                                                          pcm.data_ptr(), _lib.stream_ptr(enhanced.device)))
        return pcm

    @staticmethod
    def write_wav(path, pcm, sr: int = 16000) -> None:
        """16-bit mono PCM file with the standard library (the reference uses soundfile, base_inferencer.py:183-187)."""
        import wave
        data = pcm.cpu().numpy() if isinstance(pcm, torch.Tensor) else np.asarray(pcm)
        with wave.open(str(path), "wb") as f:
            f.setnchannels(1)
            f.setsampwidth(2)
            f.setframerate(int(sr))
            f.writeframes(np.ascontiguousarray(data, dtype="<i2").tobytes())

    # ------------------------------------------------------------------ wav files (base_inferencer.py:163-195, dataset_inference.py:39-43)
    @staticmethod
    def mono(wav: np.ndarray) -> np.ndarray:
        """float32 [C, N] -> [N]: the channels averaged like librosa.load(mono=True)."""
        return wav[0] if len(wav) == 1 else np.ascontiguousarray(wav.T).mean(axis=1).astype(np.float32)

    @staticmethod
    def load_wav(path, sr: int = 16000) -> np.ndarray:
        """Mono float32 waveform at ``sr`` from a PCM wav file (8/16/24/32-bit; channels averaged like librosa).  The reference calls
        ``librosa.load(path, sr=sr)`` (dataset_inference.py:41): same int -> float scaling (1/32768 for 16-bit); when the
        file's rate differs, a windowed-sinc polyphase resampler stands in for librosa's soxr (not bit-identical to it -
        the hot-path parity contract starts at the 16 kHz waveform).  The resampling here is ``resample`` on the host;
        ``enhance_files(..., resample_on_device=True)`` runs the same filter on the device instead."""
        wav, rate = read_wav(path)
        y = Inferencer.mono(wav)
        if rate != sr:
            y = Inferencer.resample(y, rate, sr)
        return np.ascontiguousarray(y, dtype=np.float32)

    @staticmethod
    def resample(y: np.ndarray, sr_in: int, sr_out: int, zeros: int = 24) -> np.ndarray:
        """Band-limited (hann-windowed sinc) polyphase resampling on the host, in float64 with [n_out, 2 * half]
        temporaries.  ``acoustics.resample.resample_batch`` computes the same outputs for a batch of clips on the device
        (fsn_resample), equal to these to float32 rounding."""
        from math import gcd
        g = gcd(int(sr_in), int(sr_out))
        up, down = sr_out // g, sr_in // g
        cutoff = min(1.0, up / down)
        half = int(np.ceil(zeros / cutoff))
        n_out = int(np.ceil(len(y) * up / down))
        t_out = np.arange(n_out, dtype=np.float64) * down / up  # positions in input samples
        base = np.floor(t_out).astype(np.int64)
        k = np.arange(-half + 1, half + 1)
        idx = base[:, None] + k[None, :]
        d = t_out[:, None] - idx
        w = cutoff * np.sinc(cutoff * d) * (0.5 + 0.5 * np.cos(np.pi * np.clip(d / half, -1, 1)))
        ok = (idx >= 0) & (idx < len(y))
        vals = np.where(ok, y[np.clip(idx, 0, len(y) - 1)], 0.0)
        return (vals * w).sum(axis=1).astype(np.float32)

    @torch.no_grad()
    def enhance_files(self, paths, output_dir, batch_size: int = 64, sr=None, max_padding: float = 0.0,
                      resample_on_device: bool = False):
        """Batched form of the host loop of base_inferencer.py:163-195: ``plan_batches`` groups the files, each batch
        goes through ONE fused library call (pinned staging buffer -> H2D -> the model's enhance_pcm -> int16 D2H), and
        ``<output_dir>/<stem>.wav`` is written as 16-bit PCM like the reference.  Returns the written paths.

        ``max_padding == 0`` (default): batches of equal-length clips only.  ``max_padding > 0`` (improved_fullsubnet,
        and fullsubnet and fullband_baseline with a power-of-two n_fft; other models keep equal-length batches): clips of
        different lengths share a batch, padded to its longest clip by at most that fraction of the batch's samples,
        through fsn_enhance / fsn_improved_enhance / fsn_fullband_enhance.  Every file is bit-identical either way: each
        clip is bounded by its own length in the length-dependent kernels.

        ``resample_on_device``: files are read and mixed to mono on the host as ``load_wav`` does, and each batch is
        assembled on the device by ``resample_batch`` (fsn_resample, one call per input rate): files at another rate are
        resampled there, in float64 like ``resample`` and equal to it to float32 rounding, and files at ``sr`` are copied
        with their bits.  Batches are planned on the same lengths, so files at ``sr`` come out byte-identical to the
        default, and resampled ones within an int16 step of it."""
        from pathlib import Path
        sr = int(sr or self.sr)
        out_dir = Path(output_dir)
        out_dir.mkdir(parents=True, exist_ok=True)
        if resample_on_device:
            from .acoustics.resample import resample_batch, resampled_length
            clips, rates = [], []
            for p in paths:
                wav, rate = read_wav(p)
                clips.append((Path(p), self.mono(wav)))
                rates.append(rate)
            lens = [resampled_length(len(y), rate, sr) for (_, y), rate in zip(clips, rates)]
        else:
            clips = [(Path(p), self.load_wav(p, sr)) for p in paths]
            lens = [len(y) for _, y in clips]
        written = [None] * len(clips)
        for chunk in plan_batches(lens, batch_size, max_padding if self.supports_lengths() else 0.0):
            L = max(lens[i] for i in chunk)
            mixed = any(lens[i] != L for i in chunk)
            if resample_on_device:  # every row written, 0 past each clip
                stage = torch.empty(len(chunk), L, dtype=torch.float32, device=self.device)
                resample_batch([clips[i][1] for i in chunk], [rates[i] for i in chunk], sr, self.device, out=stage)
            else:
                stage = (torch.zeros if mixed else torch.empty)(len(chunk), L, dtype=torch.float32).pin_memory()
                for r, i in enumerate(chunk):
                    stage[r, :lens[i]] = torch.from_numpy(clips[i][1])
            pcm = self.enhance_to_pcm(stage, lengths=[lens[i] for i in chunk] if mixed else None).cpu().numpy()
            for r, i in enumerate(chunk):
                dst = out_dir / f"{clips[i][0].stem}.wav"
                self.write_wav(dst, pcm[r, :lens[i]], sr)
                written[i] = dst
        return written

    @torch.no_grad()
    def __call__(self, clips):
        """Host loop of base_inferencer.py:163-195 without the wav I/O: yields (enhanced float32, int16 PCM
        scaled as base_inferencer.py:181-182) per clip."""
        out = []
        for noisy in clips:
            enhanced = getattr(self, self.inference_config["type"])(noisy.to(self.device),
                                                                    self.inference_config.get("args", {}))
            amp = np.iinfo(np.int16).max
            pcm = np.int16(0.8 * amp * enhanced / np.max(np.abs(enhanced)))
            out.append((enhanced, pcm))
        return out
