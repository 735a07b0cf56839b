"""Training data with the mixing on the device.

``snr_mix``: the arithmetic of ``Dataset.snr_mix`` (recipes/dns_interspeech_2020/dataset_train.py:136-199) for a batch
of (clean, noise) pairs, so that an 8-GPU trainer does not need the 16-48 CPU dataloader workers per GPU the
reference's on-the-fly mixing would take (SURVEY 8f rank 4).

``Dataset``: drop-in for ``dataset_train.Dataset`` (same constructor arguments, same random draws from the global
``random`` / ``np.random`` streams in the same order).  File selection, cropping and the draws stay on the host (cheap);
an item is the crops and the draws as fixed-shape arrays, and ``Trainer`` mixes the collated batch on the device."""
from __future__ import annotations

import os
import random
from typing import Optional

import numpy as np
import torch

from . import _lib
from .utils import read_wav


def snr_mix(clean_y: torch.Tensor, noise_y: torch.Tensor, snr, target_dB_FS: float, noisy_target_dB_FS,
            rir: Optional[torch.Tensor] = None, rir_len: Optional[torch.Tensor] = None, eps: float = 1e-6):
    """clean_y, noise_y [B,L] (CUDA float32); snr, noisy_target_dB_FS: [B] (the values the reference draws with
    ``random.choice(snr_list)`` and ``np.random.randint(target - floating, target + floating)``); rir [B,Lr] with
    rir_len [B] int32 (0 = no reverberation for that clip) or None.  Returns (noisy_y, clean_y), both [B,L]."""
    clean_y = _lib.require_cuda(clean_y, "clean_y")
    noise_y = _lib.require_cuda(noise_y, "noise_y")
    assert clean_y.shape == noise_y.shape and clean_y.dim() == 2, "Inequality: clean / noise shapes"
    B, L = clean_y.shape
    dev = clean_y.device
    snr_t = torch.as_tensor(snr, dtype=torch.float32, device=dev).reshape(-1).expand(B).contiguous()
    nt_t = torch.as_tensor(noisy_target_dB_FS, dtype=torch.float32, device=dev).reshape(-1).expand(B).contiguous()
    lib = _lib.load()
    with torch.cuda.device(dev):
        st = _lib.stream_ptr(dev)
        if rir is not None:
            rir = _lib.require_cuda(rir, "rir")
            assert rir.dim() == 2 and rir.shape[0] == B
            rl = None if rir_len is None else rir_len.to(device=dev, dtype=torch.int32).contiguous()
            rev = torch.empty_like(clean_y)
            _lib.check(lib.fsn_rir_convolve(clean_y.data_ptr(), rir.data_ptr(), _lib.ptr(rl), B, L, rir.shape[1],
                                            rev.data_ptr(), st))
            clean_y = rev
        noisy, clean = torch.empty_like(clean_y), torch.empty_like(clean_y)
        _lib.check(lib.fsn_snr_mix(clean_y.data_ptr(), noise_y.data_ptr(), snr_t.data_ptr(), nt_t.data_ptr(),
                                   float(target_dB_FS), float(eps), B, L, noisy.data_ptr(), clean.data_ptr(), st))
    return noisy, clean


def _expand(path) -> str:
    return os.path.abspath(os.path.expanduser(path))


def _resampled_length(n: int, rate: int, sr: int) -> int:
    """Length of an ``n``-sample signal at ``rate`` after ``Inferencer.resample`` to ``sr``."""
    if rate == sr:
        return n
    from math import gcd
    g = gcd(int(rate), int(sr))
    return int(np.ceil(n * (sr // g) / (rate // g)))


def load_wav(path, sr: int = 16000) -> np.ndarray:
    """float32 [C, N] at ``sr`` from a PCM wav file, every channel kept (``librosa.load(path, mono=False, sr=sr)``, with
    librosa's int -> float scaling).  When the file's rate differs, each channel goes through the windowed-sinc resampler
    of ``Inferencer.resample`` on the host, which stands in for librosa's soxr and is not bit-identical to it
    (``Dataset(resample_on_device=True)`` runs the same filter on the device for the preloaded lists)."""
    y, rate = read_wav(_expand(path))
    if rate != sr:
        from .inferencer import Inferencer
        y = np.stack([Inferencer.resample(c, rate, sr) for c in y])
    return y


class Dataset(torch.utils.data.Dataset):
    """Drop-in for ``recipes/dns_interspeech_2020/dataset_train.py::Dataset``: a TOML switches to it with
    ``[train_dataset] path = "fullsubnet_b200.dataset.Dataset"`` and the same ``[train_dataset.args]``.

    ``__getitem__`` makes the reference's draws from the global ``random`` and ``np.random`` streams, in its order and
    under its conditions (clean crop start, noise files, noise crop start, SNR, reverberation, RIR file, RIR channel,
    noisy target dBFS), so a seeded run selects the reference's items.  It does no arithmetic on the audio and returns
    what the reference passes to ``snr_mix``, as fixed-shape arrays the default collate stacks:

    * ``clean``, ``noise``: float32 [L], L = int(sub_sample_length * sr);
    * ``rir``: float32 [Lr_max], the chosen RIR channel zero-padded to the longest RIR of the list (read from the files
      at construction); ``rir_len``: int32, 0 when the item has no reverberation;
    * ``snr``, ``noisy_target_dB_FS``, ``target_dB_FS``: float32.

    ``Trainer`` turns such a batch into ``(noisy, clean)`` on the device with ``snr_mix``.  A clean or noise file with
    more than one channel is refused (the reference asserts on the first and silently interleaves the second); a RIR
    file may have several channels, one of which each reverberant item draws.  ``pre_load_*`` holds the waveforms in host
    memory, read by ``num_workers`` threads.  Files at another sample rate are resampled as ``load_wav`` says.

    ``resample_on_device`` (a keyword after the reference's arguments): the preloaded lists are resampled on the current
    CUDA device by ``resample_batch`` (fsn_resample, every RIR channel a clip), equal to the host resampler to float32
    rounding, and kept as host arrays as before; lengths, and so every draw, are the host's.  Lists that are not
    preloaded load in the DataLoader workers, where CUDA cannot run, and keep the host resampler."""

    def __init__(self, clean_dataset, clean_dataset_limit, clean_dataset_offset, noise_dataset, noise_dataset_limit,
                 noise_dataset_offset, rir_dataset, rir_dataset_limit, rir_dataset_offset, snr_range, reverb_proportion,
                 silence_length, target_dB_FS, target_dB_FS_floating_value, sub_sample_length, sr,
                 pre_load_clean_dataset, pre_load_noise, pre_load_rir, num_workers, resample_on_device=False):
        super().__init__()
        self.sr = sr
        self.num_workers = num_workers
        self.resample_on_device = bool(resample_on_device)
        clean = self._offset_and_limit(self._read_list(clean_dataset), clean_dataset_offset, clean_dataset_limit)
        noise = self._offset_and_limit(self._read_list(noise_dataset), noise_dataset_offset, noise_dataset_limit)
        rir = self._offset_and_limit(self._read_list(rir_dataset), rir_dataset_offset, rir_dataset_limit)
        self.clean_dataset_list = self._preload(clean, "clean") if pre_load_clean_dataset else clean
        self.noise_dataset_list = self._preload(noise, "noise") if pre_load_noise else noise
        self.rir_dataset_list = self._preload(rir, "rir") if pre_load_rir else rir
        self.snr_list = self._parse_snr_range(snr_range)
        assert 0 <= reverb_proportion <= 1, "reverb_proportion must be in [0, 1]"
        self.reverb_proportion = reverb_proportion
        self.silence_length = silence_length
        self.target_dB_FS = target_dB_FS
        self.target_dB_FS_floating_value = target_dB_FS_floating_value
        self.sub_sample_length = sub_sample_length
        self.length = len(self.clean_dataset_list)
        self.rir_length = max([self._rir_frames(r) for r in self.rir_dataset_list], default=0)

    # ------------------------------------------------------------------ the reference's argument checks
    @staticmethod
    def _offset_and_limit(dataset_list, offset, limit):
        dataset_list = dataset_list[offset:]
        return dataset_list[:limit] if limit else dataset_list

    @staticmethod
    def _parse_snr_range(snr_range):
        assert len(snr_range) == 2, f"snr_range must be [low, high], got {snr_range}"
        low, high = snr_range
        assert low <= high, f"snr_range: low {low} is larger than high {high}"
        return list(range(low, high + 1))

    @staticmethod
    def _read_list(path):
        with open(_expand(path), "r") as f:
            return [line.rstrip("\n") for line in f]

    # ------------------------------------------------------------------ waveforms
    def _preload(self, paths, kind):
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(max_workers=max(1, int(self.num_workers or 1))) as pool:
            if self.resample_on_device:
                waves = self._resample_on_device(list(pool.map(lambda p: read_wav(_expand(p)), paths)))
            else:
                waves = list(pool.map(lambda p: load_wav(p, self.sr), paths))
        if kind != "rir":
            waves = [self._mono(w, p, kind) for p, w in zip(paths, waves)]
        return [(p, w) for p, w in zip(paths, waves)]

    def _resample_on_device(self, files, batch_size: int = 32):
        """(float32 [C, N], rate) per file -> float32 [C, n] at ``sr``: the channels of files at another rate go through
        ``resample_batch`` on the current CUDA device, in batches of clips of similar length (``plan_batches``)."""
        from .acoustics.resample import resample_batch
        from .inferencer import plan_batches
        clips = [(f, c) for f, (w, rate) in enumerate(files) if rate != self.sr for c in range(w.shape[0])]
        device = torch.device("cuda", torch.cuda.current_device())
        out = {}
        for chunk in plan_batches([files[f][0].shape[1] for f, _ in clips], batch_size, 0.5):
            picked = [clips[i] for i in chunk]
            ys = resample_batch([files[f][0][c] for f, c in picked], [files[f][1] for f, _ in picked], self.sr, device)
            out.update((fc, y.cpu().numpy()) for fc, y in zip(picked, ys))
        return [w if rate == self.sr else np.stack([out[f, c] for c in range(w.shape[0])])
                for f, (w, rate) in enumerate(files)]

    @staticmethod
    def _mono(wav, path, kind) -> np.ndarray:
        if wav.shape[0] != 1:
            raise ValueError(f"{kind} file {path} has {wav.shape[0]} channels; {kind} files must be mono")
        return wav[0]

    def _load(self, entry, kind) -> np.ndarray:
        """A list entry (a path, or a preloaded (path, waveform) pair) as a waveform: [N] for clean and noise, [C, N]
        for a RIR."""
        if isinstance(entry, tuple):
            return entry[1]
        wav = load_wav(entry, self.sr)
        return wav if kind == "rir" else self._mono(wav, entry, kind)

    def _rir_frames(self, entry) -> int:
        if isinstance(entry, tuple):
            return entry[1].shape[-1]
        import wave
        with wave.open(_expand(entry), "rb") as f:
            return _resampled_length(f.getnframes(), f.getframerate(), self.sr)

    # ------------------------------------------------------------------ items
    def __len__(self):
        return self.length

    def _select_noise_y(self, target_length):
        pieces, n = [], 0
        silence = int(self.sr * self.silence_length)
        remaining = target_length
        while remaining > 0:
            y = self._load(random.choice(self.noise_dataset_list), "noise")
            pieces.append(y)
            remaining -= len(y)
            if remaining > 0:  # a silence between noise files; the last one may be partial
                k = min(remaining, silence)
                pieces.append(np.zeros(k, dtype=np.float32))
                remaining -= k
        noise = np.concatenate(pieces).astype(np.float32, copy=False)
        if len(noise) > target_length:
            start = np.random.randint(len(noise) - target_length)
            noise = noise[start:start + target_length]
        return noise

    def __getitem__(self, item):
        L = int(self.sub_sample_length * self.sr)
        clean = self._load(self.clean_dataset_list[item], "clean")
        if len(clean) > L:
            start = np.random.randint(len(clean) - L)
            clean = clean[start:start + L]
        elif len(clean) < L:
            clean = np.concatenate([clean, np.zeros(L - len(clean), dtype=np.float32)])
        noise = self._select_noise_y(L)
        snr = random.choice(self.snr_list)
        use_reverb = bool(np.random.random(1) < self.reverb_proportion)
        rir = np.zeros(self.rir_length, dtype=np.float32)
        rir_len = 0
        if use_reverb:
            r = self._load(random.choice(self.rir_dataset_list), "rir")
            if r.shape[0] > 1:
                r = r[np.random.randint(0, r.shape[0])]
            r = r.reshape(-1)
            rir_len = len(r)
            rir[:rir_len] = r
        t, f = self.target_dB_FS, self.target_dB_FS_floating_value
        noisy_target_dB_FS = np.random.randint(t - f, t + f)
        return {"clean": np.ascontiguousarray(clean, dtype=np.float32),
                "noise": np.ascontiguousarray(noise, dtype=np.float32),
                "rir": rir, "rir_len": np.int32(rir_len), "snr": np.float32(snr),
                "noisy_target_dB_FS": np.float32(noisy_target_dB_FS), "target_dB_FS": np.float32(t)}


def mix_batch(batch: dict, device, eps: float = 1e-6):
    """A collated ``Dataset`` batch -> (noisy [B,L], clean [B,L]) on ``device``: ``fsn_rir_convolve`` on the
    reverberant rows and ``fsn_snr_mix`` on all of them.  Copies to the device and launches only; never waits on it."""
    target = batch["target_dB_FS"]
    target = float(target.reshape(-1)[0]) if isinstance(target, torch.Tensor) else float(np.asarray(target).reshape(-1)[0])
    to = lambda k: torch.as_tensor(batch[k]).to(device, non_blocking=True)  # noqa: E731
    clean, noise = to("clean"), to("noise")
    rir = batch["rir"]
    has_rir = rir.shape[-1] > 0
    return snr_mix(clean, noise, to("snr"), target, to("noisy_target_dB_FS"),
                   rir=to("rir") if has_rir else None, rir_len=to("rir_len") if has_rir else None, eps=eps)
