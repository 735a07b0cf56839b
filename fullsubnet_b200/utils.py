"""audio_zen/utils.py: initialize_module (:70-105, the reference's plugin mechanism) and
prepare_device (:135-162)."""
from __future__ import annotations

import importlib
from typing import Optional

import torch


def initialize_module(path: str, args: Optional[dict] = None, initialize: bool = True):
    module_path = ".".join(path.split(".")[:-1])
    class_or_function_name = path.split(".")[-1]
    module = importlib.import_module(module_path)
    class_or_function = getattr(module, class_or_function_name)
    if initialize:
        return class_or_function(**args) if args else class_or_function()
    return class_or_function


def prepare_device(n_gpu: int, keep_reproducibility=False):
    if n_gpu == 0:
        raise RuntimeError("fullsubnet_b200 has no CPU path: a CUDA device (H100) is required.")
    return torch.device("cuda:0")


def read_wav(path):
    """PCM wav file (8/16/24/32-bit) with the standard library: (float32 [C, N], sample rate).  Integer samples are
    scaled like librosa / soundfile: 1/128 around 128 for 8-bit, 1/32768 for 16-bit, 1/2^23 for 24-bit, 1/2^31 for
    32-bit."""
    import wave

    import numpy as np
    with wave.open(str(path), "rb") as f:
        nch, width, rate, n = f.getnchannels(), f.getsampwidth(), f.getframerate(), f.getnframes()
        raw = f.readframes(n)
    if width == 2:
        y = np.frombuffer(raw, dtype="<i2").astype(np.float32) / 32768.0
    elif width == 1:
        y = (np.frombuffer(raw, dtype=np.uint8).astype(np.float32) - 128.0) / 128.0
    elif width == 4:
        y = np.frombuffer(raw, dtype="<i4").astype(np.float32) / 2147483648.0
    elif width == 3:
        b = np.frombuffer(raw, dtype=np.uint8).reshape(-1, 3).astype(np.int32)
        v = b[:, 0] | (b[:, 1] << 8) | (b[:, 2] << 16)
        y = (np.where(v >= 1 << 23, v - (1 << 24), v)).astype(np.float32) / 8388608.0
    else:
        raise NotImplementedError(f"wav sample width {width}")
    return np.ascontiguousarray(y.reshape(-1, nch).T), rate
