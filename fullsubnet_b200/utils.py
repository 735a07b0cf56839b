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
