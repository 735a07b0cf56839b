"""fullsubnet_b200 - H100 (sm_90a) implementation of FullSubNet's enhancement hot path behind
the reference's own Python API (Audio-WestlakeU/FullSubNet, recipes/dns_interspeech_2020).

Layout mirrors the reference so that TOML ``path`` strings keep working:
    fullsubnet_b200.acoustics.feature   <- audio_zen/acoustics/feature.py  (stft, istft, drop_band)
    fullsubnet_b200.acoustics.mask      <- audio_zen/acoustics/mask.py     (cIRM build / (de)compress)
    fullsubnet_b200.fullsubnet.model    <- recipes/dns_interspeech_2020/fullsubnet/model.py (Model)
    fullsubnet_b200.inferencer          <- recipes/dns_interspeech_2020/inferencer.py (Inferencer)

All device work is done by libfsn_b200.so (hand-written CUDA, C ABI in include/fsn_b200.h);
there is no CPU or PyTorch fallback: CPU tensors and a missing library raise.
"""
from . import _lib  # noqa: F401

__all__ = ["_lib"]
__version__ = "0.1.0"
