"""TEST INFRASTRUCTURE ONLY - CPU restatement of recipes/dns_interspeech_2020/fast_fullsubnet/model.py:143-202 with the
norm the constructor's ``norm_type`` selects (BaseModel.norm_wrapper, audio_zen/model/base_model.py:356-372):
``offline_laplace_norm`` or ``cumulative_laplace_norm`` (base_model.py:220-251), applied to the mel spectrogram
(model.py:170) and to the down-sampled bottleneck input (model.py:186-187).  The building blocks are those of
``oracle/fast_fullsubnet_oracle.py``; pinned against the unmodified reference through
``oracle/make_golden_fast_cum.py`` -> ``tests/golden/fast_cum.npz``.  Runs in the dtype of its inputs (float64 autograd
needs ``torch.set_default_dtype(torch.float64)`` for the LSTM's zero initial state)."""
from __future__ import annotations

from typing import Dict, Optional

import torch

from .fast_fullsubnet_oracle import DEFAULT_FAST_ARGS, _seq, real_time_downsampling, real_time_upsampling
from .fullsubnet_oracle import cumulative_laplace_norm, freq_unfold, offline_laplace_norm

NORMS = {"offline_laplace_norm": offline_laplace_norm, "cumulative_laplace_norm": cumulative_laplace_norm}


def fast_model_forward(mix_mag: torch.Tensor, sd: Dict[str, torch.Tensor], args: Optional[dict] = None) -> torch.Tensor:
    """fast_fullsubnet/model.py:143-202 with args["norm_type"].  mix_mag [B,1,F,T] -> [B,2,F,T]."""
    a = dict(DEFAULT_FAST_ARGS)
    a.update(args or {})
    norm = NORMS[a["norm_type"]]
    la, S = a["look_ahead"], a["shrink_size"]
    Nn, Ne, M = a["noisy_input_num_neighbors"], a["encoder_output_num_neighbors"], a["num_mels"]
    x = torch.nn.functional.pad(mix_mag, [0, la])
    B, C, F, T = x.shape
    assert C == 1
    mel = (x.transpose(-1, -2) @ sd["mel_scale.fb"]).transpose(-1, -2)  # [B,1,M,T]  (model.py:166)
    e1 = _seq(norm(mel).reshape(B, -1, T), sd, "encoder.0.", 1, None, False)
    enc_out = _seq(e1, sd, "encoder.1.", 1, "ReLU", True).reshape(B, 1, -1, T)  # [B,1,M,T]
    bn_in = torch.cat([freq_unfold(mel, Nn).reshape(B, M, 2 * Nn + 1, T),
                       freq_unfold(enc_out, Ne).reshape(B, M, 2 * Ne + 1, T)], dim=2)
    K = bn_in.shape[2]
    # [B,M,K,Ts]: the cumulative norm takes one scale per (clip, mel row, shrunk step) over the K features
    bn_shr = norm(real_time_downsampling(bn_in, S))
    bn_out = _seq(bn_shr.reshape(B * M, K, -1), sd, "bottleneck.", a["bottleneck_num_layers"], "ReLU", True)
    bn_up = real_time_upsampling(bn_out.reshape(B, M, 1, -1).permute(0, 2, 1, 3), S, T)  # [B,1,M,T]
    dec_in = torch.cat([enc_out, bn_up], dim=2).reshape(B, -1, T)
    d1 = _seq(dec_in, sd, "decoder_lstm.0.", 1, None, False)
    d2 = _seq(d1, sd, "decoder_lstm.1.", 1, None, True)  # [B, 2F, T]
    return d2.reshape(B, 2, F, T)[:, :, :, la:]
