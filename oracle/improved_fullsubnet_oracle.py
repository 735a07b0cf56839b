"""TEST INFRASTRUCTURE ONLY - CPU fp32 restatement of recipes/dns_interspeech_2020/improved_fullsubnet/model.py
(SURVEY 8a row A14, BASELINE config 5).  Pinned against the unmodified reference through
``oracle/make_golden.py`` -> ``tests/golden/improved.npz``."""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import numpy as np
import torch

from . import fullsubnet_oracle as O

EPSILON = float(np.finfo(np.float32).eps)  # improved_fullsubnet/model.py:23

DEFAULT_IMPROVED_ARGS = dict(  # improved_fullsubnet/model.py:453-471 (16 kHz defaults)
    n_fft=512, hop_length=128, win_length=512, fdrc=0.5, num_freqs=257, freq_cutoffs=[20, 80],
    sb_num_center_freqs=[1, 4, 8], sb_num_neighbor_freqs=[15, 15, 15], fb_num_center_freqs=[1, 4, 8],
    fb_num_neighbor_freqs=[15, 15, 15], fb_hidden_size=512, sb_hidden_size=384, sequence_model="LSTM",
    fb_output_activate_function=False, sb_output_activate_function=False, norm_type="offline_laplace_norm",
)
# BASELINE config 5 wording (48 kHz, n_fft = 1024): valid constructor of SURVEY 8a row A14
ARGS_48K_1024 = dict(DEFAULT_IMPROVED_ARGS, n_fft=1024, hop_length=512, win_length=1024, num_freqs=513,
                     freq_cutoffs=[32, 128, 256], sb_num_center_freqs=[1, 4, 16, 64],
                     sb_num_neighbor_freqs=[15, 15, 15, 15], fb_num_center_freqs=[1, 4, 16, 64],
                     fb_num_neighbor_freqs=[15, 15, 15, 15])
# the reference's own 48 kHz example (improved_fullsubnet/model.py:603-620): n_fft = 960 is not a power of two
ARGS_48K_960 = dict(DEFAULT_IMPROVED_ARGS, n_fft=960, hop_length=480, win_length=960, num_freqs=481,
                    freq_cutoffs=[20, 120, 240], sb_num_center_freqs=[1, 4, 20, 60],
                    sb_num_neighbor_freqs=[15, 15, 15, 15], fb_num_center_freqs=[1, 4, 20, 60],
                    fb_num_neighbor_freqs=[15, 15, 15, 15])


def offline_laplace_norm(x: torch.Tensor) -> torch.Tensor:
    """improved_fullsubnet/model.py:129-152: per-clip mean over every non-batch axis, eps = float32 eps."""
    mu = x.mean(dim=list(range(1, x.dim())), keepdim=True)
    return x / (mu + EPSILON)


def section_bounds(num_freqs_used: int, cutoffs: List[int]):
    """model.py:412-423: [0,c0), [c0,c1), ..., [c_last, F)."""
    lo = [0] + list(cutoffs)
    hi = list(cutoffs) + [num_freqs_used]
    return list(zip(lo, hi))


def freq_unfold(x: torch.Tensor, lo: int, hi: int, center: int, neigh: int) -> torch.Tensor:
    """model.py:321-405.  x [B,1,F,T] -> [B,N,1,center+2*neigh,T]; unit n covers rows
    lo + n*center - neigh ... lo + (n+1)*center + neigh - 1, reflected (no edge repeat) at row 0 for the first
    section and at row F-1 for the last one."""
    B, C, F, T = x.shape
    assert C == 1
    if (hi - lo) % center != 0:
        raise ValueError("The number of center frequencies should be divisible by the subband freqency interval.")
    n_units = (hi - lo) // center
    width = center + 2 * neigh
    rows = lo + torch.arange(n_units)[:, None] * center - neigh + torch.arange(width)[None, :]  # [N,W]
    rows = torch.where(rows < 0, -rows, rows)
    rows = torch.where(rows >= F, 2 * (F - 1) - rows, rows)
    out = x[:, 0][:, rows, :]  # [B,N,W,T]
    return out.unsqueeze(2)


def seq_time_major(x: torch.Tensor, sd, prefix: str, act) -> torch.Tensor:
    """improved model's own SequenceModel (model.py:26-122): [B,F,T] -> LSTM(2 layers, time-major) -> Linear."""
    o = O.lstm_stack(x.permute(0, 2, 1), sd, prefix + "sequence_model.", num_layers=2)
    o = o @ sd[prefix + "fc_output_layer.weight"].t() + sd[prefix + "fc_output_layer.bias"]
    if act == "ReLU":
        o = torch.relu(o)
    elif act == "Tanh":
        o = torch.tanh(o)
    elif act == "ReLU6":
        o = torch.clamp(o, 0, 6)
    elif act:
        raise NotImplementedError(act)
    return o.permute(0, 2, 1)


def improved_forward(y: torch.Tensor, sd: Dict[str, torch.Tensor], args: Optional[dict] = None,
                     return_crm: bool = False):
    """improved_fullsubnet/model.py:541-591: waveform [B,L] (or [B,1,L]) -> enhanced waveform [B,1,L]."""
    a = dict(DEFAULT_IMPROVED_ARGS)
    a.update(args or {})
    assert y.dim() in (2, 3), "Input must be 2D (B, T) or 3D tensor (B, 1, T)"
    if y.dim() == 3:
        assert y.size(1) == 1
        y = y.squeeze(1)
    mag, _, real, imag = O.stft(y, a["n_fft"], a["hop_length"], a["win_length"])  # [B,F,T]
    noisy = (mag.unsqueeze(1) ** a["fdrc"])[..., :-1, :]  # model.py:564-565
    B, _, Fu, T = noisy.shape
    fb_in = offline_laplace_norm(noisy).reshape(B, Fu, T)
    fb_out = seq_time_major(fb_in, sd, "fb_model.", a["fb_output_activate_function"]).reshape(B, 1, Fu, T)
    outs = []
    for s, (lo, hi) in enumerate(section_bounds(Fu, a["freq_cutoffs"])):
        cs, ns = a["sb_num_center_freqs"][s], a["sb_num_neighbor_freqs"][s]
        cf, nf = a["fb_num_center_freqs"][s], a["fb_num_neighbor_freqs"][s]
        nsb = freq_unfold(noisy, lo, hi, cs, ns)
        fsb = freq_unfold(fb_out, lo, hi, cf, nf)
        inp = offline_laplace_norm(torch.cat([nsb, fsb], dim=-2))  # [B,N,1,W,T]  (model.py:442-443)
        Bn, N, _, W, _ = inp.shape
        o = seq_time_major(inp.reshape(Bn * N, W, T), sd, f"sb_model.sb_models.{s}.", a["sb_output_activate_function"])
        o = o.reshape(Bn, N, 2, -1, T).permute(0, 2, 1, 3, 4).reshape(Bn, 2, -1, T)  # model.py:239-247
        outs.append(o)
    crm = torch.cat(outs, dim=-2)
    crm = torch.nn.functional.pad(crm, (0, 0, 0, 1))  # Nyquist row of zeros (model.py:572)
    er, ei = crm[:, 0] * real, crm[:, 1] * imag  # element-wise, not a complex product (model.py:575-576)
    wav = O.istft((er, ei), a["n_fft"], a["hop_length"], a["win_length"], length=y.shape[-1], input_type="real_imag")
    wav = wav.unsqueeze(1)
    return (wav, crm) if return_crm else wav


def improved_state_dict_shapes(args: Optional[dict] = None):
    a = dict(DEFAULT_IMPROVED_ARGS)
    a.update(args or {})
    Fu, Hf, Hs = a["num_freqs"] - 1, a["fb_hidden_size"], a["sb_hidden_size"]
    out = []

    def seq(pre, In, H, Out):
        r = []
        for l in range(2):
            k = In if l == 0 else H
            r += [(f"{pre}sequence_model.weight_ih_l{l}", (4 * H, k)), (f"{pre}sequence_model.weight_hh_l{l}", (4 * H, H)),
                  (f"{pre}sequence_model.bias_ih_l{l}", (4 * H,)), (f"{pre}sequence_model.bias_hh_l{l}", (4 * H,))]
        return r + [(f"{pre}fc_output_layer.weight", (Out, H)), (f"{pre}fc_output_layer.bias", (Out,))]

    out += seq("fb_model.", Fu, Hf, Fu)
    for s in range(len(a["sb_num_center_freqs"])):
        W = (a["sb_num_center_freqs"][s] + 2 * a["sb_num_neighbor_freqs"][s]) + \
            (a["fb_num_center_freqs"][s] + 2 * a["fb_num_neighbor_freqs"][s])
        out += seq(f"sb_model.sb_models.{s}.", W, Hs, 2 * a["sb_num_center_freqs"][s])
    return out


def make_improved_state_dict(seed: int = 0, args: Optional[dict] = None) -> Dict[str, torch.Tensor]:
    rng = np.random.default_rng(seed)
    sd = {}
    for name, shape in improved_state_dict_shapes(args):
        if "sequence_model" in name:
            k = 1.0 / math.sqrt(shape[0] // 4)
        elif name.endswith("fc_output_layer.weight"):
            k = 1.0 / math.sqrt(shape[1])
        else:
            k = 1.0 / math.sqrt(sd[name.replace("bias", "weight")].shape[1])
        sd[name] = torch.from_numpy(rng.uniform(-k, k, size=shape).astype(np.float32))
    return sd
