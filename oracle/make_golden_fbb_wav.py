"""TEST INFRASTRUCTURE ONLY.  ``tests/golden/fullband_baseline_wav.npz``: the UNMODIFIED upstream fullband_baseline Model
(recipes/dns_interspeech_2020/fullband_baseline/model.py) inside the reference ``Inferencer.full_band_crm_mask`` flow
on CPU (SURVEY 8c: stft -> model -> decompress_cIRM -> complex product -> istft), one clip at a time, for clips of
different lengths (none a multiple of the hop):
  small  F=33, H=32, ReLU, cumulative norm, n_fft 64
  full   F=257, H=512, offline norm, n_fft 512: weight set ``wa`` (seed 11) and ``wb`` (the same with
         ``fc_output_layer`` scaled by ``wb_gain``, the first of WB_GAINS whose cRM reaches the +-9.9 clip of
         decompress_cIRM)
Keys per set: ``<tag>_y`` [B, L_max] (rows zero past their length), ``<tag>_lengths``, ``<tag>_wav`` [B, L_max] and
``<tag>_crm`` [B, 2, F, T_max] (both zero past each clip).   Run:  python oracle/make_golden_fbb_wav.py
"""
from __future__ import annotations

import importlib.util
import os
import sys
from functools import partial

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

WB_GAINS = (100.0, 110.0, 120.0, 130.0, 140.0, 150.0, 160.0, 180.0, 200.0)
SETS = {"small": dict(n_fft=64, lengths=(1201, 900, 1043)),
        "wa": dict(n_fft=512, lengths=(8001, 5555, 6789)),
        "wb": dict(n_fft=512, lengths=(8001, 5555, 6789))}


def main():
    from make_golden import REF, import_reference
    from oracle import fullband_baseline_oracle as BO
    from oracle import fullsubnet_oracle as O
    feature, _, _, Inferencer = import_reference()
    spec = importlib.util.spec_from_file_location(
        "fbb_model", os.path.join(REF, "recipes", "dns_interspeech_2020", "fullband_baseline", "model.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    torch.set_num_threads(8)
    small = dict(BO.DEFAULT_FBB_ARGS, num_freqs=33, hidden_size=32, output_activate_function="ReLU",
                 norm_type="cumulative_laplace_norm")
    res = {}
    for tag, s in SETS.items():
        a = small if tag == "small" else dict(BO.DEFAULT_FBB_ARGS)
        gain = 1.0
        if tag == "wb":
            gain = next(g for g in WB_GAINS if np.abs(reference(a, g, s, feature, mod, Inferencer, O, BO)[2]).max() > 9.9)
            res["wb_gain"] = np.float32(gain)
        y, wav, crm = reference(a, gain, s, feature, mod, Inferencer, O, BO)
        lens = s["lengths"]
        res[tag + "_y"], res[tag + "_lengths"] = y, np.asarray(lens, np.int32)
        res[tag + "_wav"], res[tag + "_crm"] = wav, crm
        print(tag, "crm max", float(np.abs(crm).max()), "wav max", float(np.abs(wav).max()))
    assert np.abs(res["wb_crm"]).max() > 9.9, "wb must reach the clip of decompress_cIRM"
    out = os.path.join(ROOT, "tests", "golden", "fullband_baseline_wav.npz")
    np.savez_compressed(out, **res)
    print(out, os.path.getsize(out), "wb_gain", float(res["wb_gain"]))


def reference(a, fc_gain, s, feature, mod, Inferencer, O, BO):
    """(y, wav, crm) of one weight set: the reference model in full_band_crm_mask, one clip at a time."""
    sd = BO.make_fbb_state_dict(seed=11, args=a)
    for k in ("fullband_model.fc_output_layer.weight", "fullband_model.fc_output_layer.bias"):
        sd[k] = sd[k] * fc_gain
    m = mod.Model(**a).eval()
    m.load_state_dict(sd, strict=True)
    n_fft, lens = s["n_fft"], s["lengths"]
    hop = n_fft // 2
    inf = Inferencer.__new__(Inferencer)  # no dataset / checkpoint (SURVEY 8c recipe)
    inf.model, inf.device = m, torch.device("cpu")
    inf.torch_stft = partial(feature.stft, n_fft=n_fft, hop_length=hop, win_length=n_fft)
    inf.torch_istft = partial(feature.istft, n_fft=n_fft, hop_length=hop, win_length=n_fft)
    L_max, B, F = max(lens), len(lens), n_fft // 2 + 1
    y = np.zeros((B, L_max), np.float32)
    wav = np.zeros((B, L_max), np.float32)
    crm = np.zeros((B, 2, F, 1 + L_max // hop), np.float32)
    for b, L in enumerate(lens):
        yb = O.make_noisy(1, L, seed=23 + b, speechlike=True)
        with torch.no_grad():
            crm_b = m(feature.stft(yb, n_fft, hop, n_fft)[0].unsqueeze(1))
            wav[b, :L] = inf.full_band_crm_mask(yb, {})
        y[b, :L] = yb.numpy()[0]
        crm[b, :, :, :crm_b.shape[-1]] = crm_b.numpy()[0]
    return y, wav, crm


if __name__ == "__main__":
    main()
