"""TEST INFRASTRUCTURE ONLY.  Generates ``tests/golden/train_fbb.npz``: two optimisation steps of
recipes/dns_interspeech_2020/fullband_baseline/trainer.py:32-71 run with the UNMODIFIED upstream fullband_baseline Model /
stft / cIRM from ``/root/reference`` on CPU (AMP off, no drop_band - this trainer has none), torch.nn.MSELoss
(audio_zen/loss.py:4), clip_grad_norm_(10) and Adam(lr 1e-3, betas (0.9, 0.999)) (fullband_baseline/train.toml).

Model: the recipe's args (oracle.fullband_baseline_oracle.DEFAULT_FBB_ARGS: F = 257, H = 512, LSTM, no activation,
look_ahead 2, offline norm), weights from make_fbb_state_dict(seed=5), imported the way make_golden_fbb.py does.
Data: 3 clips x 0.5 s (T = 32 frames + 2 look-ahead).  The inputs are not stored: the tests regenerate them with
oracle.make_noisy(seed) and check the stored fingerprint.  Gradients and parameters are stored as every SUBSAMPLE-th
element (parameters after step 0: every 4 * SUBSAMPLE-th) plus the per-tensor L2 norm of the gradient.

Run:  python oracle/make_golden_train_fbb.py
"""
from __future__ import annotations

import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

SUBSAMPLE = 97
SEEDS = dict(weights=5, noisy=61, clean=62)
CLIPS, SAMPLES = 3, 8000


def fingerprint(y: torch.Tensor) -> np.ndarray:
    a = y.numpy().astype(np.float64)
    return np.concatenate([a.reshape(-1)[:8], [a.sum(), np.abs(a).sum()]])


def inputs():
    from oracle import fullsubnet_oracle as O
    noisy = O.make_noisy(CLIPS, SAMPLES, seed=SEEDS["noisy"], speechlike=True)
    clean = 0.5 * O.make_noisy(CLIPS, SAMPLES, seed=SEEDS["clean"], speechlike=True)
    return noisy, clean


def main():
    from make_golden import REF, import_reference
    from oracle import fullband_baseline_oracle as BO
    feature, mask, _, _ = import_reference()
    spec = importlib.util.spec_from_file_location(
        "fbb_model", os.path.join(REF, "recipes", "dns_interspeech_2020", "fullband_baseline", "model.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    torch.set_num_threads(8)
    args = dict(BO.DEFAULT_FBB_ARGS)
    model = mod.Model(**args).train()
    model.load_state_dict(BO.make_fbb_state_dict(seed=SEEDS["weights"], args=args), strict=True)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3, betas=(0.9, 0.999))
    loss_fn = torch.nn.MSELoss()
    noisy, clean = inputs()
    out = {"noisy_fp": fingerprint(noisy), "clean_fp": fingerprint(clean)}
    loss, gnorm = [], []
    for it in range(2):
        opt.zero_grad()
        noisy_mag, _, nr, ni = feature.stft(noisy, 512, 256, 512)
        _, _, cr, ci = feature.stft(clean, 512, 256, 512)
        cirm = mask.build_complex_ideal_ratio_mask(nr, ni, cr, ci)
        crm = model(noisy_mag.unsqueeze(1)).permute(0, 2, 3, 1)
        l = loss_fn(cirm, crm)
        l.backward()
        if it == 0:
            out["cirm"] = cirm.detach().numpy().copy()
            out["crm"] = crm.detach().numpy().copy()
            for k, p in model.named_parameters():
                g = p.grad.detach().numpy()
                out["gsub." + k] = g.reshape(-1)[::SUBSAMPLE].copy()
                out["gl2." + k] = np.array(np.sqrt((g.astype(np.float64) ** 2).sum()))
        loss.append(float(l.detach()))
        gnorm.append(float(torch.nn.utils.clip_grad_norm_(model.parameters(), 10)))
        opt.step()
        for k, p in model.named_parameters():  # after step 0 sparser: the file stays under 1 MB
            out[f"p{it}." + k] = p.detach().numpy().reshape(-1)[::SUBSAMPLE * (4 if it == 0 else 1)].copy()
    out["loss"], out["gnorm"] = np.array(loss), np.array(gnorm)
    print("fullband_baseline train: loss", loss, "gnorm", gnorm)
    path = os.path.join(ROOT, "tests", "golden", "train_fbb.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
