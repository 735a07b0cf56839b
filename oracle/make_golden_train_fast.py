"""TEST INFRASTRUCTURE ONLY.  Generates ``tests/golden/train_fast.npz``: two optimisation steps of
recipes/dns_interspeech_2020/fast_fullsubnet/trainer.py:45-56 run with the UNMODIFIED upstream fast Model / stft / cIRM
from ``/root/reference`` on CPU (AMP off, no drop_band - the fast trainer has none), torch.nn.MSELoss
(audio_zen/loss.py:4), clip_grad_norm_(10) and Adam(lr 1e-3, betas (0.9, 0.999)) (train_shrinkSize2.toml).

Model: the recipe's args (oracle.fast_fullsubnet_oracle.DEFAULT_FAST_ARGS), weights from make_fast_state_dict(seed=3).
Data: 3 clips x 0.5 s (T = 32 frames + 2 look-ahead, 18 shrunk steps, the last one a single frame).  The inputs are not stored: the tests
regenerate them with oracle.make_noisy(seed) and check the stored fingerprint.  Gradients and parameters are stored as
every SUBSAMPLE-th element (parameters after step 0: every 4 * SUBSAMPLE-th) plus the per-tensor L2 norm of the
gradient.

Run:  python oracle/make_golden_train_fast.py
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

SUBSAMPLE = 97
SEEDS = dict(weights=3, noisy=51, clean=52)
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
    from make_golden import import_reference
    from oracle import fast_fullsubnet_oracle as FO
    feature, mask, _, _ = import_reference()
    ti = types.ModuleType("torchinfo"); ti.summary = lambda *a, **k: None
    sys.modules.setdefault("torchinfo", ti)
    from fast_fullsubnet.model import Model as FastModel
    torch.set_num_threads(8)
    args = dict(FO.DEFAULT_FAST_ARGS)
    model = FastModel(**args).train()
    model.load_state_dict(FO.make_fast_state_dict(seed=SEEDS["weights"], args=args), strict=True)
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
    print("fast train: loss", loss, "gnorm", gnorm)
    path = os.path.join(ROOT, "tests", "golden", "train_fast.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
