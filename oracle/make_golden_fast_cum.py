"""TEST INFRASTRUCTURE ONLY.  Generates ``tests/golden/fast_cum.npz``: recipes/dns_interspeech_2020/fast_fullsubnet/model.py
built with ``norm_type="cumulative_laplace_norm"`` (audio_zen/model/base_model.py:220-251 on the mel spectrogram and on the
down-sampled bottleneck input) from the UNMODIFIED upstream code in ``/root/reference``, on CPU.

Inference: the recipe's args (oracle.fast_fullsubnet_oracle.DEFAULT_FAST_ARGS, shrink 2, look-ahead 2), weights
make_fast_state_dict(seed=3), Model.eval() on the noisy magnitude of 3 clips at two lengths: 4000 samples (T = 16, T' = 18:
a short last down-sampling block) and 4256 samples (T = 17, T' = 19: a full last block), each at B = 1 (the first clip) and
B = 3.  Stored: the magnitudes ``mag_T{16,17}`` and the outputs ``out_b1_T*`` / ``out_b3_T*``.

Training: two optimisation steps exactly as oracle/make_golden_train_fast.py (3 clips x 0.5 s, weights seed 3, MSELoss,
clip_grad_norm_(10), Adam(1e-3)) on the cumulative-norm model.  The inputs and the cIRM target are those of
``train_fast.npz`` (checked here, not stored again); stored: ``crm`` of step 0, every SUBSAMPLE-th gradient element and
the per-tensor L2 norms of step 0, the parameters after step 0 (every 4 * SUBSAMPLE-th) and step 1 (every SUBSAMPLE-th),
the losses and the clipped gradient norms.

Run:  python oracle/make_golden_fast_cum.py
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

SUBSAMPLE = 291
LENGTHS = {16: 4000, 17: 4256}  # frames T -> samples (hop 256)
NOISY_SEED = 13


def cum_args():
    from oracle import fast_fullsubnet_oracle as FO
    return dict(FO.DEFAULT_FAST_ARGS, norm_type="cumulative_laplace_norm")


def main():
    from make_golden import import_reference
    from oracle import fast_fullsubnet_oracle as FO
    from oracle import fullsubnet_oracle as O
    from oracle import make_golden_train_fast as MG
    feature, mask, _, _ = import_reference()
    ti = types.ModuleType("torchinfo"); ti.summary = lambda *a, **k: None
    sys.modules.setdefault("torchinfo", ti)
    from fast_fullsubnet.model import Model as FastModel
    torch.set_num_threads(8)
    args = cum_args()
    out = {}
    # ---- inference
    model = FastModel(**args).eval()
    model.load_state_dict(FO.make_fast_state_dict(seed=3, args=args), strict=True)
    for T, L in LENGTHS.items():
        y = O.make_noisy(3, L, seed=NOISY_SEED, speechlike=True)
        mag = feature.stft(y, 512, 256, 512)[0]
        assert mag.shape[-1] == T, mag.shape
        with torch.no_grad():
            out[f"out_b1_T{T}"] = model(mag[:1].unsqueeze(1)).numpy()
            out[f"out_b3_T{T}"] = model(mag.unsqueeze(1)).numpy()
        out[f"mag_T{T}"] = mag.numpy()
        print(f"T={T}: out range", float(out[f"out_b3_T{T}"].min()), float(out[f"out_b3_T{T}"].max()))
    # ---- two training steps (make_golden_train_fast.main with the cumulative norm)
    model = FastModel(**args).train()
    model.load_state_dict(FO.make_fast_state_dict(seed=MG.SEEDS["weights"], args=args), strict=True)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3, betas=(0.9, 0.999))
    loss_fn = torch.nn.MSELoss()
    noisy, clean = MG.inputs()
    g_fast = np.load(os.path.join(ROOT, "tests", "golden", "train_fast.npz"))
    assert np.array_equal(MG.fingerprint(noisy), g_fast["noisy_fp"]) and np.array_equal(MG.fingerprint(clean), g_fast["clean_fp"])
    loss, gnorm = [], []
    for it in range(2):
        opt.zero_grad()
        noisy_mag, _, nr, ni = feature.stft(noisy, 512, 256, 512)
        _, _, cr, ci = feature.stft(clean, 512, 256, 512)
        cirm = mask.build_complex_ideal_ratio_mask(nr, ni, cr, ci)
        assert np.array_equal(cirm.numpy(), g_fast["cirm"])
        crm = model(noisy_mag.unsqueeze(1)).permute(0, 2, 3, 1)
        l = loss_fn(cirm, crm)
        l.backward()
        if it == 0:
            out["crm"] = crm.detach().numpy().copy()
            for k, p in model.named_parameters():
                g = p.grad.detach().numpy()
                out["gsub." + k] = g.reshape(-1)[::SUBSAMPLE].copy()
                out["gl2." + k] = np.array(np.sqrt((g.astype(np.float64) ** 2).sum()))
        loss.append(float(l.detach()))
        gnorm.append(float(torch.nn.utils.clip_grad_norm_(model.parameters(), 10)))
        opt.step()
        for k, p in model.named_parameters():
            out[f"p{it}." + k] = p.detach().numpy().reshape(-1)[::SUBSAMPLE * (4 if it == 0 else 1)].copy()
    out["loss"], out["gnorm"] = np.array(loss), np.array(gnorm)
    print("fast cum train: loss", loss, "gnorm", gnorm)
    path = os.path.join(ROOT, "tests", "golden", "fast_cum.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
