"""TEST INFRASTRUCTURE ONLY.  Generates ``tests/golden/train_imp.npz`` and ``tests/golden/train_imp_960.npz``: optimisation
steps of the UNMODIFIED upstream improved_fullsubnet Model (recipes/dns_interspeech_2020/improved_fullsubnet/model.py:452-591)
from ``/root/reference`` on CPU, imported the way make_golden.py / make_golden_imp960.py do.

Upstream ships no trainer for this model (it is a differentiable module, wav in and wav out), so the objective is the
simplest one on the waveform: torch.nn.MSELoss(enhanced, clean), then clip_grad_norm_(10) and Adam(lr 1e-3, betas
(0.9, 0.999)).  The drop-in does not depend on the loss.

  train_imp.npz      16 kHz defaults (oracle.improved_fullsubnet_oracle.DEFAULT_IMPROVED_ARGS), 3 clips x 0.5 s (T = 63),
                     two steps: enhanced output of step 0, gradients of step 0, loss and gradient norm of both steps,
                     parameters after each step
  train_imp_960.npz  ARGS_48K_960 (n_fft = 960, the direct-DFT path), 2 clips x 0.25 s (T = 26), one step: gradients,
                     loss and gradient norm
Weights from make_improved_state_dict(seed=5).  The inputs are not stored: the tests regenerate them with
oracle.make_noisy(seed) and check the stored fingerprint.  Gradients and parameters are stored as every SUBSAMPLE-th
element (parameters after step 0: every 4 * SUBSAMPLE-th) plus the per-tensor L2 norm of the gradient, so that each file
stays under 1 MB for these ~10 M-parameter models.

Run:  python oracle/make_golden_train_imp.py
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

SUBSAMPLE = 127
SEEDS = dict(weights=5, noisy=71, clean=72)
CASES = {  # golden name: (args name in improved_fullsubnet_oracle, clips, samples, steps)
    "train_imp": ("DEFAULT_IMPROVED_ARGS", 3, 8000, 2),
    "train_imp_960": ("ARGS_48K_960", 2, 12000, 1),
}


def fingerprint(y: torch.Tensor) -> np.ndarray:
    a = y.numpy().astype(np.float64)
    return np.concatenate([a.reshape(-1)[:8], [a.sum(), np.abs(a).sum()]])


def inputs(name: str = "train_imp"):
    from oracle import fullsubnet_oracle as O
    _, clips, samples, _ = CASES[name]
    noisy = O.make_noisy(clips, samples, seed=SEEDS["noisy"], speechlike=True)
    clean = 0.5 * O.make_noisy(clips, samples, seed=SEEDS["clean"], speechlike=True)
    return noisy, clean


def args_of(name: str) -> dict:
    from oracle import improved_fullsubnet_oracle as IO
    return dict(getattr(IO, CASES[name][0]))


def main():
    from make_golden import import_reference
    from oracle import improved_fullsubnet_oracle as IO
    import_reference()
    from improved_fullsubnet.model import Model as ImpModel
    torch.set_num_threads(8)
    for name, (_, _, _, steps) in CASES.items():
        args = args_of(name)
        model = ImpModel(**args).train()
        assert [k for k, _ in IO.improved_state_dict_shapes(args)] == list(model.state_dict().keys())
        model.load_state_dict(IO.make_improved_state_dict(seed=SEEDS["weights"], args=args), strict=True)
        opt = torch.optim.Adam(model.parameters(), lr=1e-3, betas=(0.9, 0.999))
        loss_fn = torch.nn.MSELoss()
        noisy, clean = inputs(name)
        out = {"noisy_fp": fingerprint(noisy), "clean_fp": fingerprint(clean)}
        loss, gnorm = [], []
        for it in range(steps):
            opt.zero_grad()
            enhanced = model(noisy)
            l = loss_fn(enhanced, clean.unsqueeze(1))
            l.backward()
            if it == 0:
                out["enhanced"] = enhanced.detach().numpy().copy()
                for k, p in model.named_parameters():
                    g = p.grad.detach().numpy()
                    out["gsub." + k] = g.reshape(-1)[::SUBSAMPLE].copy()
                    out["gl2." + k] = np.array(np.sqrt((g.astype(np.float64) ** 2).sum()))
            loss.append(float(l.detach()))
            gnorm.append(float(torch.nn.utils.clip_grad_norm_(model.parameters(), 10)))
            opt.step()
            if steps > 1:
                for k, p in model.named_parameters():  # after step 0 sparser: the file stays under 1 MB
                    out[f"p{it}." + k] = p.detach().numpy().reshape(-1)[::SUBSAMPLE * (4 if it == 0 else 1)].copy()
        out["loss"], out["gnorm"] = np.array(loss), np.array(gnorm)
        print(name, "loss", loss, "gnorm", gnorm)
        path = os.path.join(ROOT, "tests", "golden", name + ".npz")
        np.savez_compressed(path, **out)
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
