"""bench_valid.py - one validation epoch (Trainer._validation_epoch) on one GPU: the B = 1 loop of the reference against
the grouped path.  Prints one JSON line per (model, item set), then one summary line with the card.

Item sets (16 kHz, seeded, clean speech-like signal plus noise; the dataloader yields B = 1 items from host memory):
  dns10s   150 "With_reverb" + 150 "No_reverb" clips of 10 s, the shape of the DNS synthetic test set the recipes
           validate on;
  mixed    300 clips of distinct lengths uniform in 1 - 10 s.

Models: fullsubnet (inference.toml arguments, weights W-a, the default precision "auto": f16x3_tc), fullband_baseline
(full-size arguments, fp32) and fast_fullsubnet (its default arguments; equal-length groups only).

"loop" is the per-item body that _validation_epoch ran before it was grouped (two STFTs, cIRM, Model.forward at B = 1,
MSE, decompress, complex product, iSTFT, SI-SDR, per item), kept here as the baseline.  "grouped" is
Trainer._validation_epoch with [trainer.validation] batch_size / max_padding at their defaults.  The two are timed
alternately, --rounds times each, host clock around the whole epoch (which ends in a device-to-host copy); the medians
and the ranges are reported, and the per-type losses of the two must agree to 1e-6 relative, the scores to 1e-3 dB.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

SR = 16000
N_FFT, HOP, WIN = 512, 256, 512


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001 - reported as unknown
        return {"name": torch.cuda.get_device_name(), "power_limit": f"not read ({type(e).__name__})"}


def items(which: str, n: int, seed: int):
    from oracle import fullsubnet_oracle as O
    rng = np.random.default_rng(seed)
    if which == "dns10s":
        lens = [10 * SR] * n
    else:
        lens = (rng.permutation(9 * SR + 1)[:n] + SR).tolist()
    base = O.make_noisy(n, 10 * SR, seed=seed, speechlike=True) * 0.5
    out = []
    for i, L in enumerate(lens):
        clean = base[i:i + 1, :L].clone()
        noisy = clean + torch.from_numpy(0.05 * rng.standard_normal((1, L)).astype(np.float32))
        out.append((noisy, clean, [f"clip{i}"], ["With_reverb" if i < n // 2 else "No_reverb"]))
    return out


def make_model(name: str, dev):
    if name == "fullsubnet":
        from fullsubnet_b200.fullsubnet.model import Model
        from oracle import fullsubnet_oracle as O
        m = Model(**O.DEFAULT_MODEL_ARGS)
        m.load_state_dict(O.make_state_dict(seed=0), strict=True)
    elif name == "fullband_baseline":
        from fullsubnet_b200.fullband_baseline.model import Model
        from oracle import fullband_baseline_oracle as BO
        m = Model(**BO.DEFAULT_FBB_ARGS)
        m.load_state_dict(BO.make_fbb_state_dict(seed=11), strict=True)
    else:
        from fullsubnet_b200.fast_fullsubnet.model import Model
        from oracle import fast_fullsubnet_oracle as FO
        m = Model(**FO.DEFAULT_FAST_ARGS)
        m.load_state_dict(FO.make_fast_state_dict(seed=0), strict=True)
    return m.to(dev)


@torch.no_grad()
def loop_epoch(tr):
    """The per-item validation loop the Trainer ran before grouping (the reference's B = 1 loop on the device)."""
    from fullsubnet_b200.acoustics.mask import build_complex_ideal_ratio_mask, decompress_cIRM
    from fullsubnet_b200.trainer import si_sdr
    types = ("With_reverb", "No_reverb")
    zero = lambda: torch.zeros((), device=tr.device)  # noqa: E731
    loss_total, n_items = zero(), 0
    loss_list = {k: zero() for k in types}
    score_list = {k: zero() for k in types}
    count = {k: 0 for k in types}
    model = tr.core
    was_training = model.training
    model.eval()
    for noisy, clean, name, speech_type in tr.valid_dataloader:
        speech_type = speech_type[0]
        noisy = noisy.to(tr.device, non_blocking=True)
        clean = clean.to(tr.device, non_blocking=True)
        noisy_mag, _, noisy_real, noisy_imag = tr.torch_stft(noisy)
        _, _, clean_real, clean_imag = tr.torch_stft(clean)
        cIRM = build_complex_ideal_ratio_mask(noisy_real, noisy_imag, clean_real, clean_imag)
        cRM = model(noisy_mag.unsqueeze(1)).permute(0, 2, 3, 1)
        loss = tr.loss_function(cIRM, cRM)
        cRM = decompress_cIRM(cRM)
        enhanced_real = cRM[..., 0] * noisy_real - cRM[..., 1] * noisy_imag
        enhanced_imag = cRM[..., 1] * noisy_real + cRM[..., 0] * noisy_imag
        enhanced = tr.torch_istft((enhanced_real, enhanced_imag), length=noisy.size(-1), input_type="real_imag")
        loss_total += loss
        n_items += 1
        loss_list[speech_type] += loss
        score_list[speech_type] += si_sdr(clean, enhanced)[0]
        count[speech_type] += 1
    model.train(was_training)
    n = max(1, n_items)
    return {"loss_total": float(loss_total) / n, "loss": {k: float(loss_list[k]) / n for k in types},
            "si_sdr": {k: (float(score_list[k]) / count[k] if count[k] else 0.0) for k in types}}


def grouped_epoch(tr):
    tr._validation_epoch(1)
    return tr.last_validation


def timed(fn, tr):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn(tr)  # ends in a device-to-host copy of the results
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="fullsubnet,fullband_baseline,fast_fullsubnet")
    ap.add_argument("--sets", default="dns10s,mixed")
    ap.add_argument("--items", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_valid.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.trainer import Trainer
    sets = {s: items(s, args.items, seed=1 + k) for k, s in enumerate(args.sets.split(","))}
    for name in args.models.split(","):
        model = make_model(name, dev)
        for s, its in sets.items():
            cfg = {"meta": {"use_amp": False, "save_dir": "/nonexistent", "experiment_name": "bench_valid"},
                   "acoustics": {"n_fft": N_FFT, "hop_length": HOP, "win_length": WIN},
                   "trainer": {"train": {"epochs": 1, "save_checkpoint_interval": 1, "clip_grad_norm_value": 10},
                               "validation": {"validation_interval": 1, "save_max_metric_score": True}}}
            tr = Trainer(None, 0, cfg, False, False, model, mse_loss(), torch.optim.SGD(model.parameters(), lr=0.0), [],
                         its)
            times = {"loop": [], "grouped": []}
            res = {}
            for r in range(args.rounds + 1):  # round 0 warms both up
                for which, fn in (("loop", loop_epoch), ("grouped", grouped_epoch)):
                    dt, res[which] = timed(fn, tr)
                    if r:
                        times[which].append(dt)
            a, b = res["loop"], res["grouped"]
            assert abs(a["loss_total"] - b["loss_total"]) <= 1e-6 * abs(a["loss_total"]), (a, b)
            for k in a["si_sdr"]:
                assert abs(a["si_sdr"][k] - b["si_sdr"][k]) <= 1e-3, (a, b)
            med = {k: float(np.median(v)) for k, v in times.items()}
            print(json.dumps({
                "model": name, "set": s, "items": len(its), "seconds_of_audio": sum(x[0].shape[-1] for x in its) / SR,
                "loop_s": round(med["loop"], 4), "loop_range_s": [round(min(times["loop"]), 4), round(max(times["loop"]), 4)],
                "grouped_s": round(med["grouped"], 4),
                "grouped_range_s": [round(min(times["grouped"]), 4), round(max(times["grouped"]), 4)],
                "speedup": round(med["loop"] / med["grouped"], 2),
                "batch_size": tr.validation_batch_size, "max_padding": tr.validation_max_padding,
                "loss_total": b["loss_total"], "si_sdr_with_reverb": b["si_sdr"]["With_reverb"]}), flush=True)
        del model
        torch.cuda.empty_cache()
    print(json.dumps({"card": card(), "rounds": args.rounds}))


if __name__ == "__main__":
    main()
