"""bench_data.py - the training data path at the recipes' shapes: fullsubnet_b200.dataset.Dataset on the host, the mixing
(fsn_rir_convolve + fsn_snr_mix) on the device, and the fullsubnet training step fed by it.

The corpus is synthetic, seeded and written to a temporary directory: int16 wav files at 16 kHz (clean 4-8 s, noise
1-10 s, RIRs 0.25-1 s, a quarter of them 2-channel), the args of fullsubnet/train.toml (3.072 s crops, SNR -5..20,
75 % reverberant, 0.2 s silences, -25 +- 10 dBFS).  Three measurements, printed as one JSON line:

* host: ms per item of ``Dataset.__getitem__`` (file reads, crops and draws; one process, like one DataLoader worker),
  against the CPU arithmetic the reference's worker does on the same items (``scipy.signal.fftconvolve`` with the RIR +
  ``oracle/mix_oracle.snr_mix``);
* device: ms per batch of 32 of the mixing on device-resident batches (CUDA events), on the corpus's batches and on the
  worst case, every reverberant row with a 1 s RIR;
* step: the fullsubnet training step (recipe model, default precision) per batch of 32, fed by collated Dataset batches
  from host memory (H2D + mixing inside), by the same batches pre-mixed in host memory, and pre-mixed on the device.

Usage: python bench_data.py [--steps K] [--warmup W] [--items N]
"""
from __future__ import annotations

import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import time
import wave

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

SR, B = 16000, 32
ARGS = dict(clean_dataset_limit=False, clean_dataset_offset=0, noise_dataset_limit=False, noise_dataset_offset=0,
            rir_dataset_limit=False, rir_dataset_offset=0, snr_range=[-5, 20], reverb_proportion=0.75,
            silence_length=0.2, target_dB_FS=-25, target_dB_FS_floating_value=10, sub_sample_length=3.072, sr=SR,
            pre_load_clean_dataset=False, pre_load_noise=False, pre_load_rir=False, num_workers=4)


def write_wav(path, y):
    y = np.atleast_2d(y)
    with wave.open(path, "wb") as f:
        f.setnchannels(y.shape[0])
        f.setsampwidth(2)
        f.setframerate(SR)
        f.writeframes(np.ascontiguousarray(np.clip(np.round(y * 32768), -32768, 32767).astype("<i2").T).tobytes())


def write_corpus(root, n_clean=96, n_noise=24, n_rir=16, seed=0):
    rng = np.random.default_rng(seed)
    lists = {"clean": [], "noise": [], "rir": []}
    for i in range(n_clean):
        n = int(rng.integers(4 * SR, 8 * SR))
        t = np.arange(n) / SR
        y = 0.2 * np.sin(2 * np.pi * rng.uniform(100, 400) * t) * (0.6 + 0.4 * np.sin(2 * np.pi * 3 * t))
        lists["clean"].append(os.path.join(root, f"c{i}.wav"))
        write_wav(lists["clean"][-1], y + 0.01 * rng.standard_normal(n))
    for i in range(n_noise):
        lists["noise"].append(os.path.join(root, f"n{i}.wav"))
        write_wav(lists["noise"][-1], 0.2 * rng.standard_normal(int(rng.integers(1 * SR, 10 * SR))))
    for i in range(n_rir):
        n = SR if i == 0 else int(rng.integers(SR // 4, SR + 1))
        c = 2 if i % 4 == 3 else 1
        r = 0.3 * rng.standard_normal((c, n)) * np.exp(-np.arange(n) / (n / 6.0))
        r[:, 0] = 0.9
        lists["rir"].append(os.path.join(root, f"r{i}.wav"))
        write_wav(lists["rir"][-1], r)
    args = dict(ARGS)
    for k, paths in lists.items():
        args[f"{k}_dataset"] = os.path.join(root, f"{k}.txt")
        with open(args[f"{k}_dataset"], "w") as f:
            f.write("\n".join(paths) + "\n")
    return args


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power, clock = [s.strip() for s in out.stdout.strip().split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001 - the card name from torch is still worth reporting
        return {"name": torch.cuda.get_device_name(), "power_limit": f"not read ({type(e).__name__})"}


def host_costs(ds, n_items):
    """ms per item: Dataset.__getitem__, and the reference's CPU arithmetic (fftconvolve + snr_mix) on its output."""
    from scipy import signal

    from oracle.mix_oracle import snr_mix
    random.seed(1)
    np.random.seed(1)
    items, t0 = [], time.perf_counter()
    for i in range(n_items):
        items.append(ds[i % len(ds)])
    t_item = (time.perf_counter() - t0) / n_items
    t0 = time.perf_counter()
    for it in items:
        clean = it["clean"]
        n = int(it["rir_len"])
        if n:
            clean = signal.fftconvolve(clean, it["rir"][:n])[:len(clean)]
        snr_mix(clean, it["noise"], float(it["snr"]), -25, float(it["noisy_target_dB_FS"]))
    t_mix = (time.perf_counter() - t0) / n_items
    return t_item, t_mix


def events_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--items", type=int, default=64)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_data.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    from torch.utils.data import DataLoader

    from fullsubnet_b200.dataset import Dataset, mix_batch
    from fullsubnet_b200.fullsubnet.model import Model
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.optim import FusedClipAdam
    from fullsubnet_b200.trainer import Trainer
    from oracle import fullsubnet_oracle as O

    with tempfile.TemporaryDirectory() as tmp:
        ds = Dataset(**write_corpus(tmp))
        t_item, t_mix = host_costs(ds, a.items)
        random.seed(0)
        np.random.seed(0)
        n_batches = max(2, min(4, a.steps))
        loader = DataLoader(ds, batch_size=B, shuffle=True, num_workers=0, drop_last=True)
        batches = [b for _, b in zip(range(n_batches), loader)]
    L = batches[0]["clean"].shape[1]

    # device mixing, batches resident on the device
    dev_batches = [{k: v if k == "target_dB_FS" else v.to(dev) for k, v in b.items()} for b in batches]
    worst = dict(dev_batches[0])
    rl = torch.zeros(B, dtype=torch.int32)
    rl[:B * 3 // 4] = SR
    worst["rir_len"] = rl.to(dev)
    worst["rir"] = torch.randn(B, SR, generator=torch.Generator().manual_seed(3)).mul_(0.05).to(dev)
    it = iter(range(1 << 30))
    ms_mix = events_ms(lambda: mix_batch(dev_batches[next(it) % len(dev_batches)], dev), 5 * a.steps, a.warmup)
    ms_mix_worst = events_ms(lambda: mix_batch(worst, dev), 5 * a.steps, a.warmup)
    rir_rows = [int((b["rir_len"] > 0).sum()) for b in batches]
    rir_taps = [float(b["rir_len"][b["rir_len"] > 0].float().mean()) for b in batches]

    # the training step
    model = Model(**dict(O.DEFAULT_MODEL_ARGS, weight_init=False))
    model.load_state_dict(O.make_state_dict(seed=0), strict=True)
    model = model.to(dev).train()
    cfg = {"meta": {"use_amp": False, "save_dir": tempfile.gettempdir(), "experiment_name": "bench_data"},
           "acoustics": {"n_fft": 512, "hop_length": 256, "win_length": 512},
           "trainer": {"train": {"epochs": 1, "save_checkpoint_interval": 1, "clip_grad_norm_value": 10}}}
    tr = Trainer(None, 0, cfg, False, False, model, mse_loss(), FusedClipAdam(model.parameters(), lr=1e-3), None, None)
    premixed_dev = [mix_batch(b, dev) for b in batches]
    premixed_host = [(n.cpu(), c.cpu()) for n, c in premixed_dev]
    k = iter(range(1 << 30))
    steps = {
        "dataset_batch_from_host": lambda: tr.train_step(batches[next(k) % len(batches)]),
        "premixed_from_host": lambda: tr.train_step(*premixed_host[next(k) % len(batches)]),
        "premixed_on_device": lambda: tr.train_step(*premixed_dev[next(k) % len(batches)]),
    }
    ms_step = {name: [] for name in steps}
    for _ in range(2):  # alternate the three feeds, twice
        for name, fn in steps.items():
            ms_step[name].append(events_ms(fn, a.steps, a.warmup))
    ms_step = {name: min(v) for name, v in ms_step.items()}
    share = ms_mix / ms_step["premixed_on_device"]
    print(json.dumps({
        "metric": "ms_per_batch", "card": card(), "host_cores": os.cpu_count(), "batch": B, "clip_samples": L,
        "precision": model._resolve_train_precision(),
        "host_ms_per_item": {"dataset_getitem": 1e3 * t_item, "reference_arithmetic_fftconvolve_snr_mix": 1e3 * t_mix,
                             "items": a.items},
        "device_mix_ms_per_batch": {"corpus_batches": ms_mix, "reverberant_rows": rir_rows,
                                    "mean_rir_taps": rir_taps, "worst_case_24_rows_1s_rir": ms_mix_worst},
        "step_ms": ms_step, "mix_share_of_step": share,
        "mix_share_of_step_worst_case": ms_mix_worst / ms_step["premixed_on_device"]}))


if __name__ == "__main__":
    main()
