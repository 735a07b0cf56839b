"""bench_stoi.py - STOI on one GPU (fsn_stoi) against the float64 host oracle, and the cost of STOI in a validation epoch.
Prints one JSON line per measurement, then one line with the card.

  fsn_stoi   300 clips of distinct lengths uniform in 1 - 10 s, and 300 clips of exactly 10 s (the DNS validation
             shape), 16 kHz, speech-like clean plus noise; CUDA events around --iters calls after --warmup calls.  Work
             and bytes are computed from the shapes (the resampler's taps, the DFT of bins 7 .. 218 of every frame, the
             segment correlations; float32 inputs read once, the float64 intermediates written and read once), with
             every frame counted as kept.
  oracle     oracle/stoi_oracle.py (float64 numpy / scipy, one process) on --oracle-clips clips of each set, scaled to
             300 clips.  It is this project's oracle, not pystoi.
  validation Trainer._validation_epoch in bench_valid.py's setup (fullsubnet, 300 x 10 s, defaults), with and without
             "STOI" in [trainer.visualization] metrics, alternated --rounds times, host clock around each epoch.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

SR = 16000


def clips(which: str, n: int, seed: int):
    from oracle.stoi_oracle import speechlike
    rng = np.random.default_rng(seed)
    lens = [10 * SR] * n if which == "dns10s" else (rng.permutation(9 * SR + 1)[:n] + SR).tolist()
    base = speechlike(10 * SR, seed=seed)
    out = []
    for i, L in enumerate(lens):
        x = np.roll(base, 997 * i)[:L] * np.float32(0.5 + rng.random())
        y = x + np.float32(0.05) * rng.standard_normal(L).astype(np.float32)
        out.append((x, y))
    return out


def work(lens):
    """(float64 multiply-adds, bytes) of one fsn_stoi call on clips of these lengths, from the shapes."""
    flops, nbytes = 0, 0
    for L in lens:
        Lr = -(-5 * L // 8)
        nf = max(0, -(-(Lr - 256) // 128))
        T = max(0, nf - 1)
        flops += 2 * Lr * (581 // 5 + 1)           # resampler: ~117 taps per output sample, two signals
        flops += nf * 256                           # frame energies
        flops += 2 * T * 212 * 256 * 2              # DFT of bins 7..218, re and im, two signals
        flops += max(0, T - 29) * 15 * 30 * 8       # segment correlations
        nbytes += 2 * 4 * L                         # float32 inputs
        nbytes += 2 * 8 * Lr * 2 + 2 * 8 * Lr * 2   # resampled and compacted, written and read
        nbytes += 2 * 8 * 15 * T * 2                # band magnitudes
    return flops, nbytes


def time_stoi(pairs, dev, warmup, iters):
    from fullsubnet_b200.metrics import stoi
    lens = [len(x) for x, _ in pairs]
    L = max(lens)
    c = torch.zeros(len(pairs), L)
    e = torch.zeros(len(pairs), L)
    for b, (x, y) in enumerate(pairs):
        c[b, :len(x)] = torch.from_numpy(x)
        e[b, :len(y)] = torch.from_numpy(y)
    c, e = c.to(dev), e.to(dev)
    lengths = lens if min(lens) != max(lens) else None
    for _ in range(warmup):
        out = stoi(c, e, lengths)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(iters):
        t0.record()
        out = stoi(c, e, lengths)
        t1.record()
        t1.synchronize()
        times.append(t0.elapsed_time(t1) / 1e3)
    return times, out.cpu().numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--oracle-clips", type=int, default=6)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-validation", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_stoi.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    from oracle import stoi_oracle as S
    for k, which in enumerate(("mixed", "dns10s")):
        pairs = clips(which, args.clips, seed=1 + k)
        times, out = time_stoi(pairs, dev, args.warmup, args.iters)
        lens = [len(x) for x, _ in pairs]
        flops, nbytes = work(lens)
        med = float(np.median(times))
        sub = pairs[:args.oracle_clips]
        t = time.perf_counter()
        ref = [S.stoi(x, y, SR) for x, y in sub]
        t_oracle = time.perf_counter() - t
        err = max(abs(float(out[i]) - ref[i]) for i in range(len(sub)))
        print(json.dumps({
            "what": "fsn_stoi", "set": which, "clips": len(pairs), "seconds_of_audio": sum(lens) / SR,
            "gpu_s": round(med, 5), "gpu_range_s": [round(min(times), 5), round(max(times), 5)],
            "float64_fma_per_call": flops, "bytes_per_call": nbytes,
            "achieved_fp64_gflops": round(2 * flops / med / 1e9, 1), "achieved_gb_s": round(nbytes / med / 1e9, 1),
            "oracle_host_s_scaled": round(t_oracle / len(sub) * len(pairs), 2), "oracle_clips_timed": len(sub),
            "worst_abs_vs_oracle": err, "mean_stoi": float(np.mean(out))}), flush=True)
    if not args.skip_validation:
        import bench_valid as BV
        from fullsubnet_b200.loss import mse_loss
        from fullsubnet_b200.trainer import Trainer
        model = BV.make_model("fullsubnet", dev)
        its = BV.items("dns10s", args.clips, seed=1)
        trainers = {}
        for name, metrics in (("without_stoi", None), ("with_stoi", ["WB_PESQ", "NB_PESQ", "STOI", "SI_SDR"])):
            trainer = {"train": {"epochs": 1, "save_checkpoint_interval": 1, "clip_grad_norm_value": 10},
                       "validation": {"validation_interval": 1, "save_max_metric_score": True}}
            if metrics:
                trainer["visualization"] = {"metrics": metrics}
            cfg = {"meta": {"use_amp": False, "save_dir": "/nonexistent", "experiment_name": "bench_stoi"},
                   "acoustics": {"n_fft": BV.N_FFT, "hop_length": BV.HOP, "win_length": BV.WIN}, "trainer": trainer}
            trainers[name] = Trainer(None, 0, cfg, False, False, model, mse_loss(),
                                     torch.optim.SGD(model.parameters(), lr=0.0), [], its)
        times = {k: [] for k in trainers}
        for r in range(args.rounds + 1):  # round 0 warms both up
            for name, tr in trainers.items():
                dt, _ = BV.timed(BV.grouped_epoch, tr)
                if r:
                    times[name].append(dt)
        a, b = trainers["without_stoi"].last_validation, trainers["with_stoi"].last_validation
        assert a["si_sdr"] == b["si_sdr"] and a["loss"] == b["loss"]
        med = {k: float(np.median(v)) for k, v in times.items()}
        print(json.dumps({
            "what": "validation_epoch", "model": "fullsubnet", "set": "dns10s", "items": len(its),
            **{f"{k}_s": round(v, 4) for k, v in med.items()},
            **{f"{k}_range_s": [round(min(v), 4), round(max(v), 4)] for k, v in times.items()},
            "stoi": b["stoi"]}), flush=True)
    from bench_valid import card
    print(json.dumps({"card": card()}))


if __name__ == "__main__":
    main()
