"""bench_fast_cum.py - cost of fast_fullsubnet's cumulative_laplace_norm against the offline norm on one GPU.  Prints one
JSON line.

Two workloads, each timed for both norms, the two norms alternating round by round in one process (the spread between
rounds is reported with the medians):
  inference  BASELINE config 4: Model.forward on the noisy magnitude of 512 x 4 s clips (T = 251 frames), default
             precision ("auto" = f16x3_tc)
  training   the recipe's step (train_shrinkSize2.toml): 72 x 3.072 s clips (T = 193), Model.forward in train mode + MSE
             against the cIRM + backward + FusedClipAdam, tf32_tc
Device time from CUDA events around each step, a 256 MiB write between timed steps (no L2 reuse across steps).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

os.environ.setdefault("PYTORCH_CUDA_ALLOC_CONF", "expandable_segments:True")
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

N_FFT, HOP, WIN = 512, 256, 512
NORMS = ("offline_laplace_norm", "cumulative_laplace_norm")


def power_limit_w(index: int):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(index)],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:  # noqa: BLE001 - reported as unknown
        return None


def build(norm, dev, train_precision=None):
    from fullsubnet_b200.fast_fullsubnet.model import Model
    from oracle import fast_fullsubnet_oracle as FO
    args = dict(FO.DEFAULT_FAST_ARGS, norm_type=norm)
    m = Model(**args)
    m.load_state_dict(FO.make_fast_state_dict(seed=0, args=args), strict=True)
    if train_precision:
        m.train_precision = train_precision
        return m.to(dev).train()
    return m.to(dev).eval()


def spectra(B, samples, dev):
    from fullsubnet_b200.acoustics.feature import stft
    from fullsubnet_b200.acoustics.mask import build_complex_ideal_ratio_mask
    from oracle import fullsubnet_oracle as O  # inputs generator only
    noisy = O.make_noisy(B, samples, seed=0, speechlike=True).to(dev)
    clean = (0.5 * O.make_noisy(B, samples, seed=100, speechlike=True)).to(dev)
    nm, _, nr, ni = stft(noisy, N_FFT, HOP, WIN)
    _, _, cr, ci = stft(clean, N_FFT, HOP, WIN)
    return nm.unsqueeze(1), build_complex_ideal_ratio_mask(nr, ni, cr, ci)


def timed(fn, steps, flush):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    total = 0.0
    for _ in range(steps):
        flush.zero_()
        ev0.record()
        fn()
        ev1.record()
        torch.cuda.synchronize()
        total += ev0.elapsed_time(ev1)
    return total / steps


def compare(make_step, rounds, steps, warmup, flush):
    """make_step(norm) -> a callable running one step; the norms alternate within every round."""
    fns = {n: make_step(n) for n in NORMS}
    for n in NORMS:
        for _ in range(warmup):
            fns[n]()
    torch.cuda.synchronize()
    ms = {n: [] for n in NORMS}
    for _ in range(rounds):
        for n in NORMS:
            ms[n].append(timed(fns[n], steps, flush))
    res = {n: {"ms_median": statistics.median(v), "ms_min": min(v), "ms_max": max(v)} for n, v in ms.items()}
    off, cum = res[NORMS[0]]["ms_median"], res[NORMS[1]]["ms_median"]
    res["cumulative_over_offline"] = cum / off
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--infer-batch", type=int, default=512)
    ap.add_argument("--train-batch", type=int, default=72)
    a = ap.parse_args()
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.optim import FusedClipAdam
    dev = torch.device("cuda", torch.cuda.current_device())
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    mag, _ = spectra(a.infer_batch, 64000, dev)  # 4 s: T = 251

    def infer_step(norm):
        m = build(norm, dev)

        def step():
            with torch.no_grad():
                m(mag)
        return step

    infer = compare(infer_step, a.rounds, a.steps, a.warmup, flush)
    infer["precision"] = build(NORMS[0], dev)._resolve_precision()
    del mag
    torch.cuda.empty_cache()

    nm, cirm = spectra(a.train_batch, 49152, dev)  # 3.072 s: T = 193

    def train_step(norm):
        m = build(norm, dev, "tf32_tc")
        opt, loss_fn = FusedClipAdam(m.parameters(), lr=1e-3, max_norm=10.0), mse_loss()

        def step():
            opt.zero_grad()
            loss_fn(cirm, m(nm).permute(0, 2, 3, 1)).backward()
            opt.step()
        return step

    train = compare(train_step, a.rounds, a.steps, a.warmup, flush)
    train["precision"] = "tf32_tc"
    print(json.dumps({
        "workloads": {
            "inference": dict(infer, shape=f"{a.infer_batch} x 4 s (T = 251), Model.forward on the noisy magnitude"),
            "training": dict(train, shape=f"{a.train_batch} x 3.072 s (T = 193), forward + MSE + backward + FusedClipAdam"),
        },
        "rounds": a.rounds, "steps_per_round": a.steps, "warmup": a.warmup,
        "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index or 0)}))


if __name__ == "__main__":
    main()
