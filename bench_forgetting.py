"""bench_forgetting.py - cost of fullsubnet's forgetting_norm against cumulative_laplace_norm on one GPU.  Prints one JSON
line.

One fullsubnet enhance call (wav -> wav, fsn_enhance) of 256 x 4 s clips (T = 251) with each norm, on each inference
precision (fp32, f16x3_tc, f16_tc); the two norms alternate round by round in one process and the spread between rounds
is reported with the medians.  Device time from CUDA events around each call, a 256 MiB write between timed calls (no
L2 reuse across calls).  The power limit and the SM clock are read with nvidia-smi queries and reported beside the times.
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

NORMS = ("cumulative_laplace_norm", "forgetting_norm")
PRECISIONS = ("fp32", "f16x3_tc", "f16_tc")


def smi(field: str, index: int):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={field}", "--format=csv,noheader,nounits", "-i", str(index)],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:  # noqa: BLE001 - reported as unknown
        return None


def build(norm, precision, dev):
    from fullsubnet_b200.fullsubnet.model import Model
    from oracle import fullsubnet_oracle as O
    args = dict(O.DEFAULT_MODEL_ARGS, norm_type=norm)
    m = Model(**args, precision=precision)
    m.load_state_dict(O.make_state_dict(seed=0, args=args), strict=True)
    return m.to(dev).eval()


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=256)
    a = ap.parse_args()
    from oracle import fullsubnet_oracle as O  # inputs generator only
    dev = torch.device("cuda", torch.cuda.current_device())
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    y = O.make_noisy(a.batch, 64000, seed=0, speechlike=True).to(dev)  # 4 s: T = 251
    res = {}
    for prec in PRECISIONS:
        fns = {}
        for n in NORMS:
            m = build(n, prec, dev)

            def step(m=m):
                with torch.no_grad():
                    m.enhance(y)
            fns[n] = step
        for n in NORMS:
            for _ in range(a.warmup):
                fns[n]()
        torch.cuda.synchronize()
        ms = {n: [] for n in NORMS}
        for _ in range(a.rounds):
            for n in NORMS:
                ms[n].append(timed(fns[n], a.steps, flush))
        r = {n: {"ms_median": statistics.median(v), "ms_min": min(v), "ms_max": max(v)} for n, v in ms.items()}
        r["forgetting_over_cumulative"] = r[NORMS[1]]["ms_median"] / r[NORMS[0]]["ms_median"]
        res[prec] = r
        del fns
        torch.cuda.empty_cache()
    idx = dev.index or 0
    print(json.dumps({
        "workload": f"fullsubnet fsn_enhance, {a.batch} x 4 s (T = 251), wav -> wav",
        "precisions": res, "rounds": a.rounds, "steps_per_round": a.steps, "warmup": a.warmup,
        "device": torch.cuda.get_device_name(dev), "power_limit_w": smi("power.limit", idx),
        "sm_clock_mhz": smi("clocks.sm", idx), "max_sm_clock_mhz": smi("clocks.max.sm", idx)}))


if __name__ == "__main__":
    main()
