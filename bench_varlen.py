"""bench_varlen.py - inference over clips of DIFFERENT lengths on one GPU.  Prints one JSON line.

Workload (--model fullsubnet, the default): a seeded set of --clips clips (default 1024) whose lengths are distinct and
uniform in 1 - 10 s at 16 kHz, the inference.toml model with weights W-a, the default precision ("auto": f16x3_tc),
wav -> enhanced wav + int16 PCM (what the file loop writes).  Two schedules of the same clips:

  exact       equal-length batches (``plan_batches(lengths, 256, 0)``): every length is distinct, so B = 1 per call
              (fsn_enhance with the int16 output), which is what the file loop does on real recordings by default;
  pad<x>      ``plan_batches(lengths, 256, x)``: length-sorted runs of <= 256 clips padded to their longest clip by at
              most a fraction x of the batch's samples, one fsn_enhance call with per-clip lengths per batch.

--model improved_fullsubnet --variant k16|k48|k48_960: the same schedules for improved_fullsubnet with bench.py's
constructor arguments and weights of that variant, the precision of --precision (default "auto": tf32_tc), clip
lengths distinct and uniform in 1 - 10 s at the variant's sample rate (16 or 48 kHz), fsn_improved_enhance for every
call.  On tf32_tc its sections launch kernels once per frame, and one call on a 10 s clip keeps every step's gates, so
the defaults are --clips 256 and --batch 64; f16x3_tc / f16_tc run each section in one launch and keep only the input
projection and layer 1's output of every step.

--model fullband_baseline: the same schedules and clips as fullsubnet for the paper's baseline (its full-size constructor
arguments, seed-11 weights, fp32), fsn_fullband_enhance for every call.  The JSON line also carries "per_call_64x10s":
the time of one call on 64 clips of 10 s (resident, null lengths).

Each schedule is timed twice with CUDA events around the whole schedule: "resident" (inputs already in HBM, outputs left
there) and "e2e" (pinned host float32 -> H2D -> call -> int16 D2H into pinned host memory, the file loop minus the wav
I/O).  Every clip's PCM of every schedule is compared with the exact schedule's, bit for bit.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

SR = 16000  # fullsubnet; improved_fullsubnet: the variant's rate
GAIN = 0.8 * 32767.0


def power_limit_w(index: int):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(index)],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:  # noqa: BLE001 - reported as unknown
        return None


def clip_lengths(n: int, seed: int, sr: int = SR):
    rng = np.random.default_rng(seed)
    return (rng.permutation(9 * sr + 1)[:n] + sr).tolist()  # distinct, uniform in [1 s, 10 s]


class Schedule:
    """The batches of one schedule with their staging buffers (device and pinned host), built outside the timing."""

    def __init__(self, name, plan, lens, clips, dev):
        self.name, self.plan, self.lens = name, plan, lens
        self.batches = []
        for idx in plan:
            L = max(lens[i] for i in idx)
            host = torch.zeros(len(idx), L, dtype=torch.float32).pin_memory()
            for r, i in enumerate(idx):
                host[r, :lens[i]] = clips[i]
            mixed = any(lens[i] != L for i in idx)
            self.batches.append(dict(idx=idx, L=L, lengths=[lens[i] for i in idx] if mixed else None, host=host,
                                     dev=host.to(dev), pcm_host=torch.empty(len(idx), L, dtype=torch.int16).pin_memory()))
        self.samples = sum(lens[i] for idx in plan for i in idx)
        self.padded = sum(len(b["idx"]) * b["L"] for b in self.batches)

    def run(self, m, e2e):
        outs = []
        for b in self.batches:
            x = b["host"].to(b["dev"].device, non_blocking=True) if e2e else b["dev"]
            pcm = m.enhance_pcm(x, gain=GAIN, lengths=b["lengths"])[1]
            if e2e:
                b["pcm_host"].copy_(pcm, non_blocking=True)
            outs.append(pcm)
        return outs


def time_schedule(m, s, e2e, reps):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        ev0.record()
        s.run(m, e2e)
        ev1.record()
        torch.cuda.synchronize()
        ms.append(ev0.elapsed_time(ev1))
    return ms


def make_model(a, dev):
    """(model, sample rate, workload description) of --model / --variant"""
    from oracle import fullsubnet_oracle as O  # weights / inputs generator only
    if a.model == "fullband_baseline":
        from fullsubnet_b200.fullband_baseline.model import Model as FbbModel
        from oracle import fullband_baseline_oracle as BO
        m = FbbModel(**BO.DEFAULT_FBB_ARGS)
        m.load_state_dict(BO.make_fbb_state_dict(seed=11), strict=True)
        return m.to(dev).eval(), SR, "fullband_baseline (F=257, H=512, 3 layers, offline norm), seed-11 weights"
    if a.model == "fullsubnet":
        from fullsubnet_b200.fullsubnet.model import Model
        m = Model(**O.DEFAULT_MODEL_ARGS)
        m.load_state_dict(O.make_state_dict(seed=0), strict=True)
        return m.to(dev).eval(), SR, "fullsubnet inference.toml, W-a"
    from fullsubnet_b200.improved_fullsubnet.model import Model as ImpModel
    from oracle import improved_fullsubnet_oracle as IO
    imp_args = {"k48": IO.ARGS_48K_1024, "k48_960": IO.ARGS_48K_960, "k16": IO.DEFAULT_IMPROVED_ARGS}[a.variant]
    m = ImpModel(**imp_args)  # the constructor arguments and weights of bench.py --variant
    m.load_state_dict(IO.make_improved_state_dict(seed=5, args=imp_args), strict=True)
    m.precision = a.precision
    sr = 16000 if a.variant == "k16" else 48000
    return m.to(dev).eval(), sr, (f"improved_fullsubnet {a.variant} (n_fft={imp_args['n_fft']}, "
                                  f"hop={imp_args['hop_length']})")


def per_call_ms(m, dev, reps):
    """Best-of-reps time of one enhance_pcm call on 64 clips of 10 s (null lengths, inputs and outputs in HBM)."""
    from oracle import fullsubnet_oracle as O  # inputs generator only
    x = O.make_noisy(64, 10 * SR, seed=64, speechlike=True).to(dev)
    m.enhance_pcm(x, gain=GAIN)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(max(reps, 3)):
        ev0.record()
        m.enhance_pcm(x, gain=GAIN)
        ev1.record()
        torch.cuda.synchronize()
        ms.append(ev0.elapsed_time(ev1))
    return {"ms": min(ms), "ms_all": ms}


def main():
    from fullsubnet_b200 import _lib
    from fullsubnet_b200.inferencer import plan_batches
    from oracle import fullsubnet_oracle as O  # weights / inputs generator only
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--model", default="fullsubnet", choices=["fullsubnet", "improved_fullsubnet", "fullband_baseline"])
    ap.add_argument("--variant", default="k48", choices=["k48", "k48_960", "k16"],
                    help="improved_fullsubnet constructor args (as bench.py --variant)")
    ap.add_argument("--precision", default="auto", choices=["auto", "fp32", "tf32_tc", "f16x3_tc", "f16_tc"],
                    help="improved_fullsubnet's precision (auto: tf32_tc)")
    ap.add_argument("--clips", type=int, default=None, help="default 1024 (fullsubnet), 256 (improved_fullsubnet)")
    ap.add_argument("--batch", type=int, default=None, help="default 256 (fullsubnet), 64 (improved_fullsubnet)")
    ap.add_argument("--max-padding", type=float, nargs="+", default=[0.05, 0.1, 0.25])
    ap.add_argument("--steps", type=int, default=1, help="timed repetitions of every schedule")
    ap.add_argument("--warmup", type=int, default=1, help="untimed repetitions of every schedule")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    improved = a.model == "improved_fullsubnet"
    assert improved or a.precision == "auto", "--precision applies to --model improved_fullsubnet"
    a.clips = a.clips or (256 if improved else 1024)
    a.batch = a.batch or (64 if improved else 256)
    assert a.gpus == 1, "bench_varlen.py measures one GPU"
    assert torch.cuda.is_available(), "bench_varlen.py needs a CUDA device"
    dev = torch.device("cuda", torch.cuda.current_device())
    lib = _lib.load()
    m, sr, what = make_model(a, dev)
    lens = clip_lengths(a.clips, a.seed, sr)
    noise = O.make_noisy(1, max(lens), seed=a.seed + 1, speechlike=True, sr=sr)[0]
    rng = np.random.default_rng(a.seed + 2)
    clips = [noise[int(rng.integers(0, max(lens) - L + 1)):][:L] * float(rng.uniform(0.3, 1.0)) for L in lens]

    schedules = [Schedule("exact", plan_batches(lens, a.batch, 0.0), lens, clips, dev)]
    for mp in a.max_padding:
        schedules.append(Schedule(f"pad{mp:g}", plan_batches(lens, a.batch, mp), lens, clips, dev))
    audio_s = sum(lens) / sr
    res, ref = {}, None
    for s in schedules:
        for _ in range(a.warmup):
            s.run(m, False)
        n0 = lib.fsn_total_launch_count()
        outs = s.run(m, False)
        torch.cuda.synchronize()
        launches = int(lib.fsn_total_launch_count() - n0)
        per_clip = {i: pcm[r, :lens[i]] for b, pcm in zip(s.batches, outs) for r, i in enumerate(b["idx"])}
        if ref is None:
            ref = per_clip
        identical = all(torch.equal(per_clip[i], ref[i]) for i in range(len(lens)))
        r = {"calls": len(s.batches), "max_batch": max(len(b["idx"]) for b in s.batches), "gpu_launches": launches,
             "padded_fraction": 1.0 - s.samples / s.padded, "pcm_identical_to_exact": identical}
        for mode in ("resident", "e2e"):
            ms = time_schedule(m, s, mode == "e2e", a.steps)
            best = min(ms)
            r[mode] = {"ms": best, "ms_all": ms, "clips_per_sec": len(lens) / (best * 1e-3),
                       "xRT": audio_s / (best * 1e-3)}
        res[s.name] = r
        del outs, per_clip
    best_name = max((n for n in res if n != "exact"), key=lambda n: res[n]["e2e"]["clips_per_sec"])
    best = res[best_name]
    config = {"workload": f"{a.clips} clips, distinct lengths uniform in 1-10 s at {sr // 1000} kHz ({audio_s:.0f} s of "
                          f"audio), {what}, wav -> enhanced + int16 PCM",
              "precision": m._resolve_precision(), "batch": a.batch, "seed": a.seed}
    extra = {}
    if improved:
        config.update(model=a.model, variant=a.variant)
    if a.model == "fullband_baseline":
        config.update(model=a.model)
        extra["per_call_64x10s"] = per_call_ms(m, dev, a.steps)
    print(json.dumps({
        "metric": "clips_per_sec", "value": best["e2e"]["clips_per_sec"], "unit": "clips/s", "n_gpus": 1,
        "steps": a.steps, "warmup": a.warmup, "higher_is_better": True, "best_schedule": best_name,
        "speedup_vs_exact_e2e": best["e2e"]["clips_per_sec"] / res["exact"]["e2e"]["clips_per_sec"],
        "speedup_vs_exact_resident": best["resident"]["clips_per_sec"] / res["exact"]["resident"]["clips_per_sec"],
        "config": config,
        "schedules": res, **extra,
        "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index or 0)}))


if __name__ == "__main__":
    main()
