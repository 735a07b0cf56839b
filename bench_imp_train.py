"""bench_imp_train.py - improved_fullsubnet TRAINING step on one GPU (16 kHz defaults of improved_fullsubnet/model.py:453-471:
n_fft 512 / hop 128, sections [0,20) [20,80) [80,256) with centre widths 1 / 4 / 8 and 15 neighbours, fb_hidden 512,
sb_hidden 384, LSTM, offline norm).  Prints one JSON line.

Upstream ships no trainer for this model, so one "step" is the simplest wav-domain loop a user writes around the
differentiable module: Model.forward (wav -> enhanced wav, T = 385 frames per 3.072 s clip) -> torch.nn.MSELoss against the
clean wav -> backward (iSTFT adjoint and BPTT in libfsn_b200) -> FusedClipAdam (clip 10, Adam 1e-3).  Both training
precisions are measured (fp32 and tf32_tc), each after its own warm-up; device time from CUDA events with a 256 MiB write
between timed steps (no L2 reuse across steps).  Algorithmic work per step = 3 x forward = 3 * B * T * 221.79 MFLOP
(SURVEY 8d: forward FLOPs per frame of the default model).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

os.environ.setdefault("PYTORCH_CUDA_ALLOC_CONF", "expandable_segments:True")
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

SAMPLES = 49152  # 3.072 s at 16 kHz
HOP = 128
FLOP_FWD_PER_FRAME = 221.79e6


def power_limit_w(index: int):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(index)],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:  # noqa: BLE001 - reported as unknown
        return None


def measure(prec, B, steps, warmup, dev, flush):
    from fullsubnet_b200 import _lib
    from fullsubnet_b200.improved_fullsubnet.model import Model
    from fullsubnet_b200.optim import FusedClipAdam
    from oracle import fullsubnet_oracle as O  # inputs generator only
    from oracle import improved_fullsubnet_oracle as IO  # weights generator only
    lib = _lib.load()
    args = dict(IO.DEFAULT_IMPROVED_ARGS)
    model = Model(**args)
    model.load_state_dict(IO.make_improved_state_dict(seed=0, args=args), strict=True)
    model.train_precision = prec
    model = model.to(dev).train()
    opt = FusedClipAdam(model.parameters(), lr=1e-3, max_norm=10.0)
    loss_fn = torch.nn.MSELoss()
    noisy = O.make_noisy(B, SAMPLES, seed=0, speechlike=True).to(dev)
    clean = (0.5 * O.make_noisy(B, SAMPLES, seed=100, speechlike=True)).to(dev).unsqueeze(1)
    T = 1 + SAMPLES // HOP

    def step():
        opt.zero_grad(set_to_none=False)
        loss = loss_fn(model(noisy), clean)
        loss.backward()
        opt.step()
        return loss

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    total = 0.0
    for _ in range(steps):  # the flush write is outside the timed window
        flush.zero_()
        ev0.record()
        loss = step()
        ev1.record()
        torch.cuda.synchronize()
        total += ev0.elapsed_time(ev1)
    ms = total / steps
    # forward / backward split of one step (same inputs, its own events)
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    flush.zero_()
    opt.zero_grad(set_to_none=False)
    e[0].record()
    out = model(noisy)
    e[1].record()
    loss_fn(out, clean).backward()
    e[2].record()
    torch.cuda.synchronize()
    n0 = lib.fsn_total_launch_count()
    step()
    torch.cuda.synchronize()
    launches = int(lib.fsn_total_launch_count() - n0)
    d = model._train_desc()
    ws = int(lib.fsn_improved_train_workspace_bytes(C.byref(d), B, SAMPLES))
    flops = 3.0 * B * T * FLOP_FWD_PER_FRAME
    res = {"ms_per_step": ms, "frames_per_sec": B * T / (ms * 1e-3), "fwd_ms": e[0].elapsed_time(e[1]),
           "fwd_bwd_ms": e[0].elapsed_time(e[2]), "gpu_launches": launches, "workspace_bytes": ws,
           "tflops": flops / (ms * 1e-3) / 1e12, "loss": float(loss.detach())}
    del opt, model, out, noisy, clean
    torch.cuda.empty_cache()
    return res, T, flops


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=32)
    a = ap.parse_args()
    assert a.gpus == 1, "bench_imp_train.py measures one GPU"
    dev = torch.device("cuda", torch.cuda.current_device())
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    res = {}
    for prec in ("fp32", "tf32_tc"):
        res[prec], T, flops = measure(prec, a.batch, a.steps, a.warmup, dev, flush)
    best = res["tf32_tc"]
    print(json.dumps({
        "metric": "frames_per_sec", "value": best["frames_per_sec"], "unit": "frames/s", "n_gpus": 1, "steps": a.steps,
        "warmup": a.warmup, "ms_per_step": best["ms_per_step"], "higher_is_better": True,
        "config": {"workload": f"improved_fullsubnet training step (16 kHz defaults), batch={a.batch} x 3.072 s synthetic "
                               f"clips, T={T}, forward + MSE on the waveform + backward + FusedClipAdam",
                   "flops_per_step": flops, "l2": "256 MiB flush write between timed steps"},
        "precisions": res,
        "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index or 0)}))


if __name__ == "__main__":
    main()
