"""bench_fbb_train.py - fullband_baseline TRAINING step on one GPU (the recipe fullband_baseline/train.toml: batch 100 x 3.072 s
clips, F = 257, H = 512, 3 LSTM layers, look_ahead 2, offline norm, cIRM MSE loss, clip 10 + Adam 1e-3).  Prints one JSON
line.

One "step" = Trainer.train_step (fullband_baseline/trainer.py:32-71): STFT of noisy + clean -> cIRM target -> Model.forward
(T = 193 frames, Tp = 195 with look-ahead) -> MSE -> backward (BPTT in libfsn_b200) -> FusedClipAdam.  Both training
precisions are measured (fp32 and tf32_tc), each after its own warm-up; device time from CUDA events with a 256 MiB write
between timed steps (no L2 reuse across steps).  Algorithmic work per step = 3 x forward = 3 * 100 * 195 * 12.06 MFLOP =
0.71 TFLOP (forward FLOPs per frame: LSTM 2 * 4H * (F + H) + 2 * 2 * 4H * 2H, Linear 2 * 2F * H).
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

SR, N_FFT, HOP, WIN = 16000, 512, 256, 512
SAMPLES = 49152  # 3.072 s (train.toml: sub_sample_length)
F, H = 257, 512
FLOP_FWD_PER_FRAME = 2 * 4 * H * (F + H) + 2 * (2 * 4 * H * 2 * H) + 2 * 2 * F * H  # 12.06 M


def power_limit_w(index: int):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(index)],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:  # noqa: BLE001 - reported as unknown
        return None


def measure(prec, B, steps, warmup, dev, flush, save_dir):
    from fullsubnet_b200 import _lib
    from fullsubnet_b200.acoustics.feature import stft
    from fullsubnet_b200.acoustics.mask import build_complex_ideal_ratio_mask
    from fullsubnet_b200.fullband_baseline.model import Model
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.optim import FusedClipAdam
    from fullsubnet_b200.trainer import Trainer
    from oracle import fullband_baseline_oracle as BO
    from oracle import fullsubnet_oracle as O  # weights / inputs generator only
    lib = _lib.load()
    args = dict(BO.DEFAULT_FBB_ARGS)
    model = Model(**args)
    model.load_state_dict(BO.make_fbb_state_dict(seed=0, args=args), strict=True)
    model.train_precision = prec
    model = model.to(dev).train()
    cfg = {"meta": {"use_amp": True, "save_dir": save_dir, "experiment_name": "bench"},
           "acoustics": {"n_fft": N_FFT, "hop_length": HOP, "win_length": WIN},
           "trainer": {"train": {"epochs": 1, "save_checkpoint_interval": 1, "clip_grad_norm_value": 10}}}
    trainer = Trainer(None, dev.index or 0, cfg, False, False, model, mse_loss(), FusedClipAdam(model.parameters(), lr=1e-3),
                      None, None)
    noisy = O.make_noisy(B, SAMPLES, seed=0, speechlike=True).to(dev)
    clean = (0.5 * O.make_noisy(B, SAMPLES, seed=100, speechlike=True)).to(dev)
    T = 1 + SAMPLES // HOP
    for _ in range(warmup):
        trainer.train_step(noisy, clean)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    total = 0.0
    for _ in range(steps):  # the flush write is outside the timed window
        flush.zero_()
        ev0.record()
        loss = trainer.train_step(noisy, clean)
        ev1.record()
        torch.cuda.synchronize()
        total += ev0.elapsed_time(ev1)
    ms = total / steps
    # forward / backward split of one step (same inputs, its own events)
    nm, _, nr, ni = stft(noisy, N_FFT, HOP, WIN)
    _, _, cr, ci = stft(clean, N_FFT, HOP, WIN)
    cirm = build_complex_ideal_ratio_mask(nr, ni, cr, ci)
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    flush.zero_()
    e[0].record()
    out = model(nm.unsqueeze(1))
    e[1].record()
    mse_loss()(cirm, out.permute(0, 2, 3, 1)).backward()
    e[2].record()
    torch.cuda.synchronize()
    n0 = lib.fsn_total_launch_count()
    trainer.train_step(noisy, clean)
    torch.cuda.synchronize()
    launches = int(lib.fsn_total_launch_count() - n0)
    d = model._desc(_lib.PREC[model._resolve_train_precision()])
    ws = int(lib.fsn_fullband_train_workspace_bytes(C.byref(d), B, T))
    flops = 3.0 * B * (T + args["look_ahead"]) * FLOP_FWD_PER_FRAME
    res = {"ms_per_step": ms, "frames_per_sec": B * T / (ms * 1e-3), "fwd_ms": e[0].elapsed_time(e[1]),
           "fwd_bwd_ms": e[0].elapsed_time(e[2]), "gpu_launches": launches, "workspace_bytes": ws,
           "tflops": flops / (ms * 1e-3) / 1e12, "loss": float(loss)}
    del trainer, model, out, noisy, clean
    torch.cuda.empty_cache()
    return res, T, flops


def main():
    import tempfile
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=100)
    a = ap.parse_args()
    assert a.gpus == 1, "bench_fbb_train.py measures one GPU"
    dev = torch.device("cuda", torch.cuda.current_device())
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    res = {}
    with tempfile.TemporaryDirectory(prefix="fsn_bench_fbb_") as save_dir:  # the Trainer's (unused) checkpoint directory
        for prec in ("fp32", "tf32_tc"):
            res[prec], T, flops = measure(prec, a.batch, a.steps, a.warmup, dev, flush, save_dir)
    best = res["tf32_tc"]
    print(json.dumps({
        "metric": "frames_per_sec", "value": best["frames_per_sec"], "unit": "frames/s", "n_gpus": 1, "steps": a.steps,
        "warmup": a.warmup, "ms_per_step": best["ms_per_step"], "higher_is_better": True,
        "config": {"workload": f"fullband_baseline training step (train.toml), batch={a.batch} x 3.072 s synthetic clips, "
                               f"T={T}, Trainer.train_step + FusedClipAdam",
                   "flops_per_step": flops, "l2": "256 MiB flush write between timed steps"},
        "precisions": res,
        "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index or 0)}))


if __name__ == "__main__":
    main()
