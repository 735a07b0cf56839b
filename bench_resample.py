"""bench_resample.py - resampling wav files to 16 kHz on one GPU (fsn_resample) against the host resampler, and its
effect on the wav -> wav file loop.  Prints one JSON line per measurement, then one line with the card.

  resample   one clip of --durations seconds at 44.1 and 48 kHz (seeded noise), to 16 kHz with zeros = 24:
             host  Inferencer.resample (float64 numpy), host clock over --host-iters calls; peak host memory from
                   tracemalloc (numpy's and Python's allocations);
             device resample_batch on that clip (pinned staging, H2D, fsn_resample), host clock around calls that end in
                   a device synchronise, after --warmup calls; kernel alone with CUDA events over --iters calls.  Peak
                   host memory from tracemalloc (pageable), plus the pinned staging buffer, 4 bytes per input sample.
  files      Inferencer.enhance_files on --files seeded 1 - 10 s 48 kHz mono files (fullsubnet, default arguments,
             precision "auto", seeded weights), batch size 64, with and without resample_on_device, at max_padding 0
             and 0.05; clips/s = files / wall time of the call, the files read, enhanced and written (to a temporary
             directory).  Each configuration runs once after one warm-up call on the first 8 files.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import tracemalloc

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def clip(n: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(n) + 0.3 * np.sin(np.arange(n) * 0.013)
    return (0.5 * x / np.abs(x).max()).astype(np.float32)


def bench_resample(dev, sr_in: int, seconds: int, args) -> dict:
    from fullsubnet_b200 import _lib
    from fullsubnet_b200.acoustics.resample import resample_batch, resampled_length
    from fullsubnet_b200.inferencer import Inferencer
    x = clip(sr_in * seconds, seed=sr_in + seconds)
    rec = {"what": "resample", "sr_in": sr_in, "sr_out": 16000, "seconds": seconds, "zeros": 24}
    if seconds <= args.host_max_seconds:
        tracemalloc.start()
        t0 = time.perf_counter()
        for _ in range(args.host_iters):
            ref = Inferencer.resample(x, sr_in, 16000)
        rec["host_s"] = (time.perf_counter() - t0) / args.host_iters
        rec["host_peak_mb"] = tracemalloc.get_traced_memory()[1] / 2 ** 20
        tracemalloc.stop()
    else:
        ref = None
    for _ in range(args.warmup):
        resample_batch([x], sr_in, 16000, dev)
    torch.cuda.synchronize(dev)
    tracemalloc.start()
    t0 = time.perf_counter()
    for _ in range(args.iters):
        y = resample_batch([x], sr_in, 16000, dev)[0]
        torch.cuda.synchronize(dev)
    rec["device_s"] = (time.perf_counter() - t0) / args.iters
    rec["device_peak_mb"] = tracemalloc.get_traced_memory()[1] / 2 ** 20
    rec["device_pinned_mb"] = 4 * len(x) / 2 ** 20
    tracemalloc.stop()
    # the kernel alone: one fsn_resample call on a device-resident input
    lib = _lib.load()
    xd = torch.from_numpy(x)[None].to(dev)
    n_out = resampled_length(len(x), sr_in, 16000)
    yd = torch.empty(1, n_out, device=dev)
    nb = lib.fsn_resample_workspace_bytes(1, len(x), sr_in, 16000, 24)
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    st = _lib.stream_ptr(dev)
    call = lambda: _lib.check(lib.fsn_resample(xd.data_ptr(), None, 1, len(x), sr_in, 16000, 24, yd.data_ptr(),  # noqa
                                               n_out, ws.data_ptr(), nb, st))
    for _ in range(args.warmup):
        call()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.iters):
        call()
    e1.record()
    torch.cuda.synchronize(dev)
    rec["kernel_ms"] = e0.elapsed_time(e1) / args.iters
    if ref is not None:
        got = y.cpu().numpy()
        rec["max_abs_diff_over_max_x"] = float(np.abs(got.astype(np.float64) - ref).max() / np.abs(x).max())
        rec["bit_identical_fraction"] = float((got.view(np.int32) == ref.view(np.int32)).mean())
        rec["speedup"] = rec["host_s"] / rec["device_s"]
    return rec


def bench_files(dev, args) -> list:
    from fullsubnet_b200.fullsubnet.model import Model
    from fullsubnet_b200.inferencer import Inferencer
    from oracle import fullsubnet_oracle as O
    m = Model(**O.DEFAULT_MODEL_ARGS, precision="auto")
    m.load_state_dict(O.make_state_dict(seed=0), strict=True)
    inf = Inferencer(model=m.to(dev).eval(), device=dev)
    rng = np.random.default_rng(1)
    out = []
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for i in range(args.files):
            n = int(rng.integers(48000, 480001))
            p = os.path.join(tmp, f"in_{i:04d}.wav")
            inf.write_wav(p, np.round(clip(n, seed=1000 + i) * 32767).astype(np.int16), 48000)
            paths.append(p)
        seconds = sum(os.path.getsize(p) - 44 for p in paths) / 2 / 48000
        for mp in (0.0, 0.05):
            for on_device in (False, True):
                inf.enhance_files(paths[:8], os.path.join(tmp, "warm"), max_padding=mp, resample_on_device=on_device)
                torch.cuda.synchronize(dev)
                t0 = time.perf_counter()
                inf.enhance_files(paths, os.path.join(tmp, "out"), max_padding=mp, resample_on_device=on_device)
                wall = time.perf_counter() - t0
                out.append({"what": "enhance_files", "files": args.files, "audio_s": round(seconds, 1), "sr_in": 48000,
                            "max_padding": mp, "resample_on_device": on_device, "wall_s": wall,
                            "clips_per_s": args.files / wall})
    return out


def card(index: int) -> dict:
    try:
        q = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = "nvidia-smi unavailable"
    return {"what": "card", "nvidia_smi": q, "torch_name": torch.cuda.get_device_name(index)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--durations", type=int, nargs="+", default=[10, 60])
    ap.add_argument("--host-max-seconds", type=int, default=60, help="skip the host resampler on longer clips")
    ap.add_argument("--host-iters", type=int, default=1)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--files", type=int, default=48)
    ap.add_argument("--skip-files", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_resample.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    for seconds in args.durations:
        for sr in (44100, 48000):
            print(json.dumps(bench_resample(dev, sr, seconds, args)), flush=True)
    if not args.skip_files:
        for rec in bench_files(dev, args):
            print(json.dumps(rec), flush=True)
    print(json.dumps(card(0)), flush=True)


if __name__ == "__main__":
    main()
