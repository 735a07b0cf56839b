"""Chunked streaming throughput of fullband_baseline (fsn_fullband_stream_step), fullsubnet (fsn_stream_step, --model
fullsubnet, precision="fp32") or fast_fullsubnet (fsn_fast_stream_step, --model fast_fullsubnet): ms per call, audio
seconds enhanced per wall second and concurrent real-time streams for slots x K, with the whole-clip fp32 rate of the
same process beside it (fsn_fullband_enhance; fullsubnet: fsn_enhance; fast_fullsubnet: Inferencer.enhance_batch).  For
fullsubnet and fast_fullsubnet each line also says whether every slot stays real-time; for fast_fullsubnet it gives the
bottleneck's share of the call's GPU time, from a torch.profiler pass of its own after the timed calls.  fullsubnet and
fast_fullsubnet with --precision f16x3_tc / f16_tc stream on the tensor cores (fsn_stream_tc_step, fsn_fast_stream_tc_step),
give the launches per call, and the whole-clip rate beside them is of that precision (fast_fullsubnet: also at B = 256).  Prints one JSON line per configuration and a header line with the GPU,
power limit and clocks.

    python bench_stream.py [--model fullband_baseline] [--precision fp32] [--slots 1 64 256] [--ks 1 4 16 64]
                           [--calls 20] [--warmup 3]"""
from __future__ import annotations

import argparse
import json
import subprocess

import torch

from fullsubnet_b200 import _lib

SR, HOP = 16000, 256


def gpu_info():
    try:
        q = "name,power.limit,clocks.max.sm,clocks.sm"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except Exception as e:  # the numbers still stand; say the query failed
        return {"error": str(e)}


def model(name, norm, dev, precision="fp32"):
    if name == "fast_fullsubnet":
        from fullsubnet_b200.fast_fullsubnet.model import Model
        from oracle import fast_fullsubnet_oracle as FO
        args = dict(FO.DEFAULT_FAST_ARGS, norm_type=norm)
        m = Model(**args, precision=precision)
        m.load_state_dict(FO.make_fast_state_dict(seed=11, args=args), strict=True)
        return m.to(dev).eval()
    if name == "fullsubnet":
        from fullsubnet_b200.fullsubnet.model import Model
        from oracle import fullsubnet_oracle as O
        args = dict(O.DEFAULT_MODEL_ARGS, norm_type=norm)
        m = Model(**args, precision=precision)
        m.load_state_dict(O.make_state_dict(seed=11, args=args), strict=True)
        return m.to(dev).eval()
    from fullsubnet_b200.fullband_baseline.model import Model
    from oracle import fullband_baseline_oracle as BO
    args = dict(BO.DEFAULT_FBB_ARGS, norm_type=norm)
    m = Model(**args)
    m.load_state_dict(BO.make_fbb_state_dict(seed=11, args=args), strict=True)
    return m.to(dev).eval()


def bottleneck_share(step, calls=3):
    """Share of the GPU time of `calls` streaming calls spent in fast_fullsubnet's bottleneck: the kernels and copies
    from fast_stream_open_kernel up to fast_stream_dec_input_kernel, over all of them (on the tensor cores: the input
    and norm kernels, the one sb_phased_lstm_tc_kernel launch and the output carry)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            step()
        torch.cuda.synchronize()
    evs = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                 key=lambda e: e.time_range.start)
    total = inside = 0.0
    on = False
    for e in evs:
        if "fast_stream_open_kernel" in e.name:
            on = True
        elif "fast_stream_dec_input_kernel" in e.name:
            on = False
        d = e.time_range.elapsed_us()
        total += d
        inside += d if on else 0.0
    return round(inside / total, 3) if total > 0 else None


def time_ms(fn, calls, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, nargs="+", default=[1, 64, 256])
    ap.add_argument("--ks", type=int, nargs="+", default=[1, 4, 16, 64])
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--norm", default="cumulative_laplace_norm")
    ap.add_argument("--model", default="fullband_baseline", choices=["fullband_baseline", "fullsubnet", "fast_fullsubnet"])
    # fullsubnet and fast_fullsubnet: f16x3_tc / f16_tc stream on the tensor cores (Streamer(tensor_cores=True)), and
    # the whole-clip rate is of the same precision
    ap.add_argument("--precision", default="fp32", choices=["fp32", "f16x3_tc", "f16_tc"])
    a = ap.parse_args()
    assert a.precision == "fp32" or a.model != "fullband_baseline", "--precision is for fullsubnet and fast_fullsubnet"
    tc = a.precision != "fp32"
    assert torch.cuda.is_available(), "bench_stream.py needs a CUDA device"
    dev = torch.device("cuda:0")
    from fullsubnet_b200.stream import Streamer
    fast = a.model == "fast_fullsubnet"
    m = model(a.model, a.norm, dev, a.precision)
    print(json.dumps({"gpu": gpu_info(), "model": a.model, "precision": a.precision, "norm": a.norm}))
    lib = _lib.load()
    g = torch.Generator(device="cpu").manual_seed(0)
    for slots in a.slots:
        s = Streamer(m, slots, tensor_cores=tc)
        for K in a.ks:
            x = (0.1 * torch.randn(slots, K * HOP, generator=g)).to(dev)
            s.step(x, [1] * slots)
            ms = time_ms(lambda: s.step(x), a.calls, a.warmup)
            chunk_ms = 1000.0 * K * HOP / SR
            audio_rate = slots * chunk_ms / ms
            rt = slots if ms <= chunk_ms else int(slots * chunk_ms / ms)
            line = {"slots": slots, "K": K, "ms_per_call": round(ms, 3), "chunk_ms": chunk_ms,
                    "audio_s_per_s": round(audio_rate, 1), "realtime_streams": rt, "delay": s.delay}
            if a.model != "fullband_baseline":
                line["all_realtime"] = ms <= chunk_ms
            if tc:
                line["launches_per_call"] = int(lib.fsn_last_launch_count())
            if fast:
                line["bottleneck_share"] = bottleneck_share(lambda: s.step(x))
            print(json.dumps(line))
        del s
        torch.cuda.empty_cache()
    if fast:
        from fullsubnet_b200.inferencer import Inferencer
        whole = Inferencer(model=m, device=dev).enhance_batch
    else:
        whole = m.enhance
    for B in ((1, 64, 256) if fast and tc else (1, 64)):
        y = (0.1 * torch.randn(B, 4 * SR, generator=g)).to(dev)
        ms = time_ms(lambda: whole(y), max(3, a.calls // 4), a.warmup)
        print(json.dumps({"whole_clip": True, "B": B, "clip_s": 4.0, "ms_per_call": round(ms, 3),
                          "audio_s_per_s": round(B * 4000.0 / ms, 1)}))


if __name__ == "__main__":
    main()
