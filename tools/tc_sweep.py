"""GPU timing sweep of the sub-band stage (sb_lstm_tc_kernel) at the bench.py headline shape: B = 256 x 4 s clips,
H = 384, precisions f16x3_tc and f16_tc, x FSN_TC_CLUSTER 1 / 2 / 4, x FSN_TC_STAGES 2 / 3 / 4.

  python tools/tc_sweep.py [--precisions f16x3_tc,f16_tc] [--clusters 1,2,4] [--stages 2,3,4] [--batch 256] [--runs 2]

The switches are read once per process, so every setting runs in a subprocess of its own.  FSN_TC_CLUSTER = CL is
the number of CTA pairs that share each half's weight stream by multicast: a hardware cluster is 2 CL CTAs.  Each
setting prints the stage time from the library's stage events (fsn_set_profiling / fsn_last_stage_ms(2)), the time per
ring stage in SM cycles next to the shared-memory budget of DESIGN 4.1, the resident clusters
(cudaOccupancyMaxActiveClusters) and the waves they give, and the median SM clock sampled during the timed calls.
Card name and power limit are read once.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SR, HOP, CLIP_SECONDS, LA = 16000, 256, 4, 2
H, NB, KS, W_TILE = 384, 32, 32, 16384  # NB rows per CTA pair; a stage is 4 gates x 64 units x 32 k of fp16
A_BYTES = 64 * 16 * 2  # A operand of one m64n32k16 (weights), read from shared memory
B_BYTES = 32 * 16 * 2  # B operand (state)
SMEM_BYTES_PER_CLK = 128


def shape(x3: bool):
    """Ring stages, MMAs and shared-memory bytes per CTA and LSTM step (both layers, the CTA's H / 128 slices of 64
    hidden units: half of the units of its pair)."""
    mt, nkb = H // 128, (1 + H // KS) + 2 * H // KS
    stages = mt * nkb * (2 if x3 else 1)
    mmas = mt * nkb * 8 * (3 if x3 else 1)  # 4 gates x 2 k16 per k range; X3: hi.hi, hi.lo, lo.hi
    smem = stages * W_TILE + mmas * (A_BYTES + B_BYTES)
    return stages, mmas, smem


def smi(query: str) -> list[str]:
    out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={query}", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True, check=True).stdout
    return [c.strip() for c in out.strip().split(",")]


def child(prec: str, batch: int, runs: int) -> None:
    sys.path.insert(0, ROOT)
    import torch
    from fullsubnet_b200 import _lib
    from fullsubnet_b200.fullsubnet.model import Model
    from oracle import fullsubnet_oracle as O
    dev = torch.device("cuda:0")
    lib = _lib.load()
    m = Model(**O.DEFAULT_MODEL_ARGS, precision=prec)
    m.load_state_dict(O.make_state_dict(0))
    m = m.to(dev).eval()
    y = O.make_noisy(batch, SR * CLIP_SECONDS, seed=1).to(dev)
    m.enhance(y)
    torch.cuda.synchronize()
    q = subprocess.Popen(["nvidia-smi", "--id=0", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-lms",
                          "100"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    lib.fsn_set_profiling(1)
    ms = []
    for _ in range(runs):
        m.enhance(y)
        torch.cuda.synchronize()
        ms.append(lib.fsn_last_stage_ms(2))
    lib.fsn_set_profiling(0)
    q.terminate()
    clocks = sorted(float(v) for v in q.communicate()[0].split() if v.replace(".", "").isdigit())
    st, cl = int(os.environ["FSN_TC_STAGES"]), int(os.environ["FSN_TC_CLUSTER"])
    n = C.c_int(0)
    _lib.check(lib.fsn_debug_sb_lstm_tc_max_clusters(H, 1 if prec == "f16x3_tc" else 0, st, cl, C.byref(n)))
    print(json.dumps({"ms": ms, "sm_mhz": clocks[len(clocks) // 2] if clocks else None, "resident_clusters": n.value}))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--precisions", default="f16x3_tc,f16_tc")
    ap.add_argument("--clusters", default="1,2,4")
    ap.add_argument("--stages", default="2,3,4")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        child(args.child, args.batch, args.runs)
        return
    name, plimit, maxclk = smi("name,power.limit,clocks.max.sm")
    print(f"# {name}, power limit {plimit} W, max SM clock {maxclk} MHz", flush=True)
    T = 1 + SR * CLIP_SECONDS // HOP
    steps = T + LA
    pairs = -(-args.batch * 257 // NB)
    print(f"# B = {args.batch} x {CLIP_SECONDS} s, {steps} LSTM steps, {pairs} CTA pairs of {NB} rows", flush=True)
    for prec in args.precisions.split(","):
        x3 = prec == "f16x3_tc"
        n_st, mmas, smem = shape(x3)
        budget = smem / SMEM_BYTES_PER_CLK
        print(f"# {prec}: {n_st} stages, {mmas} MMAs, {smem / 1e6:.2f} MB of shared-memory traffic per CTA-step "
              f"-> budget {budget / 1e3:.0f} k cycles per step, {budget / n_st:.0f} cycles per stage", flush=True)
        for cl in (int(c) for c in args.clusters.split(",")):
            for st in (int(s) for s in args.stages.split(",")):
                env = dict(os.environ, FSN_TC_CLUSTER=str(cl), FSN_TC_STAGES=str(st))
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", prec, "--batch",
                                    str(args.batch), "--runs", str(args.runs)], env=env, capture_output=True, text=True)
                if p.returncode:
                    print(f"{prec:9s} CL={cl} stages={st}: FAILED\n{p.stdout[-2000:]}{p.stderr[-2000:]}", flush=True)
                    continue
                r = json.loads(p.stdout.strip().splitlines()[-1])
                ms = min(r["ms"])
                clusters = -(-pairs // cl)
                waves = -(-clusters // r["resident_clusters"]) if r["resident_clusters"] > 0 else None
                mhz = r["sm_mhz"] or float(maxclk)
                cyc = ms * 1e-3 * mhz * 1e6 / (waves * steps * n_st) if waves else float("nan")
                print(f"{prec:9s} CL={cl} stages={st}: {ms:9.1f} ms  (runs {', '.join(f'{v:.1f}' for v in r['ms'])})  "
                      f"{cyc:6.0f} cycles/stage (budget {budget / n_st:.0f})  resident clusters "
                      f"{r['resident_clusters']:3d} -> {waves} waves  SM {mhz:.0f} MHz", flush=True)


if __name__ == "__main__":
    main()
