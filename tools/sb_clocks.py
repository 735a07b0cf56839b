"""Where the cycles of the sub-band kernel (sb_lstm_tc_kernel) go, from the cycle stamps of its PROBE instantiation
(fsn_debug_sb_lstm_tc_probe), at the bench.py headline shape: 256 x 4 s clips, 257 bins, H = 384, 253 LSTM steps.

  python tools/sb_clocks.py [--precisions f16x3_tc,f16_tc] [--batch 256] [--ctas 8] [--stages 0] [--cluster 0]

The first `--ctas` CTAs record every loop iteration.  Per CTA and step the tool prints the step time, and per ring stage
the cycles spent in each wait of the consumer warpgroup that holds the ring, next to the 192-cycle tensor bound (12
m64n32k16 at 16 cycles, single pass 8) and the shared-memory bound of DESIGN 4.1 (operand reads + TMA writes at
128 B/clk).  Card name, power limit and the median SM clock of the timed calls are read in the same run.  It also times
the production instantiation on the same inputs, so the probe's own cost is visible.
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, F, NS, NF, LA, STEPS, KS = 384, 257, 15, 0, 2, 253, 32
FIELDS = ["t_begin", "t_mma0", "t_mma1", "t_end", "operand", "turn", "w_full", "wait_group", "group_lat", "stages",
          "cell", "l1_done", "h1_empty", "h0_empty", "fc_done", "gt_begin"]
F_ = {n: i for i, n in enumerate(FIELDS)}


def smi(query: str) -> list[str]:
    out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={query}", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True, check=True).stdout
    return [c.strip() for c in out.strip().split(",")]


def budget(x3: bool):
    """stages, MMAs, tensor and shared-memory cycles per ring stage (DESIGN 4.1)"""
    mt, nkb = H // 128, (1 + H // KS) + 2 * H // KS
    stages = mt * nkb * (2 if x3 else 1)
    mmas = mt * nkb * 8 * (3 if x3 else 1)
    smem = stages * 16384 + mmas * (64 * 16 * 2 + 32 * 16 * 2)
    return stages, mmas, mmas * 16 / stages, smem / 128 / stages


def run(lib, dev, x3, B, ctas, stages, cluster, probe, reps=1):
    from fullsubnet_b200 import _lib
    g = torch.Generator().manual_seed(0)
    k = 1.0 / H ** 0.5
    ksb = 2 * NS + 1 + 2 * NF + 1
    w = {}
    for layer in range(2):
        w[f"ih{layer}"] = ((torch.rand(4 * H, ksb if layer == 0 else H, generator=g) * 2 - 1) * k).to(dev)
        w[f"hh{layer}"] = ((torch.rand(4 * H, H, generator=g) * 2 - 1) * k).to(dev)
        w[f"bi{layer}"] = ((torch.rand(4 * H, generator=g) * 2 - 1) * k).to(dev)
        w[f"bh{layer}"] = ((torch.rand(4 * H, generator=g) * 2 - 1) * k).to(dev)
    fcw, fcb = ((torch.rand(2, H, generator=g) * 2 - 1) * k).to(dev), torch.zeros(2, device=dev)
    s = _lib.SeqWeights()
    for layer in range(2):
        s.w_ih[layer], s.w_hh[layer] = w[f"ih{layer}"].data_ptr(), w[f"hh{layer}"].data_ptr()
        s.b_ih[layer], s.b_hh[layer] = w[f"bi{layer}"].data_ptr(), w[f"bh{layer}"].data_ptr()
    s.fc_w, s.fc_b = fcw.data_ptr(), fcb.data_ptr()
    magT = torch.randn(B, STEPS, F, generator=g).abs().to(dev)
    fbT = torch.relu(torch.randn(B, STEPS, F, generator=g)).to(dev)
    inv2 = (torch.rand(B, generator=g) + 0.3).to(dev)
    packed = torch.empty(lib.fsn_debug_sb_lstm_tc_packed_bytes(H, int(x3)), dtype=torch.uint8, device=dev)
    crm = torch.empty(B, 2, F, STEPS - LA, device=dev)
    its = STEPS + 1
    stamps = torch.zeros(ctas, its, 2, _lib.SB_PROBE_SLOTS, _lib.SB_PROBE_FIELDS, dtype=torch.int64, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    common = (C.byref(s), H, NS, NF, 2, 0, int(x3), magT.data_ptr(), fbT.data_ptr(), B, F, STEPS, 1, inv2.data_ptr(),
              None, LA, STEPS, 1, stages, cluster, packed.data_ptr(), crm.data_ptr())
    ms = []
    for _ in range(reps + 1):  # the first call warms up
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        if probe:
            _lib.check(lib.fsn_debug_sb_lstm_tc_probe(*common, stamps.data_ptr(), ctas, its, st))
        else:
            _lib.check(lib.fsn_debug_sb_lstm_tc(*common, st))
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))  # includes the weight packing (a few microseconds)
    return ms[1:], stamps.cpu().numpy(), crm.cpu()


def report(prec, x3, st, ms_prod, ms_probe, mhz):
    n_st, mmas, tensor, smem = budget(x3)
    ctas, its = st.shape[0], st.shape[1]
    mt = H // 128
    prod = st[:, :, 0, st.shape[3] - 1, :]    # [cta, it, field]: the producer has the last slot (MAX_MT)
    cons = st[:, :, :, :mt, :]                 # [cta, it, layer, m, field]
    steady = slice(2, its - 2)                 # full iterations (both layers), away from the start and the end
    step = (prod[:, steady, F_["t_end"]] - prod[:, steady, F_["t_begin"]]).astype(np.float64)
    # consecutive producer iteration starts: the CTA's step period
    period = np.diff(prod[:, :, F_["t_begin"]].astype(np.float64), axis=1)[:, steady]
    c = cons[:, steady].astype(np.float64)
    per_step = lambda f: c[..., F_[f]].sum(axis=(2, 3)).mean()  # summed over layers and warpgroups, mean over CTAs, steps
    stage_sum = per_step("stages")
    print(f"{prec}: {n_st} stages and {mmas} m64n32k16 per CTA and step; bounds per stage: tensor {tensor:.0f} cycles, "
          f"shared memory {smem:.0f} cycles")
    print(f"  kernel: production {min(ms_prod):.1f} ms, probe {min(ms_probe):.1f} ms; SM clock {mhz:.0f} MHz")
    print(f"  step period (producer) {period.mean():9.0f} cycles = {period.mean() / n_st:6.1f} per stage"
          f"   ({ctas} CTAs x {step.shape[1]} steps, spread p10 {np.percentile(period, 10):.0f} / "
          f"p90 {np.percentile(period, 90):.0f})")
    mma_win = (c[..., F_["t_mma1"]] - c[..., F_["t_mma0"]]).sum(axis=(2, 3)).mean()
    rows = [
        ("MMA window (turn to wait_group 0, summed over warpgroups)", mma_win),
        ("  w_full waits (stage not landed)", per_step("w_full")),
        ("  wgmma.wait_group", per_step("wait_group")),
        ("  commit -> next stage's wait<1> returns (bounds retire)", per_step("group_lat")),
        ("turn waits", per_step("turn")),
        ("operand waits (x_full, h0_ready, h1_ready)", per_step("operand")),
        ("cell + h stores + exchange issue", per_step("cell")),
        ("l1_done waits", per_step("l1_done")),
        ("h1_empty waits", per_step("h1_empty")),
        ("h0_empty waits", per_step("h0_empty")),
        ("fc_done waits", per_step("fc_done")),
        ("producer w_empty waits", prod[:, steady, F_["operand"]].astype(np.float64).mean()),
    ]
    for name, v in rows:
        print(f"  {name:58s} {v:9.0f} cycles/step  {v / stage_sum:6.1f} per stage")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--precisions", default="f16x3_tc,f16_tc")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--ctas", type=int, default=8)
    ap.add_argument("--stages", type=int, default=0, help="ring depth, 0 = FSN_TC_STAGES / default")
    ap.add_argument("--cluster", type=int, default=0, help="CTA pairs per cluster, 0 = FSN_TC_CLUSTER / default")
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    dev = torch.device("cuda:0")
    name, plimit = smi("name,power.limit")
    print(f"# {name}, power limit {plimit} W; B = {args.batch} x 4 s, F = {F}, H = {H}, {STEPS} steps", flush=True)
    for prec in args.precisions.split(","):
        x3 = prec == "f16x3_tc"
        q = subprocess.Popen(["nvidia-smi", "--id=0", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-lms",
                              "100"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        try:
            ms_prod, _, crm_prod = run(lib, dev, x3, args.batch, args.ctas, args.stages, args.cluster, False, args.reps)
            ms_probe, st, crm_probe = run(lib, dev, x3, args.batch, args.ctas, args.stages, args.cluster, True,
                                          args.reps)
        finally:
            q.terminate()
            sampled = q.communicate()[0]
        clocks = sorted(float(v) for v in sampled.split() if v.replace(".", "").isdigit())
        mhz = clocks[len(clocks) // 2] if clocks else float("nan")
        assert torch.equal(crm_prod, crm_probe), "the probe instantiation changed the output bits"
        report(prec, x3, st, ms_prod, ms_probe, mhz)


if __name__ == "__main__":
    main()
