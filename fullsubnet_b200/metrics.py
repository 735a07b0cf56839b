"""audio_zen/metrics.py on the GPU: SI-SDR and STOI of batches of clips with per-clip lengths (fsn_si_sdr_lengths,
fsn_stoi), the module's numpy-facing ``SI_SDR`` / ``STOI`` functions, and ``python -m fullsubnet_b200.metrics``, the
GPU counterpart of tools/calculate_metrics.py for these two metrics.  PESQ (ITU-T P.862) is not built here: the CLI
refuses WB_PESQ / NB_PESQ by name."""
from __future__ import annotations

import argparse
import csv
import sys
from pathlib import Path

import numpy as np
import torch

from . import _lib

STOI_RATES = (16000, 10000)
PESQ_METRICS = ("WB_PESQ", "NB_PESQ")
METRICS = ("SI_SDR", "STOI")


def stoi(reference: torch.Tensor, estimation: torch.Tensor, lengths=None, sr: int = 16000) -> torch.Tensor:
    """pystoi's stoi(reference, estimation, sr, extended=False) per clip on the device: [B,L] x [B,L] -> [B] float32
    (fsn_stoi, float64 inside).  ``lengths`` (B ints, max L): clip b is row b's first lengths[b] samples, and out[b]
    equals the call on it alone.  ``sr`` 16000 or 10000.  Runs on the caller's current stream."""
    reference = _lib.require_cuda(reference, "reference")
    estimation = _lib.require_cuda(estimation, "estimation")
    assert reference.shape == estimation.shape and reference.dim() == 2
    B, L = reference.shape
    lens = None if lengths is None else _lib.lengths_table(lengths, B, L)
    lib = _lib.load()
    nbytes = _lib.check_workspace(lib.fsn_stoi_workspace_bytes(B, L, int(sr)))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=reference.device)
    out = torch.empty(B, dtype=torch.float32, device=reference.device)
    with torch.cuda.device(reference.device):
        _lib.check(lib.fsn_stoi(reference.data_ptr(), estimation.data_ptr(), None if lens is None else lens.ctypes.data,
                                B, L, int(sr), out.data_ptr(), ws.data_ptr(), nbytes, _lib.stream_ptr(reference.device)))
    return out


def _device() -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError("fullsubnet_b200: the metrics run on a CUDA device; this package has no CPU path.")
    return torch.device("cuda", torch.cuda.current_device())


def _pair(ref, est):
    ref = torch.as_tensor(np.asarray(ref, dtype=np.float32)).reshape(1, -1)
    est = torch.as_tensor(np.asarray(est, dtype=np.float32)).reshape(1, -1)
    dev = _device()
    return ref.to(dev), est.to(dev)


def SI_SDR(reference, estimation, sr=16000) -> float:
    """audio_zen/metrics.py:SI_SDR for one pair of 1-D numpy clips, computed on the current CUDA device."""
    from .trainer import si_sdr
    ref, est = _pair(reference, estimation)
    return float(si_sdr(ref, est)[0])


def STOI(ref, est, sr=16000) -> float:
    """audio_zen/metrics.py:STOI (pystoi, extended=False) for one pair of 1-D numpy clips, on the current CUDA device."""
    ref, est = _pair(ref, est)
    return float(stoi(ref, est, sr=sr)[0])


# ---------------------------------------------------------------------------------------------- tools/calculate_metrics.py
def pair_files(reference_dir, estimated_dir):
    """[(basename, reference path, estimated path)] of the wav files under both directories (recursively), paired by
    basename like tools/calculate_metrics.py; every basename must be in both, and only once in each."""
    def by_name(d):
        files = sorted(Path(d).expanduser().rglob("*.wav"))
        names = {}
        for f in files:
            if f.stem in names:
                raise ValueError(f"{f.stem} is in {d} twice: {names[f.stem]} and {f}")
            names[f.stem] = f
        return names
    ref, est = by_name(reference_dir), by_name(estimated_dir)
    if not ref:
        raise ValueError(f"no wav files under {reference_dir}")
    if set(ref) != set(est):
        only_ref, only_est = sorted(set(ref) - set(est)), sorted(set(est) - set(ref))
        raise ValueError(f"unpaired files: only in the reference directory {only_ref[:5]}, only in the estimated "
                         f"directory {only_est[:5]}")
    return [(k, ref[k], est[k]) for k in sorted(ref)]


def parse_metrics(names: str):
    out = []
    for m in (s.strip() for s in names.split(",") if s.strip()):
        if m in PESQ_METRICS:
            raise ValueError(f"{m}: PESQ (ITU-T P.862) is not computed by fullsubnet_b200; use the reference's "
                             "tools/calculate_metrics.py for it")
        if m not in METRICS:
            raise ValueError(f"unknown metric {m}; supported: {', '.join(METRICS)}")
        out.append(m)
    if not out:
        raise ValueError("no metric given")
    return out


def compute_files(pairs, metrics, sr: int = 16000, batch_size: int = 64, max_padding: float = 0.25, device=None):
    """{metric: float32 [len(pairs)]} of each pair, in the order of ``pairs``.  Each clip is the reference truncated to
    the estimate's length (or the estimate to the reference's, whichever is shorter), as the reference's tool compares
    ref[:len(est)] with est; clips are grouped by ``plan_batches`` and scored with per-clip lengths."""
    from .inferencer import Inferencer, plan_batches
    from .trainer import si_sdr
    dev = device or _device()
    clips = []
    for _, r, e in pairs:
        ref, est = Inferencer.load_wav(r, sr), Inferencer.load_wav(e, sr)
        n = min(len(ref), len(est))
        clips.append((ref[:n], est[:n]))
    lens = [len(r) for r, _ in clips]
    out = {m: np.empty(len(clips), dtype=np.float32) for m in metrics}
    for g in plan_batches(lens, batch_size, max_padding):
        L = max(lens[i] for i in g)
        ref = torch.zeros(len(g), L)
        est = torch.zeros(len(g), L)
        for k, i in enumerate(g):
            ref[k, :lens[i]] = torch.from_numpy(clips[i][0])
            est[k, :lens[i]] = torch.from_numpy(clips[i][1])
        ref, est = ref.to(dev), est.to(dev)
        g_lens = [lens[i] for i in g]
        for m in metrics:
            v = si_sdr(ref, est, g_lens) if m == "SI_SDR" else stoi(ref, est, g_lens, sr)
            out[m][g] = v.cpu().numpy()
    return out


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="python -m fullsubnet_b200.metrics",
                                 description="SI_SDR and STOI of estimated wav files against reference wav files, "
                                             "paired by basename, on the GPU.")
    ap.add_argument("-R", "--reference", required=True, help="directory of reference (clean) wav files")
    ap.add_argument("-E", "--estimated", required=True, help="directory of estimated wav files")
    ap.add_argument("-M", "--metric_types", default="SI_SDR,STOI", help="comma-separated: SI_SDR, STOI")
    ap.add_argument("--sr", type=int, default=16000, choices=STOI_RATES)
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--max-padding", type=float, default=0.25)
    ap.add_argument("--csv", default="metrics.csv", help="where the per-file values go (default: ./metrics.csv)")
    args = ap.parse_args(argv)
    try:
        metrics = parse_metrics(args.metric_types)
        pairs = pair_files(args.reference, args.estimated)
    except ValueError as e:
        ap.error(str(e))
    values = compute_files(pairs, metrics, args.sr, args.batch_size, args.max_padding)
    for m in metrics:
        print(f"{m}: {float(np.mean(values[m].astype(np.float64)))}")
    path = Path(args.csv)
    with open(path, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(["Speech", *metrics])
        for i, (name, _, _) in enumerate(pairs):
            w.writerow([name, *(repr(float(values[m][i])) for m in metrics)])
    print(f"per-file values: {path}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
