"""``Inferencer.resample`` on the device for a batch of clips: ``fsn_resample``, one call per input rate, the weights
and sums in float64 as the host computes them (DESIGN 4.10.1).  Outputs equal the host's to float32 rounding: almost
every sample has the host's bits, the rest differ by one rounding step."""
from __future__ import annotations

from math import gcd

import numpy as np
import torch

from .. import _lib


def resampled_length(n: int, sr_in: int, sr_out: int) -> int:
    """Samples of an ``n``-sample clip at ``sr_in`` after resampling to ``sr_out``: ceil(n * up / down) in integers, as
    ``fsn_resample`` computes it (the length ``Inferencer.resample`` returns while n * up < 2^53)."""
    g = gcd(int(sr_in), int(sr_out))
    up, down = int(sr_out) // g, int(sr_in) // g
    return -(-int(n) * up // down)


def resample_batch(ys, sr_in, sr_out: int, device, zeros: int = 24, out: torch.Tensor = None):
    """``Inferencer.resample(y, rate, sr_out, zeros)`` for every 1-D float32 host array of ``ys`` on ``device``: a list
    of 1-D device tensors, clip i's resampled samples.  ``sr_in``: one rate for all clips, or one per clip.  The inputs
    are staged through one pinned buffer, and the clips of each rate go through one ``fsn_resample`` call; a clip at
    ``sr_out`` is copied with its bits.  ``out`` (optional): a contiguous float32 [len(ys), L] device tensor to fill, L at
    least the longest result; row i gets clip i, 0 past its length, and the returned tensors are views of it.  Runs on
    the device's current stream and never waits on it."""
    ys = [np.ascontiguousarray(y, dtype=np.float32) for y in ys]
    if any(y.ndim != 1 for y in ys):
        raise ValueError("resample_batch takes 1-D waveforms")
    rates = [int(sr_in)] * len(ys) if np.ndim(sr_in) == 0 else [int(r) for r in sr_in]
    if len(rates) != len(ys):
        raise ValueError(f"{len(rates)} sample rates for {len(ys)} clips")
    if not ys:
        return []
    sr_out, device = int(sr_out), torch.device(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    n_out = [resampled_length(len(y), r, sr_out) for y, r in zip(ys, rates)]
    if out is None:
        out = torch.empty(len(ys), max(n_out), dtype=torch.float32, device=device)
    elif out.dim() != 2 or out.shape[0] != len(ys) or out.dtype != torch.float32 or not out.is_contiguous() \
            or out.device != device:
        raise ValueError(f"out must be a contiguous float32 [{len(ys)}, L] tensor on {device}")
    groups = {}
    for i, r in enumerate(rates):
        groups.setdefault(r, []).append(i)
    shapes = {r: (len(rows), max(len(ys[i]) for i in rows)) for r, rows in groups.items()}
    stage = torch.empty(sum(B * N for B, N in shapes.values()), dtype=torch.float32, pin_memory=True)
    lib = _lib.load()
    off = 0
    with torch.cuda.device(device):
        st = _lib.stream_ptr(device)
        for r, rows in groups.items():
            B, N = shapes[r]
            x = stage[off:off + B * N].view(B, N)  # past each clip's length the kernel reads nothing
            off += B * N
            for j, i in enumerate(rows):
                x[j, :len(ys[i])] = torch.from_numpy(ys[i])
            x = x.to(device, non_blocking=True)
            lens = np.ascontiguousarray([len(ys[i]) for i in rows], dtype=np.int32)
            nbytes = _lib.check_workspace(lib.fsn_resample_workspace_bytes(B, N, r, sr_out, int(zeros)))
            ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
            y = out if B == len(ys) else torch.empty(B, out.shape[1], dtype=torch.float32, device=device)
            _lib.check(lib.fsn_resample(x.data_ptr(), lens.ctypes.data, B, N, r, sr_out, int(zeros), y.data_ptr(),
                                        y.shape[1], ws.data_ptr(), nbytes, st))
            if y is not out:
                out.index_copy_(0, torch.tensor(rows, device=device), y)
    return [out[i, :n] for i, n in enumerate(n_out)]
