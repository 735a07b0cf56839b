"""forgetting_norm (audio_zen/model/base_model.py:102-151) restated for the tests, in float32 and float64.

The reference loops over frames with

    alp = torch.min(torch.tensor([(t - 1) / (t + 1), alpha]))      t < 192: a float32 tensor
    mu  = alp * mu + (1 - alp) * mean_t                              every operation in float32
    mu  = alpha * mu + (1 - alpha) * mean_t                          t >= 192: Python doubles on float32 tensors

so a_t = float32(min((t-1)/(t+1), alpha)) and b_t = 1 - a_t rounded in float32 for t < 192 (a_0 = -1, b_0 = 2; a_1 = 0),
then a = float32(alpha) and b = float32(1 - alpha) with 1 - alpha evaluated in double.  ``coefficients`` gives exactly
these; ``forgetting_norm`` in float32 runs the reference's operations in its order (bit-identical to it, pinned by
tests/test_cpu_forgetting.py against tests/golden/forgetting.npz), and in float64 the same recurrence on the same
coefficients, the reference for the GPU kernels' error bounds.
"""
from __future__ import annotations

import numpy as np
import torch

SAMPLE_LENGTH = 192
EPS = 1e-10


def coefficients(T: int):
    """float32 (a [T], b [T]) of mu_t = a_t mu_{t-1} + b_t m_t as the reference rounds them."""
    alpha = (SAMPLE_LENGTH - 1) / (SAMPLE_LENGTH + 1)
    a = np.empty(T, np.float32)
    b = np.empty(T, np.float32)
    for t in range(T):
        if t < SAMPLE_LENGTH:
            a[t] = min(np.float32((t - 1) / (t + 1)), np.float32(alpha))
            b[t] = np.float32(1) - a[t]
        else:
            a[t] = np.float32(alpha)
            b[t] = np.float32(1 - alpha)
    return a, b


def frame_means(x: torch.Tensor) -> torch.Tensor:
    """m [B, T]: mean over the C*F features of each frame of x [B, C, F, T], one torch.mean per frame slice as the
    reference takes it (a mean over the whole [B, C*F, T] tensor at once reduces in another order)."""
    B, C, F, T = x.shape
    flat = x.reshape(B, C * F, T)
    return torch.stack([torch.mean(flat[:, :, t], dim=1) for t in range(T)], dim=-1)


def running_mean(m: torch.Tensor) -> torch.Tensor:
    """mu [B, T] of the frame means m [B, T] in m's dtype; float32 follows the reference's operation order."""
    a, b = coefficients(m.shape[-1])
    mus = []
    mu = torch.zeros_like(m[:, 0])
    for t in range(m.shape[-1]):
        at = torch.tensor(float(a[t]), dtype=m.dtype)
        bt = torch.tensor(float(b[t]), dtype=m.dtype)
        mu = at * mu + bt * m[:, t]
        mus.append(mu)
    return torch.stack(mus, dim=-1)


def forgetting_norm(x: torch.Tensor):
    """(x / (mu + 1e-10), mu) for x [B, C, F, T]; mu [B, T].  Differentiable (float64 autograd of the adjoint tests)."""
    mu = running_mean(frame_means(x))
    return x / (mu[:, None, None, :] + EPS), mu


def scale(mu: torch.Tensor) -> torch.Tensor:
    """the multiplier the library stores per (clip, frame): 1 / (mu + 1e-10), rounded in mu's dtype."""
    return 1.0 / (mu + EPS)
