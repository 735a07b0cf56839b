"""Mirror of audio_zen/loss.py:3-4.  ``mse_loss()`` builds the module the trainer calls as
``loss_function(cIRM, cRM)`` (fullsubnet/trainer.py:61) with cIRM [B,F,T,2] and cRM = Model.forward's [B,2,F,T]
output permuted to [B,F,T,2]; value and gradient come from one fused kernel pair (fsn_mse_loss)."""
from __future__ import annotations

import torch

from . import _lib


class _FusedMSE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, cirm, crm_bcft):
        """cirm [B,F,T,2] contiguous, crm_bcft [B,2,F,T] contiguous -> scalar."""
        B, Fs, T, _ = cirm.shape
        lib = _lib.load()
        device = cirm.device
        with torch.cuda.device(device):
            loss = torch.empty((), dtype=torch.float32, device=device)
            dcrm = torch.empty_like(crm_bcft)
            scratch = torch.empty(lib.fsn_mse_loss_scratch_bytes(), dtype=torch.uint8, device=device)
            _lib.check(lib.fsn_mse_loss(cirm.data_ptr(), crm_bcft.data_ptr(), B, Fs, T, loss.data_ptr(), dcrm.data_ptr(),
                                        scratch.data_ptr(), scratch.numel(), _lib.stream_ptr(device)))
        ctx.save_for_backward(dcrm)
        return loss

    @staticmethod
    def backward(ctx, g):
        (dcrm,) = ctx.saved_tensors
        d = dcrm * g
        return (-d.permute(0, 2, 3, 1) if ctx.needs_input_grad[0] else None), (d if ctx.needs_input_grad[1] else None)


class MSELoss(torch.nn.Module):
    """torch.nn.MSELoss() (mean reduction) for the trainer's (cIRM, cRM) pair."""

    def forward(self, input, target):
        assert input.shape == target.shape and input.dim() == 4 and input.shape[-1] == 2, \
            "expects cIRM / cRM of shape [B, F, T, 2]"
        a = _lib.require_cuda(input, "input")
        b = _lib.require_cuda(target, "target")
        # exactly one side is the model output (a permuted [B,2,F,T] tensor); the other is the constant target
        if b.requires_grad or not a.requires_grad:
            return _FusedMSE.apply(a.contiguous(), b.permute(0, 3, 1, 2).contiguous())
        return _FusedMSE.apply(b.contiguous(), a.permute(0, 3, 1, 2).contiguous())


def cirm_mse_per_clip(noisy, clean, crm, n_fft, hop_length, win_length, lengths=None) -> torch.Tensor:
    """Validation loss of B clips in one call (fsn_cirm_mse_per_clip): noisy, clean [B,L] and the model output crm
    [B,2,F,T] on them -> loss [B], where loss[b] equals ``MSELoss()(cIRM, cRM)`` of the trainer on clip b alone, bit
    for bit.  ``lengths`` (B ints, max L): clip b is row b's first lengths[b] samples and its 1 + lengths[b] //
    hop_length frames of crm."""
    noisy = _lib.require_cuda(noisy, "noisy")
    clean = _lib.require_cuda(clean, "clean")
    crm = _lib.require_cuda(crm, "crm")
    B, L = noisy.shape
    assert clean.shape == (B, L) and crm.shape == (B, 2, n_fft // 2 + 1, 1 + L // hop_length), (clean.shape, crm.shape)
    lens = None if lengths is None else _lib.lengths_table(lengths, B, L)
    lib = _lib.load()
    device = noisy.device
    with torch.cuda.device(device):
        n = _lib.check_workspace(lib.fsn_cirm_mse_per_clip_workspace_bytes(B, L, n_fft, hop_length))
        ws = torch.empty(n, dtype=torch.uint8, device=device)
        loss = torch.empty(B, dtype=torch.float32, device=device)
        _lib.check(lib.fsn_cirm_mse_per_clip(noisy.data_ptr(), clean.data_ptr(), None if lens is None else lens.ctypes.data,
                                             B, L, n_fft, hop_length, win_length, crm.data_ptr(), loss.data_ptr(),
                                             ws.data_ptr(), n, _lib.stream_ptr(device)))
    return loss


mse_loss = MSELoss
l1_loss = torch.nn.L1Loss
