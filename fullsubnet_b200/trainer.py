"""Mirror of recipes/dns_interspeech_2020/fullsubnet/trainer.py:14-181 (and of fast_fullsubnet/trainer.py and
fullband_baseline/trainer.py:32-71, the same loop without drop_band) on top of
audio_zen/trainer/base_trainer.py:28-218 - the parts of the trainer that are arithmetic on the hot path (SURVEY 8a row
A11, 8f rank 4): mixing of a Dataset batch, STFT of noisy/clean, cIRM target + drop_band, Model.forward, MSE,
backward, gradient mean over ranks, clip, Adam; and the B=1 validation loop (enhance + loss + SI-SDR, all on the device).

Same constructor arguments and config keys as the reference, so `train.py:65-80` can construct it unchanged
(``meta.use_amp`` is accepted: the kernels compute in fp32 / tf32, at least the precision of the reference's fp16
autocast, so the GradScaler is the identity and ``scaler`` stays an empty dict in the checkpoint schema
{epoch, best_score, optimizer, scaler, model} of base_trainer.py:208-218).  TensorBoard, audio / spectrogram
visualisation and the third-party CPU metrics STOI / PESQ (base_trainer.py:277-370) are outside the hot path.

Two gradient paths, both ONE all-reduce of gradients per step (SURVEY 8e):
  * ``model`` wrapped in DistributedDataParallel exactly like base_trainer.py:32 - the autograd Function behind
    Model.forward delivers the gradients to DDP's hooks, DDP averages them; nothing else is reduced here;
  * plain ``model`` on every rank (default): rank 0's parameters are broadcast once at construction (what DDP's
    constructor does), ``model.flat_grad()`` makes every ``p.grad`` a view of one flat buffer, ``dist.all_reduce``
    moves that buffer once per step, and FusedClipAdam folds the 1/world mean into its clip coefficient."""
from __future__ import annotations

from functools import partial
from pathlib import Path

import torch

from . import _lib
from .acoustics.feature import drop_band, istft, stft
from .acoustics.mask import build_complex_ideal_ratio_mask, decompress_cIRM
from .dataset import mix_batch
from .optim import FusedClipAdam


def unwrap(model):
    """The fullsubnet Model behind an optional DistributedDataParallel wrapper (base_trainer.py:32)."""
    return model.module if isinstance(model, torch.nn.parallel.DistributedDataParallel) else model


def broadcast_parameters(model, dist, src: int = 0) -> None:
    """What DistributedDataParallel does at construction: every rank starts from rank ``src``'s parameters/buffers."""
    with torch.no_grad():
        for t in list(model.parameters()) + list(model.buffers()):
            dist.broadcast(t.data, src)


def si_sdr(reference: torch.Tensor, estimation: torch.Tensor) -> torch.Tensor:
    """audio_zen/metrics.py:6-31 on the device: [B,L] x [B,L] -> [B] dB (fsn_si_sdr)."""
    reference = _lib.require_cuda(reference, "reference")
    estimation = _lib.require_cuda(estimation, "estimation")
    assert reference.shape == estimation.shape and reference.dim() == 2
    out = torch.empty(reference.shape[0], dtype=torch.float32, device=reference.device)
    with torch.cuda.device(reference.device):
        _lib.check(_lib.load().fsn_si_sdr(reference.data_ptr(), estimation.data_ptr(), reference.shape[0],
                                          reference.shape[1], out.data_ptr(), _lib.stream_ptr(reference.device)))
    return out


class Trainer:
    def __init__(self, dist, rank, config, resume, only_validation, model, loss_function, optimizer,
                 train_dataloader, validation_dataloader=None):
        self.dist, self.rank = dist, rank
        self.device = torch.device("cuda", rank)
        self.is_ddp = isinstance(model, torch.nn.parallel.DistributedDataParallel)
        self.model = model if self.is_ddp else model.cuda(rank)
        self.core = unwrap(self.model)
        self.loss_function = loss_function
        self.optimizer = optimizer
        self.world_size = dist.get_world_size() if dist is not None and dist.is_initialized() else 1
        if self.world_size > 1 and not self.is_ddp:
            broadcast_parameters(self.core, dist)
        self.use_amp = config["meta"].get("use_amp", False)
        ac = config["acoustics"]
        self.torch_stft = partial(stft, n_fft=ac["n_fft"], hop_length=ac["hop_length"], win_length=ac["win_length"])
        self.torch_istft = partial(istft, n_fft=ac["n_fft"], hop_length=ac["hop_length"], win_length=ac["win_length"])
        self.train_config = config["trainer"]["train"]
        self.epochs = self.train_config["epochs"]
        self.save_checkpoint_interval = self.train_config["save_checkpoint_interval"]
        self.clip_grad_norm_value = self.train_config["clip_grad_norm_value"]
        assert self.save_checkpoint_interval >= 1, \
            "Check the 'save_checkpoint_interval' parameter in the config. It should be large than one."
        self.validation_config = config["trainer"].get("validation", {})
        self.validation_interval = self.validation_config.get("validation_interval", 1)
        self.save_max_metric_score = self.validation_config.get("save_max_metric_score", True)
        self.only_validation = only_validation
        self.start_epoch = 1
        self.best_score = float("-inf") if self.save_max_metric_score else float("inf")
        self.save_dir = Path(config["meta"]["save_dir"]).expanduser().absolute() / config["meta"]["experiment_name"]
        self.checkpoints_dir = self.save_dir / "checkpoints"
        self.train_dataloader = train_dataloader
        self.valid_dataloader = validation_dataloader
        self.last_validation = None
        if isinstance(optimizer, FusedClipAdam):
            optimizer.max_norm = self.clip_grad_norm_value
        if resume:
            self._resume_checkpoint()

    # ------------------------------------------------------------------ one optimisation step (trainer.py:41-71)
    def train_step(self, noisy, clean=None):
        """One step on ``(noisy, clean)`` [B,L], or on a batch of ``fullsubnet_b200.dataset.Dataset`` items passed as
        ``noisy`` (a dict): moved to the device and mixed there (``dataset.mix_batch``) before the same step."""
        model, core = self.model, self.core
        self.optimizer.zero_grad(set_to_none=False)
        if isinstance(noisy, dict):
            assert clean is None, "a Dataset batch carries its own clean speech"
            noisy, clean = mix_batch(noisy, self.device)
        noisy = noisy.to(self.device, non_blocking=True)
        clean = clean.to(self.device, non_blocking=True)
        noisy_mag, _, noisy_real, noisy_imag = self.torch_stft(noisy)
        _, _, clean_real, clean_imag = self.torch_stft(clean)
        cIRM = build_complex_ideal_ratio_mask(noisy_real, noisy_imag, clean_real, clean_imag)  # [B, F, T, 2]
        if hasattr(core, "num_groups_in_drop_band"):  # fullsubnet; fast_fullsubnet/trainer.py:45-56 has no drop_band
            cIRM = drop_band(cIRM.permute(0, 3, 1, 2), core.num_groups_in_drop_band).permute(0, 2, 3, 1)
        cRM = model(noisy_mag.unsqueeze(1)).permute(0, 2, 3, 1)
        loss = self.loss_function(cIRM, cRM)
        loss.backward()  # under DDP the gradient mean over ranks happens in here (base_trainer.py:32)
        scale = 1.0
        if self.world_size > 1 and not self.is_ddp:  # the same mean as ONE collective over the flat buffer
            flat = core.flat_grad()
            self.dist.all_reduce(flat)
            scale = 1.0 / self.world_size
        if isinstance(self.optimizer, FusedClipAdam):
            self.optimizer.step(grad_scale=scale)
        else:
            if scale != 1.0:
                for p in core.parameters():
                    p.grad.mul_(scale)
            torch.nn.utils.clip_grad_norm_(core.parameters(), self.clip_grad_norm_value)
            self.optimizer.step()
        return loss.detach()

    # ------------------------------------------------------------------ validation (trainer.py:78-181), B = 1 loop
    @torch.no_grad()
    def _validation_epoch(self, epoch):
        """Per item (noisy [1,L], clean [1,L], name, speech_type): cIRM loss of the B=1 forward (no drop_band, like the
        reference at B=1), enhanced waveform through decompress / complex product / iSTFT, SI-SDR on the device.
        Returns the mean SI-SDR of the "With_reverb" items (the reference's score, trainer.py:181); per-type losses
        and scores stay in ``self.last_validation``.  No host synchronisation inside the loop."""
        types = ("With_reverb", "No_reverb")
        zero = lambda: torch.zeros((), device=self.device)  # noqa: E731
        loss_total, n_items = zero(), 0
        loss_list = {k: zero() for k in types}
        score_list = {k: zero() for k in types}
        count = {k: 0 for k in types}
        model = self.core
        was_training = model.training
        model.eval()
        for noisy, clean, name, speech_type in self.valid_dataloader:
            assert len(name) == 1, "The batch size for the validation stage must be one."
            speech_type = speech_type[0]
            noisy = noisy.to(self.device, non_blocking=True)
            clean = clean.to(self.device, non_blocking=True)
            noisy_mag, _, noisy_real, noisy_imag = self.torch_stft(noisy)
            _, _, clean_real, clean_imag = self.torch_stft(clean)
            cIRM = build_complex_ideal_ratio_mask(noisy_real, noisy_imag, clean_real, clean_imag)
            cRM = model(noisy_mag.unsqueeze(1)).permute(0, 2, 3, 1)
            loss = self.loss_function(cIRM, cRM)
            cRM = decompress_cIRM(cRM)
            enhanced_real = cRM[..., 0] * noisy_real - cRM[..., 1] * noisy_imag
            enhanced_imag = cRM[..., 1] * noisy_real + cRM[..., 0] * noisy_imag
            enhanced = self.torch_istft((enhanced_real, enhanced_imag), length=noisy.size(-1), input_type="real_imag")
            assert noisy.shape == clean.shape == enhanced.shape
            loss_total += loss
            n_items += 1
            loss_list[speech_type] += loss
            score_list[speech_type] += si_sdr(clean, enhanced)[0]
            count[speech_type] += 1
        model.train(was_training)
        n = max(1, n_items)
        self.last_validation = {
            "loss_total": float(loss_total) / n,
            "loss": {k: float(loss_list[k]) / n for k in types},  # divided by len(dataloader) like trainer.py:163-168
            "si_sdr": {k: (float(score_list[k]) / count[k] if count[k] else 0.0) for k in types},
            "items": dict(count)}
        return self.last_validation["si_sdr"]["With_reverb"]

    def _is_best_epoch(self, score, save_max_metric_score=True):
        """base_trainer.py:254-266"""
        if save_max_metric_score and score >= self.best_score:
            self.best_score = score
            return True
        if not save_max_metric_score and score <= self.best_score:
            self.best_score = score
            return True
        return False

    def _train_epoch(self, epoch):
        loss_total = torch.zeros((), device=self.device)
        for batch in self.train_dataloader:  # (noisy, clean), or a dict of Dataset items that train_step mixes
            loss_total += self.train_step(batch) if isinstance(batch, dict) else self.train_step(*batch)
        return float(loss_total) / max(1, len(self.train_dataloader))  # the step loop itself never synchronises

    def train(self):
        """base_trainer.py:372-417: epochs of training; rank 0 checkpoints and validates (no barrier afterwards,
        like the reference)."""
        for epoch in range(self.start_epoch, self.epochs + 1):
            if self.only_validation and self.rank == 0:
                self.core.eval()
                self._validation_epoch(epoch)
                continue
            self.model.train()
            self.last_epoch_loss = self._train_epoch(epoch)
            if self.rank == 0 and self.save_checkpoint_interval != 0 and epoch % self.save_checkpoint_interval == 0:
                self._save_checkpoint(epoch)
            if (self.rank == 0 and self.valid_dataloader is not None and self.validation_interval
                    and epoch % self.validation_interval == 0):
                score = self._validation_epoch(epoch)
                if self._is_best_epoch(score, save_max_metric_score=self.save_max_metric_score):
                    self._save_checkpoint(epoch, is_best_epoch=True)

    # ------------------------------------------------------------------ checkpoints (base_trainer.py:170-252)
    def _save_checkpoint(self, epoch, is_best_epoch=False):
        state = {"epoch": epoch, "best_score": self.best_score, "optimizer": self.optimizer.state_dict(), "scaler": {},
                 "model": self.core.state_dict()}  # model.module.state_dict() under DDP (base_trainer.py:213-216)
        self.checkpoints_dir.mkdir(parents=True, exist_ok=True)
        torch.save(state, (self.checkpoints_dir / "latest_model.tar").as_posix())
        torch.save(state["model"], (self.checkpoints_dir / f"model_{str(epoch).zfill(4)}.pth").as_posix())
        if is_best_epoch:
            torch.save(state, (self.checkpoints_dir / "best_model.tar").as_posix())

    def _resume_checkpoint(self):
        path = self.checkpoints_dir.expanduser().absolute() / "latest_model.tar"
        assert path.exists(), f"{path} does not exist, can not load latest checkpoint."
        ckpt = torch.load(path.as_posix(), map_location="cpu")
        self.start_epoch = ckpt["epoch"] + 1
        self.best_score = ckpt["best_score"]
        self.optimizer.load_state_dict(ckpt["optimizer"])
        self.core.load_state_dict(ckpt["model"])
