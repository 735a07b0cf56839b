"""Mirror of recipes/dns_interspeech_2020/fullsubnet/trainer.py:14-181 (and of fast_fullsubnet/trainer.py and
fullband_baseline/trainer.py:32-71, the same loop without drop_band) on top of
audio_zen/trainer/base_trainer.py:28-218 - the parts of the trainer that are arithmetic on the hot path (SURVEY 8a row
A11, 8f rank 4): mixing of a Dataset batch, STFT of noisy/clean, cIRM target + drop_band, Model.forward, MSE,
backward, gradient mean over ranks, clip, Adam; and the validation loop, its B=1 items enhanced in groups (enhance +
per-clip loss + SI-SDR, all on the device).

Same constructor arguments and config keys as the reference, so `train.py:65-80` can construct it unchanged
(``meta.use_amp`` is accepted: the kernels compute in fp32 / tf32, at least the precision of the reference's fp16
autocast, so the GradScaler is the identity and ``scaler`` stays an empty dict in the checkpoint schema
{epoch, best_score, optimizer, scaler, model} of base_trainer.py:208-218).  TensorBoard, audio / spectrogram
visualisation and PESQ (base_trainer.py:277-370) are outside the hot path.  STOI is computed on the device
(``metrics.stoi``) for the noisy and the enhanced clip of every validation item when the recipe's
``[trainer.visualization] metrics`` list names it, as base_trainer.py:316-370 does.

Two gradient paths, both ONE all-reduce of gradients per step (SURVEY 8e):
  * ``model`` wrapped in DistributedDataParallel exactly like base_trainer.py:32 - the autograd Function behind
    Model.forward delivers the gradients to DDP's hooks, DDP averages them; nothing else is reduced here;
  * plain ``model`` on every rank (default): rank 0's parameters are broadcast once at construction (what DDP's
    constructor does), ``model.flat_grad()`` makes every ``p.grad`` a view of one flat buffer, ``dist.all_reduce``
    moves that buffer once per step, and FusedClipAdam folds the 1/world mean into its clip coefficient."""
from __future__ import annotations

from functools import partial
from pathlib import Path

import numpy as np
import torch

from . import _lib
from .acoustics.feature import drop_band, istft, stft
from .acoustics.mask import build_complex_ideal_ratio_mask
from .dataset import mix_batch
from .inferencer import Inferencer, plan_batches
from .loss import MSELoss, cirm_mse_per_clip
from .metrics import stoi
from .optim import FusedClipAdam


def unwrap(model):
    """The fullsubnet Model behind an optional DistributedDataParallel wrapper (base_trainer.py:32)."""
    return model.module if isinstance(model, torch.nn.parallel.DistributedDataParallel) else model


def broadcast_parameters(model, dist, src: int = 0) -> None:
    """What DistributedDataParallel does at construction: every rank starts from rank ``src``'s parameters/buffers."""
    with torch.no_grad():
        for t in list(model.parameters()) + list(model.buffers()):
            dist.broadcast(t.data, src)


def si_sdr(reference: torch.Tensor, estimation: torch.Tensor, lengths=None) -> torch.Tensor:
    """audio_zen/metrics.py:6-31 on the device: [B,L] x [B,L] -> [B] dB (fsn_si_sdr).  ``lengths`` (B ints, max L):
    clip b is row b's first lengths[b] samples, and out[b] equals the call on it alone (fsn_si_sdr_lengths)."""
    reference = _lib.require_cuda(reference, "reference")
    estimation = _lib.require_cuda(estimation, "estimation")
    assert reference.shape == estimation.shape and reference.dim() == 2
    B, L = reference.shape
    lens = None if lengths is None else _lib.lengths_table(lengths, B, L)
    out = torch.empty(B, dtype=torch.float32, device=reference.device)
    with torch.cuda.device(reference.device):
        _lib.check(_lib.load().fsn_si_sdr_lengths(reference.data_ptr(), estimation.data_ptr(),
                                                  None if lens is None else lens.ctypes.data, B, L, out.data_ptr(),
                                                  _lib.stream_ptr(reference.device)))
    return out


def validation_groups(inferencer, lengths, batch_size: int, max_padding: float):
    """The groups of validation items (indices into ``lengths``) that share one enhance call: ``plan_batches``, with
    clips of different lengths together only where the model's fused call takes per-clip lengths
    (``Inferencer.supports_lengths``); fast_fullsubnet gets equal-length groups, as in ``enhance_files``."""
    return plan_batches(lengths, batch_size, max_padding if inferencer.supports_lengths() else 0.0)


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
        self.acoustics = ac
        self.train_config = config["trainer"]["train"]
        self.epochs = self.train_config["epochs"]
        self.save_checkpoint_interval = self.train_config["save_checkpoint_interval"]
        self.clip_grad_norm_value = self.train_config["clip_grad_norm_value"]
        assert self.save_checkpoint_interval >= 1, \
            "Check the 'save_checkpoint_interval' parameter in the config. It should be large than one."
        self.validation_config = config["trainer"].get("validation", {})
        self.validation_interval = self.validation_config.get("validation_interval", 1)
        self.save_max_metric_score = self.validation_config.get("save_max_metric_score", True)
        # validation items per enhance call, and how much padding lets clips of different lengths share one
        self.validation_batch_size = self.validation_config.get("batch_size", 32)
        self.validation_max_padding = self.validation_config.get("max_padding", 0.25)
        plan_batches([], self.validation_batch_size, self.validation_max_padding)  # refuses bad values here
        # the recipes' [trainer.visualization] metrics list: "STOI" there adds the STOI of noisy and enhanced speech
        visualization = config["trainer"].get("visualization", {}) or {}
        self.validation_stoi = "STOI" in (visualization.get("metrics") or ())
        self.last_validation_stoi = None  # per-item (enhanced, noisy) STOI of the last validation, dataloader order
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

    # ------------------------------------------------------------------ validation (trainer.py:78-181), in groups
    @torch.no_grad()
    def _validation_items(self):
        """The validation dataloader's items (noisy [1,L], clean [1,L], name, speech_type) evaluated in groups
        (``validation_groups``): one fused enhance call per group (the model's mask + iSTFT, as
        Inferencer.enhance_batch), then ``cirm_mse_per_clip`` and ``si_sdr`` over each clip's own length, and with
        ``validation_stoi`` the STOI of the enhanced and of the noisy clip (``metrics.stoi``).  Returns (loss float32 [N],
        SI-SDR float32 [N], speech types) in dataloader order, after ONE device-to-host copy; the STOI rows go to
        ``last_validation_stoi`` ({"enhanced": [N], "noisy": [N]}, None without STOI).  Each loss equals the reference's
        B=1 ``loss_function(cIRM, cRM)`` on that item alone (no drop_band), bit for bit."""
        if not isinstance(self.loss_function, (MSELoss, torch.nn.MSELoss)) or \
                getattr(self.loss_function, "reduction", "mean") != "mean":
            raise NotImplementedError("fullsubnet_b200: validation computes the recipes' mean-squared cIRM loss only")
        ac = self.acoustics
        n_fft, hop, win = ac["n_fft"], ac["hop_length"], ac["win_length"]
        inferencer = Inferencer(config={"acoustics": ac}, model=self.core, device=self.device)
        noisy_items, clean_items, item_types = [], [], []
        for noisy, clean, name, speech_type in self.valid_dataloader:
            assert len(name) == 1, "The batch size for the validation stage must be one."
            assert noisy.shape == clean.shape and noisy.shape[0] == 1
            noisy_items.append(noisy.to(self.device, non_blocking=True).reshape(-1))
            clean_items.append(clean.to(self.device, non_blocking=True).reshape(-1))
            item_types.append(speech_type[0])
        lens = [x.numel() for x in noisy_items]
        groups = validation_groups(inferencer, lens, self.validation_batch_size, self.validation_max_padding)
        order = [i for g in groups for i in g]
        rows = 4 if self.validation_stoi else 2
        # loss, SI-SDR (, STOI enhanced, STOI noisy) in group order
        values = torch.empty(rows, len(order), dtype=torch.float32, device=self.device)
        pos = 0
        for g in groups:
            g_lens = [lens[i] for i in g]
            lengths = g_lens if min(g_lens) != max(g_lens) else None
            noisy = torch.nn.utils.rnn.pad_sequence([noisy_items[i] for i in g], batch_first=True)
            clean = torch.nn.utils.rnn.pad_sequence([clean_items[i] for i in g], batch_first=True)
            enhanced, crm = inferencer.enhance_batch(noisy, lengths=lengths, return_crm=True)
            values[0, pos:pos + len(g)] = cirm_mse_per_clip(noisy, clean, crm, n_fft, hop, win, lengths)
            values[1, pos:pos + len(g)] = si_sdr(clean, enhanced, lengths)
            if self.validation_stoi:
                values[2, pos:pos + len(g)] = stoi(clean, enhanced, lengths)
                values[3, pos:pos + len(g)] = stoi(clean, noisy, lengths)
            pos += len(g)
        per_item = np.empty((rows, len(order)), dtype=np.float32)
        per_item[:, order] = values.cpu().numpy()
        self.last_validation_stoi = {"enhanced": per_item[2], "noisy": per_item[3]} if self.validation_stoi else None
        return per_item[0], per_item[1], item_types

    def _validation_epoch(self, epoch):
        """Loss and SI-SDR of every validation item (``_validation_items``), summed per speech type in float32 in
        dataloader order like the reference's B=1 loop.  Returns the mean SI-SDR of the "With_reverb" items (the
        reference's score, trainer.py:181); per-type losses and scores stay in ``self.last_validation``, with the per-type
        mean STOI of the noisy and the enhanced items under "stoi" when the recipe's visualization metrics name STOI."""
        types = ("With_reverb", "No_reverb")
        model = self.core
        was_training = model.training
        model.eval()
        try:
            loss, score, item_types = self._validation_items()
        finally:
            model.train(was_training)
        zero = np.float32(0.0)
        loss_total, loss_list, score_list = zero, {k: zero for k in types}, {k: zero for k in types}
        count = {k: 0 for k in types}
        for i, speech_type in enumerate(item_types):
            loss_total += loss[i]
            loss_list[speech_type] += loss[i]
            score_list[speech_type] += score[i]
            count[speech_type] += 1
        n = max(1, len(item_types))
        self.last_validation = {
            "loss_total": float(loss_total) / n,
            "loss": {k: float(loss_list[k]) / n for k in types},  # divided by len(dataloader) like trainer.py:163-168
            "si_sdr": {k: (float(score_list[k]) / count[k] if count[k] else 0.0) for k in types},
            "items": dict(count)}
        if self.validation_stoi:
            st = self.last_validation_stoi
            sums = {k: {"noisy": zero, "enhanced": zero} for k in types}
            for i, speech_type in enumerate(item_types):
                sums[speech_type]["noisy"] += st["noisy"][i]
                sums[speech_type]["enhanced"] += st["enhanced"][i]
            self.last_validation["stoi"] = {
                k: {w: (float(sums[k][w]) / count[k] if count[k] else 0.0) for w in ("noisy", "enhanced")} for k in types}
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
