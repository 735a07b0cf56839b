"""Training from fullsubnet_b200.dataset.Dataset with the mixing on the device: collated items of the golden corpus,
mixed by the Trainer, against the (noisy, clean) of the unmodified reference Dataset (tests/golden/dataset_train.npz,
within the 2e-5 relative max of tests/golden/mix.npz); a step on a Dataset batch is bit for bit the step on the
(noisy, clean) that dataset.snr_mix makes from it, for every model the Trainer trains; an epoch over a DataLoader of the
Dataset never waits on the device inside the step loop."""
import random

import numpy as np
import pytest
import torch
from torch.utils.data import DataLoader

from conftest import rel_max
from oracle import make_golden_dataset as MG

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    return MG.write_corpus(str(tmp_path_factory.mktemp("corpus")))


def trainer_for(model, n_fft, tmp_path, epochs=1):
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.optim import FusedClipAdam
    from fullsubnet_b200.trainer import Trainer
    cfg = {"meta": {"use_amp": False, "save_dir": str(tmp_path), "experiment_name": "d"},
           "acoustics": {"n_fft": n_fft, "hop_length": n_fft // 2, "win_length": n_fft},
           "trainer": {"train": {"epochs": epochs, "save_checkpoint_interval": 1, "clip_grad_norm_value": 10}}}
    return Trainer(None, 0, cfg, False, False, model, mse_loss(), FusedClipAdam(model.parameters(), lr=1e-3), None, None)


def fullsubnet(dev, prec):
    from fullsubnet_b200.fullsubnet.model import Model
    from oracle import fullsubnet_oracle as O
    from oracle.make_golden_train import SMALL
    m = Model(**SMALL)
    m.load_state_dict(O.make_state_dict(seed=7, args=SMALL, sb_fc_gain=8.0), strict=True)
    m.train_precision = prec
    return m.to(dev).train(), 64


def fast_fullsubnet(dev, prec):
    from fullsubnet_b200.fast_fullsubnet.model import Model
    from oracle import fast_fullsubnet_oracle as FO
    a = dict(FO.DEFAULT_FAST_ARGS, shrink_size=3, look_ahead=1, encoder_output_num_neighbors=1, bottleneck_hidden_size=128)
    m = Model(**a)
    m.load_state_dict(FO.make_fast_state_dict(seed=3, args=a), strict=True)
    m.train_precision = prec
    return m.to(dev).train(), 512


def fullband_baseline(dev, prec):
    from fullsubnet_b200.fullband_baseline.model import Model
    from oracle import fullband_baseline_oracle as BO
    a = dict(BO.DEFAULT_FBB_ARGS, num_freqs=33, hidden_size=32)
    m = Model(**a)
    m.load_state_dict(BO.make_fbb_state_dict(seed=5, args=a), strict=True)
    m.train_precision = prec
    return m.to(dev).train(), 64


def test_collated_items_mixed_by_trainer_match_reference(golden, corpus, dev):
    from fullsubnet_b200.dataset import Dataset, mix_batch
    g = golden("dataset_train")
    ds = Dataset(**corpus)
    random.seed(int(g["seed"]))
    np.random.seed(int(g["seed"]))
    batches = list(DataLoader(ds, batch_size=8, shuffle=False, num_workers=0))
    assert len(batches) == len(g["clean"]) // 8
    for j, batch in enumerate(batches):
        noisy, clean = mix_batch(batch, dev)
        for r in range(8):
            i = 8 * j + r
            assert rel_max(noisy[r].cpu(), g["noisy"][i]) < 2e-5, i
            assert rel_max(clean[r].cpu(), g["clean_out"][i]) < 2e-5, i


def synthetic_batch(B=4, L=8000, Lr=1700, seed=0):
    """A collated Dataset batch (CPU tensors) with reverberant and dry rows."""
    rng = np.random.default_rng(seed)
    t = np.arange(L) / 16000
    clean = np.stack([0.3 * np.sin(2 * np.pi * (200 + 50 * b) * t) * (0.5 + 0.5 * np.sin(2 * np.pi * 4 * t))
                      + 0.01 * rng.standard_normal(L) for b in range(B)]).astype(np.float32)
    rir_len = np.array([600, 0, 1700, 0][:B], np.int32)
    rir = np.zeros((B, Lr), np.float32)
    for b, n in enumerate(rir_len):
        rir[b, :n] = rng.standard_normal(n) * np.exp(-np.arange(n) / (n / 5.0))
        rir[b, :1] = 0.9
    f = lambda v: torch.from_numpy(np.asarray(v, np.float32))  # noqa: E731
    return {"clean": f(clean), "noise": f(0.2 * rng.standard_normal((B, L))), "rir": f(rir),
            "rir_len": torch.from_numpy(rir_len), "snr": f(rng.integers(-5, 21, B)),
            "noisy_target_dB_FS": f(rng.integers(-35, -15, B)), "target_dB_FS": f(np.full(B, -25))}


@pytest.mark.parametrize("build,prec", [(fullsubnet, "fp32"), (fullsubnet, "tf32_tc"), (fast_fullsubnet, "fp32"),
                                        (fullband_baseline, "fp32")])
def test_dataset_batch_step_equals_premixed_step(dev, tmp_path, build, prec):
    from fullsubnet_b200.dataset import snr_mix
    batch = synthetic_batch()
    m1, n_fft = build(dev, prec)
    m2, _ = build(dev, prec)
    t1, t2 = trainer_for(m1, n_fft, tmp_path / "a"), trainer_for(m2, n_fft, tmp_path / "b")
    noisy, clean = snr_mix(batch["clean"].to(dev), batch["noise"].to(dev), batch["snr"].to(dev), -25.0,
                           batch["noisy_target_dB_FS"].to(dev), rir=batch["rir"].to(dev), rir_len=batch["rir_len"])
    for _ in range(2):
        l1 = t1.train_step(batch)
        l2 = t2.train_step(noisy, clean)
        assert torch.equal(l1, l2), (float(l1), float(l2))
        for (k, p1), p2 in zip(m1.named_parameters(), m2.parameters()):
            assert torch.equal(p1.grad, p2.grad), k
            assert torch.equal(p1, p2), k


def test_epoch_over_dataset_loader_never_synchronises(corpus, dev, tmp_path):
    """Trainer.train() over DataLoader(Dataset): with CUDA's sync debug mode set to "error" for the whole step loop (the
    epoch's final loss read-back is outside it), mixing and steps never wait on the device."""
    from fullsubnet_b200.dataset import Dataset

    class Guarded:
        def __init__(self, loader):
            self.loader = loader

        def __len__(self):
            return len(self.loader)

        def __iter__(self):
            torch.cuda.set_sync_debug_mode("error")
            try:
                yield from self.loader
            finally:
                torch.cuda.set_sync_debug_mode("default")

    ds = Dataset(**dict(corpus, reverb_proportion=0.75))
    random.seed(0)
    np.random.seed(0)
    loader = DataLoader(ds, batch_size=6, shuffle=True, num_workers=0, drop_last=True)
    m, n_fft = fullsubnet(dev, "tf32_tc")
    tr = trainer_for(m, n_fft, tmp_path)
    tr.train_dataloader = Guarded(loader)
    before = [p.detach().clone() for p in m.parameters()]
    tr.train()
    assert torch.cuda.get_sync_debug_mode() == 0
    assert np.isfinite(tr.last_epoch_loss) and tr.last_epoch_loss > 0
    assert any(not torch.equal(a, p) for a, p in zip(before, m.parameters()))
    assert (tmp_path / "d" / "checkpoints" / "latest_model.tar").exists()
