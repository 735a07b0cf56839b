"""CPU-only checks of validation in groups: the workspace query of fsn_cirm_mse_per_clip, the argument checks of it and of
fsn_si_sdr_lengths (all answered before any CUDA call), and the grouping of the validation items."""
import ctypes as C
import random

import pytest
import torch


def _mse_call(lib, lengths, L_max, n_fft=512, hop=256, win=512, loss=None, ptrs=16):
    arr = None if lengths is None else (C.c_int32 * len(lengths))(*lengths)
    B = len(lengths) if lengths is not None else 2
    return lib.fsn_cirm_mse_per_clip(ptrs, ptrs, arr, B, L_max, n_fft, hop, win, ptrs, loss, None, 0, None)


def test_cirm_mse_workspace_query_needs_no_gpu():
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    n = lib.fsn_cirm_mse_per_clip_workspace_bytes(4, 64000, 512, 256)
    # four spectra [B, F, T] of float32, 1024 partials and a length per clip, each rounded up to 256 bytes
    assert n >= 4 * (4 * 257 * 251 * 4) + 4 * 1024 * 4 + 4 * 4
    assert lib.fsn_cirm_mse_per_clip_workspace_bytes(8, 64000, 512, 256) > n
    assert lib.fsn_cirm_mse_per_clip_workspace_bytes(4, 48000, 960, 480) > 0  # the direct DFT
    assert lib.fsn_cirm_mse_per_clip_workspace_bytes(4, 64000, 501, 256) == 0  # an n_fft the STFT does not take
    assert lib.fsn_last_error_code() == _lib.FSN_ERR_UNSUPPORTED
    assert lib.fsn_cirm_mse_per_clip_workspace_bytes(0, 64000, 512, 256) == 0
    assert lib.fsn_cirm_mse_per_clip_workspace_bytes(4, 256, 512, 256) == 0  # L_max <= n_fft/2


def test_cirm_mse_rejects_bad_arguments_before_any_cuda_call():
    """No workspace, no device: every one of these fails on its argument check."""
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    assert _mse_call(lib, [4000, 256, 3000], 4000, loss=16) == _lib.FSN_ERR_SHAPE  # too short: <= n_fft/2
    assert b"clip 1" in lib.fsn_last_error()
    assert _mse_call(lib, [4000, 4001, 3000], 4000, loss=16) == _lib.FSN_ERR_SHAPE  # longer than the row
    assert b"clip 1" in lib.fsn_last_error()
    assert _mse_call(lib, [3900, 257, 3000], 4000, loss=16) == _lib.FSN_ERR_SHAPE  # max(lengths) != L_max
    assert b"3900" in lib.fsn_last_error()
    assert _mse_call(lib, [200, 200], 200, loss=16) == _lib.FSN_ERR_SHAPE  # L_max <= n_fft/2
    assert _mse_call(lib, [4000, 3000], 4000, n_fft=501, loss=16) == _lib.FSN_ERR_UNSUPPORTED
    assert b"n_fft=501" in lib.fsn_last_error()
    assert _mse_call(lib, [4000, 3000], 4000, n_fft=4096, loss=16) == _lib.FSN_ERR_UNSUPPORTED
    assert _mse_call(lib, [4000, 3000], 4000, hop=0, loss=16) == _lib.FSN_ERR_SHAPE
    assert _mse_call(lib, [4000, 3000], 4000, loss=None) == _lib.FSN_ERR_SHAPE  # no output
    assert _mse_call(lib, [4000, 3000], 4000, loss=16, ptrs=None) == _lib.FSN_ERR_SHAPE  # no inputs
    # valid arguments reach the workspace check, the last one before the first launch (stand-in pointers, never read)
    assert _mse_call(lib, [4000, 257, 3000], 4000, loss=16) == _lib.FSN_ERR_WORKSPACE
    assert _mse_call(lib, None, 4000, loss=16) == _lib.FSN_ERR_WORKSPACE


def test_si_sdr_lengths_rejects_bad_lengths_before_any_cuda_call():
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    for lens, L_max in (([100, 0], 100), ([100, 101], 100), ([-1, 50], 100)):
        arr = (C.c_int32 * len(lens))(*lens)
        assert lib.fsn_si_sdr_lengths(16, 16, arr, len(lens), L_max, 16, None) == _lib.FSN_ERR_SHAPE
        assert b"clip" in lib.fsn_last_error()
    arr = (C.c_int32 * 1)(10)
    assert lib.fsn_si_sdr_lengths(16, 16, arr, 0, 10, 16, None) == _lib.FSN_ERR_SHAPE
    assert lib.fsn_si_sdr_lengths(16, 16, arr, 1, 0, 16, None) == _lib.FSN_ERR_SHAPE


def test_python_wrappers_refuse_host_tensors():
    from fullsubnet_b200.loss import cirm_mse_per_clip
    from fullsubnet_b200.trainer import si_sdr
    x = torch.zeros(2, 1000)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        cirm_mse_per_clip(x, x, torch.zeros(2, 2, 257, 4), 512, 256, 512, [1000, 900])
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        si_sdr(x, x, [1000, 900])


def _models():
    from fullsubnet_b200.fast_fullsubnet.model import Model as Fast
    from fullsubnet_b200.fullband_baseline.model import Model as Fbb
    from fullsubnet_b200.fullsubnet.model import Model as Fsn
    from oracle import fast_fullsubnet_oracle as FO
    from oracle import fullband_baseline_oracle as BO
    from oracle import fullsubnet_oracle as O
    return {"fullsubnet": Fsn(**O.DEFAULT_MODEL_ARGS), "fullband_baseline": Fbb(**BO.DEFAULT_FBB_ARGS),
            "fast_fullsubnet": Fast(**FO.DEFAULT_FAST_ARGS)}


@pytest.mark.parametrize("batch_size", [1, 3, 1000])
@pytest.mark.parametrize("max_padding", [0.0, 0.25])
def test_grouping_covers_every_item_once(batch_size, max_padding):
    """Each validation item is in exactly one group; fast_fullsubnet (no fused call) and every model at a
    non-power-of-two n_fft get equal-length groups."""
    from fullsubnet_b200.inferencer import Inferencer
    from fullsubnet_b200.trainer import validation_groups
    rng = random.Random(5)
    lens = [rng.choice([16000, 16001, 24000, 160000]) if rng.random() < 0.5 else rng.randint(16000, 160000)
            for _ in range(300)]
    for name, m in _models().items():
        for n_fft in (512, 960):
            ac = {"n_fft": n_fft, "hop_length": n_fft // 2, "win_length": n_fft}
            inf = Inferencer(config={"acoustics": ac}, model=m, device="cpu")
            groups = validation_groups(inf, lens, batch_size, max_padding)
            assert sorted(i for g in groups for i in g) == list(range(len(lens))), (name, n_fft)
            mixed_ok = name != "fast_fullsubnet" and n_fft == 512
            for g in groups:
                assert 1 <= len(g) <= batch_size
                Lm = max(lens[i] for i in g)
                assert len(g) * Lm - sum(lens[i] for i in g) <= max_padding * len(g) * Lm
                if not (mixed_ok and max_padding > 0):
                    assert len({lens[i] for i in g}) == 1, (name, n_fft, g)


def test_validation_keys_have_defaults_and_are_checked():
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.trainer import Trainer
    from oracle import fullsubnet_oracle as O
    from fullsubnet_b200.fullsubnet.model import Model

    class CpuModel(Model):
        def cuda(self, device=None):  # the Trainer's constructor moves the model; nothing here needs a device
            return self

    def make(validation):
        cfg = {"meta": {"save_dir": "/nonexistent", "experiment_name": "v"},
               "acoustics": {"n_fft": 512, "hop_length": 256, "win_length": 512},
               "trainer": {"train": {"epochs": 1, "save_checkpoint_interval": 1, "clip_grad_norm_value": 10},
                           "validation": validation}}
        m = CpuModel(**O.DEFAULT_MODEL_ARGS)
        return Trainer(None, 0, cfg, False, False, m, mse_loss(), torch.optim.SGD(m.parameters(), lr=0.0), [], None)

    t = make({"validation_interval": 1, "save_max_metric_score": True})  # a reference config without the new keys
    assert t.validation_batch_size >= 1 and 0.0 <= t.validation_max_padding < 1.0
    t = make({"batch_size": 4, "max_padding": 0.0})
    assert (t.validation_batch_size, t.validation_max_padding) == (4, 0.0)
    with pytest.raises(ValueError):
        make({"batch_size": 0})
    with pytest.raises(ValueError):
        make({"max_padding": 1.0})
