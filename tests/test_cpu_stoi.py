"""CPU-only checks of STOI: the float64 oracle's properties (and, where pystoi is installed, the oracle against it), the
argument checks of fsn_stoi / fsn_debug_stoi_stages and its workspace query (all answered before any CUDA call), the
Python wrappers' checks, the Trainer's opt-in key and the metrics CLI's file pairing and refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import stoi_oracle as S
from oracle.stoi_oracle import speechlike

PINNED_BANDS = [(7, 9), (9, 11), (11, 14), (14, 17), (17, 22), (22, 27), (27, 34), (34, 43), (43, 55), (55, 69),
                (69, 87), (87, 109), (109, 138), (138, 174), (174, 219)]


def test_oracle_identity_scale_and_silence():
    x = speechlike(16000 * 2, seed=1)
    assert abs(S.stoi(x, x) - 1.0) < 1e-12
    assert abs(S.stoi(x, 3.7 * x) - 1.0) < 1e-12
    assert S.stoi(np.zeros_like(x), x) == 0.0  # every frame kept, every correlation 0
    assert S.stoi(x, np.zeros_like(x)) == 0.0
    noisy = x + np.random.default_rng(2).standard_normal(len(x)).astype(np.float32) * 0.05
    assert 0.0 < S.stoi(x, noisy) < 1.0


def test_oracle_fewer_than_30_frames_gives_1e_5():
    # 29 STFT frames after removal need n_kept = 30 frames of the clean clip, all kept: 10 kHz, 31 * 128 + 1 samples
    n = (30 + 1) * 128 + 1
    x = speechlike(n, seed=3, sr=10000) + 0.05
    st = S.stages(x, x, 10000)
    assert st["mask"].all() and st["mask"].size == 30
    assert st["bands"][0].shape == (15, 29)
    assert S.stoi(x, x, 10000) == 1e-5
    x = speechlike(n + 128, seed=3, sr=10000) + 0.05  # 30 frames
    assert abs(S.stoi(x, x, 10000) - 1.0) < 1e-12


def test_oracle_resampled_length_filter_and_bands():
    for L in (410, 411, 16000, 12345, 160000):
        assert len(S.resample(np.zeros(L, np.float32), 16000)) == -(-5 * L // 8)
    p, q, h, beta = S.resample_filter(16000)
    assert (p, q, len(h)) == (5, 8, 581)
    assert abs(beta - 5.65326) < 1e-12
    assert S.band_edges() == PINNED_BANDS
    assert S.min_length(16000) == 410 and S.min_length(10000) == 257
    with pytest.raises(ValueError):
        S.stoi(np.zeros(409), np.zeros(409))


def test_oracle_matches_pystoi():
    pystoi = pytest.importorskip("pystoi")
    rng = np.random.default_rng(4)
    for sr, n in ((16000, 40000), (16000, 23456), (10000, 30000)):
        x = speechlike(n, seed=int(rng.integers(1 << 30)), sr=sr)
        x[n // 3:n // 2] = 0.0
        y = x + 0.1 * rng.standard_normal(n).astype(np.float32)
        got, want = S.stoi(x, y, sr), pystoi.stoi(x, y, sr, extended=False)
        assert abs(got - want) < 1e-10, (sr, n, got, want)


# ---------------------------------------------------------------------------------------------- the C ABI, no GPU
def _call(lib, lengths, L_max, sr=16000, B=None, ptrs=16, out=16, ws=16, ws_bytes=0):
    arr = None if lengths is None else (C.c_int32 * len(lengths))(*lengths)
    B = (len(lengths) if lengths is not None else 2) if B is None else B
    return lib.fsn_stoi(ptrs, ptrs, arr, B, L_max, sr, out, ws, ws_bytes, None)


def test_stoi_workspace_query_needs_no_gpu_and_is_monotone():
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    n = lib.fsn_stoi_workspace_bytes(4, 160000, 16000)
    assert n >= 4 * 32 * 100000  # two float64 signals, resampled and compacted
    prev_b = 0
    for B in (1, 2, 3, 8, 300):
        cur = lib.fsn_stoi_workspace_bytes(B, 16000, 16000)
        assert cur > prev_b
        prev_b = cur
    prev_l = 0
    for L in (410, 411, 1000, 1001, 16000, 160000):
        cur = lib.fsn_stoi_workspace_bytes(3, L, 16000)
        assert cur >= prev_l
        prev_l = cur
    assert lib.fsn_stoi_workspace_bytes(3, 160000, 10000) > lib.fsn_stoi_workspace_bytes(3, 160000, 16000)
    assert lib.fsn_stoi_workspace_bytes(4, 16000, 8000) == 0
    assert lib.fsn_last_error_code() == _lib.FSN_ERR_UNSUPPORTED
    assert lib.fsn_stoi_workspace_bytes(0, 16000, 16000) == 0
    assert lib.fsn_last_error_code() == _lib.FSN_ERR_SHAPE
    assert lib.fsn_stoi_workspace_bytes(4, 409, 16000) == 0
    assert lib.fsn_stoi_workspace_bytes(4, 256, 10000) == 0
    assert lib.fsn_stoi_workspace_bytes(4, 257, 10000) > 0


def test_stoi_rejects_bad_arguments_before_any_cuda_call():
    """No workspace, no device: every one of these fails on its argument check."""
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    assert _call(lib, [4000, 409, 3000], 4000) == _lib.FSN_ERR_SHAPE  # one sample short of a frame at 16 kHz
    assert b"clip 1" in lib.fsn_last_error() and b"410" in lib.fsn_last_error()
    assert _call(lib, [4000, 256, 3000], 4000, sr=10000) == _lib.FSN_ERR_SHAPE
    assert b"clip 1" in lib.fsn_last_error() and b"257" in lib.fsn_last_error()
    assert _call(lib, [4000, 4001], 4000) == _lib.FSN_ERR_SHAPE  # longer than the row
    assert b"clip 1" in lib.fsn_last_error()
    assert _call(lib, [4000, 0], 4000) == _lib.FSN_ERR_SHAPE
    assert _call(lib, [4000, 3000], 4000, sr=8000) == _lib.FSN_ERR_UNSUPPORTED
    assert b"8000" in lib.fsn_last_error()
    assert _call(lib, [4000, 3000], 4000, sr=44100) == _lib.FSN_ERR_UNSUPPORTED
    assert _call(lib, None, 4000, B=0) == _lib.FSN_ERR_SHAPE
    assert _call(lib, None, 4000, B=-3) == _lib.FSN_ERR_SHAPE
    assert _call(lib, None, 409) == _lib.FSN_ERR_SHAPE
    assert _call(lib, [4000, 3000], 4000, ptrs=None) == _lib.FSN_ERR_SHAPE
    assert _call(lib, [4000, 3000], 4000, out=None) == _lib.FSN_ERR_SHAPE
    # valid arguments reach the workspace check, the last one before the first launch (stand-in pointers, never read)
    assert _call(lib, [4000, 410, 3000], 4000) == _lib.FSN_ERR_WORKSPACE
    assert _call(lib, None, 4000) == _lib.FSN_ERR_WORKSPACE
    need = lib.fsn_stoi_workspace_bytes(2, 4000, 16000)
    assert _call(lib, None, 4000, ws_bytes=need - 1) == _lib.FSN_ERR_WORKSPACE
    assert _call(lib, None, 4000, ws=None, ws_bytes=need) == _lib.FSN_ERR_WORKSPACE
    # the hook checks the same, and its stage buffers
    arr = (C.c_int32 * 2)(4000, 409)
    assert lib.fsn_debug_stoi_stages(16, 16, arr, 2, 4000, 16000, 16, 16, 16, 16, 16, 16, 16, need, None) == \
        _lib.FSN_ERR_SHAPE
    assert b"clip 1" in lib.fsn_last_error()
    assert lib.fsn_debug_stoi_stages(16, 16, None, 2, 4000, 16000, 16, None, 16, 16, 16, 16, 16, 1 << 40, None) == \
        _lib.FSN_ERR_SHAPE
    assert lib.fsn_debug_stoi_stages(16, 16, None, 2, 4000, 16000, 16, 16, 16, 16, 16, 16, 16, 0, None) == \
        _lib.FSN_ERR_WORKSPACE


def test_python_wrappers_check_lengths_and_refuse_host_tensors():
    from fullsubnet_b200 import metrics
    x = torch.zeros(2, 1000)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        metrics.stoi(x, x, [1000, 900])
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        metrics.stoi(x, x)
    from fullsubnet_b200 import _lib
    with pytest.raises(ValueError, match="entries"):
        _lib.lengths_table([1000], 2, 1000)
    with pytest.raises(ValueError, match="exceeds"):
        _lib.lengths_table([1000, 1001], 2, 1000)
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="no CPU path"):
            metrics.STOI(np.zeros(1000, np.float32), np.zeros(1000, np.float32))
        with pytest.raises(RuntimeError, match="no CPU path"):
            metrics.SI_SDR(np.zeros(1000, np.float32), np.zeros(1000, np.float32))


def _cpu_trainer(trainer_cfg):
    from fullsubnet_b200.fullsubnet.model import Model
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.trainer import Trainer
    from oracle import fullsubnet_oracle as O

    class CpuModel(Model):
        def cuda(self, device=None):  # the Trainer's constructor moves the model; nothing here needs a device
            return self

    cfg = {"meta": {"save_dir": "/nonexistent", "experiment_name": "v"},
           "acoustics": {"n_fft": 512, "hop_length": 256, "win_length": 512},
           "trainer": dict({"train": {"epochs": 1, "save_checkpoint_interval": 1, "clip_grad_norm_value": 10},
                            "validation": {"validation_interval": 1}}, **trainer_cfg)}
    m = CpuModel(**O.DEFAULT_MODEL_ARGS)
    return Trainer(None, 0, cfg, False, False, m, mse_loss(), torch.optim.SGD(m.parameters(), lr=0.0), [], None)


def test_trainer_reads_the_recipes_visualization_metrics():
    assert not _cpu_trainer({}).validation_stoi
    assert not _cpu_trainer({"visualization": {"n_samples": 10}}).validation_stoi
    assert not _cpu_trainer({"visualization": {"metrics": ["SI_SDR", "WB_PESQ"]}}).validation_stoi
    t = _cpu_trainer({"visualization": {"n_samples": 10, "num_workers": 36,
                                        "metrics": ["WB_PESQ", "NB_PESQ", "STOI", "SI_SDR"]}})
    assert t.validation_stoi and t.last_validation_stoi is None


def _write(path, n, seed):
    from fullsubnet_b200.inferencer import Inferencer
    path.parent.mkdir(parents=True, exist_ok=True)
    Inferencer.write_wav(path, (speechlike(n, seed) * 32767).astype(np.int16))


def test_cli_pairs_files_by_basename_and_refuses_pesq(tmp_path):
    from fullsubnet_b200 import metrics
    ref, est = tmp_path / "clean", tmp_path / "enhanced"
    for i, name in enumerate(("b_2", "a_1", "c_3")):
        _write(ref / f"{name}.wav", 4000 + i, i)
        _write(est / "sub" / f"{name}.wav", 4000 + i, 10 + i)
    pairs = metrics.pair_files(ref, est)
    assert [p[0] for p in pairs] == ["a_1", "b_2", "c_3"]
    assert all(p[1].stem == p[2].stem == p[0] and p[1].parent == ref for p in pairs)
    _write(est / "d_4.wav", 4000, 1)
    with pytest.raises(ValueError, match="d_4"):
        metrics.pair_files(ref, est)
    for name in ("WB_PESQ", "NB_PESQ"):
        with pytest.raises(ValueError, match="PESQ"):
            metrics.parse_metrics(f"SI_SDR,{name}")
        with pytest.raises(SystemExit):
            metrics.main(["-R", str(ref), "-E", str(est), "-M", name])
    with pytest.raises(ValueError, match="unknown metric"):
        metrics.parse_metrics("ESTOI")
    assert metrics.parse_metrics("STOI, SI_SDR") == ["STOI", "SI_SDR"]
