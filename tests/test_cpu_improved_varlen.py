"""CPU-only checks of improved_fullsubnet's clips-of-different-lengths entry point (fsn_improved_enhance): its workspace
query and argument checks answer before any CUDA call, the Python ``lengths`` argument, and the Inferencer's rules for a
model that computes its own STFT."""
import ctypes as C

import pytest
import torch


def _model(args=None):
    from fullsubnet_b200.improved_fullsubnet.model import Model
    from oracle import improved_fullsubnet_oracle as IO
    return Model(**(args or IO.DEFAULT_IMPROVED_ARGS))


def _call(lib, d, lengths, L_max, enhanced=None):
    arr = (C.c_int32 * len(lengths))(*lengths)
    return lib.fsn_improved_enhance(C.byref(d), None, None, arr, len(lengths), L_max, enhanced, None, None, 1.0, None, 0,
                                    None)


def test_improved_enhance_workspace_query_needs_no_gpu():
    from fullsubnet_b200 import _lib
    from oracle import improved_fullsubnet_oracle as IO
    lib = _lib.load()
    for prec in ("fp32", "tf32_tc"):
        d = _model()._desc(prec)
        n = lib.fsn_improved_enhance_workspace_bytes(C.byref(d), 4, 64000)
        # the forward's workspace plus the per-clip peak and length table
        assert n > lib.fsn_improved_workspace_bytes(C.byref(d), 4, 64000) > 0
        assert lib.fsn_improved_enhance_workspace_bytes(C.byref(d), 8, 64000) > n
    d960 = _model(IO.ARGS_48K_960)._desc("tf32_tc")
    assert lib.fsn_improved_enhance_workspace_bytes(C.byref(d960), 4, 48000) > 0
    bad = _model(dict(IO.DEFAULT_IMPROVED_ARGS, n_fft=1536, win_length=1536, num_freqs=769))._desc("fp32")
    assert lib.fsn_improved_enhance_workspace_bytes(C.byref(bad), 4, 48000) == 0
    assert lib.fsn_last_error_code() == _lib.FSN_ERR_UNSUPPORTED


def test_improved_enhance_checks_arguments_before_any_cuda_call():
    """No workspace, no weights, no device: every one of these fails on its argument check."""
    from fullsubnet_b200 import _lib
    from oracle import improved_fullsubnet_oracle as IO
    lib = _lib.load()
    d = _model()._desc("tf32_tc")
    assert _call(lib, d, [16000, 256, 3000], 16000) == _lib.FSN_ERR_SHAPE  # too short: <= n_fft/2
    assert b"clip 1" in lib.fsn_last_error()
    assert _call(lib, d, [16000, 16001, 3000], 16000) == _lib.FSN_ERR_SHAPE  # longer than the row
    assert b"clip 1" in lib.fsn_last_error()
    assert _call(lib, d, [15000, 257, 3000], 16000) == _lib.FSN_ERR_SHAPE  # max(lengths) != L_max
    assert b"15000" in lib.fsn_last_error()
    # valid lengths reach the workspace check, the last one before the first launch; n_fft 960 included (a stand-in
    # output pointer, never written: the call returns before any CUDA call)
    assert _call(lib, d, [16000, 257, 3000], 16000, enhanced=16) == _lib.FSN_ERR_WORKSPACE
    d960 = _model(IO.ARGS_48K_960)._desc("fp32")
    assert _call(lib, d960, [48000, 480], 48000) == _lib.FSN_ERR_SHAPE
    assert b"clip 1" in lib.fsn_last_error()
    assert _call(lib, d960, [48000, 481], 48000, enhanced=16) == _lib.FSN_ERR_WORKSPACE
    # null lengths: every clip L_max samples
    assert lib.fsn_improved_enhance(C.byref(d960), None, None, None, 2, 48000, 16, None, None, 1.0, None, 0,
                                    None) == _lib.FSN_ERR_WORKSPACE


def test_improved_python_lengths_argument_is_checked():
    m = _model()
    y = torch.zeros(3, 4000)
    for fn in (m.enhance, m.enhance_pcm):
        with pytest.raises(ValueError, match="entries"):
            fn(y, lengths=[4000, 3000])
        with pytest.raises(ValueError, match="exceeds"):
            fn(y, lengths=[4000, 4001, 300])
        with pytest.raises(ValueError):
            fn(y, lengths=torch.tensor([4000.0, 3000.0, 300.0]))
        with pytest.raises(RuntimeError, match="CUDA tensor"):  # valid lengths reach the device check
            fn(y, lengths=torch.tensor([4000, 3000, 300]))


def test_inferencer_rules_for_waveform_models():
    from fullsubnet_b200.fast_fullsubnet.model import Model as Fast
    from fullsubnet_b200.inferencer import Inferencer
    from oracle import fast_fullsubnet_oracle as FO
    from oracle import improved_fullsubnet_oracle as IO
    for args in (IO.DEFAULT_IMPROVED_ARGS, IO.ARGS_48K_1024, IO.ARGS_48K_960):
        inf = Inferencer.__new__(Inferencer)
        inf.model, inf.n_fft = _model(args), args["n_fft"]
        assert inf.supports_lengths(), args["n_fft"]
    fast = Inferencer.__new__(Inferencer)
    fast.model, fast.n_fft = Fast(**FO.DEFAULT_FAST_ARGS), 512
    assert not fast.supports_lengths()
    # the model's own STFT sets n_fft / hop / window; a config that disagrees is refused
    m = _model(IO.ARGS_48K_960)
    inf = Inferencer(model=m, device="cpu")
    assert (inf.n_fft, inf.hop_length, inf.win_length) == (960, 480, 960)
    cfg = {"acoustics": {"n_fft": 960, "hop_length": 480, "win_length": 960, "sr": 48000}}
    inf = Inferencer(config=cfg, model=m, device="cpu")
    assert (inf.n_fft, inf.hop_length, inf.sr) == (960, 480, 48000)
    for bad in ({"n_fft": 512, "hop_length": 256, "win_length": 512, "sr": 16000}, {"hop_length": 240}):
        with pytest.raises(ValueError, match="hop_length"):
            Inferencer(config={"acoustics": bad}, model=m, device="cpu")
