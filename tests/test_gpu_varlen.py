"""Clips of different lengths in one fullsubnet call (fsn_enhance with lengths): every clip of a mixed batch is
bit-identical to the same clip enhanced alone, whatever its length, its neighbours or the samples past its end; the file
loop's mixed-length batches write the same files as equal-length batches; and the Inferencer's int16 output takes the
fused call at every n_fft."""
import numpy as np
import pytest
import torch

from conftest import WB_GAIN, rel_l2, rel_max

pytestmark = pytest.mark.gpu

CRM_TOL = 1e-3
WAV_TOL = 1e-4
HOP = 256

# the shortest clip (n_fft/2 + 1), a multiple of hop, hop*k - 1, odd and even frame counts, a spread of 0.5 - 4 s, L_max
LENGTHS = [257, HOP * 40, HOP * 50 - 1, HOP * 30 + 5, HOP * 41 + 3, 8000, 23456, 40001, 51234, 64000]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _model(args, sd, dev, precision):
    from fullsubnet_b200.fullsubnet.model import Model
    m = Model(**args, precision=precision)
    m.load_state_dict(sd, strict=True)
    return m.to(dev).eval()


def _mixed_batch(lengths, seed):
    """[B, max(lengths)] rows of independent clips; the tail of every row is NaN or +-1e30 (never read)."""
    from oracle import fullsubnet_oracle as O
    L_max = max(lengths)
    y = O.make_noisy(len(lengths), L_max, seed=seed, speechlike=True)
    fills = (float("nan"), 1e30, -1e30)
    for b, Lb in enumerate(lengths):
        y[b, Lb:] = fills[b % 3]
    return y


def _check_against_single_calls(m, y, lengths, n_fft=512, hop=HOP, win=512):
    yd = y.to(m.fb_model.sequence_model.weight_ih_l0.device)
    B, L_max = yd.shape
    T_max = 1 + L_max // hop
    enh, crm = m.enhance(yd, n_fft, hop, win, return_crm=True, lengths=lengths)
    enh2, pcm = m.enhance_pcm(yd, n_fft, hop, win, lengths=lengths)
    assert enh.shape == (B, L_max) and crm.shape == (B, 2, n_fft // 2 + 1, T_max) and pcm.shape == (B, L_max)
    assert torch.isfinite(enh).all() and torch.isfinite(crm).all()
    assert torch.equal(enh, enh2)
    for b, Lb in enumerate(lengths):
        Tb = 1 + Lb // hop
        one, crm1 = m.enhance(yd[b:b + 1, :Lb], n_fft, hop, win, return_crm=True)
        one2, pcm1 = m.enhance_pcm(yd[b:b + 1, :Lb], n_fft, hop, win)
        assert torch.equal(enh[b, :Lb], one[0]), (b, Lb)
        assert torch.equal(crm[b, :, :, :Tb], crm1[0]), (b, Lb)
        assert torch.equal(pcm[b, :Lb], pcm1[0]) and torch.equal(one2, one), (b, Lb)
        assert not enh[b, Lb:].any() and not crm[b, :, :, Tb:].any() and not pcm[b, Lb:].any(), (b, Lb)
    return enh, crm


@pytest.mark.parametrize("norm", ["offline_laplace_norm", "cumulative_laplace_norm"])
@pytest.mark.parametrize("precision", ["fp32", "f16x3_tc", "f16_tc"])
@pytest.mark.parametrize("gain", [1.0, WB_GAIN], ids=["wa", "wb"])
def test_mixed_batch_equals_single_clip_calls(dev, norm, precision, gain):
    from oracle import fullsubnet_oracle as O
    args = dict(O.DEFAULT_MODEL_ARGS, norm_type=norm)
    m = _model(args, O.make_state_dict(seed=0, args=args, sb_fc_gain=gain), dev, precision)
    _check_against_single_calls(m, _mixed_batch(LENGTHS, seed=3), LENGTHS)


def test_gru_mixed_batch_equals_single_clip_calls(dev):
    """The small GRU model on the fp32 kernels (n_fft 64, hop 32: 33 bins)."""
    from oracle import fullsubnet_oracle as O
    args = dict(num_freqs=33, look_ahead=2, sequence_model="GRU", fb_num_neighbors=0, sb_num_neighbors=3,
                fb_output_activate_function="ReLU", sb_output_activate_function=False, fb_model_hidden_size=32,
                sb_model_hidden_size=24, norm_type="offline_laplace_norm", num_groups_in_drop_band=2, weight_init=False)
    m = _model(args, O.make_state_dict(seed=7, args=args), dev, "auto")
    assert m._resolve_precision() == "fp32"
    lengths = [33, 32 * 20, 32 * 31 - 1, 32 * 17 + 5, 1000, 2345, 4000]
    _check_against_single_calls(m, _mixed_batch(lengths, seed=9), lengths, 64, 32, 64)


@pytest.mark.parametrize("precision", ["fp32", "auto", "f16_tc"])
def test_equal_lengths_give_the_fixed_length_call(dev, precision):
    from oracle import fullsubnet_oracle as O
    m = _model(dict(O.DEFAULT_MODEL_ARGS), O.make_state_dict(seed=0), dev, precision)
    y = O.make_noisy(3, 6000, seed=5, speechlike=True).to(dev)
    enh, crm = m.enhance(y, return_crm=True, lengths=[6000] * 3)
    ref, ref_crm = m.enhance(y, return_crm=True)
    assert torch.equal(enh, ref) and torch.equal(crm, ref_crm)
    enh2, pcm = m.enhance_pcm(y, lengths=torch.tensor([6000] * 3))
    ref2, ref_pcm = m.enhance_pcm(y)
    assert torch.equal(enh2, ref2) and torch.equal(pcm, ref_pcm)


@pytest.mark.parametrize("precision,crm_tol", [("fp32", 5e-5), ("f16x3_tc", 5e-5)])
def test_mixed_batch_matches_reference(dev, precision, crm_tol):
    """Two clips of a mixed batch against the reference flow on each clip alone: the north-star gates (cRM <= 1e-3
    relative, held to 5e-5 here; waveform <= 1e-4 absolute)."""
    from oracle import fullsubnet_oracle as O
    m = _model(dict(O.DEFAULT_MODEL_ARGS), O.make_state_dict(seed=0), dev, precision)
    lengths = [20000, 9001, 14336]
    y = _mixed_batch(lengths, seed=13)
    enh, crm = m.enhance(y.to(dev), return_crm=True, lengths=lengths)
    sd = O.make_state_dict(0)
    for b in (0, 1):
        Lb, Tb = lengths[b], 1 + lengths[b] // HOP
        ref_wav, ref_crm = O.enhance(y[b:b + 1, :Lb], sd, return_crm=True)
        got = crm[b:b + 1, :, :, :Tb].cpu()
        assert rel_max(got, ref_crm) < crm_tol and rel_l2(got, ref_crm) < crm_tol, b
        assert np.abs(enh[b:b + 1, :Lb].cpu().numpy() - ref_wav.numpy()).max() < WAV_TOL, b


def test_full_size_mixed_batch(dev):
    """256 clips of 1 - 4 s in one call: finite outputs, the shortest / longest / a middle clip equal their single-clip
    calls, and one clip placed twice among neighbours of different lengths gives the same bits both times."""
    from oracle import fullsubnet_oracle as O
    m = _model(dict(O.DEFAULT_MODEL_ARGS), O.make_state_dict(seed=0), dev, "auto")
    rng = np.random.default_rng(77)
    lengths = rng.integers(16000, 64001, size=256).tolist()
    lengths[7] = lengths[200] = 33333
    y = O.make_noisy(256, max(lengths), seed=77)
    y[200] = y[7]
    for b, Lb in enumerate(lengths):
        y[b, Lb:] = float("nan")
    yd = y.to(dev)
    out, crm = m.enhance(yd, return_crm=True, lengths=lengths)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and torch.isfinite(crm).all()
    assert torch.equal(out[7], out[200]) and torch.equal(crm[7], crm[200])
    assert lengths[6] != lengths[199] and lengths[8] != lengths[201]
    for i in (int(np.argmin(lengths)), int(np.argmax(lengths)), 131):
        Lb, Tb = lengths[i], 1 + lengths[i] // HOP
        single, crm1 = m.enhance(yd[i:i + 1, :Lb], return_crm=True)
        assert torch.equal(single[0], out[i, :Lb]) and torch.equal(crm1[0], crm[i, :, :, :Tb]), i


def test_file_loop_mixed_length_batches(dev, tmp_path, monkeypatch):
    """enhance_files(max_padding=0.5) writes the same bytes as equal-length batches (max_padding=0), within 1 LSB of the
    reference host loop, with one library call per planned batch."""
    import wave
    from fullsubnet_b200.inferencer import Inferencer, plan_batches
    from oracle import fullsubnet_oracle as O
    m = _model(dict(O.DEFAULT_MODEL_ARGS), O.make_state_dict(seed=0), dev, "auto")
    inf = Inferencer(model=m, device=dev)
    lens = [6000, 4000, 7777, 5120, 4999, 9000]
    paths = []
    for i, L in enumerate(lens):
        y = O.make_noisy(1, L, seed=50 + i, speechlike=True)[0].numpy()
        p = tmp_path / f"n{i}.wav"
        inf.write_wav(p, np.round(y / np.abs(y).max() * 20000).astype(np.int16), 16000)
        paths.append(p)
    calls = []
    orig = inf.enhance_to_pcm
    monkeypatch.setattr(inf, "enhance_to_pcm", lambda x, lengths=None: calls.append(lengths) or orig(x, lengths=lengths))
    mixed = inf.enhance_files(paths, tmp_path / "mixed", batch_size=3, max_padding=0.5)
    plan = plan_batches(lens, 3, 0.5)
    assert len(calls) == len(plan) < len(lens) and any(c is not None for c in calls)
    calls.clear()
    exact = inf.enhance_files(paths, tmp_path / "exact", batch_size=3, max_padding=0.0)
    assert len(calls) == len(lens) and all(c is None for c in calls)
    amp = np.iinfo(np.int16).max
    for p, q, r in zip(paths, mixed, exact):
        assert q.name == r.name == p.name and q.read_bytes() == r.read_bytes()
        noisy = torch.from_numpy(inf.load_wav(p, 16000))[None].to(dev)
        enhanced = inf.full_band_crm_mask(noisy, {})
        ref = np.int16(0.8 * amp * enhanced / np.max(np.abs(enhanced)))
        with wave.open(str(q)) as f:
            got = np.frombuffer(f.readframes(f.getnframes()), dtype="<i2")
        assert got.shape == ref.shape
        assert np.abs(got.astype(np.int32) - ref).max() <= 1


@pytest.mark.parametrize("which", ["fullsubnet", "fullband_baseline"])
def test_inferencer_pcm_at_n_fft_960_equals_the_two_pass_path(dev, which):
    """n_fft 960 (direct DFT): Inferencer.enhance_to_pcm takes the model's fused enhance_pcm, and its int16 output is
    enhance_batch followed by the two-pass fsn_peak_normalize_int16, bit for bit."""
    from fullsubnet_b200 import _lib
    from fullsubnet_b200.inferencer import Inferencer
    from oracle import fullsubnet_oracle as O
    if which == "fullsubnet":
        args = dict(O.DEFAULT_MODEL_ARGS, num_freqs=481)
        m = _model(args, O.make_state_dict(seed=0, args=args), dev, "auto")
    else:
        from fullsubnet_b200.fullband_baseline.model import Model
        from oracle import fullband_baseline_oracle as BO
        args = dict(BO.DEFAULT_FBB_ARGS, num_freqs=481)
        m = Model(**args)
        m.load_state_dict(BO.make_fbb_state_dict(seed=11, args=args), strict=True)
        m = m.to(dev).eval()
    cfg = {"acoustics": {"n_fft": 960, "hop_length": 480, "win_length": 960, "sr": 48000}}
    inf = Inferencer(config=cfg, model=m, device=dev)
    B, L = 3, 48000 + 123
    y = O.make_noisy(B, L, seed=21, speechlike=True, sr=48000)
    pcm = inf.enhance_to_pcm(y)
    enhanced = inf.enhance_batch(y)
    ref = torch.empty_like(pcm)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().fsn_peak_normalize_int16(enhanced.data_ptr(), B, L, 0.8 * float(np.iinfo(np.int16).max),
                                                      ref.data_ptr(), _lib.stream_ptr(dev)))
    assert pcm.dtype == torch.int16 and pcm.shape == (B, L)
    assert torch.equal(pcm, ref)
