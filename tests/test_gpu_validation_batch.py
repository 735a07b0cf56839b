"""Validation in groups: fsn_cirm_mse_per_clip and fsn_si_sdr_lengths on a mixed-length batch equal the B = 1 calls on
each clip bit for bit (and a float64 evaluation of the same formulas within fp32 tolerance), and Trainer._validation_epoch
gives every item the loss of the reference's op-by-op B = 1 evaluation, bit for bit, whatever the grouping."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N_FFT, HOP, WIN = 512, 256, 512
# not multiples of the hop, the shortest clip the STFT takes (n_fft/2 + 1), repeated lengths (equal-length groups of
# fast_fullsubnet), and one clip at L_max
LENGTHS = [12345, 16000, 8005, 16000, 257, 12345, 9999, 16000, 4097]
# |SI-SDR(fused waveform) - SI-SDR(op-by-op waveform)| in dB: the fused iSTFT applies the mask inside the transform,
# the op-by-op path rounds each product in its own pass, so the waveforms differ in the last bits (DESIGN 4.11).
# Measured at most 1.9e-6 dB on these items (fullband_baseline; H100 SXM, 700 W); the bound keeps 50x of margin and
# stays 10x inside the 1e-3 dB that test_trainer_with_validation_loader allows.
SCORE_TOL = 1e-4


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _clips(lengths, seed):
    """noisy, clean [B, L_max] rows; the tail of every row past its clip is NaN (never read)."""
    from oracle import fullsubnet_oracle as O
    L = max(lengths)
    clean = O.make_noisy(len(lengths), L, seed=seed, speechlike=True) * 0.5
    g = torch.Generator().manual_seed(seed + 1)
    noisy = clean + 0.05 * torch.randn(len(lengths), L, generator=g)
    for b, Lb in enumerate(lengths):
        noisy[b, Lb:] = float("nan")
        clean[b, Lb:] = float("nan")
    return noisy, clean


def _fullsubnet(dev, norm, precision):
    from fullsubnet_b200.fullsubnet.model import Model
    from oracle import fullsubnet_oracle as O
    args = dict(O.DEFAULT_MODEL_ARGS, norm_type=norm)
    m = Model(**args, precision=precision)
    m.load_state_dict(O.make_state_dict(seed=0, args=args), strict=True)
    return m.to(dev)


def _fbb(dev):
    from fullsubnet_b200.fullband_baseline.model import Model
    from oracle import fullband_baseline_oracle as BO
    m = Model(**BO.DEFAULT_FBB_ARGS)
    m.load_state_dict(BO.make_fbb_state_dict(seed=5, args=dict(BO.DEFAULT_FBB_ARGS)), strict=True)
    return m.to(dev)


def _fast(dev):
    from fullsubnet_b200.fast_fullsubnet.model import Model
    from oracle import fast_fullsubnet_oracle as FO
    m = Model(**FO.DEFAULT_FAST_ARGS)
    m.load_state_dict(FO.make_fast_state_dict(seed=3, args=dict(FO.DEFAULT_FAST_ARGS)), strict=True)
    return m.to(dev)


MODELS = {"fsn_offline_f16x3": lambda d: _fullsubnet(d, "offline_laplace_norm", "f16x3_tc"),
          "fsn_offline_fp32": lambda d: _fullsubnet(d, "offline_laplace_norm", "fp32"),
          "fsn_cum_f16x3": lambda d: _fullsubnet(d, "cumulative_laplace_norm", "f16x3_tc"),
          "fsn_cum_fp32": lambda d: _fullsubnet(d, "cumulative_laplace_norm", "fp32"),
          "fullband_baseline": _fbb, "fast_fullsubnet": _fast}


def _op_by_op(model, noisy, clean):
    """The B = 1 validation body of fullsubnet/trainer.py:146-165 through the drop-in functions: (loss, SI-SDR)."""
    from fullsubnet_b200.acoustics.feature import istft, stft
    from fullsubnet_b200.acoustics.mask import build_complex_ideal_ratio_mask, decompress_cIRM
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.trainer import si_sdr
    noisy_mag, _, nr, ni = stft(noisy, N_FFT, HOP, WIN)
    _, _, cr, ci = stft(clean, N_FFT, HOP, WIN)
    cirm = build_complex_ideal_ratio_mask(nr, ni, cr, ci)
    crm = model(noisy_mag.unsqueeze(1)).permute(0, 2, 3, 1)
    loss = mse_loss()(cirm, crm)
    crm = decompress_cIRM(crm)
    er = crm[..., 0] * nr - crm[..., 1] * ni
    ei = crm[..., 1] * nr + crm[..., 0] * ni
    enhanced = istft((er, ei), N_FFT, HOP, WIN, length=noisy.size(-1), input_type="real_imag")
    return loss, si_sdr(clean, enhanced)[0]


def _trainer(model, items, tmp_path, batch_size=32, max_padding=0.25):
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.trainer import Trainer
    cfg = {"meta": {"use_amp": False, "save_dir": str(tmp_path), "experiment_name": "v"},
           "acoustics": {"n_fft": N_FFT, "hop_length": HOP, "win_length": WIN},
           "trainer": {"train": {"epochs": 1, "save_checkpoint_interval": 1, "clip_grad_norm_value": 10},
                       "validation": {"validation_interval": 1, "save_max_metric_score": True,
                                      "batch_size": batch_size, "max_padding": max_padding}}}
    return Trainer(None, 0, cfg, False, False, model, mse_loss(), torch.optim.SGD(model.parameters(), lr=0.0), [],
                   items)


def _items(lengths, seed):
    noisy, clean = _clips(lengths, seed)
    return [(noisy[i:i + 1, :Lb], clean[i:i + 1, :Lb], [f"clip{i}"], ["With_reverb" if i % 3 else "No_reverb"])
            for i, Lb in enumerate(lengths)]


def _f64_stft(y, lens):
    from oracle import fullsubnet_oracle as O
    return [O.stft(y[b:b + 1, :Lb].double(), N_FFT, HOP, WIN) for b, Lb in enumerate(lens)]


def test_per_clip_kernels_equal_single_clip_calls_and_float64(dev):
    from fullsubnet_b200.acoustics.feature import stft
    from fullsubnet_b200.acoustics.mask import build_complex_ideal_ratio_mask
    from fullsubnet_b200.loss import cirm_mse_per_clip, mse_loss
    from fullsubnet_b200.trainer import si_sdr
    noisy, clean = _clips(LENGTHS, seed=11)
    B, L = noisy.shape
    F, T = N_FFT // 2 + 1, 1 + L // HOP
    g = torch.Generator().manual_seed(2)
    crm = (2.0 * torch.rand(B, 2, F, T, generator=g) - 1.0) * 5.0
    est = torch.where(torch.isnan(clean), clean, 0.8 * clean + 0.1 * torch.randn(B, L, generator=g))
    nd, cd, crm_d, est_d = noisy.to(dev), clean.to(dev), crm.to(dev), est.to(dev)
    loss = cirm_mse_per_clip(nd, cd, crm_d, N_FFT, HOP, WIN, LENGTHS).cpu()
    score = si_sdr(cd, est_d, LENGTHS).cpu()
    for b, Lb in enumerate(LENGTHS):
        Tb = 1 + Lb // HOP
        _, _, nr, ni = stft(nd[b:b + 1, :Lb], N_FFT, HOP, WIN)
        _, _, cr, ci = stft(cd[b:b + 1, :Lb], N_FFT, HOP, WIN)
        cirm = build_complex_ideal_ratio_mask(nr, ni, cr, ci)
        one = mse_loss()(cirm, crm_d[b:b + 1, :, :, :Tb].permute(0, 2, 3, 1))
        assert torch.equal(loss[b], one.cpu()), (b, Lb, float(loss[b]), float(one))
        assert torch.equal(score[b], si_sdr(cd[b:b + 1, :Lb], est_d[b:b + 1, :Lb])[0].cpu()), (b, Lb)
    # the same formulas in float64
    from oracle import fullsubnet_oracle as O
    n64, c64 = _f64_stft(noisy, LENGTHS), _f64_stft(clean, LENGTHS)
    for b, Lb in enumerate(LENGTHS):
        Tb = 1 + Lb // HOP
        a, bb, c, d = n64[b][2][0], n64[b][3][0], c64[b][2][0], c64[b][3][0]
        den = a * a + bb * bb + float(np.finfo(np.float32).eps)
        cirm = torch.stack([O.compress_cIRM((a * c + bb * d) / den), O.compress_cIRM((a * d - bb * c) / den)])
        want = float(((crm[b, :, :, :Tb].double() - cirm) ** 2).mean())
        assert abs(float(loss[b]) - want) <= 1e-4 * want, (b, float(loss[b]), want)
        r, e = clean[b, :Lb].double(), est[b, :Lb].double()
        p = (r @ e) / (r @ r) * r
        want = 10.0 * np.log10(float((p @ p) / ((e - p) @ (e - p))))
        assert abs(float(score[b]) - want) < 2e-3, (b, float(score[b]), want)


def test_lengthless_calls_are_the_fixed_length_calls(dev):
    from fullsubnet_b200.loss import cirm_mse_per_clip
    from fullsubnet_b200.trainer import si_sdr
    noisy, clean = (t.to(dev) for t in _clips([6000] * 3, seed=4))
    crm = torch.rand(3, 2, N_FFT // 2 + 1, 1 + 6000 // HOP, device=dev)
    assert torch.equal(cirm_mse_per_clip(noisy, clean, crm, N_FFT, HOP, WIN),
                       cirm_mse_per_clip(noisy, clean, crm, N_FFT, HOP, WIN, [6000] * 3))
    assert torch.equal(si_sdr(clean, noisy), si_sdr(clean, noisy, [6000] * 3))


@pytest.mark.parametrize("which", list(MODELS))
def test_validation_items_equal_op_by_op(dev, which, tmp_path):
    """Every item's loss is the op-by-op B = 1 loss bit for bit; its SI-SDR is within SCORE_TOL of the op-by-op one."""
    m = MODELS[which](dev)
    items = _items(LENGTHS, seed=7)
    tr = _trainer(m, items, tmp_path)
    loss, score, types = tr._validation_items()
    assert types == [it[3][0] for it in items]
    m.eval()
    diffs = []
    with torch.no_grad():
        for i, (noisy, clean, _, _) in enumerate(items):
            want_loss, want_score = _op_by_op(m, noisy.to(dev), clean.to(dev))
            assert loss[i] == want_loss.cpu().numpy(), (which, i, loss[i], float(want_loss))
            diffs.append(abs(float(score[i]) - float(want_score)))
    print(f"{which}: max |SI-SDR difference| {max(diffs):.3e} dB")
    assert max(diffs) <= SCORE_TOL, (which, diffs)


@pytest.mark.parametrize("which", ["fsn_offline_f16x3", "fast_fullsubnet"])
def test_results_do_not_depend_on_grouping(dev, which, tmp_path):
    m = MODELS[which](dev).train()
    items = _items(LENGTHS, seed=8)
    ref = None
    for batch_size in (1, 3, len(items)):
        for max_padding in (0.0, 0.25):
            tr = _trainer(m, items, tmp_path, batch_size, max_padding)
            m.train()
            score = tr._validation_epoch(1)
            assert m.training  # restored
            got = (tr._validation_items(), tr.last_validation, score)
            if ref is None:
                ref = got
                continue
            assert all(np.array_equal(a, b) for a, b in zip(got[0][:2], ref[0][:2])), (batch_size, max_padding)
            assert got[1] == ref[1] and got[2] == ref[2], (batch_size, max_padding)


def test_validation_epoch_sums_in_dataloader_order(dev, tmp_path):
    """last_validation is the reference's float32 sums of the per-item values, in dataloader order."""
    m = MODELS["fsn_offline_f16x3"](dev)
    items = _items(LENGTHS, seed=9)
    tr = _trainer(m, items, tmp_path)
    loss, score, types = tr._validation_items()
    s = tr._validation_epoch(1)
    v = tr.last_validation
    tot, per_loss, per_score = np.float32(0), {}, {}
    for i, t in enumerate(types):
        tot += loss[i]
        per_loss[t] = per_loss.get(t, np.float32(0)) + loss[i]
        per_score[t] = per_score.get(t, np.float32(0)) + score[i]
    n = len(types)
    assert v["loss_total"] == float(tot) / n
    assert v["loss"] == {k: float(per_loss[k]) / n for k in ("With_reverb", "No_reverb")}
    assert v["items"] == {k: types.count(k) for k in ("With_reverb", "No_reverb")}
    assert s == v["si_sdr"]["With_reverb"] == float(per_score["With_reverb"]) / types.count("With_reverb")
