"""GPU parity: libfsn_b200 (through the reference-API host) vs. the golden fixtures produced by
the unmodified reference and vs. the oracle on the same seeded inputs.

Tolerances (BASELINE.json north_star): cRM <= 1e-3 relative to max|ref| (and rel-L2 <= 1e-3);
enhanced waveform <= 1e-4 absolute.  The fp32 path is held to much tighter bounds."""
import numpy as np
import pytest
import torch

from conftest import rel_max, rel_l2, WB_GAIN

pytestmark = pytest.mark.gpu

CRM_TOL = 1e-3
WAV_TOL = 1e-4


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def T(x, dev):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def small_args():
    return dict(num_freqs=33, look_ahead=2, sequence_model="LSTM", fb_num_neighbors=0, sb_num_neighbors=3,
                fb_output_activate_function="ReLU", sb_output_activate_function=False,
                fb_model_hidden_size=32, sb_model_hidden_size=24, norm_type="offline_laplace_norm",
                num_groups_in_drop_band=2, weight_init=False)


def make_model(args, sd, dev, precision):
    from fullsubnet_b200.fullsubnet.model import Model
    m = Model(**args, precision=precision)
    m.load_state_dict(sd, strict=True)
    return m.to(dev).eval()


# ------------------------------------------------------------------ A1 / A9: STFT, iSTFT
def test_stft_matches_reference(golden, dev):
    from fullsubnet_b200.acoustics.feature import stft
    g = golden("dsp")
    mag, phase, real, imag = stft(T(g["y"], dev), 512, 256, 512)
    assert mag.shape == g["mag"].shape
    assert rel_max(real.cpu(), g["real"]) < 5e-6 and rel_max(imag.cpu(), g["imag"]) < 5e-6
    assert rel_max(mag.cpu(), g["mag"]) < 5e-6
    sel = g["mag"] > 1e-2 * g["mag"].max()
    # phase compared directly, not modulo 2 pi: a negative Re with Im exactly 0 (DC, Nyquist) is +pi in both.  Only bins
    # whose non-zero Im is too small for its float32 sign to be certain sit on the branch cut and are left out.
    cut = (g["real"] < 0) & (g["imag"] != 0) & (np.abs(g["imag"]) < 1e-5 * g["mag"].max())
    d = phase.cpu().numpy() - g["phase"]
    assert np.abs(d[sel & ~cut]).max() < 1e-4
    mag3 = stft(T(g["y3"], dev), 512, 256, 512)[0]  # [B,C,T] input (feature.py:30-31,43-44)
    assert mag3.shape == g["mag3"].shape and rel_max(mag3.cpu(), g["mag3"]) < 5e-6
    _, _, rs, is_ = stft(T(g["y"], dev), 64, 32, 64)
    assert rel_max(rs.cpu(), g["real_s"]) < 5e-6 and rel_max(is_.cpu(), g["imag_s"]) < 5e-6


def test_istft_matches_reference(golden, dev):
    from fullsubnet_b200.acoustics.feature import istft
    g = golden("dsp")
    L = g["y"].shape[-1]
    w = istft((T(g["real"], dev), T(g["imag"], dev)), 512, 256, 512, length=L, input_type="real_imag")
    assert rel_max(w.cpu(), g["wav_rt"]) < 1e-5
    w2 = istft(torch.complex(T(g["real"], dev), T(g["imag"], dev)), 512, 256, 512)
    assert w2.shape == g["wav_nolen"].shape and rel_max(w2.cpu(), g["wav_nolen"]) < 1e-5
    mag = np.hypot(g["real"], g["imag"]).astype(np.float32)
    w3 = istft((T(mag, dev), T(g["phase"], dev)), 512, 256, 512, length=L, input_type="mag_phase")
    assert rel_max(w3.cpu(), g["wav_rt"]) < 1e-5
    w4 = istft((T(g["real_s"], dev), T(g["imag_s"], dev)), 64, 32, 64, length=L, input_type="real_imag")
    assert rel_max(w4.cpu(), g["wav_s"]) < 1e-5


@pytest.mark.parametrize("L", [257, 511, 4096, 64000])
def test_stft_istft_roundtrip_and_oracle(dev, L):
    from fullsubnet_b200.acoustics.feature import stft, istft
    from oracle import fullsubnet_oracle as O
    y = O.make_noisy(2, L, seed=L)
    mag, _, re, im = stft(y.to(dev), 512, 256, 512)
    om, _, ore, oim = O.stft(y, 512, 256, 512)
    assert mag.shape == om.shape
    scale = float(om.max())  # Im can be identically ~0 (L=257: the reflect-padded frame is symmetric)
    assert np.abs(re.cpu().numpy() - ore.numpy()).max() < 5e-6 * scale
    assert np.abs(im.cpu().numpy() - oim.numpy()).max() < 5e-6 * scale
    assert rel_max(mag.cpu(), om) < 5e-6
    back = istft((re, im), 512, 256, 512, length=L, input_type="real_imag").cpu().numpy()
    # size-independent property: identity.  Only on the samples covered by full window overlap, hop*(T-1):
    # past that the window-square envelope tends to 0 and y*w^2/w^2 is ill-conditioned (in torch.istft too).
    n_ok = 256 * (mag.shape[-1] - 1)
    assert np.abs(back[:, :n_ok] - y.numpy()[:, :n_ok]).max() < 5e-6
    oback = O.istft((ore, oim), 512, 256, 512, length=L, input_type="real_imag").numpy()
    assert np.abs(back - oback)[:, :n_ok].max() < 5e-6 and back.shape == oback.shape


# ------------------------------------------------------------------ masks, drop_band
def test_masks_and_drop_band_match_reference(golden, dev):
    from fullsubnet_b200.acoustics import mask, feature
    g = golden("dsp")
    assert rel_max(mask.decompress_cIRM(T(g["m"], dev)).cpu(), g["dec"]) < 2e-6
    assert rel_max(mask.compress_cIRM(T(g["big"], dev)).cpu(), g["comp"]) < 2e-6
    _, _, cr, ci = feature.stft(T(g["yc"], dev), 512, 256, 512)
    cirm = mask.build_complex_ideal_ratio_mask(T(g["real"], dev), T(g["imag"], dev), cr, ci)
    assert cirm.shape == g["cirm"].shape
    assert np.abs(cirm.cpu().numpy() - g["cirm"]).max() < 5e-3  # ill-conditioned where |noisy| ~ 0
    assert np.median(np.abs(cirm.cpu().numpy() - g["cirm"])) < 1e-5
    assert np.array_equal(feature.drop_band(T(g["xb"], dev), 2).cpu().numpy(), g["db2"])  # bit-exact index op
    assert np.array_equal(feature.drop_band(T(g["xb"], dev), 3).cpu().numpy(), g["db3"])
    nan = torch.tensor([float("nan"), 20.0, -20.0, 0.0], device=dev)
    ref = np.array([0.0, 52.93305, -52.93305, 0.0], dtype=np.float32)
    assert np.allclose(mask.decompress_cIRM(nan).cpu().numpy(), ref, rtol=1e-5)


# ------------------------------------------------------------------ Model.forward
@pytest.mark.parametrize("precision", ["fp32"])
def test_small_model_matches_reference(golden, dev, precision):
    g = golden("model_small")
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd.")}
    m = make_model(small_args(), sd, dev, precision)
    mag = T(g["mag"], dev).unsqueeze(1)
    with torch.no_grad():
        assert rel_max(m(mag[:1]).cpu(), g["crm_b1"]) < 2e-5
        out = m(mag)  # B=3 -> drop_band G=2, batch order [0,2,1], 16 of 33 bins
        assert out.shape == g["crm_g2"].shape
        assert rel_max(out.cpu(), g["crm_g2"]) < 2e-5
        m.num_groups_in_drop_band = 1
        assert rel_max(m(mag).cpu(), g["crm_g1"]) < 2e-5
        m.num_groups_in_drop_band = 3
        with pytest.raises(AssertionError):
            m(mag)  # B == G (feature.py:317-319)


def _full_model(dev, gain, precision):
    from oracle import fullsubnet_oracle as O
    return make_model(dict(O.DEFAULT_MODEL_ARGS), O.make_state_dict(seed=0, sb_fc_gain=gain), dev, precision)


@pytest.mark.parametrize("precision,crm_tol", [("fp32", 5e-5), ("f16x3_tc", 5e-5), ("auto", 5e-5)])
@pytest.mark.parametrize("tag,gain", [("wa", 1.0), ("wb", WB_GAIN)])
def test_full_model_and_inferencer_match_reference(golden, dev, tag, gain, precision, crm_tol):
    """Both north-star gates (cRM <= 1e-3 rel -- held to 5e-5 here -- and waveform <= 1e-4 abs) on BOTH weight
    sets, W-b being the set whose cRM reaches the +-9.9 clip where decompress_cIRM has gain ~100
    (mask.py:58-63).  `auto` (the default precision) resolves to the error-compensated tensor-core path."""
    from fullsubnet_b200.acoustics.feature import stft
    from fullsubnet_b200.inferencer import Inferencer
    g = golden("model_full")
    m = _full_model(dev, gain, precision)
    if precision == "auto":
        assert m._resolve_precision() == "f16x3_tc"
    y = T(g["y"], dev)
    ref_crm, ref_wav = g[f"{tag}_crm"], g[f"{tag}_wav"]
    with torch.no_grad():
        mag = stft(y, 512, 256, 512)[0]
        crm = torch.cat([m(mag[i:i + 1].unsqueeze(1)) for i in range(2)], 0)
    assert rel_max(crm.cpu(), ref_crm) < crm_tol and rel_l2(crm.cpu(), ref_crm) < crm_tol
    inf = Inferencer(model=m, device=dev)
    wav = np.stack([inf.full_band_crm_mask(y[i:i + 1], {}) for i in range(2)])  # op-by-op reference flow
    fused, crm2 = m.enhance(y, return_crm=True)  # one fsn_enhance call, batched
    assert rel_max(crm2.cpu(), ref_crm) < crm_tol
    assert np.abs(wav - ref_wav).max() < WAV_TOL
    assert np.abs(fused.cpu().numpy() - ref_wav).max() < WAV_TOL


def test_single_pass_f16_is_opt_in_and_meets_the_mask_gate(golden, dev):
    """precision="f16_tc" (one fp16 MMA pass, 3x the speed) is never chosen by `auto`.  It meets the cRM gate on both
    weight sets and the waveform gate on W-a; on W-b its 11-bit operand rounding is amplified x100 by
    decompress_cIRM near the clip, which is exactly why the default is the compensated path."""
    g = golden("model_full")
    y = T(g["y"], dev)
    for tag, gain in (("wa", 1.0), ("wb", WB_GAIN)):
        m = _full_model(dev, gain, "f16_tc")
        fused, crm = m.enhance(y, return_crm=True)
        assert rel_max(crm.cpu(), g[f"{tag}_crm"]) < CRM_TOL and rel_l2(crm.cpu(), g[f"{tag}_crm"]) < CRM_TOL
        if tag == "wa":
            assert np.abs(fused.cpu().numpy() - g["wa_wav"]).max() < WAV_TOL


@pytest.mark.parametrize("precision,tol", [("fp32", 2e-5), ("f16x3_tc", 2e-5), ("f16_tc", WAV_TOL)])
def test_batched_equals_loop_of_single_clips(dev, precision, tol):
    """SURVEY fact 4: batched inference == loop of B=1 calls (drop_band off)."""
    from oracle import fullsubnet_oracle as O
    m = _full_model(dev, 1.0, precision)
    y = O.make_noisy(3, 4000, seed=11, speechlike=True).to(dev)
    batched = m.enhance(y)
    single = torch.cat([m.enhance(y[i:i + 1]) for i in range(3)], 0)
    assert np.abs(batched.cpu().numpy() - single.cpu().numpy()).max() < 2e-6  # tiling-independent
    ref = O.enhance(y.cpu(), O.make_state_dict(0))
    assert np.abs(batched.cpu().numpy() - ref.numpy()).max() < tol


def test_tc_drop_band_training_layout_and_unsupported_shapes(golden, dev):
    """f16_tc with B>1, G=2 reproduces the drop_band batch permutation; unsupported hidden sizes raise."""
    from oracle import fullsubnet_oracle as O
    m = _full_model(dev, 1.0, "f16_tc")
    y = O.make_noisy(3, 3000, seed=21, speechlike=True)
    mag = O.stft(y, 512, 256, 512)[0].unsqueeze(1)
    ref = O.model_forward(mag, O.make_state_dict(0))  # G=2 -> [3,2,128,T], batch order [0,2,1]
    with torch.no_grad():
        out = m(mag.to(dev))
    assert out.shape == ref.shape
    assert rel_max(out.cpu(), ref) < CRM_TOL and rel_l2(out.cpu(), ref) < CRM_TOL
    g = golden("model_small")
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd.")}
    small = make_model(small_args(), sd, dev, "f16_tc")  # hidden 24: not a multiple of 128
    with pytest.raises(NotImplementedError), torch.no_grad():
        small(T(g["mag"], dev).unsqueeze(1)[:1])
    auto = make_model(small_args(), sd, dev, "auto")  # auto falls back to the fp32 kernels
    with torch.no_grad():
        assert rel_max(auto(T(g["mag"], dev).unsqueeze(1)[:1]).cpu(), g["crm_b1"]) < 2e-5
    # with grad enabled the same call runs the activation-saving training kernels (fp32 here) and is differentiable
    auto.train_precision = "fp32"
    tr = auto(T(g["mag"], dev).unsqueeze(1)[:1])
    assert tr.requires_grad and rel_max(tr.detach().cpu(), g["crm_b1"]) < 2e-5


def test_full_size_batch_properties(dev):
    """BASELINE configs[1] size (256 x 4 s) through size-independent properties: finite output, tiling
    independence (a clip's result does not depend on where it sits in the batch / which CTA tile its
    sub-band units land in), duplicate clips give bit-identical outputs, first/middle/last clip match the
    oracle within the north-star tolerances."""
    from oracle import fullsubnet_oracle as O
    m = _full_model(dev, 1.0, "auto")
    B, L = 256, 64000
    y = O.make_noisy(B, L, seed=77)
    y[200] = y[7]  # duplicate clip at another batch position (different tile alignment: 7*257 vs 200*257 mod 32)
    yd = y.to(dev)
    out, crm = m.enhance(yd, return_crm=True)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and torch.isfinite(crm).all()
    assert torch.equal(out[7], out[200]) and torch.equal(crm[7], crm[200])
    for i in (0, 131, 255):
        single, crm1 = m.enhance(yd[i:i + 1], return_crm=True)
        assert torch.equal(single[0], out[i]) and torch.equal(crm1[0], crm[i])
    sd = O.make_state_dict(0)
    ref_wav, ref_crm = O.enhance(y[255:256], sd, return_crm=True)
    assert rel_max(crm[255:256].cpu(), ref_crm) < CRM_TOL and rel_l2(crm[255:256].cpu(), ref_crm) < CRM_TOL
    assert np.abs(out[255:256].cpu().numpy() - ref_wav.numpy()).max() < WAV_TOL


# ------------------------------------------------------------------ fast_fullsubnet (config 4, A13)
@pytest.mark.parametrize("precision,tol", [("fp32", 5e-5), ("f16x3_tc", 5e-5), ("f16_tc", CRM_TOL)])
def test_fast_fullsubnet_matches_reference(golden, dev, precision, tol):
    from fullsubnet_b200.fast_fullsubnet.model import Model
    from oracle import fast_fullsubnet_oracle as FO
    g = golden("fast_full")
    m = Model(**FO.DEFAULT_FAST_ARGS, precision=precision)
    m.load_state_dict(FO.make_fast_state_dict(seed=3), strict=True)
    m = m.to(dev).eval()
    mag = T(g["mag"], dev).unsqueeze(1)
    with torch.no_grad():
        o1 = m(mag[:1])
        o3 = m(mag)
    assert o3.shape == g["out_b3"].shape
    e1, e3 = rel_max(o1.cpu(), g["out_b1"]), rel_max(o3.cpu(), g["out_b3"])
    print(f"fast_fullsubnet {precision}: max-rel {e1:.2e} / {e3:.2e}, rel-l2 {rel_l2(o3.cpu(), g['out_b3']):.2e}")
    assert e1 < tol and e3 < tol
    assert rel_l2(o3.cpu(), g["out_b3"]) < tol
    # odd / even frame counts exercise the last (short) down-sampling block
    for Tn in (7, 8):
        x = torch.rand(2, 1, 257, Tn)
        ref = FO.fast_model_forward(x, FO.make_fast_state_dict(seed=3))
        with torch.no_grad():
            got = m(x.to(dev))
        assert rel_max(got.cpu(), ref) < tol, Tn
    # the inference kernels are built for LSTM only: a GRU model is refused before any kernel reads its [3H, K] weights
    gru = Model(**dict(FO.DEFAULT_FAST_ARGS, sequence_model="GRU"), precision=precision).to(dev).eval()
    with pytest.raises(NotImplementedError), torch.no_grad():
        gru(mag[:1])


# ------------------------------------------------------------------ improved_fullsubnet (config 5, A14)
@pytest.mark.parametrize("prec", ["fp32", "tf32_tc"])
@pytest.mark.parametrize("tag", ["k16", "k48"])
def test_improved_fullsubnet_matches_reference(golden, dev, tag, prec):
    from fullsubnet_b200.improved_fullsubnet.model import Model
    from oracle import improved_fullsubnet_oracle as IO
    g = golden("improved")
    args = IO.DEFAULT_IMPROVED_ARGS if tag == "k16" else IO.ARGS_48K_1024
    m = Model(**args)
    m.load_state_dict(IO.make_improved_state_dict(seed=5, args=args), strict=True)
    m.precision = prec
    m = m.to(dev).eval()
    y = T(g[tag + "_y"], dev)
    with torch.no_grad():
        wav = m(y)
        wav3 = m(y.unsqueeze(1)[:1])
    assert wav.shape == g[tag + "_wav"].shape
    err = np.abs(wav.cpu().numpy() - g[tag + "_wav"]).max()
    print(f"improved_fullsubnet {tag} {prec}: waveform max-abs {err:.2e} (scale {np.abs(g[tag + '_wav']).max():.2e})")
    if prec == "fp32":
        assert err < 1e-6
    assert err < WAV_TOL
    assert np.abs(wav3.cpu().numpy() - g[tag + "_wav"][:1]).max() < WAV_TOL
    # bad section geometry: ValueError like the reference (model.py:341-345)
    bad = Model(**dict(args, freq_cutoffs=[21] + list(args["freq_cutoffs"][1:]))).to(dev).eval()
    with pytest.raises(ValueError), torch.no_grad():
        bad(y)


@pytest.mark.parametrize("prec", ["fp32", "tf32_tc"])
def test_improved_fullsubnet_tanh_head_matches_oracle(golden, dev, prec):
    """sb_output_activate_function="Tanh": the section heads apply it (improved_fullsubnet/model.py:69-74)."""
    from fullsubnet_b200.improved_fullsubnet.model import Model
    from oracle import improved_fullsubnet_oracle as IO
    args = dict(IO.DEFAULT_IMPROVED_ARGS, sb_output_activate_function="Tanh")
    sd = IO.make_improved_state_dict(seed=5, args=args)
    for k in sd:  # heads 4x the init scale: the Tanh bends their outputs, a head without it misses by >> WAV_TOL
        if k.startswith("sb_model.") and "fc_output_layer" in k:
            sd[k] = sd[k] * 4.0
    m = Model(**args)
    m.load_state_dict(sd, strict=True)
    m.precision = prec
    m = m.to(dev).eval()
    y = torch.from_numpy(np.asarray(golden("improved")["k16_y"]))
    ref = IO.improved_forward(y, sd, args).numpy()
    with torch.no_grad():
        wav = m(y.to(dev))
    err = np.abs(wav.cpu().numpy() - ref).max()
    print(f"improved_fullsubnet Tanh head {prec}: waveform max-abs {err:.2e} (scale {np.abs(ref).max():.2e})")
    if prec == "fp32":
        assert err < 1e-6
    assert err < WAV_TOL


# ------------------------------------------------------------------ cumulative_laplace_norm (SURVEY 8f rank 1)
def test_cumulative_laplace_norm_matches_reference(golden, dev):
    from fullsubnet_b200.fullsubnet.model import Model
    from oracle import fullsubnet_oracle as O
    g = golden("model_cum")
    args = dict(small_args(), norm_type="cumulative_laplace_norm")
    m = make_model(args, O.make_state_dict(seed=7, args=args), dev, "auto")
    assert m._resolve_precision() == "fp32"  # hidden 24: the tensor-core kernels do not cover it
    mag = T(g["small_mag"], dev).unsqueeze(1)
    with torch.no_grad():
        assert rel_max(m(mag[:1]).cpu(), g["small_b1"]) < 2e-5
        assert rel_max(m(mag).cpu(), g["small_g2"]) < 2e-5  # B=3: drop_band + per-unit running means
    full = dict(O.DEFAULT_MODEL_ARGS, norm_type="cumulative_laplace_norm")
    for prec, tol in (("fp32", 5e-5), ("auto", 5e-5), ("f16_tc", CRM_TOL)):
        # auto = the compensated tensor-core path: per-step unit scales inside the tensor-core gather warp
        mf = make_model(full, O.make_state_dict(seed=0, args=full, sb_fc_gain=60.0), dev, prec)
        if prec == "auto":
            assert mf._resolve_precision() == "f16x3_tc"
        wav, crm = mf.enhance(T(g["full_y"], dev), return_crm=True)
        assert rel_max(crm.cpu(), g["full_crm"]) < tol, prec
        if prec != "f16_tc":
            assert np.abs(wav.cpu().numpy() - g["full_wav"]).max() < WAV_TOL, prec
        # a batch large enough for the tensor-core full-band path (time-major per-(step, clip) scales): every copy of
        # the clip gives the single-clip result
        y = T(g["full_y"], dev)
        wav_b = mf.enhance(y.repeat(10, 1))  # 20 clips: c0, c1, c0, c1, ...
        assert np.abs(wav_b.cpu().numpy() - np.tile(g["full_wav"], (10, 1))).max() < (
            WAV_TOL if prec != "f16_tc" else 1e-2), prec


# ------------------------------------------------------------------ n_fft = 960 (the direct-DFT policy of fsn_dsp.cu)
def test_non_power_of_two_stft_istft(golden, dev):
    from fullsubnet_b200.acoustics.feature import stft, istft
    g = golden("improved_960")
    mag, _, re, im = stft(T(g["y"], dev), 960, 480, 960)
    assert mag.shape == g["mag"].shape
    scale = float(np.abs(g["mag"]).max())
    assert np.abs(re.cpu().numpy() - g["real"]).max() < 2e-5 * scale
    assert np.abs(im.cpu().numpy() - g["imag"]).max() < 2e-5 * scale
    assert rel_max(mag.cpu(), g["mag"]) < 2e-5
    back = istft((re * 0.5 - im * 0.25, im * 0.5 + re * 0.25), 960, 480, 960, length=12000, input_type="real_imag")
    n_ok = 480 * (mag.shape[-1] - 1)
    assert np.abs(back.cpu().numpy() - g["back"])[:, :n_ok].max() < 2e-5 * max(1.0, float(np.abs(g["back"]).max()))


def test_improved_fullsubnet_960_matches_reference(golden, dev):
    from fullsubnet_b200.improved_fullsubnet.model import Model
    from oracle import improved_fullsubnet_oracle as IO
    g = golden("improved_960")
    m = Model(**IO.ARGS_48K_960)
    m.load_state_dict(IO.make_improved_state_dict(seed=5, args=IO.ARGS_48K_960), strict=True)
    m = m.to(dev).eval()
    with torch.no_grad():
        wav = m(T(g["y"], dev))
    err = np.abs(wav.cpu().numpy() - g["wav"]).max()
    print(f"improved_fullsubnet n_fft=960: waveform max-abs {err:.2e} (scale {np.abs(g['wav']).max():.2e})")
    assert err < WAV_TOL


# ------------------------------------------------------------------ fullband_baseline (SURVEY 8f rank 3)
def test_fullband_baseline_matches_reference(golden, dev):
    from fullsubnet_b200.fullband_baseline.model import Model
    from oracle import fullband_baseline_oracle as BO
    g = golden("fullband_baseline")
    small = dict(BO.DEFAULT_FBB_ARGS, num_freqs=33, hidden_size=32, output_activate_function="ReLU",
                 norm_type="cumulative_laplace_norm")
    for tag, a in (("small", small), ("full", dict(BO.DEFAULT_FBB_ARGS))):
        m = Model(**a)
        m.load_state_dict(BO.make_fbb_state_dict(seed=11, args=a), strict=True)
        m = m.to(dev).eval()
        with torch.no_grad():
            out = m(T(g[tag + "_mag"], dev))
            one = m(T(g[tag + "_mag"], dev)[1:2])
        assert out.shape == g[tag + "_out"].shape
        assert rel_max(out.cpu(), g[tag + "_out"]) < 2e-5, tag
        assert rel_max(one.cpu(), g[tag + "_out"][1:2]) < 2e-5, tag
    gru = Model(**dict(small, sequence_model="GRU")).to(dev).eval()  # LSTM inference kernels only
    with pytest.raises(NotImplementedError), torch.no_grad():
        gru(T(g["small_mag"], dev))


# ------------------------------------------------------------------ host loop: int16 scaling (SURVEY 8f rank 2)
def test_peak_normalize_int16_matches_numpy(dev, tmp_path):
    from fullsubnet_b200.inferencer import Inferencer
    from oracle import fullsubnet_oracle as O
    m = _full_model(dev, 1.0, "auto")
    inf = Inferencer(model=m, device=dev)
    y = O.make_noisy(3, 6000, seed=5, speechlike=True)
    pcm = inf.enhance_to_pcm(y).cpu().numpy()
    enhanced = inf.enhance_batch(y).cpu().numpy()
    amp = np.iinfo(np.int16).max
    for i in range(3):  # base_inferencer.py:181-182 per clip
        ref = np.int16(0.8 * amp * enhanced[i] / np.max(np.abs(enhanced[i])))
        assert np.array_equal(pcm[i], ref), int(np.abs(pcm[i].astype(np.int32) - ref).max())
    assert np.abs(pcm).max(axis=1).tolist() == [26213] * 3
    inf.write_wav(tmp_path / "a.wav", pcm[0], 16000)
    import wave
    with wave.open(str(tmp_path / "a.wav")) as f:
        assert f.getframerate() == 16000 and f.getnframes() == 6000 and f.getsampwidth() == 2


# ------------------------------------------------------------------ GRU cell (SURVEY 8f rank 3)
def test_gru_model_matches_reference(golden, dev):
    """sequence_model="GRU" (audio_zen/model/module/sequence_model.py:59-66): fp32 kernels, 3-gate weights, both the
    Model.forward contract (B=1, B=3 with drop_band) and the fused wav -> wav call; training is reported as not built."""
    from oracle import fullsubnet_oracle as O
    g = golden("model_gru")
    args = dict(small_args(), sequence_model="GRU")
    m = make_model(args, O.make_state_dict(seed=7, args=args), dev, "auto")
    assert m._resolve_precision() == "fp32"
    assert m.fb_model.sequence_model.weight_ih_l0.shape == (3 * 32, 33)
    mag = T(g["small_mag"], dev).unsqueeze(1)
    with torch.no_grad():
        assert rel_max(m(mag[:1]).cpu(), g["small_b1"]) < 2e-5
        assert rel_max(m(mag).cpu(), g["small_g2"]) < 2e-5
    full = dict(O.DEFAULT_MODEL_ARGS, sequence_model="GRU")
    mf = make_model(full, O.make_state_dict(seed=0, args=full, sb_fc_gain=60.0), dev, "auto")
    wav, crm = mf.enhance(T(g["full_y"], dev), return_crm=True)
    assert rel_max(crm.cpu(), g["full_crm"]) < 5e-5
    assert np.abs(wav.cpu().numpy() - g["full_wav"]).max() < WAV_TOL
    with pytest.raises(NotImplementedError), torch.no_grad():
        make_model(full, O.make_state_dict(seed=0, args=full), dev, "f16_tc")(torch.rand(1, 1, 257, 4, device=dev))
    with pytest.raises(NotImplementedError):
        m.train()(mag)  # BPTT is built for the LSTM recipe


def test_batched_file_loop_matches_reference_host_loop(dev, tmp_path):
    """Inferencer.enhance_files: wav files of two different lengths -> grouped batches -> fsn_enhance with pcm (int16
    scaling fused behind the iSTFT) -> wav files; every file equals the reference's per-file flow
    (base_inferencer.py:172-187: full_band_crm_mask on that clip alone, int16(0.8 * 32767 * y / max|y|))."""
    import wave
    from fullsubnet_b200.inferencer import Inferencer
    from oracle import fullsubnet_oracle as O
    m = _full_model(dev, 1.0, "auto")
    inf = Inferencer(model=m, device=dev)
    lens = [6000, 4000, 6000, 6000, 4000]
    paths = []
    for i, L in enumerate(lens):
        y = O.make_noisy(1, L, seed=50 + i, speechlike=True)[0].numpy()
        p = tmp_path / f"n{i}.wav"
        inf.write_wav(p, np.round(y / np.abs(y).max() * 20000).astype(np.int16), 16000)
        paths.append(p)
    out = inf.enhance_files(paths, tmp_path / "enh", batch_size=2)
    amp = np.iinfo(np.int16).max
    for p, q in zip(paths, out):
        noisy = torch.from_numpy(inf.load_wav(p, 16000))[None].to(dev)
        enhanced = inf.full_band_crm_mask(noisy, {})
        ref = np.int16(0.8 * amp * enhanced / np.max(np.abs(enhanced)))
        with wave.open(str(q)) as f:
            got = np.frombuffer(f.readframes(f.getnframes()), dtype="<i2")
            assert f.getframerate() == 16000
        assert q.name == p.name and got.shape == ref.shape
        assert np.abs(got.astype(np.int32) - ref).max() <= 1, int(np.abs(got.astype(np.int32) - ref).max())
    # fused peak == separate peak-normalise kernel, bit for bit
    y = O.make_noisy(3, 6000, seed=5, speechlike=True).to(dev)
    enh, pcm = m.enhance_pcm(y)
    from fullsubnet_b200 import _lib
    pcm2 = torch.empty_like(pcm)
    _lib.check(_lib.load().fsn_peak_normalize_int16(enh.data_ptr(), 3, 6000, 0.8 * 32767.0, pcm2.data_ptr(),
                                                    torch.cuda.current_stream().cuda_stream))
    assert torch.equal(pcm, pcm2) and torch.equal(enh, m.enhance(y))
