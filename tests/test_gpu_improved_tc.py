"""improved_fullsubnet on the fp16 tensor cores (precision "f16x3_tc" / "f16_tc"): each sub-band section runs its input
projection on the tf32 GEMM, both LSTM layers of all steps in one persistent wgmma launch (sb_proj_lstm_tc_kernel) and
its head once over all steps.  Checked against the reference fixtures and the CPU oracle, the section recurrence alone
against a float64 LSTM, the bit identities the file loop relies on (batch invariance, mixed lengths with the int16
output), and the fp32 / tf32_tc paths against outputs stored from the build before these precisions existed."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import rel_l2, rel_max

pytestmark = pytest.mark.gpu

WAV_TOL = 1e-4   # waveform max-abs against the reference fixtures (as tests/test_gpu_parity.py)
CRM_TOL = 1e-3   # cRM relative max / relative L2 against the CPU oracle
# f16_tc (single fp16 pass) meets the same gates: measured on an H100 80GB HBM3 over the fixtures below, worst waveform
# 1.1e-5 max-abs and worst cRM 7.2e-4 rel max / 5.2e-4 rel L2 (f16x3_tc: 1.2e-7, 7.5e-6, 5.1e-6)
TC = ["f16x3_tc", "f16_tc"]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _args(tag):
    from oracle import improved_fullsubnet_oracle as IO
    return {"k16": IO.DEFAULT_IMPROVED_ARGS, "k48": IO.ARGS_48K_1024, "k48_960": IO.ARGS_48K_960}[tag]


def _model(tag, precision, dev):
    from fullsubnet_b200.improved_fullsubnet.model import Model
    from oracle import improved_fullsubnet_oracle as IO
    m = Model(**_args(tag))
    m.load_state_dict(IO.make_improved_state_dict(seed=5, args=_args(tag)), strict=True)
    m.precision = precision
    return m.to(dev).eval()


def _fixture(golden, case):
    """(variant, input [B, L], reference waveform [B, 1, L]) of one fixture case."""
    from oracle import fullsubnet_oracle as O
    if case in ("k16", "k48"):
        g = golden("improved")
        return case, torch.from_numpy(np.asarray(g[case + "_y"])), np.asarray(g[case + "_wav"])
    if case == "960":
        g = golden("improved_960")
        return "k48_960", torch.from_numpy(np.asarray(g["y"])), np.asarray(g["wav"])
    tag = case[:-3]  # "<variant>_2s": tests/test_gpu_config_length.py's 2 s clip
    L = 32000 if tag == "k16" else 96000
    return tag, O.make_noisy(1, L, seed=44, speechlike=True), np.asarray(golden("improved_2s")[tag + "_wav"])


@pytest.mark.parametrize("precision", TC)
@pytest.mark.parametrize("case", ["k16", "k48", "960", "k16_2s", "k48_2s", "k48_960_2s"])
def test_matches_reference_fixtures_and_oracle(golden, dev, case, precision):
    from oracle import improved_fullsubnet_oracle as IO
    tag, y, ref_wav = _fixture(golden, case)
    m = _model(tag, precision, dev)
    assert m._resolve_precision() == precision
    with torch.no_grad():
        wav, crm = m(y.to(dev), return_crm=True)
    _, ref_crm = IO.improved_forward(y, IO.make_improved_state_dict(seed=5, args=_args(tag)), _args(tag), return_crm=True)
    e_wav = float(np.abs(wav.cpu().numpy() - ref_wav).max())
    e_max, e_l2 = rel_max(crm.cpu(), ref_crm), rel_l2(crm.cpu(), ref_crm)
    print(f"improved {case} {precision}: waveform max-abs {e_wav:.2e}, cRM rel max {e_max:.2e} rel L2 {e_l2:.2e}")
    assert wav.shape == ref_wav.shape and e_wav < WAV_TOL
    assert e_max < CRM_TOL and e_l2 < CRM_TOL


def _lstm64(x, w):
    """float64 2-layer LSTM over x [T, R, W] with the torch gate order (i, f, g, o) -> h1 [T, R, H]."""
    T, R, _ = x.shape
    H = w["w_hh0"].shape[1]
    h = [torch.zeros(R, H, dtype=torch.float64) for _ in range(2)]
    c = [torch.zeros(R, H, dtype=torch.float64) for _ in range(2)]
    out = []
    for t in range(T):
        inp = x[t]
        for l in range(2):
            g = inp @ w[f"w_ih{l}"].T + h[l] @ w[f"w_hh{l}"].T + w[f"b_ih{l}"] + w[f"b_hh{l}"]
            i, f, gg, o = g.split(H, dim=1)
            c[l] = torch.sigmoid(f) * c[l] + torch.sigmoid(i) * torch.tanh(gg)
            h[l] = torch.sigmoid(o) * torch.tanh(c[l])
            inp = h[l]
        out.append(h[1])
    return torch.stack(out)


def _run_section_hook(dev, W, R, T, H, x3, seed, stages=0, cluster=0):
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(seed)
    k = 1.0 / np.sqrt(H)
    shapes = {"w_ih0": (4 * H, W), "w_hh0": (4 * H, H), "b_ih0": (4 * H,), "b_hh0": (4 * H,),
              "w_ih1": (4 * H, H), "w_hh1": (4 * H, H), "b_ih1": (4 * H,), "b_hh1": (4 * H,)}
    w = {n: (torch.rand(s, generator=g, dtype=torch.float64) * 2 - 1) * k for n, s in shapes.items()}
    x = torch.rand(T, R, W, generator=g, dtype=torch.float64) * 2.0  # section inputs are non-negative magnitudes
    wd = {n: v.float().to(dev).contiguous() for n, v in w.items()}
    sw = _lib.SeqWeights()
    for l in range(2):
        sw.w_ih[l], sw.w_hh[l] = wd[f"w_ih{l}"].data_ptr(), wd[f"w_hh{l}"].data_ptr()
        sw.b_ih[l], sw.b_hh[l] = wd[f"b_ih{l}"].data_ptr(), wd[f"b_hh{l}"].data_ptr()
    d = _lib.ImprovedDesc(n_fft=512, hop_length=128, win_length=512, num_freqs=257, fdrc=0.5, num_sections=1,
                          fb_hidden=512, sb_hidden=H, precision=_lib.PREC["f16x3_tc" if x3 else "f16_tc"])
    d.sb_num_center[0], d.fb_num_center[0] = 1, 1
    packed = torch.empty(lib.fsn_improved_packed_bytes(C.byref(d), 0), dtype=torch.uint8, device=dev)
    n = _lib.check_workspace(lib.fsn_debug_imp_section_lstm_tc_workspace_bytes(R, T, W, H, int(x3)))
    ws = torch.empty(n, dtype=torch.uint8, device=dev)
    xd = x.float().to(dev).contiguous()
    h1 = torch.full((T, R, H), float("nan"), device=dev)
    _lib.check(lib.fsn_debug_imp_section_lstm_tc(C.byref(sw), W, H, int(x3), xd.data_ptr(), R, T, stages, cluster,
                                                 packed.data_ptr(), h1.data_ptr(), ws.data_ptr(), n,
                                                 _lib.stream_ptr(dev)))
    torch.cuda.synchronize()
    return h1.cpu().double(), _lstm64(x.float().double(), {n: v.float().double() for n, v in w.items()})


@pytest.mark.parametrize("x3", [True, False], ids=["f16x3_tc", "f16_tc"])
@pytest.mark.parametrize("W,R,T", [(62, 70, 9), (68, 33, 9), (76, 64, 5), (100, 45, 5), (180, 96, 4), (188, 17, 6),
                                   (62, 5, 1), (188, 1, 3)])
def test_section_recurrence_against_float64(dev, W, R, T, x3):
    """Widths of every shipped section (62 / 68 / 76 at k16, up to 180 at n_fft 960 and 188 at n_fft 1024); R a
    multiple of 32 or not, R < 32 and T = 1."""
    h1, ref = _run_section_hook(dev, W, R, T, 384, x3, seed=W * 1000 + R + T)
    err = float((h1 - ref).abs().max())
    print(f"section recurrence W={W} R={R} T={T} {'f16x3_tc' if x3 else 'f16_tc'}: h1 max-abs {err:.2e}")
    assert torch.isfinite(h1).all()
    # measured on an H100: at most 1.3e-6 (f16x3_tc) and 1.3e-4 (f16_tc)
    assert err < (2e-5 if x3 else 5e-4), err


@pytest.mark.parametrize("stages,cluster", [(2, 1), (3, 2), (4, 4)])
def test_section_recurrence_launch_configurations(dev, stages, cluster):
    """The ring depths and cluster sizes the kernel accepts give the bits of the default configuration."""
    a, ref = _run_section_hook(dev, 76, 150, 4, 384, True, seed=3, stages=stages, cluster=cluster)
    b, _ = _run_section_hook(dev, 76, 150, 4, 384, True, seed=3)
    assert torch.equal(a, b)
    assert float((a - ref).abs().max()) < 2e-5


@pytest.mark.parametrize("tag", ["k16", "k48_960"])
@pytest.mark.parametrize("precision", TC)
def test_forward_is_batch_invariant(dev, tag, precision):
    from oracle import fullsubnet_oracle as O
    m = _model(tag, precision, dev)
    y = O.make_noisy(3, 3 * m.hop_length * 40 + 11, seed=21, speechlike=True).to(dev)
    with torch.no_grad():
        out = m(y)
        for i in range(3):
            assert torch.equal(out[i:i + 1], m(y[i:i + 1])), i


@pytest.mark.parametrize("tag", ["k16", "k48_960"])
@pytest.mark.parametrize("precision", TC)
def test_mixed_lengths_equal_single_clip_calls(dev, tag, precision):
    from oracle import fullsubnet_oracle as O
    m = _model(tag, precision, dev)
    hop, n_fft = m.hop_length, m.n_fft
    sr = 16000 if tag == "k16" else 48000
    lengths = [n_fft // 2 + 1, hop * 20, hop * 25 - 1, sr // 2 + 7, sr]
    y = O.make_noisy(len(lengths), max(lengths), seed=3, speechlike=True, sr=sr)
    for b, Lb in enumerate(lengths):
        y[b, Lb:] = float("nan")  # never read
    yd = y.to(dev)
    enh, crm = m.enhance(yd, lengths=lengths, return_crm=True)
    enh2, pcm = m.enhance_pcm(yd, lengths=lengths)
    assert torch.isfinite(enh).all() and torch.equal(enh, enh2)
    for b, Lb in enumerate(lengths):
        Tb = 1 + Lb // hop
        with torch.no_grad():
            one, crm1 = m(yd[b:b + 1, :Lb], return_crm=True)
        _, pcm1 = m.enhance_pcm(yd[b:b + 1, :Lb])
        assert torch.equal(enh[b, :Lb], one[0, 0]), (b, Lb)
        assert torch.equal(crm[b, :, :, :Tb], crm1[0]), (b, Lb)
        assert torch.equal(pcm[b, :Lb], pcm1[0]), (b, Lb)
        assert not enh[b, Lb:].any() and not pcm[b, Lb:].any(), (b, Lb)


def test_packed_images_follow_the_parameters(dev):
    """A weight update rebuilds the section images: the output changes with it and returns with the old weights."""
    from oracle import fullsubnet_oracle as O
    m = _model("k16", "f16x3_tc", dev)
    y = O.make_noisy(1, 8000, seed=9, speechlike=True).to(dev)
    with torch.no_grad():
        a = m(y)
        w = m.sb_model.sb_models[1].sequence_model.weight_hh_l0
        keep = w.clone()
        w.mul_(0.5)
        b = m(y)
        w.copy_(keep)
        c = m(y)
    assert not torch.equal(a, b) and torch.equal(a, c)


@pytest.mark.parametrize("precision", ["fp32", "tf32_tc"])
def test_fp32_and_tf32_paths_are_unchanged(golden, dev, precision):
    """Bit-identical to the waveforms the build before the fp16 precisions computed (tests/golden/improved_tc_parent.npz,
    stored from that build on an H100 with this input)."""
    g = golden("improved_tc_parent")
    for tag, key in (("k16", "improved"), ("k48_960", "improved_960")):
        y = golden(key)["k16_y" if tag == "k16" else "y"]
        m = _model(tag, precision, dev)
        with torch.no_grad():
            wav = m(torch.from_numpy(np.asarray(y)).to(dev))
        assert np.array_equal(wav.cpu().numpy(), g[f"{tag}_{precision}"]), (tag, precision)
