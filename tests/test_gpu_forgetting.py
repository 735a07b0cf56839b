"""forgetting_norm (audio_zen/model/base_model.py:102-151) on the GPU: the forward scan and the second norm's adjoint alone
against float64 (oracle/forgetting_oracle.py), fullsubnet and fullband_baseline against the unmodified reference
(tests/golden/forgetting.npz, model_forget_{wa,wb}.npz) under the existing gates, and the per-clip-length bit-exactness
of fsn_enhance / fsn_fullband_enhance."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import WB_GAIN, rel_l2, rel_max

pytestmark = pytest.mark.gpu

CRM_TOL, WAV_TOL = 1e-3, 1e-4
GRAD_TOL = {"fp32": 2e-4, "tf32_tc": 1e-2}
LOSS_TOL = {"fp32": 1e-5, "tf32_tc": 1e-3}
GUARD = 12345.5
EDGE_T = (1, 2, 191, 192, 193, 4000)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _lib():
    from fullsubnet_b200 import _lib
    return _lib, _lib.load()


def _guarded(n, dev):
    buf = torch.full((n + 64,), GUARD, dtype=torch.float32, device=dev)
    return buf, buf[:n]


def _scale_hook(x, x2, N, N2, cnt, lengths=None, hop=0, la=0):
    """x, x2 [B, T, F] device float32 -> (scale [T, B], mu [T, B], guard buffers)"""
    _l, lib = _lib()
    B, T, F = x.shape
    dev = x.device
    sbuf, scale = _guarded(T * B, dev)
    mbuf, mu = _guarded(T * B, dev)
    fs = torch.empty(B * T * 2, device=dev)
    fs2 = torch.empty(B * T * 2, device=dev) if x2 is not None else None
    lens_dev = torch.zeros(B, dtype=torch.int32, device=dev)
    lens = (C.c_int32 * B)(*lengths) if lengths is not None else None
    _l.check(lib.fsn_debug_forgetting_scale(x.data_ptr(), N, x2.data_ptr() if x2 is not None else None, N2, B, T, F, T * F,
                                            F, cnt, lens, lens_dev.data_ptr(), hop, la, fs.data_ptr(),
                                            fs2.data_ptr() if fs2 is not None else None, scale.data_ptr(), mu.data_ptr(),
                                            _l.stream_ptr(dev)))
    torch.cuda.synchronize()
    return scale.view(T, B).cpu(), mu.view(T, B).cpu(), sbuf, mbuf


def _ref_mu(x, x2, N, N2, cnt):
    """float64 mu [T, B] of the frame sums (closed-form reflect counts at site 2) on the library's coefficients"""
    from oracle import forgetting_oracle as FO
    from oracle import fullsubnet_oracle as O
    x = x.double()
    if x2 is None:
        s = x.sum(-1)
    else:
        F = x.shape[-1]
        s = (x * torch.from_numpy(O.reflect_count(F, N)).double()).sum(-1) + \
            (x2.double() * torch.from_numpy(O.reflect_count(F, N2)).double()).sum(-1)
    return FO.running_mean(s / cnt).T  # [T, B]


@pytest.mark.parametrize("site", [1, 2])
@pytest.mark.parametrize("T", EDGE_T)
def test_scale_hook_against_float64(dev, site, T):
    from oracle import forgetting_oracle as FO
    B, F, N, N2 = 3, 33, 3, 0
    g = torch.Generator().manual_seed(T * 10 + site)
    x = torch.rand(B, T, F, generator=g) * 2.0
    x2 = torch.rand(B, T, F, generator=g) * 0.5 if site == 2 else None
    cnt = float(F) if site == 1 else float(F * (2 * N + 1 + 2 * N2 + 1))
    xd, x2d = x.to(dev), (x2.to(dev) if x2 is not None else None)
    scale, mu, sbuf, mbuf = _scale_hook(xd, x2d, N, N2, cnt)
    assert (sbuf[T * B:] == GUARD).all() and (mbuf[T * B:] == GUARD).all()
    ref_mu = _ref_mu(x, x2, N, N2, cnt)
    err_mu = float(((mu.double() - ref_mu).abs() / ref_mu.abs()).max())
    err_s = float(((scale.double() - FO.scale(ref_mu)).abs() / FO.scale(ref_mu).abs()).max())
    # three roundings per step carried with gain a ~ alpha: at most 3 * 2^-24 / (1 - alpha) ~ 1.7e-5 relative
    print(f"[forgetting scale] site {site} T={T}: mu rel {err_mu:.2e}, scale rel {err_s:.2e} (bound 2e-5)")
    assert err_mu < 2e-5 and err_s < 2e-5
    # bit-identical repeated runs; a clip alone gives the bits it gets in the batch
    s2, m2, _, _ = _scale_hook(xd, x2d, N, N2, cnt)
    assert torch.equal(s2, scale) and torch.equal(m2, mu)
    s1, m1, _, _ = _scale_hook(xd[1:2].contiguous(), x2d[1:2].contiguous() if x2d is not None else None, N, N2, cnt)
    assert torch.equal(s1[:, 0], scale[:, 1]) and torch.equal(m1[:, 0], mu[:, 1])


@pytest.mark.parametrize("T", [193, 4000])
def test_scale_hook_lengths(dev, T):
    """With lengths, clip b is scanned over its own 1 + lengths[b]/hop + la frames only: those get the bits of the
    unbounded scan and of the clip alone, later entries stay untouched."""
    B, F, hop, la = 3, 17, 32, 2
    g = torch.Generator().manual_seed(T)
    lengths = [(T - 1 - la) * hop, (T // 2) * hop + 5, 7]
    x = (torch.rand(B, T, F, generator=g) * 2.0).to(dev)
    full, _, _, _ = _scale_hook(x, None, 0, 0, float(F))
    part, _, _, _ = _scale_hook(x, None, 0, 0, float(F), lengths, hop, la)
    for b, Lb in enumerate(lengths):
        Tb = 1 + Lb // hop + la
        assert torch.equal(part[:Tb, b], full[:Tb, b]), b
        assert (part[Tb:, b] == GUARD).all(), b
        alone, _, _, _ = _scale_hook(x[b:b + 1, :Tb].contiguous(), None, 0, 0, float(F))
        assert torch.equal(alone[:, 0], full[:Tb, b]), b


def _bwd_reference(raw, z, dX, B, F, G, Ns, act):
    """float64 autograd of <dX, X> through drop_band(forgetting_norm(cat(unfold(raw), unfold(fb)))), fb = act(z), Nf = 0.
    raw, z [Tp,B,F]; dX [Tp,R,K].  Returns (dz, X, scale [Tp,B] float64, mid)."""
    from oracle import forgetting_oracle as FO
    from oracle import fullsubnet_oracle as O
    z = z.double().clone().requires_grad_(True)
    fb = torch.relu(z) if act == 1 else z
    mag4 = raw.double().permute(1, 2, 0).unsqueeze(1)        # [B,1,F,Tp]
    fb4 = fb.permute(1, 2, 0).unsqueeze(1)
    u = torch.cat([O.freq_unfold(mag4, Ns).reshape(B, F, 2 * Ns + 1, -1),
                   O.freq_unfold(fb4, 0).reshape(B, F, 1, -1)], dim=2)   # [B,F,K,Tp]
    xn, mu = FO.forgetting_norm(u)
    if G > 1:
        src_b, src_f = O.drop_band_index_map(B, F, G)
        xn = torch.stack([xn[src_b[i]][src_f[i]] for i in range(B)])   # [B,Fsub,K,Tp]
    K = 2 * Ns + 2
    X = xn.permute(3, 0, 1, 2).reshape(raw.shape[0], -1, K)              # [Tp,R,K]
    (X * dX.double()).sum().backward()
    return z.grad, X.detach(), FO.scale(mu.detach()).T.contiguous(), fb.detach()


@pytest.mark.parametrize("G", [1, 2, 3])
@pytest.mark.parametrize("Tp", EDGE_T[:5] + (600,))
def test_adjoint_hook_against_float64_autograd(dev, G, Tp):
    _l, lib = _lib()
    B, F, Ns, act = 5, 13, 2, 1
    g = torch.Generator().manual_seed(Tp * 7 + G)
    raw = torch.rand(Tp, B, F, generator=g) + 0.05
    z = torch.randn(Tp, B, F, generator=g)
    Fsub = F // G if G > 1 else F
    R, K = B * Fsub, 2 * Ns + 2
    dX = torch.randn(Tp, R, K, generator=g)
    ref_dz, X, scale, fb = _bwd_reference(raw, z, dX, B, F, G, Ns, act)
    mbuf, mid = _guarded(Tp * B, dev)
    zbuf, dz = _guarded(Tp * B * F, dev)
    args = [dX.to(dev).contiguous(), X.float().to(dev).contiguous(), fb.float().to(dev).contiguous(),
            scale.float().to(dev).contiguous()]
    _l.check(lib.fsn_debug_forgetting_bwd(*[a.data_ptr() for a in args], B, F, G, Tp, Ns, act, mid.data_ptr(),
                                          dz.data_ptr(), _l.stream_ptr(dev)))
    torch.cuda.synchronize()
    assert (mbuf[Tp * B:] == GUARD).all() and (zbuf[Tp * B * F:] == GUARD).all()
    got = dz.view(Tp, B, F).cpu().double()
    # conditioning: the same adjoint with every term taken in magnitude (|dX|, and the recurrence on |<dX, X>|)
    from oracle import forgetting_oracle as FO
    a, bc = FO.coefficients(Tp)
    from oracle import fullsubnet_oracle as O
    if G > 1:
        src_b, _ = O.drop_band_index_map(B, F, G)
    else:
        src_b = np.arange(B)
    dot = np.zeros((Tp, B))
    ad = (dX.double().abs() * X.abs()).view(Tp, B, Fsub * K).sum(-1).numpy()
    for bq in range(B):
        dot[:, src_b[bq]] = ad[:, bq]
    s = scale.numpy()
    gacc = np.zeros(B)
    mid_abs = np.zeros((Tp, B))
    for t in range(Tp - 1, -1, -1):
        an = abs(float(a[t + 1])) if t + 1 < Tp else 0.0
        gacc = s[t] * dot[t] + an * gacc
        mid_abs[t] = abs(float(bc[t])) * gacc / (F * K)
    # direct term |dX[., K-1]| s_t plus the recurrence taken in magnitude
    cond = float(dX[:, :, K - 1].abs().max()) * float(s.max()) + float(mid_abs.max())
    err = float(np.abs(got.numpy() - ref_dz.numpy()).max())
    print(f"[forgetting bwd] G={G} Tp={Tp}: dz max err {err:.2e}, conditioning {cond:.2e}, ratio {err / cond:.2e} "
          f"(bound 3e-5)")
    assert err <= 3e-5 * cond
    # two runs give the same bits
    dz2 = torch.empty_like(dz)
    mid2 = torch.empty_like(mid)
    _l.check(lib.fsn_debug_forgetting_bwd(*[a.data_ptr() for a in args], B, F, G, Tp, Ns, act, mid2.data_ptr(),
                                          dz2.data_ptr(), _l.stream_ptr(dev)))
    torch.cuda.synchronize()
    assert torch.equal(dz2, dz) and torch.equal(mid2, mid)


# ------------------------------------------------------------------ whole models against the unmodified reference
def _fsn(args, sd, dev, precision):
    from fullsubnet_b200.fullsubnet.model import Model
    m = Model(**args, precision=precision)
    m.load_state_dict(sd, strict=True)
    return m.to(dev).eval()


@pytest.mark.parametrize("prec", ["fp32", "f16x3_tc", "f16_tc"])
@pytest.mark.parametrize("tag", ["wa", "wb"])
def test_fullsubnet_matches_reference(golden, dev, tag, prec):
    """1 clip, T = 202 (T' = 204: both sides of the t = 192 switch), weight sets W-a and W-b, every inference precision;
    a batch of 6 copies gives every copy the single-clip bits."""
    from oracle import fullsubnet_oracle as O
    from oracle.make_golden_forgetting import FULL_LEN
    from oracle.make_golden_long import fingerprint
    g = golden(f"model_forget_{tag}")
    y = O.make_noisy(1, FULL_LEN, seed=73, speechlike=True)
    assert np.allclose(fingerprint(y), g["y_fp"], rtol=1e-6)
    args = dict(O.DEFAULT_MODEL_ARGS, norm_type="forgetting_norm")
    m = _fsn(args, O.make_state_dict(seed=0, args=args, sb_fc_gain=1.0 if tag == "wa" else WB_GAIN), dev, prec)
    assert m._resolve_precision() == prec
    wav, crm = m.enhance(y.to(dev), return_crm=True)
    crm_err, wav_err = rel_max(crm.cpu(), g["crm"]), float(np.abs(wav.cpu().numpy() - g["wav"]).max())
    print(f"[forgetting fullsubnet] {tag} {prec}: cRM rel max {crm_err:.2e}, waveform max-abs {wav_err:.2e}")
    assert crm_err < CRM_TOL
    if prec != "f16_tc" or tag == "wa":  # f16_tc on W-b: 11-bit operands amplified x100 by decompress_cIRM (as offline)
        assert wav_err < WAV_TOL
    wav6 = m.enhance(y.to(dev).repeat(6, 1))
    assert all(torch.equal(wav6[i], wav[0]) for i in range(6))


@pytest.mark.parametrize("prec", ["fp32", "f16x3_tc"])
def test_fullsubnet_enhance_lengths_bit_exact(dev, prec):
    """fsn_enhance with mixed lengths gives each clip the bits of a call on that clip alone; with null lengths every clip
    gets the bits of stft -> Model.forward -> istft on that clip (the three-call path)."""
    from fullsubnet_b200 import _lib
    from oracle import fullsubnet_oracle as O
    args = dict(O.DEFAULT_MODEL_ARGS, norm_type="forgetting_norm")
    m = _fsn(args, O.make_state_dict(seed=0, args=args), dev, prec)
    lengths = [256 * 230 + 17, 256 * 100 + 3, 256 * 193 - 1]
    y = O.make_noisy(3, max(lengths), seed=81, speechlike=True)
    for b, Lb in enumerate(lengths):
        y[b, Lb:] = float("nan")
    yd = y.to(dev)
    enh, crm = m.enhance(yd, return_crm=True, lengths=lengths)
    for b, Lb in enumerate(lengths):
        one, crm1 = m.enhance(yd[b:b + 1, :Lb], return_crm=True)
        assert torch.equal(enh[b, :Lb], one[0]) and torch.equal(crm[b, :, :, :1 + Lb // 256], crm1[0]), b
    lib = _lib.load()
    L = 256 * 200 + 5
    yy = O.make_noisy(3, L, seed=82, speechlike=True).to(dev)
    enh0, crm0 = m.enhance(yy, return_crm=True)
    F, T = 257, 1 + L // 256
    for b in range(3):
        buf = torch.empty(3, 1, F, T, device=dev)
        out = torch.empty(1, L, device=dev)
        st = _lib.stream_ptr(dev)
        _lib.check(lib.fsn_stft(yy[b:b + 1].contiguous().data_ptr(), 1, L, 512, 256, 512, buf[0].data_ptr(), None,
                                buf[1].data_ptr(), buf[2].data_ptr(), None, 0, st))
        with torch.no_grad():
            c = m(buf[0].unsqueeze(1)).contiguous()
        _lib.check(lib.fsn_istft(buf[1].data_ptr(), buf[2].data_ptr(), 1, c.data_ptr(), 1, T, 512, 256, 512, L,
                                 out.data_ptr(), st))
        torch.cuda.synchronize()
        assert torch.equal(c[0], crm0[b]) and torch.equal(out[0], enh0[b]), b


def _fbb(dev):
    from fullsubnet_b200.fullband_baseline.model import Model
    from oracle import fullband_baseline_oracle as BO
    args = dict(BO.DEFAULT_FBB_ARGS, num_freqs=33, hidden_size=32, output_activate_function="ReLU",
                norm_type="forgetting_norm")
    m = Model(**args)
    m.load_state_dict(BO.make_fbb_state_dict(seed=11, args=args), strict=True)
    return m.to(dev).eval()


def test_fullband_baseline_matches_reference(golden, dev):
    """fullband_baseline wav -> wav with three clip lengths (T = 204, 160, 195) in one call against the reference run one
    clip at a time; each clip also gets the bits of its own call, and null lengths give the three-call path."""
    from fullsubnet_b200 import _lib
    g = golden("forgetting")
    m = _fbb(dev)
    lengths = g["fbb_lengths"].tolist()
    y = torch.from_numpy(g["fbb_y"]).to(dev)
    enh, crm = m.enhance(y, 64, 32, 64, return_crm=True, lengths=lengths)
    crm_err, wav_err = rel_max(crm.cpu(), g["fbb_crm"]), float(np.abs(enh.cpu().numpy() - g["fbb_wav"]).max())
    print(f"[forgetting fullband_baseline] cRM rel max {crm_err:.2e}, waveform max-abs {wav_err:.2e}")
    assert crm_err < 2e-5 and wav_err < WAV_TOL
    for b, Lb in enumerate(lengths):
        one, crm1 = m.enhance(y[b:b + 1, :Lb].contiguous(), 64, 32, 64, return_crm=True)
        assert torch.equal(enh[b, :Lb], one[0]) and torch.equal(crm[b, :, :, :1 + Lb // 32], crm1[0]), b
    lib = _lib.load()
    L = min(lengths)
    yy = y[:, :L].contiguous()
    enh0, crm0 = m.enhance(yy, 64, 32, 64, return_crm=True)
    F, T = 33, 1 + L // 32
    buf = torch.empty(3, 3, F, T, device=dev)
    out = torch.empty(3, L, device=dev)
    st = _lib.stream_ptr(dev)
    _lib.check(lib.fsn_stft(yy.data_ptr(), 3, L, 64, 32, 64, buf[0].data_ptr(), None, buf[1].data_ptr(), buf[2].data_ptr(),
                            None, 0, st))
    with torch.no_grad():
        c = m(buf[0].unsqueeze(1)).contiguous()
    _lib.check(lib.fsn_istft(buf[1].data_ptr(), buf[2].data_ptr(), 1, c.data_ptr(), 3, T, 64, 32, 64, L, out.data_ptr(),
                             st))
    torch.cuda.synchronize()
    assert torch.equal(c, crm0) and torch.equal(out, enh0)


# ------------------------------------------------------------------ training steps against the unmodified reference
@pytest.mark.parametrize("prec", ["fp32", "tf32_tc"])
def test_training_matches_reference(golden, dev, prec):
    """Two steps of the small fullsubnet at the recipe crop (5 clips, T = 193, T' = 195; drop_band G = 2)."""
    from fullsubnet_b200.acoustics.feature import drop_band, stft
    from fullsubnet_b200.acoustics.mask import build_complex_ideal_ratio_mask
    from fullsubnet_b200.fullsubnet.model import Model
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.optim import FusedClipAdam
    from oracle import fullsubnet_oracle as O
    from oracle.make_golden_train import SMALL
    g = golden("forgetting")
    args = dict(SMALL, norm_type="forgetting_norm")
    m = Model(**args)
    m.load_state_dict(O.make_state_dict(seed=7, args=args, sb_fc_gain=8.0), strict=True)
    m.train_precision = prec
    m = m.to(dev).train()
    opt = FusedClipAdam(m.parameters(), lr=1e-3, betas=(0.9, 0.999), max_norm=10.0)
    noisy, clean = torch.from_numpy(g["train_noisy"]).to(dev), torch.from_numpy(g["train_clean"]).to(dev)
    for it in range(2):
        opt.zero_grad()
        nm, _, nr, ni = stft(noisy, 64, 32, 64)
        _, _, cr, ci = stft(clean, 64, 32, 64)
        cirm = build_complex_ideal_ratio_mask(nr, ni, cr, ci)
        cirm = drop_band(cirm.permute(0, 3, 1, 2), m.num_groups_in_drop_band).permute(0, 2, 3, 1)
        crm = m(nm.unsqueeze(1)).permute(0, 2, 3, 1)
        loss = mse_loss()(cirm, crm)
        loss.backward()
        want = float(g["train_loss"][it])
        print(f"[forgetting train] {prec} step {it}: loss {float(loss.detach()):.7f} (reference {want:.7f})")
        assert abs(float(loss.detach()) - want) <= LOSS_TOL[prec] * abs(want)
        if it == 0:
            assert rel_max(crm.detach().cpu(), g["train_crm"]) < (1e-5 if prec == "fp32" else 1e-3)
            worst = 0.0
            for k, p in m.named_parameters():
                e = rel_l2(p.grad.cpu(), g["train_grad." + k])
                worst = max(worst, e)
                assert e < GRAD_TOL[prec], k
            print(f"[forgetting train] {prec}: worst gradient rel-L2 {worst:.2e}")
        opt.step()
        if prec == "fp32":
            assert abs(float(opt.last_norm[0]) - g["train_gnorm"][it]) < 1e-4 * g["train_gnorm"][it]
    if prec == "fp32":
        for k, v in m.state_dict().items():
            assert np.abs(v.cpu().numpy() - g["train_p1." + k]).max() < 2e-5, k
