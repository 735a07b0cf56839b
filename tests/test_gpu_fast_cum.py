"""fast_fullsubnet with norm_type="cumulative_laplace_norm" on the GPU: inference on every precision and the training step
(fp32, tf32_tc) against the unmodified reference (tests/golden/fast_cum.npz, oracle/make_golden_fast_cum.py), against
the oracle on other shapes (float64 autograd for the gradients), and the causality the norm exists for."""
import contextlib

import numpy as np
import pytest
import torch

from conftest import rel_l2, rel_max

pytestmark = pytest.mark.gpu

CUM = "cumulative_laplace_norm"
INFER_TOL = {"fp32": 5e-5, "f16x3_tc": 5e-5, "f16_tc": 1e-3}  # test_gpu_parity.py:test_fast_fullsubnet_matches_reference
SUB = 291  # oracle/make_golden_fast_cum.py:SUBSAMPLE
GRAD_TOL = {"fp32": 2e-4, "tf32_tc": 1e-2}  # test_gpu_fast_train.py
LOSS_TOL = {"fp32": 1e-5, "tf32_tc": 1e-3}
GNORM_TOL = {"fp32": 1e-4, "tf32_tc": 5e-3}
# shrink 3 (a short or a full last block), one frame of look-ahead, encoder-output neighbours
OTHER = dict(shrink_size=3, look_ahead=1, encoder_output_num_neighbors=1)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def fast_args(**kw):
    from oracle import fast_fullsubnet_oracle as FO
    return dict(FO.DEFAULT_FAST_ARGS, norm_type=CUM, **kw)


def build(dev, args, seed, precision=None, train_precision=None):
    from fullsubnet_b200.fast_fullsubnet.model import Model
    from oracle import fast_fullsubnet_oracle as FO
    m = Model(**args, precision=precision)
    m.load_state_dict(FO.make_fast_state_dict(seed=seed, args=args), strict=True)
    if train_precision:
        m.train_precision = train_precision
        return m.to(dev).train()
    return m.to(dev).eval()


# ------------------------------------------------------------------------------------------------------ inference
@pytest.mark.parametrize("precision", ["fp32", "f16x3_tc", "f16_tc"])
def test_inference_matches_reference(golden, dev, precision):
    from oracle import fast_fullsubnet_cum_oracle as CO
    from oracle import fast_fullsubnet_oracle as FO
    from oracle import make_golden_fast_cum as MG
    g = golden("fast_cum")
    tol = INFER_TOL[precision]
    m = build(dev, fast_args(), 3, precision)
    assert m._resolve_precision() == precision
    for T in MG.LENGTHS:  # T' = 18 (a short last down-sampling block) and 19 (a full one)
        mag = torch.from_numpy(g[f"mag_T{T}"]).to(dev).unsqueeze(1)
        with torch.no_grad():
            o1, o3 = m(mag[:1]), m(mag)
        e1, e3 = rel_max(o1.cpu(), g[f"out_b1_T{T}"]), rel_max(o3.cpu(), g[f"out_b3_T{T}"])
        print(f"fast_fullsubnet cumulative norm {precision} T={T}: max-rel {e1:.2e} / {e3:.2e}")
        assert e1 < tol and e3 < tol and rel_l2(o3.cpu(), g[f"out_b3_T{T}"]) < tol, T
    sd = FO.make_fast_state_dict(seed=3, args=fast_args())
    for T in (5, 6):  # T' = 7 (a full last block) and 8 (a single-frame one)
        x = torch.rand(2, 1, 257, T, generator=torch.Generator().manual_seed(T))
        with torch.no_grad():
            got = m(x.to(dev))
        assert rel_max(got.cpu(), CO.fast_model_forward(x, sd, fast_args())) < tol, T


@pytest.mark.parametrize("precision", ["fp32", "f16x3_tc", "f16_tc"])
def test_inference_other_config_matches_oracle(dev, precision):
    from oracle import fast_fullsubnet_cum_oracle as CO
    from oracle import fast_fullsubnet_oracle as FO
    args = fast_args(**OTHER)
    m = build(dev, args, 7, precision)
    sd = FO.make_fast_state_dict(seed=7, args=args)
    for B, T in ((2, 12), (3, 13), (1, 14)):  # T' = 13 (full last block), 14 (one frame), 15 (two frames)
        x = torch.rand(B, 1, 257, T, generator=torch.Generator().manual_seed(10 * B + T)) * 2
        with torch.no_grad():
            got = m(x.to(dev))
        e = rel_max(got.cpu(), CO.fast_model_forward(x, sd, args))
        print(f"{precision} B={B} T={T}: max-rel {e:.2e}")
        assert e < INFER_TOL[precision], (B, T, e)


@pytest.mark.parametrize("precision", ["fp32", "f16x3_tc", "f16_tc"])
@pytest.mark.parametrize("kw", [{}, OTHER], ids=["recipe", "shrink3"])
def test_inference_is_causal(dev, precision, kw):
    """Output frame t (padded frame t' = t + look_ahead) reads the encoder up to t' and the shrunk steps up to t' // S, whose
    block ends at frame t' - t' % S.  On a prefix of P frames, every output frame with t' < P whose step is not the prefix's
    last one gives the bits of the full run: both norms are running means, so nothing later reaches them."""
    args = fast_args(**kw)
    la, S = args["look_ahead"], args["shrink_size"]
    m = build(dev, args, 5, precision)
    x = torch.rand(3, 1, 257, 40, generator=torch.Generator().manual_seed(4), device="cpu").to(dev)
    with torch.no_grad():
        full = m(x)
        for P in (9, 16, 23):
            part = m(x[..., :P].contiguous())
            Ts_p = 1 + -(-(P + la - 1) // S)
            n = max(t + 1 for t in range(P) if t + la < P and (t + la) // S < Ts_p - 1)
            assert torch.equal(part[..., :n], full[..., :n]), (P, n)
            assert not torch.equal(part[..., n:], full[..., n:P]), P


# ------------------------------------------------------------------------------------------------------ training
def check_grads(m, g, prec):
    worst = 0.0
    for k, p in m.named_parameters():
        got = p.grad.cpu().numpy().reshape(-1)
        e = rel_l2(got[::SUB], g["gsub." + k])
        n = abs(np.sqrt((got.astype(np.float64) ** 2).sum()) - g["gl2." + k]) / g["gl2." + k]
        # tf32: the encoder's gradients are a small remainder of the bottleneck / decoder chain, as in test_gpu_fast_train
        tol = 5e-2 if prec == "tf32_tc" and k.startswith("encoder.") else GRAD_TOL[prec]
        assert e < tol and n < GRAD_TOL[prec], (k, e, n)
        worst = max(worst, e, n)
    return worst


@pytest.mark.parametrize("prec", ["fp32", "tf32_tc"])
def test_two_golden_training_steps_match_reference(golden, dev, prec):
    from fullsubnet_b200.acoustics.feature import stft
    from oracle import make_golden_train_fast as MGT
    g, g_fast = golden("fast_cum"), golden("train_fast")
    m = build(dev, fast_args(), MGT.SEEDS["weights"], train_precision=prec)
    noisy, _ = MGT.inputs()
    cirm = torch.from_numpy(g_fast["cirm"]).to(dev)  # the same inputs as train_fast.npz: the reference's target
    opt, loss_fn = torch.optim.Adam(m.parameters(), lr=1e-3, betas=(0.9, 0.999)), torch.nn.MSELoss()
    for it in range(2):
        opt.zero_grad()
        crm = m(stft(noisy.to(dev), 512, 256, 512)[0].unsqueeze(1)).permute(0, 2, 3, 1)
        loss = loss_fn(cirm, crm)
        loss.backward()
        assert abs(float(loss.detach()) - g["loss"][it]) <= LOSS_TOL[prec] * g["loss"][it], (it, float(loss), g["loss"][it])
        if it == 0:
            assert rel_max(crm.detach().cpu(), g["crm"]) < (1e-4 if prec == "fp32" else 5e-3)
            print(f"fast train, cumulative norm, {prec}: worst gradient error {check_grads(m, g, prec):.2e}")
        gn = float(torch.nn.utils.clip_grad_norm_(m.parameters(), 10.0))
        assert abs(gn - g["gnorm"][it]) < GNORM_TOL[prec] * g["gnorm"][it], (it, gn, g["gnorm"][it])
        opt.step()
        if prec == "fp32":  # Adam's first steps are +-lr whatever the magnitude: parameters are compared for fp32 only
            sub = SUB * (4 if it == 0 else 1)
            for k, p in m.named_parameters():
                assert np.abs(p.detach().cpu().numpy().reshape(-1)[::sub] - g[f"p{it}." + k]).max() < 2e-5, (it, k)


@contextlib.contextmanager
def default_dtype(dtype):
    old = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        yield
    finally:
        torch.set_default_dtype(old)


@pytest.mark.parametrize("prec", ["fp32", "tf32_tc"])
@pytest.mark.parametrize("B,T", [(1, 12), (2, 13), (2, 12), (1, 14)])
def test_training_matches_float64_autograd_on_other_shapes(dev, prec, B, T):
    """shrink 3 with T + 1 frames: T = 12 leaves a full last block, 13 and 14 a short one; Ne = 1 exercises the reflected
    encoder columns of the unfold transpose; bottleneck_hidden_size = 128."""
    from oracle import fast_fullsubnet_cum_oracle as CO
    from oracle import fast_fullsubnet_oracle as FO
    args = fast_args(**OTHER, bottleneck_hidden_size=128)
    sd = FO.make_fast_state_dict(seed=11, args=args)
    gen = torch.Generator().manual_seed(100 * B + T)
    x = torch.rand(B, 1, 257, T, generator=gen) * 2
    w = torch.randn(B, 2, 257, T, generator=gen)
    with default_dtype(torch.float64):
        p = {k: v.double().requires_grad_(k != "mel_scale.fb") for k, v in sd.items()}
        ref_out = CO.fast_model_forward(x.double(), p, args)
        (ref_out * w.double()).sum().backward()
    m = build(dev, args, 11, train_precision=prec)
    out = m(x.to(dev))
    (out * w.to(dev)).sum().backward()
    assert rel_max(out.detach().cpu(), ref_out.detach()) < (1e-5 if prec == "fp32" else 5e-3)
    worst = 0.0
    for k, q in m.named_parameters():
        e = rel_l2(q.grad.cpu(), p[k].grad)
        worst = max(worst, e)
        assert e < GRAD_TOL[prec], (k, e)
    print(f"B={B} T={T} {prec}: worst gradient rel-L2 against float64 {worst:.2e}")


@pytest.mark.parametrize("kw", [{}, dict(OTHER, bottleneck_hidden_size=128)], ids=["recipe", "shrink3"])
def test_train_forward_equals_inference_forward(dev, kw):
    m = build(dev, fast_args(**kw), 3, precision="fp32", train_precision="fp32")
    x = torch.rand(3, 1, 257, 20, device=dev)
    a = m(x)
    assert a.requires_grad and a.shape == (3, 2, 257, 20)
    with torch.no_grad():
        b = m(x)
    assert rel_max(a.detach().cpu(), b.cpu()) < 1e-5


@pytest.mark.parametrize("prec", ["fp32", "tf32_tc"])
def test_two_backward_runs_give_identical_bits(dev, prec):
    m = build(dev, fast_args(), 3, train_precision=prec)
    x = torch.rand(3, 1, 257, 25, device=dev)
    w = torch.randn(3, 2, 257, 25, device=dev)
    grads = []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        (m(x) * w).sum().backward()
        grads.append([p.grad.clone() for p in m.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*grads))
