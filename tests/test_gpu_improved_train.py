"""GPU training step of improved_fullsubnet (fsn_improved_train_forward / fsn_improved_train_backward behind Model.forward
with gradients enabled) against optimisation steps of the UNMODIFIED reference (tests/golden/train_imp*.npz,
oracle/make_golden_train_imp.py) and against CPU autograd of the oracle on shapes the goldens do not cover."""
import numpy as np
import pytest
import torch

from conftest import rel_l2, rel_max

pytestmark = pytest.mark.gpu

GRAD_TOL = {"fp32": 2e-4, "tf32_tc": 1e-2}
LOSS_TOL = {"fp32": 1e-5, "tf32_tc": 1e-3}
GNORM_TOL = {"fp32": 1e-4, "tf32_tc": 5e-3}
OUT_TOL = {"fp32": 1e-5, "tf32_tc": 5e-3}
HID = dict(fb_hidden_size=32, sb_hidden_size=32)
# n_fft 256 / hop 64: section 0 reflects at row 0, section 1 has no neighbours, section 2 reflects at row F-2
SMALL_256 = dict(HID, n_fft=256, hop_length=64, win_length=256, num_freqs=129, freq_cutoffs=[8, 32],
                 sb_num_center_freqs=[1, 4, 8], sb_num_neighbor_freqs=[15, 0, 7], fb_num_center_freqs=[1, 4, 8],
                 fb_num_neighbor_freqs=[15, 0, 7])


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def build(dev, prec="fp32", args=None, seed=5, sd=None):
    from fullsubnet_b200.improved_fullsubnet.model import Model
    from oracle import improved_fullsubnet_oracle as IO
    a = dict(IO.DEFAULT_IMPROVED_ARGS, **(args or {}))
    m = Model(**a)
    m.load_state_dict(sd if sd is not None else IO.make_improved_state_dict(seed=seed, args=a), strict=True)
    m.train_precision = prec
    return m.to(dev).train()


def golden_setup(golden, dev, name, prec):
    from oracle import make_golden_train_imp as MG
    g = golden(name)
    noisy, clean = MG.inputs(name)
    assert np.allclose(MG.fingerprint(noisy), g["noisy_fp"], rtol=1e-6)
    m = build(dev, prec, {k: v for k, v in MG.args_of(name).items()}, seed=MG.SEEDS["weights"])
    return g, m, noisy.to(dev), clean.to(dev).unsqueeze(1), MG.SUBSAMPLE


def check_grads(m, g, prec, sub):
    worst = 0.0
    for k, p in m.named_parameters():
        got = p.grad.cpu().numpy().reshape(-1)
        e = rel_l2(got[::sub], g["gsub." + k])
        n = abs(np.sqrt((got.astype(np.float64) ** 2).sum()) - g["gl2." + k]) / g["gl2." + k]
        worst = max(worst, e, n)
        assert e < GRAD_TOL[prec] and n < GRAD_TOL[prec], (k, e, n)
    return worst


@pytest.mark.parametrize("fused,prec", [(True, "fp32"), (False, "fp32"), (True, "tf32_tc"), (False, "tf32_tc")])
def test_two_golden_steps_match_reference(golden, dev, fused, prec):
    from fullsubnet_b200.optim import FusedClipAdam
    g, m, noisy, clean, sub = golden_setup(golden, dev, "train_imp", prec)
    if fused:
        opt = FusedClipAdam(m.parameters(), lr=1e-3, betas=(0.9, 0.999), max_norm=10.0)
    else:  # the reference's own objects on top of our Model
        opt = torch.optim.Adam(m.parameters(), lr=1e-3, betas=(0.9, 0.999))
    loss_fn = torch.nn.MSELoss()
    for it in range(2):
        opt.zero_grad()
        enhanced = m(noisy)
        loss = loss_fn(enhanced, clean)
        loss.backward()
        assert abs(float(loss.detach()) - g["loss"][it]) <= LOSS_TOL[prec] * g["loss"][it], (it, float(loss), g["loss"][it])
        if it == 0:
            assert enhanced.shape == (3, 1, 8000)
            assert rel_max(enhanced.detach().cpu(), g["enhanced"]) < (1e-4 if prec == "fp32" else 5e-3)
            worst = check_grads(m, g, prec, sub)
            print(f"improved_fullsubnet train ({'fused' if fused else 'torch'} optimiser, {prec}): worst gradient error {worst:.2e}")
        if fused:
            opt.step()
            gn = float(opt.last_norm[0])
        else:
            gn = float(torch.nn.utils.clip_grad_norm_(m.parameters(), 10.0))
            opt.step()
        assert abs(gn - g["gnorm"][it]) < GNORM_TOL[prec] * g["gnorm"][it], (it, gn, g["gnorm"][it])
        if prec == "fp32":  # Adam's first steps are +-lr whatever the magnitude: parameters are compared for fp32 only
            for k, p in m.named_parameters():
                ref = g[f"p{it}." + k]
                assert np.abs(p.detach().cpu().numpy().reshape(-1)[::sub * (4 if it == 0 else 1)] - ref).max() < 2e-5, (it, k)


@pytest.mark.parametrize("prec", ["fp32", "tf32_tc"])
def test_golden_step_n_fft_960(golden, dev, prec):
    """The reference's 48 kHz example: the STFT, iSTFT and their adjoint run on the direct DFT."""
    g, m, noisy, clean, sub = golden_setup(golden, dev, "train_imp_960", prec)
    loss = torch.nn.MSELoss()(m(noisy), clean)
    loss.backward()
    assert abs(float(loss.detach()) - g["loss"][0]) <= LOSS_TOL[prec] * g["loss"][0]
    worst = check_grads(m, g, prec, sub)
    print(f"improved_fullsubnet n_fft=960 train ({prec}): worst gradient error {worst:.2e}")


# (args, B, L): B = 1 / 3, L not a multiple of hop, n_fft 256 / 512, reflections at both ends, a section without
# neighbours, ReLU on both stacks, noisy and full-band neighbour counts that differ
CASES = {
    "n256_B1": (SMALL_256, 1, 1000),
    "n512_relu_B3": (dict(HID, fb_output_activate_function="ReLU", sb_output_activate_function="ReLU"), 3, 4037),
    "n256_mixed_B3": (dict(SMALL_256, sb_num_neighbor_freqs=[3, 0, 7], fb_num_neighbor_freqs=[15, 2, 1]), 3, 1500),
}


# ReLU on both stacks is compared in fp32 only: with random weights many outputs sit near 0, and the ~1e-3 relative error
# of tf32 moves some of them across 0, which changes their ReLU' (section 2's layer-0 input-weight gradient came out
# 1.6e-2 rel-L2 from the oracle's on an H100; 1.9e-6 in fp32)
@pytest.mark.parametrize("case,prec", [(c, p) for c in CASES for p in ("fp32", "tf32_tc") if (c, p) != ("n512_relu_B3", "tf32_tc")])
def test_matches_oracle_autograd_on_other_shapes(dev, case, prec):
    from oracle import fullsubnet_oracle as O
    from oracle import improved_fullsubnet_oracle as IO
    args, B, L = CASES[case]
    a = dict(IO.DEFAULT_IMPROVED_ARGS, **args)
    sd = IO.make_improved_state_dict(seed=11, args=a)
    y = O.make_noisy(B, L, seed=B * 7 + L, speechlike=True)
    w = torch.randn(B, 1, L, generator=torch.Generator().manual_seed(L))
    p = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ref = IO.improved_forward(y, p, a)
    (ref * w).sum().backward()
    m = build(dev, prec, args, sd=sd)
    out = m(y.to(dev))
    (out * w.to(dev)).sum().backward()
    assert out.shape == (B, 1, L)
    assert rel_max(out.detach().cpu(), ref.detach()) < OUT_TOL[prec] * (10 if prec == "fp32" else 1)
    worst = 0.0
    for k, q in m.named_parameters():
        e = rel_l2(q.grad.cpu(), p[k].grad)
        worst = max(worst, e)
        assert e < GRAD_TOL[prec], (k, e)
    print(f"{case} {prec}: worst gradient rel-L2 {worst:.2e}")


@pytest.mark.parametrize("prec", ["fp32", "tf32_tc"])
def test_train_forward_equals_inference_forward(dev, prec):
    m = build(dev, prec, HID)
    m.precision = prec
    y = torch.randn(2, 4000, device=dev) * 0.1
    a = m(y)
    assert a.requires_grad and a.shape == (2, 1, 4000)
    with torch.no_grad():
        b = m(y)
    assert rel_max(a.detach().cpu(), b.cpu()) < OUT_TOL[prec]
    m.eval()  # eval mode with gradients enabled is a training step too, like the reference module
    assert m(y).requires_grad


@pytest.mark.parametrize("prec", ["fp32", "tf32_tc"])
def test_two_backward_runs_give_identical_bits(dev, prec):
    m = build(dev, prec)
    y = torch.randn(3, 8000, device=dev) * 0.1
    w = torch.randn(3, 1, 8000, device=dev)
    grads = []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        (m(y) * w).sum().backward()
        grads.append([p.grad.clone() for p in m.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*grads))


def test_error_behaviour(dev):
    from fullsubnet_b200.improved_fullsubnet.model import Model
    from oracle import improved_fullsubnet_oracle as IO
    m = build(dev, "fp32", SMALL_256)
    y = torch.randn(2, 1000, device=dev) * 0.1
    out = m(y)
    out.sum().backward()
    with pytest.raises(RuntimeError):
        out.sum().backward()  # activations are released after the first backward
    out = m(y)
    with torch.no_grad():
        m.fb_model.fc_output_layer.bias.add_(0.0)  # in-place update between forward and backward
    with pytest.raises(RuntimeError):
        out.sum().backward()
    with pytest.raises(NotImplementedError):
        m(y, return_crm=True)
    with pytest.raises(NotImplementedError):
        m(y.clone().requires_grad_(True))  # no input gradient is computed
    frozen = build(dev, "fp32", SMALL_256)
    frozen.sb_model.sb_models[1].fc_output_layer.weight.requires_grad_(False)
    with pytest.raises(NotImplementedError):
        frozen(y)
    gru = Model(**dict(IO.DEFAULT_IMPROVED_ARGS, **SMALL_256, sequence_model="GRU")).to(dev).train()
    with pytest.raises(NotImplementedError):
        gru(y)
