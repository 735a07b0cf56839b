"""GPU training step of fullband_baseline (fsn_fullband_train_forward / fsn_fullband_train_backward behind Model.forward
with gradients enabled) against two optimisation steps of the UNMODIFIED reference (tests/golden/train_fbb.npz,
oracle/make_golden_train_fbb.py) and against CPU autograd of the oracle on shapes the golden does not cover."""
import numpy as np
import pytest
import torch

from conftest import rel_l2, rel_max

pytestmark = pytest.mark.gpu

SUB = 97  # oracle/make_golden_train_fbb.py:SUBSAMPLE
GRAD_TOL = {"fp32": 2e-4, "tf32_tc": 1e-2}
LOSS_TOL = {"fp32": 1e-5, "tf32_tc": 1e-3}
GNORM_TOL = {"fp32": 1e-4, "tf32_tc": 5e-3}
SMALL = dict(num_freqs=33, hidden_size=32)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def build(dev, prec="fp32", args=None, seed=5, sd=None):
    from fullsubnet_b200.fullband_baseline.model import Model
    from oracle import fullband_baseline_oracle as BO
    a = dict(BO.DEFAULT_FBB_ARGS, **(args or {}))
    m = Model(**a)
    m.load_state_dict(sd if sd is not None else BO.make_fbb_state_dict(seed=seed, args=a), strict=True)
    m.train_precision = prec
    return m.to(dev).train()


def golden_inputs(dev):
    from oracle import make_golden_train_fbb as MG
    noisy, clean = MG.inputs()
    return noisy.to(dev), clean.to(dev)


def forward_loss(m, noisy, cirm, loss_fn):
    """fullband_baseline/trainer.py:45-57: the target is the stored cIRM of the reference (see check_cirm)."""
    from fullsubnet_b200.acoustics.feature import stft
    noisy_mag = stft(noisy, 512, 256, 512)[0]
    crm = m(noisy_mag.unsqueeze(1)).permute(0, 2, 3, 1)
    return loss_fn(cirm, crm), crm


def check_cirm(noisy, clean, g):
    """Our cIRM against the reference's: a few bins where |noisy| is tiny amplify STFT rounding differences."""
    from fullsubnet_b200.acoustics.feature import stft
    from fullsubnet_b200.acoustics.mask import build_complex_ideal_ratio_mask
    _, _, nr, ni = stft(noisy, 512, 256, 512)
    _, _, cr, ci = stft(clean, 512, 256, 512)
    cirm = build_complex_ideal_ratio_mask(nr, ni, cr, ci)
    e = rel_l2(cirm.cpu(), g["cirm"])
    print(f"cIRM rel-L2 vs reference {e:.2e}")
    assert e < 1e-2
    return cirm


def check_grads(m, g, prec):
    worst = 0.0
    for k, p in m.named_parameters():
        got = p.grad.cpu().numpy().reshape(-1)
        e = rel_l2(got[::SUB], g["gsub." + k])
        n = abs(np.sqrt((got.astype(np.float64) ** 2).sum()) - g["gl2." + k]) / g["gl2." + k]
        worst = max(worst, e, n)
        assert e < GRAD_TOL[prec] and n < GRAD_TOL[prec], (k, e, n)
    return worst


def check_params(m, g, it, tol=2e-5):
    for k, p in m.named_parameters():
        sub = SUB * (4 if it == 0 else 1)
        assert np.abs(p.detach().cpu().numpy().reshape(-1)[::sub] - g[f"p{it}." + k]).max() < tol, (it, k)


@pytest.mark.parametrize("fused,prec", [(True, "fp32"), (False, "fp32"), (True, "tf32_tc"), (False, "tf32_tc")])
def test_two_golden_steps_match_reference(golden, dev, fused, prec):
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.optim import FusedClipAdam
    g = golden("train_fbb")
    m = build(dev, prec)
    noisy, clean = golden_inputs(dev)
    check_cirm(noisy, clean, g)
    cirm = torch.from_numpy(g["cirm"]).to(dev)
    if fused:
        opt, loss_fn = FusedClipAdam(m.parameters(), lr=1e-3, betas=(0.9, 0.999), max_norm=10.0), mse_loss()
    else:  # the reference's own objects on top of our Model
        opt, loss_fn = torch.optim.Adam(m.parameters(), lr=1e-3, betas=(0.9, 0.999)), torch.nn.MSELoss()
    for it in range(2):
        opt.zero_grad()
        loss, crm = forward_loss(m, noisy, cirm, loss_fn)
        loss.backward()
        assert abs(float(loss.detach()) - g["loss"][it]) <= LOSS_TOL[prec] * g["loss"][it], (it, float(loss), g["loss"][it])
        if it == 0:
            assert rel_max(crm.detach().cpu(), g["crm"]) < (1e-4 if prec == "fp32" else 5e-3)
            worst = check_grads(m, g, prec)
            print(f"fullband_baseline train ({'fused' if fused else 'torch'} optimiser, {prec}): worst gradient error {worst:.2e}")
        if fused:
            opt.step()
            gn = float(opt.last_norm[0])
        else:
            gn = float(torch.nn.utils.clip_grad_norm_(m.parameters(), 10.0))
            opt.step()
        assert abs(gn - g["gnorm"][it]) < GNORM_TOL[prec] * g["gnorm"][it], (it, gn, g["gnorm"][it])
        if prec == "fp32":  # Adam's first steps are +-lr whatever the magnitude: parameters are compared for fp32 only
            check_params(m, g, it)


# (activation, norm, look_ahead, B): every activation, both norms, look-ahead 0 / 1, B = 1 / 3
CASES = [(None, "offline_laplace_norm", 0, 1), ("ReLU", "cumulative_laplace_norm", 1, 3),
         ("ReLU6", "offline_laplace_norm", 1, 3), ("Tanh", "cumulative_laplace_norm", 0, 3),
         ("Tanh", "offline_laplace_norm", 1, 1)]


def check_against_oracle(dev, prec, act, norm, la, B, gain=1.0):
    """F = 33, H = 32, T = 17 against CPU autograd of the oracle; `gain` scales the output Linear's weight."""
    from oracle import fullband_baseline_oracle as BO
    args = dict(BO.DEFAULT_FBB_ARGS, **SMALL, output_activate_function=act, norm_type=norm, look_ahead=la)
    sd = BO.make_fbb_state_dict(seed=11, args=args)
    sd["fullband_model.fc_output_layer.weight"] *= gain
    T = 17
    gen = torch.Generator().manual_seed(100 * B + la)
    x = torch.rand(B, 1, 33, T, generator=gen) * 2
    w = torch.randn(B, 2, 33, T, generator=gen)
    p = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ref_out = BO.fbb_forward(x, p, args)
    (ref_out * w).sum().backward()
    m = build(dev, prec, dict(SMALL, output_activate_function=act, norm_type=norm, look_ahead=la), sd=sd)
    out = m(x.to(dev))
    (out * w.to(dev)).sum().backward()
    assert rel_max(out.detach().cpu(), ref_out.detach()) < (1e-5 if prec == "fp32" else 5e-3)
    worst = 0.0
    for k, q in m.named_parameters():
        e = rel_l2(q.grad.cpu(), p[k].grad)
        worst = max(worst, e)
        assert e < GRAD_TOL[prec], (k, e)
    print(f"{act} {norm} la={la} B={B} gain={gain} {prec}: worst gradient rel-L2 {worst:.2e}")
    return ref_out.detach()


@pytest.mark.parametrize("prec", ["fp32", "tf32_tc"])
@pytest.mark.parametrize("act,norm,la,B", CASES)
def test_matches_oracle_autograd_on_other_shapes(dev, prec, act, norm, la, B):
    check_against_oracle(dev, prec, act, norm, la, B)


def test_relu6_saturation_matches_oracle_autograd(dev):
    """ReLU6 with the output Linear scaled by 200: about a fifth of the outputs sit at 6, where act' is 0.  fp32 only: at
    this gain the ~1e-3 relative error of tf32 moves a few per cent of the pre-activations across 0 or 6, which changes
    their act' and put layer 0's input-weight gradient 4.4e-2 (rel-L2) away from the oracle's on an H100."""
    ref = check_against_oracle(dev, "fp32", "ReLU6", "offline_laplace_norm", 1, 3, gain=200.0)
    sat = float((ref >= 6).float().mean())
    assert 0.05 < sat < 0.6, sat


@pytest.mark.parametrize("args", [None, dict(SMALL, output_activate_function="Tanh", norm_type="cumulative_laplace_norm")])
def test_train_forward_equals_inference_forward(dev, args):
    m = build(dev, "fp32", args)
    F = m.num_freqs
    x = torch.rand(3, 1, F, 20, device=dev)
    a = m(x)
    assert a.requires_grad and a.shape == (3, 2, F, 20)
    with torch.no_grad():
        b = m(x)
    assert rel_max(a.detach().cpu(), b.cpu()) < 1e-5


@pytest.mark.parametrize("prec", ["fp32", "tf32_tc"])
def test_two_backward_runs_give_identical_bits(dev, prec):
    m = build(dev, prec)
    x = torch.rand(3, 1, 257, 25, device=dev)
    w = torch.randn(3, 2, 257, 25, device=dev)
    grads = []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        (m(x) * w).sum().backward()
        grads.append([p.grad.clone() for p in m.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*grads))


def test_trainer_steps_checkpoint_and_validation(golden, dev, tmp_path):
    """Two one-step epochs of the Trainer (no drop_band for this model) == two explicit steps; the loss of the second equals
    the reference's golden step 1; the checkpoint round-trips; the B = 1 validation loop runs on this model."""
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.optim import FusedClipAdam
    from fullsubnet_b200.trainer import Trainer
    g = golden("train_fbb")
    noisy, clean = golden_inputs(dev)
    cfg = {"meta": {"use_amp": True, "save_dir": str(tmp_path), "experiment_name": "b"},
           "acoustics": {"n_fft": 512, "hop_length": 256, "win_length": 512},
           "trainer": {"train": {"epochs": 2, "save_checkpoint_interval": 1, "clip_grad_norm_value": 10},
                       "validation": {"validation_interval": 2, "save_max_metric_score": True}}}
    valid = [(noisy[i:i + 1].cpu(), clean[i:i + 1].cpu(), [f"clip{i}"], ["With_reverb" if i != 1 else "No_reverb"])
             for i in range(3)]
    m = build(dev, "fp32")
    tr = Trainer(None, 0, cfg, False, False, m, mse_loss(), FusedClipAdam(m.parameters(), lr=1e-3), [(noisy.cpu(), clean.cpu())],
                 valid)
    tr.train()
    assert abs(tr.last_epoch_loss - g["loss"][1]) < 1e-4 * g["loss"][1], (tr.last_epoch_loss, g["loss"][1])
    v = tr.last_validation
    assert v["items"] == {"With_reverb": 2, "No_reverb": 1} and np.isfinite(v["loss_total"]) and m.training
    # the same two steps written out
    cirm = check_cirm(noisy, clean, g)
    m2 = build(dev, "fp32")
    opt = FusedClipAdam(m2.parameters(), lr=1e-3, max_norm=10.0)
    for _ in range(2):
        opt.zero_grad(set_to_none=False)
        forward_loss(m2, noisy, cirm, mse_loss())[0].backward()
        opt.step()
    for (k, p), p2 in zip(m.named_parameters(), m2.parameters()):
        assert torch.equal(p, p2), k
    ck = torch.load(tmp_path / "b" / "checkpoints" / "latest_model.tar", map_location="cpu")
    assert set(ck) == {"epoch", "best_score", "optimizer", "scaler", "model"} and ck["epoch"] == 2
    assert len(ck["model"]) == 14  # 3 x 4 LSTM tensors + the Linear's weight and bias
    m3 = build(dev, "fp32", seed=6)
    tr3 = Trainer(None, 0, cfg, True, False, m3, mse_loss(), FusedClipAdam(m3.parameters(), lr=1e-3), [], None)
    assert tr3.start_epoch == 3
    for k, t in m3.state_dict().items():
        assert torch.equal(t.cpu(), m.state_dict()[k].cpu()), k


def test_reference_flow_autocast_gradscaler(golden, dev):
    """fullband_baseline/trainer.py:45-71 verbatim on the drop-in Model: autocast + GradScaler + unscale_ +
    clip_grad_norm_ + torch.optim.Adam, two steps equal to the golden steps of the unmodified reference."""
    from torch.cuda.amp import GradScaler, autocast
    from fullsubnet_b200.acoustics.feature import stft
    g = golden("train_fbb")
    m = build(dev, "fp32")
    noisy, _ = golden_inputs(dev)
    cIRM = torch.from_numpy(g["cirm"]).to(dev)
    optimizer = torch.optim.Adam(m.parameters(), lr=1e-3, betas=(0.9, 0.999))
    loss_function = torch.nn.MSELoss()
    scaler = GradScaler(enabled=True)
    for it in range(2):
        optimizer.zero_grad()
        noisy_mag = stft(noisy, 512, 256, 512)[0]
        with autocast(enabled=True):
            cRM = m(noisy_mag.unsqueeze(1)).permute(0, 2, 3, 1)
            loss = loss_function(cIRM, cRM)
        scaler.scale(loss).backward()
        scaler.unscale_(optimizer)
        gn = torch.nn.utils.clip_grad_norm_(m.parameters(), 10)
        scaler.step(optimizer)
        scaler.update()
        assert abs(float(loss) - g["loss"][it]) <= 1e-5 * g["loss"][it], (it, float(loss))
        assert abs(float(gn) - g["gnorm"][it]) < 1e-4 * g["gnorm"][it]
        check_params(m, g, it)


def test_error_behaviour(dev):
    from fullsubnet_b200.fullband_baseline.model import Model
    from oracle import fullband_baseline_oracle as BO
    m = build(dev, "fp32", SMALL)
    x = torch.rand(2, 1, 33, 10, device=dev)
    out = m(x)
    out.sum().backward()
    with pytest.raises(RuntimeError):
        out.sum().backward()  # activations are released after the first backward
    out = m(x)
    with torch.no_grad():
        m.fullband_model.fc_output_layer.bias.add_(0.0)  # in-place update between forward and backward
    with pytest.raises(RuntimeError):
        out.sum().backward()
    frozen = build(dev, "fp32", SMALL)
    frozen.fullband_model.sequence_model.weight_ih_l0.requires_grad_(False)
    with pytest.raises(NotImplementedError):
        frozen(x)
    gru = Model(**dict(BO.DEFAULT_FBB_ARGS, **SMALL, sequence_model="GRU")).to(dev).train()
    with pytest.raises(NotImplementedError):
        gru(x)
