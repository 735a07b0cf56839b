"""GPU training step of fast_fullsubnet (fsn_fast_train_forward / fsn_fast_train_backward behind Model.forward in train mode)
against two optimisation steps of the UNMODIFIED reference (tests/golden/train_fast.npz, oracle/make_golden_train_fast.py)
and against CPU autograd of the oracle on shapes the goldens do not cover."""
import numpy as np
import pytest
import torch

from conftest import rel_l2, rel_max

pytestmark = pytest.mark.gpu

SUB = 97  # oracle/make_golden_train_fast.py:SUBSAMPLE
GRAD_TOL = {"fp32": 2e-4, "tf32_tc": 1e-2}
LOSS_TOL = {"fp32": 1e-5, "tf32_tc": 1e-3}
GNORM_TOL = {"fp32": 1e-4, "tf32_tc": 5e-3}
# shrink 3 (a short or a full last block), one frame of look-ahead, encoder-output neighbours, a narrower bottleneck
EXTRA_ARGS = dict(shrink_size=3, look_ahead=1, encoder_output_num_neighbors=1, bottleneck_hidden_size=128)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def build(dev, prec="fp32", args=None, seed=3):
    from fullsubnet_b200.fast_fullsubnet.model import Model
    from oracle import fast_fullsubnet_oracle as FO
    a = dict(FO.DEFAULT_FAST_ARGS, **(args or {}))
    m = Model(**a)
    m.load_state_dict(FO.make_fast_state_dict(seed=seed, args=a), strict=True)
    m.train_precision = prec
    return m.to(dev).train()


def golden_inputs(dev):
    from oracle import make_golden_train_fast as MG
    noisy, clean = MG.inputs()
    return noisy.to(dev), clean.to(dev)


def forward_loss(m, noisy, cirm, loss_fn):
    """fast_fullsubnet/trainer.py:45-56: the target is the stored cIRM of the reference (see check_cirm)."""
    from fullsubnet_b200.acoustics.feature import stft
    noisy_mag = stft(noisy, 512, 256, 512)[0]
    crm = m(noisy_mag.unsqueeze(1)).permute(0, 2, 3, 1)
    return loss_fn(cirm, crm), crm


def check_cirm(noisy, clean, g):
    """Our cIRM against the reference's: a few frame-0 bins where |noisy| ~ 1e-4 amplify STFT rounding differences."""
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
    worst, errs = 0.0, []
    for k, p in m.named_parameters():
        got = p.grad.cpu().numpy().reshape(-1)
        e = rel_l2(got[::SUB], g["gsub." + k])
        n = abs(np.sqrt((got.astype(np.float64) ** 2).sum()) - g["gl2." + k]) / g["gl2." + k]
        worst = max(worst, e, n)
        errs.append((k, e, n))
    for k, e, n in errs:
        # tf32: the encoder's gradients are a small remainder of the bottleneck / decoder chain (second-norm mean term,
        # unfold sums); at this step they sit at 1.7-3.8e-2 rel-L2 (sub-sampled) and 4e-3 in L2 norm
        tol = 5e-2 if prec == "tf32_tc" and k.startswith("encoder.") else GRAD_TOL[prec]
        assert e < tol and n < GRAD_TOL[prec], (k, e, n)
    return worst


def check_params(m, g, it, tol=2e-5):
    for k, p in m.named_parameters():
        sub = SUB * (4 if it == 0 else 1)
        assert np.abs(p.detach().cpu().numpy().reshape(-1)[::sub] - g[f"p{it}." + k]).max() < tol, (it, k)


@pytest.mark.parametrize("fused,prec", [(True, "fp32"), (False, "fp32"), (True, "tf32_tc"), (False, "tf32_tc")])
def test_two_golden_steps_match_reference(golden, dev, fused, prec):
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.optim import FusedClipAdam
    g = golden("train_fast")
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
            print(f"fast train ({'fused' if fused else 'torch'} optimiser, {prec}): worst gradient error {worst:.2e}")
        if fused:
            opt.step()
            gn = float(opt.last_norm[0])
        else:
            gn = float(torch.nn.utils.clip_grad_norm_(m.parameters(), 10.0))
            opt.step()
        assert abs(gn - g["gnorm"][it]) < GNORM_TOL[prec] * g["gnorm"][it], (it, gn, g["gnorm"][it])
        if prec == "fp32":  # Adam's first steps are +-lr whatever the magnitude: parameters are compared for fp32 only
            check_params(m, g, it)


def oracle_grads(x, sd, args, w):
    from oracle import fast_fullsubnet_oracle as FO
    p = {k: v.clone().requires_grad_(k != "mel_scale.fb") for k, v in sd.items()}
    out = FO.fast_model_forward(x, p, args)
    (out * w).sum().backward()
    return out.detach(), {k: v.grad for k, v in p.items() if k != "mel_scale.fb"}


@pytest.mark.parametrize("prec", ["fp32", "tf32_tc"])
@pytest.mark.parametrize("B,T", [(1, 12), (2, 13), (2, 12), (1, 14)])
def test_matches_oracle_autograd_on_other_shapes(dev, prec, B, T):
    """shrink 3 with T + 1 frames: T = 12 leaves a full last block, 13 and 14 a short one; Ne = 1 exercises the reflected
    encoder columns of the unfold transpose; bottleneck_hidden_size = 128."""
    from oracle import fast_fullsubnet_oracle as FO
    args = dict(FO.DEFAULT_FAST_ARGS, **EXTRA_ARGS)
    sd = FO.make_fast_state_dict(seed=11, args=args)
    gen = torch.Generator().manual_seed(100 * B + T)
    x = torch.rand(B, 1, 257, T, generator=gen) * 2
    w = torch.randn(B, 2, 257, T, generator=gen)
    ref_out, ref = oracle_grads(x, sd, args, w)
    m = build(dev, prec, EXTRA_ARGS, seed=11)
    out = m(x.to(dev))
    (out * w.to(dev)).sum().backward()
    assert rel_max(out.detach().cpu(), ref_out) < (1e-5 if prec == "fp32" else 5e-3)
    worst = 0.0
    for k, p in m.named_parameters():
        e = rel_l2(p.grad.cpu(), ref[k])
        worst = max(worst, e)
        assert e < GRAD_TOL[prec], (k, e)
    print(f"B={B} T={T} {prec}: worst gradient rel-L2 {worst:.2e}")


@pytest.mark.parametrize("args", [None, EXTRA_ARGS])
def test_train_forward_equals_inference_forward(dev, args):
    m = build(dev, "fp32", args)
    x = torch.rand(3, 1, 257, 20, device=dev)
    a = m(x)
    assert a.requires_grad and a.shape == (3, 2, 257, 20)
    m.precision = "fp32"
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
    the reference's golden step 1; the checkpoint round-trips; the B = 1 validation loop runs on the fast model."""
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.optim import FusedClipAdam
    from fullsubnet_b200.trainer import Trainer
    g = golden("train_fast")
    noisy, clean = golden_inputs(dev)
    cfg = {"meta": {"use_amp": True, "save_dir": str(tmp_path), "experiment_name": "f"},
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
    ck = torch.load(tmp_path / "f" / "checkpoints" / "latest_model.tar", map_location="cpu")
    assert set(ck) == {"epoch", "best_score", "optimizer", "scaler", "model"} and ck["epoch"] == 2
    assert len(ck["model"]) == 31  # 30 parameters + the mel filterbank buffer
    m3 = build(dev, "fp32", seed=4)
    tr3 = Trainer(None, 0, cfg, True, False, m3, mse_loss(), FusedClipAdam(m3.parameters(), lr=1e-3), [], None)
    assert tr3.start_epoch == 3
    for k, t in m3.state_dict().items():
        assert torch.equal(t.cpu(), m.state_dict()[k].cpu()), k


def test_reference_flow_autocast_gradscaler(golden, dev):
    """fast_fullsubnet/trainer.py:45-63 verbatim on the drop-in Model: autocast + GradScaler + unscale_ + clip_grad_norm_ +
    torch.optim.Adam, two steps equal to the golden steps of the unmodified reference."""
    from torch.cuda.amp import GradScaler, autocast
    from fullsubnet_b200.acoustics.feature import stft
    g = golden("train_fast")
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
    from fullsubnet_b200.fast_fullsubnet.model import Model
    from oracle import fast_fullsubnet_oracle as FO
    m = build(dev, "fp32")
    x = torch.rand(2, 1, 257, 10, device=dev)
    out = m(x)
    out.sum().backward()
    with pytest.raises(RuntimeError):
        out.sum().backward()  # activations are released after the first backward
    out = m(x)
    with torch.no_grad():
        m.bottleneck.fc_output_layer.bias.add_(0.0)  # in-place update between forward and backward
    with pytest.raises(RuntimeError):
        out.sum().backward()
    frozen = build(dev, "fp32")
    frozen.encoder[0].sequence_model.weight_ih_l0.requires_grad_(False)
    with pytest.raises(NotImplementedError):
        frozen(x)
    gru = Model(**dict(FO.DEFAULT_FAST_ARGS, sequence_model="GRU")).to(dev).train()
    with pytest.raises(NotImplementedError):
        gru(x)
