"""GPU parity of the training step (SURVEY 8a row A11, BASELINE config 3) against one step of the UNMODIFIED
reference trainer arithmetic (tests/golden/train_*.npz, oracle/make_golden_train.py) and the CPU oracle.

Gates (SURVEY 8d): loss rel <= 1e-3, per-tensor gradient rel-L2 <= 1e-2.  The fp32 kernels are held to 2e-4."""
import numpy as np
import pytest
import torch

from conftest import rel_l2, rel_max

pytestmark = pytest.mark.gpu

GRAD_TOL = {"fp32": 2e-4, "tf32_tc": 1e-2}   # tf32_tc: the north-star gate (SURVEY 8d); measured ~1e-3
LOSS_TOL = {"fp32": 1e-5, "tf32_tc": 1e-3}
SUB = 97  # oracle/make_golden_train.py:SUBSAMPLE


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def T(x, dev):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def small_args():
    from oracle.make_golden_train import SMALL
    return dict(SMALL)


def build(args, sd, dev, prec="fp32"):
    from fullsubnet_b200.fullsubnet.model import Model
    m = Model(**args)
    m.load_state_dict(sd, strict=True)
    m.train_precision = prec
    return m.to(dev).train()


def reference_like_step(model, noisy, clean, n_fft, hop, loss_fn):
    """fullsubnet/trainer.py:46-63 written against the fullsubnet_b200 mirrors of the same functions."""
    from fullsubnet_b200.acoustics.feature import drop_band, stft
    from fullsubnet_b200.acoustics.mask import build_complex_ideal_ratio_mask
    noisy_mag, _, nr, ni = stft(noisy, n_fft, hop, n_fft)
    _, _, cr, ci = stft(clean, n_fft, hop, n_fft)
    cIRM = build_complex_ideal_ratio_mask(nr, ni, cr, ci)
    cIRM = drop_band(cIRM.permute(0, 3, 1, 2), model.num_groups_in_drop_band).permute(0, 2, 3, 1)
    cRM = model(noisy_mag.unsqueeze(1)).permute(0, 2, 3, 1)
    loss = loss_fn(cIRM, cRM)
    loss.backward()
    return loss, cIRM, cRM


@pytest.mark.parametrize("fused,prec", [(True, "fp32"), (False, "fp32"), (True, "tf32_tc")])
def test_small_model_two_steps_match_reference(golden, dev, fused, prec):
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.optim import FusedClipAdam
    from oracle import fullsubnet_oracle as O
    g = golden("train_small")
    args = small_args()
    m = build(args, O.make_state_dict(seed=7, args=args, sb_fc_gain=8.0), dev, prec)
    noisy, clean = T(g["noisy"], dev), T(g["clean"], dev)
    if fused:
        opt, loss_fn = FusedClipAdam(m.parameters(), lr=1e-3, betas=(0.9, 0.999), max_norm=10.0), mse_loss()
    else:  # the reference's own objects on top of our Model: drop-in check of the autograd seam
        opt, loss_fn = torch.optim.Adam(m.parameters(), lr=1e-3, betas=(0.9, 0.999)), torch.nn.MSELoss()
    for it in range(2):
        opt.zero_grad()
        loss, cirm, crm = reference_like_step(m, noisy, clean, 64, 32, loss_fn)
        assert abs(float(loss.detach()) - g["loss"][it]) <= LOSS_TOL[prec] * abs(g["loss"][it]), (float(loss), g["loss"][it])
        if it == 0:
            assert rel_max(cirm.cpu(), g["cirm"]) < 5e-5  # near-0/0 bins of the ratio mask carry rounding noise
            assert rel_max(crm.detach().cpu(), g["crm"]) < (1e-5 if prec == "fp32" else 1e-3)
            worst = 0.0
            for k, p in m.named_parameters():
                e = rel_l2(p.grad.cpu(), g["grad." + k])
                worst = max(worst, e)
                assert e < GRAD_TOL[prec], (k, e)
            print(f"small model ({'fused' if fused else 'torch'} optimiser, {prec}): worst gradient rel-L2 {worst:.2e}")
        if prec != "fp32":
            opt.step()  # Adam's first steps are +-lr whatever the magnitude: parameters are compared for fp32 only
            continue
        if fused:
            opt.step()
            assert abs(float(opt.last_norm[0]) - g["gnorm"][it]) < 1e-4 * g["gnorm"][it]
        else:
            gn = torch.nn.utils.clip_grad_norm_(m.parameters(), 10.0)
            assert abs(float(gn) - g["gnorm"][it]) < 1e-4 * g["gnorm"][it]
            opt.step()
        for k, v in m.state_dict().items():
            assert np.abs(v.cpu().numpy() - g[f"p{it}." + k]).max() < 2e-5, (it, k)


@pytest.mark.parametrize("prec", ["fp32", "tf32_tc"])
def test_full_size_model_step_matches_reference(golden, dev, prec):
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.optim import FusedClipAdam
    from oracle import fullsubnet_oracle as O
    g = golden("train_full")
    args = dict(O.DEFAULT_MODEL_ARGS, weight_init=False)
    m = build(args, O.make_state_dict(seed=0, args=args, sb_fc_gain=40.0), dev, prec)
    opt = FusedClipAdam(m.parameters(), lr=1e-3, max_norm=10.0)
    loss, _, _ = reference_like_step(m, T(g["noisy"], dev), T(g["clean"], dev), 512, 256, mse_loss())
    assert abs(float(loss.detach()) - g["loss"][0]) <= LOSS_TOL[prec] * g["loss"][0], float(loss)
    worst = 0.0
    for k, p in m.named_parameters():
        got = p.grad.cpu().numpy().reshape(-1)
        e = rel_l2(got[::SUB], g["gsub." + k])
        n = abs(np.sqrt((got.astype(np.float64) ** 2).sum()) - g["gl2." + k]) / g["gl2." + k]
        worst = max(worst, e, n)
        assert e < GRAD_TOL[prec] and n < GRAD_TOL[prec], (k, e, n)
    print(f"full-size model ({prec}): worst gradient error {worst:.2e}, loss {float(loss):.6f} (ref {g['loss'][0]:.6f})")
    opt.step()  # norm 19.9 > 10: the clip is active
    tol = 1e-4 if prec == "fp32" else 5e-3
    assert abs(float(opt.last_norm[0]) - g["gnorm"][0]) < tol * g["gnorm"][0]
    assert abs(float(opt.last_norm[1]) - 10.0 / (g["gnorm"][0] + 1e-6)) < tol
    if prec != "fp32":
        return
    for k, v in m.state_dict().items():
        assert np.abs(v.cpu().numpy().reshape(-1)[::SUB] - g["psub." + k]).max() < 2e-5, k


def test_train_forward_equals_inference_forward(dev):
    """The activation-saving forward and the inference kernels are two implementations of model.py:72-136."""
    from oracle import fullsubnet_oracle as O
    args = small_args()
    sd = O.make_state_dict(seed=7, args=args)
    m = build(args, sd, dev)
    x = torch.rand(6, 1, 33, 21, device=dev)
    a = m(x)
    assert a.requires_grad and a.shape == (6, 2, 16, 21)
    m.precision = "fp32"
    with torch.no_grad():
        b = m(x)
    assert rel_max(a.detach().cpu(), b.cpu()) < 1e-5
    one = m(x[:1])  # B = 1: no drop_band (model.py:114)
    assert one.shape == (1, 2, 33, 21)
    one.sum().backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in m.parameters())
    with pytest.raises(RuntimeError):
        one.sum().backward()  # activations are released after the first backward


def test_mse_loss_kernel_matches_torch(dev):
    from fullsubnet_b200.loss import mse_loss
    torch.manual_seed(0)
    cirm = torch.randn(3, 17, 29, 2, device=dev)
    out = torch.randn(3, 2, 17, 29, device=dev, requires_grad=True)
    loss = mse_loss()(cirm, out.permute(0, 2, 3, 1))
    ref_in = out.detach().clone().requires_grad_(True)
    ref = torch.nn.functional.mse_loss(cirm, ref_in.permute(0, 2, 3, 1))
    (3.0 * loss).backward()
    (3.0 * ref).backward()
    assert abs(float(loss) - float(ref)) < 1e-6 * float(ref)
    assert torch.allclose(out.grad, ref_in.grad, rtol=1e-5, atol=1e-9)


def test_trainer_step_and_checkpoint_roundtrip(golden, dev, tmp_path):
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.optim import FusedClipAdam
    from fullsubnet_b200.trainer import Trainer
    from oracle import fullsubnet_oracle as O
    g = golden("train_small")
    args = small_args()
    sd = O.make_state_dict(seed=7, args=args, sb_fc_gain=8.0)
    cfg = {"meta": {"use_amp": False, "save_dir": str(tmp_path), "experiment_name": "t"},
           "acoustics": {"n_fft": 64, "hop_length": 32, "win_length": 64},
           "trainer": {"train": {"epochs": 2, "save_checkpoint_interval": 1, "clip_grad_norm_value": 10}}}
    data = [(torch.from_numpy(g["noisy"]), torch.from_numpy(g["clean"]))]
    m = build(args, sd, dev)
    tr = Trainer(None, 0, cfg, False, False, m, mse_loss(), FusedClipAdam(m.parameters(), lr=1e-3), data, None)
    tr.train()  # two epochs of one step each == the two golden steps
    for k, v in m.state_dict().items():
        assert np.abs(v.cpu().numpy() - g["p1." + k]).max() < 2e-5, k
    assert abs(tr.last_epoch_loss - g["loss"][1]) < 1e-5 * g["loss"][1]
    # resume: schema of base_trainer.py:208-218, optimiser state interchangeable with torch.optim.Adam
    ck = torch.load(tmp_path / "t" / "checkpoints" / "latest_model.tar", map_location="cpu")
    assert set(ck) == {"epoch", "best_score", "optimizer", "scaler", "model"} and ck["epoch"] == 2
    m2 = build(args, sd, dev)
    adam = torch.optim.Adam(m2.parameters(), lr=1e-3)
    adam.load_state_dict(ck["optimizer"])
    assert int(adam.state_dict()["state"][0]["step"]) == 2
    tr2 = Trainer(None, 0, cfg, True, False, m2, mse_loss(), FusedClipAdam(m2.parameters(), lr=1e-3), data, None)
    assert tr2.start_epoch == 3
    for k, v in m2.state_dict().items():
        assert torch.equal(v.cpu(), m.state_dict()[k].cpu())


def test_tf32_tensor_core_gemm_matches_truncated_reference(dev):
    """fsn_debug_tgemm: C (+)= A B^T on wgmma tf32 == fp64 GEMM of the tf32-truncated operands."""
    from fullsubnet_b200 import _lib
    lib = _lib.load()

    def trunc(x):
        return (x.view(torch.int32) & ~0x1FFF).view(torch.float32)
    torch.manual_seed(1)
    for (M, N, K, ld, acc, split) in ((128, 128, 32, 32, 0, 0), (200, 130, 100, 104, 0, 0), (256, 384, 1536, 1536, 1, 0),
                                     (300, 512, 70, 72, 1, 0), (1536, 64, 40000, 40000, 0, 1),
                                     # long K, 256 < N <= 384: the 128 x 384 tile of the weight-gradient GEMMs
                                     (1536, 384, 70000, 70000, 0, 1), (200, 300, 66000, 66000, 1, 1)):
        A, B = torch.randn(M, ld, device=dev), torch.randn(N, ld, device=dev)
        C0 = torch.randn(M, N + 8, device=dev)
        Cc = C0.clone()
        scratch = torch.empty(16 << 20, device=dev) if split else None
        _lib.check(lib.fsn_debug_tgemm(A.data_ptr(), ld, B.data_ptr(), ld, Cc.data_ptr(), N + 8, M, N, K, acc,
                                       _lib.ptr(scratch), scratch.numel() if split else 0,
                                       torch.cuda.current_stream().cuda_stream))
        ref = trunc(A[:, :K]).double() @ trunc(B[:, :K]).double().T + (C0[:, :N].double() if acc else 0)
        err = ((Cc[:, :N].double() - ref).abs().max() / ref.abs().max()).item()
        assert err < 1e-4, (M, N, K, err)
        assert torch.equal(Cc[:, N:], C0[:, N:])


def test_blocked_weight_gradient_gemm_matches_truncated_reference(dev):
    """fsn_debug_tgemm_blocked: C = A^T B over a long K through the block-tiled K-major copies (the dW_ih / dW_hh GEMMs of
    the training step; the k offsets are the one-step shift of dW_hh) == fp64 GEMM of the tf32-truncated operands."""
    from fullsubnet_b200 import _lib
    lib = _lib.load()

    def trunc(x):
        return (x.view(torch.int32) & ~0x1FFF).view(torch.float32)
    torch.manual_seed(2)
    for (M, N, K, a0, b0) in ((128, 128, 64, 0, 0), (1536, 33, 50000, 0, 0), (1536, 384, 70001, 64, 0), (2048, 257, 9000, 0, 0),
                              (2048, 512, 40010, 32, 0), (200, 130, 4100, 0, 96)):
        A, B = torch.randn(K + a0, M, device=dev), torch.randn(K + b0, N, device=dev)
        Cc = torch.full((M, N), float("nan"), device=dev)
        scratch = torch.empty((32 << 20) + (M + 128 + N + 128) * (K + 128), device=dev)
        _lib.check(lib.fsn_debug_tgemm_blocked(A.data_ptr(), B.data_ptr(), Cc.data_ptr(), M, N, K, a0, b0, scratch.data_ptr(),
                                               scratch.numel(), torch.cuda.current_stream().cuda_stream))
        ref = trunc(A[a0:]).double().T @ trunc(B[b0:]).double()
        err = ((Cc.double() - ref).abs().max() / ref.abs().max()).item()
        assert err < 1e-4, (M, N, K, a0, b0, err)


def test_reference_trainer_flow_ddp_autocast_gradscaler(golden, dev):
    """The reference's own optimisation flow (fullsubnet/trainer.py:56-69, base_trainer.py:32,46) on the drop-in Model:
    DistributedDataParallel (NCCL, world 1) + autocast + GradScaler + unscale_ + clip_grad_norm_ + torch.optim.Adam,
    two steps, equal to the golden steps of the unmodified reference."""
    import os
    import torch.distributed as dist
    from torch.cuda.amp import GradScaler, autocast
    from torch.nn.parallel import DistributedDataParallel
    from fullsubnet_b200.acoustics.feature import drop_band, stft
    from fullsubnet_b200.acoustics.mask import build_complex_ideal_ratio_mask
    from oracle import fullsubnet_oracle as O
    g = golden("train_small")
    args = small_args()
    core = build(args, O.make_state_dict(seed=7, args=args, sb_fc_gain=8.0), dev, "fp32")
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29541")
    created = not dist.is_initialized()
    if created:
        dist.init_process_group("nccl", rank=0, world_size=1, device_id=dev)
    try:
        model = DistributedDataParallel(core, device_ids=[0])
        optimizer = torch.optim.Adam(model.parameters(), lr=1e-3, betas=(0.9, 0.999))
        loss_function = torch.nn.MSELoss()
        scaler = GradScaler(enabled=True)
        noisy, clean = T(g["noisy"], dev), T(g["clean"], dev)
        for it in range(2):
            optimizer.zero_grad()
            noisy_mag, _, nr, ni = stft(noisy, 64, 32, 64)
            _, _, cr, ci = stft(clean, 64, 32, 64)
            cIRM = build_complex_ideal_ratio_mask(nr, ni, cr, ci)
            cIRM = drop_band(cIRM.permute(0, 3, 1, 2), model.module.num_groups_in_drop_band).permute(0, 2, 3, 1)
            with autocast(enabled=True):
                cRM = model(noisy_mag.unsqueeze(1)).permute(0, 2, 3, 1)
                loss = loss_function(cIRM, cRM)
            scaler.scale(loss).backward()
            scaler.unscale_(optimizer)
            gn = torch.nn.utils.clip_grad_norm_(model.parameters(), 10)
            scaler.step(optimizer)
            scaler.update()
            assert abs(float(loss) - g["loss"][it]) <= 1e-5 * abs(g["loss"][it]), (float(loss), g["loss"][it])
            assert abs(float(gn) - g["gnorm"][it]) < 1e-4 * g["gnorm"][it]
            if it == 0:
                for k, p in model.module.named_parameters():
                    assert rel_l2(p.grad.cpu(), g["grad." + k]) < GRAD_TOL["fp32"], k
            for k, v in model.module.state_dict().items():
                assert np.abs(v.cpu().numpy() - g[f"p{it}." + k]).max() < 2e-5, (it, k)
        # the Trainer accepts the DDP-wrapped model (no second all-reduce, checkpoints without the `module.` prefix)
        from fullsubnet_b200.trainer import Trainer
        cfg = {"meta": {"use_amp": True, "save_dir": "/tmp/fsn_t", "experiment_name": "ddp"},
               "acoustics": {"n_fft": 64, "hop_length": 32, "win_length": 64},
               "trainer": {"train": {"epochs": 1, "save_checkpoint_interval": 1, "clip_grad_norm_value": 10}}}
        tr = Trainer(dist, 0, cfg, False, False, model, loss_function, optimizer, [(g["noisy"], g["clean"])], None)
        assert tr.is_ddp and tr.core is core
        l3 = tr.train_step(torch.from_numpy(g["noisy"]), torch.from_numpy(g["clean"]))
        assert torch.isfinite(l3)
        tr._save_checkpoint(1)
        ck = torch.load("/tmp/fsn_t/ddp/checkpoints/latest_model.tar", map_location="cpu")
        assert all(not k.startswith("module.") for k in ck["model"])
    finally:
        if created:
            dist.destroy_process_group()


def test_si_sdr_kernel_matches_reference_formula(dev):
    """audio_zen/metrics.py:6-31 restated in numpy float32 vs fsn_si_sdr."""
    from fullsubnet_b200.trainer import si_sdr
    rng = np.random.default_rng(3)
    ref = rng.standard_normal((5, 64000)).astype(np.float32) * 0.1
    est = (0.7 * ref + 0.05 * rng.standard_normal((5, 64000))).astype(np.float32)
    est[4] = ref[4] * 1.5 + 1e-4 * rng.standard_normal(64000).astype(np.float32)  # high SI-SDR

    def SI_SDR(reference, estimation):
        estimation, reference = np.broadcast_arrays(estimation, reference)
        reference_energy = np.sum(reference ** 2, axis=-1, keepdims=True)
        optimal_scaling = np.sum(reference * estimation, axis=-1, keepdims=True) / reference_energy
        projection = optimal_scaling * reference
        noise = estimation - projection
        return 10 * np.log10(np.sum(projection ** 2, axis=-1) / np.sum(noise ** 2, axis=-1))
    got = si_sdr(torch.from_numpy(ref).to(dev), torch.from_numpy(est).to(dev)).cpu().numpy()
    want = SI_SDR(ref.astype(np.float64), est.astype(np.float64))
    assert np.abs(got - want).max() < 2e-3, (got, want)
    assert np.abs(got - SI_SDR(ref, est)).max() < 5e-3


def test_trainer_with_validation_loader(golden, dev, tmp_path):
    """train.py:65-80 always passes a validation dataloader: the B=1 validation loop (trainer.py:78-181) runs on the
    device (loss + enhance + SI-SDR) and its numbers equal the op-by-op evaluation of the same items."""
    from fullsubnet_b200.inferencer import Inferencer
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.optim import FusedClipAdam
    from fullsubnet_b200.trainer import Trainer, si_sdr
    from oracle import fullsubnet_oracle as O
    g = golden("train_small")
    args = small_args()
    sd = O.make_state_dict(seed=7, args=args, sb_fc_gain=8.0)
    cfg = {"meta": {"use_amp": False, "save_dir": str(tmp_path), "experiment_name": "v"},
           "acoustics": {"n_fft": 64, "hop_length": 32, "win_length": 64},
           "trainer": {"train": {"epochs": 1, "save_checkpoint_interval": 1, "clip_grad_norm_value": 10},
                       "validation": {"validation_interval": 1, "save_max_metric_score": True}}}
    noisy, clean = torch.from_numpy(g["noisy"]), torch.from_numpy(g["clean"])
    valid = [(noisy[i:i + 1], clean[i:i + 1], [f"clip{i}"], ["With_reverb" if i % 2 == 0 else "No_reverb"])
             for i in range(4)]
    m = build(args, sd, dev)
    tr = Trainer(None, 0, cfg, False, False, m, mse_loss(), FusedClipAdam(m.parameters(), lr=1e-3),
                 [(noisy, clean)], valid)
    tr.train()
    v = tr.last_validation
    assert v["items"] == {"With_reverb": 2, "No_reverb": 2} and np.isfinite(v["loss_total"])
    assert (tmp_path / "v" / "checkpoints" / "best_model.tar").exists() and tr.best_score == v["si_sdr"]["With_reverb"]
    assert m.training  # validation restores the training mode
    # same items through the Inferencer + SI-SDR, one by one
    inf = Inferencer(config={"acoustics": cfg["acoustics"]}, model=m, device=dev)
    scores = []
    for i in (0, 2):
        enh = torch.from_numpy(inf.full_band_crm_mask(noisy[i:i + 1].to(dev), {}))[None].to(dev)
        scores.append(float(si_sdr(clean[i:i + 1].to(dev), enh)[0]))
    assert abs(np.mean(scores) - v["si_sdr"]["With_reverb"]) < 1e-3


def test_snr_mix_kernels_match_reference(golden, dev):
    """fsn_rir_convolve + fsn_snr_mix vs the unmodified Dataset.snr_mix (tests/golden/mix.npz), all cases in ONE
    batched call (clips without reverberation have rir_len 0)."""
    from fullsubnet_b200.dataset import snr_mix
    g = golden("mix")
    cases = g["cases"]
    n = len(cases)
    Lr = max(int(c[2]) for c in cases)
    clean = torch.from_numpy(np.stack([g[f"c{i}_clean"] for i in range(n)])).to(dev)
    noise = torch.from_numpy(np.stack([g[f"c{i}_noise"] for i in range(n)])).to(dev)
    rir = torch.zeros(n, Lr)
    for i, c in enumerate(cases):
        if c[2]:
            rir[i, :c[2]] = torch.from_numpy(g[f"c{i}_rir"])
    noisy, clean_out = snr_mix(clean, noise, cases[:, 0].astype(np.float32), -25, cases[:, 1].astype(np.float32),
                               rir=rir.to(dev), rir_len=torch.from_numpy(cases[:, 2].astype(np.int32)))
    for i in range(n):
        assert rel_max(noisy[i].cpu(), g[f"c{i}_noisy"]) < 2e-5, i
        assert rel_max(clean_out[i].cpu(), g[f"c{i}_clean_out"]) < 2e-5, i
    # without any RIR the convolution is skipped entirely
    noisy2, _ = snr_mix(clean[:2], noise[:2], cases[:2, 0].astype(np.float32), -25, cases[:2, 1].astype(np.float32))
    assert torch.equal(noisy2, noisy[:2])


@pytest.mark.parametrize("prec", ["fp32", "tf32_tc"])
def test_cumulative_norm_training_matches_reference(golden, dev, prec):
    """norm_type="cumulative_laplace_norm" in the training step (train_cumulativeLaplaceNorm.toml:82): per-(step, clip) and
    per-(step, unit) running means in the forward, their suffix-sum backward; two golden steps of the unmodified reference,
    and the full-size architecture against CPU autograd of the oracle."""
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.optim import FusedClipAdam
    from oracle import fullsubnet_oracle as O
    from oracle import train_oracle as TO
    g = golden("train_cum_small")
    args = dict(small_args(), norm_type="cumulative_laplace_norm")
    m = build(args, O.make_state_dict(seed=7, args=args, sb_fc_gain=8.0), dev, prec)
    opt = FusedClipAdam(m.parameters(), lr=1e-3, betas=(0.9, 0.999), max_norm=10.0)
    noisy, clean = T(g["noisy"], dev), T(g["clean"], dev)
    for it in range(2):
        opt.zero_grad()
        loss, _, crm = reference_like_step(m, noisy, clean, 64, 32, mse_loss())
        assert abs(float(loss.detach()) - g["loss"][it]) <= LOSS_TOL[prec] * abs(g["loss"][it]), (it, float(loss), g["loss"][it])
        if it == 0:
            assert rel_max(crm.detach().cpu(), g["crm"]) < (1e-5 if prec == "fp32" else 1e-3)
            for k, p in m.named_parameters():
                assert rel_l2(p.grad.cpu(), g["grad." + k]) < GRAD_TOL[prec], k
        opt.step()
        if prec == "fp32":
            assert abs(float(opt.last_norm[0]) - g["gnorm"][it]) < 1e-4 * g["gnorm"][it]
            for k, v in m.state_dict().items():
                assert np.abs(v.cpu().numpy() - g[f"p{it}." + k]).max() < 2e-5, (it, k)
    if prec != "fp32":
        return
    full = dict(O.DEFAULT_MODEL_ARGS, weight_init=False, norm_type="cumulative_laplace_norm")
    sd = O.make_state_dict(seed=0, args=full, sb_fc_gain=40.0)
    ny, cl = O.make_noisy(3, 2048, seed=5, speechlike=True), 0.5 * O.make_noisy(3, 2048, seed=6)
    nm, cirm = TO.targets(ny, cl, 2)
    ref_loss, ref_grads, _ = TO.loss_and_grads(nm, cirm, sd, full)
    mf = build(full, sd, dev, "fp32")
    loss = mse_loss()(cirm.to(dev), mf(nm.unsqueeze(1).to(dev)).permute(0, 2, 3, 1))
    loss.backward()
    assert abs(float(loss.detach()) - float(ref_loss)) < 1e-5 * float(ref_loss)
    for k, p in mf.named_parameters():
        assert rel_l2(p.grad.cpu(), ref_grads[k]) < 2e-4, k


def test_packed_weight_cache_follows_fused_optimizer_steps(dev):
    """ADVICE r1 (high): FusedClipAdam writes parameters through raw pointers; the packed tensor-core image of the sub-band
    weights is cached on (data_ptr, _version), so the optimiser must bump the versions - otherwise a train -> infer flow in
    one process would enhance with stale sub-band weights.  infer, step, infer again: the tensor-core result must follow
    the fp32 kernels (which read the live parameters) both times, and must have changed."""
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.optim import FusedClipAdam
    from oracle import fullsubnet_oracle as O
    from oracle import train_oracle as TO
    args = dict(O.DEFAULT_MODEL_ARGS, weight_init=False)
    m = build(args, O.make_state_dict(seed=0, args=args, sb_fc_gain=40.0), dev, "fp32")
    y = O.make_noisy(2, 4000, seed=3, speechlike=True).to(dev)

    def both():
        m.eval()
        m.precision = "auto"
        tc = m.enhance(y, return_crm=True)[1]
        m.precision = "fp32"
        ref = m.enhance(y, return_crm=True)[1]
        m.train()
        return tc, ref
    tc0, ref0 = both()
    assert rel_max(tc0.cpu(), ref0.cpu()) < 5e-5
    opt = FusedClipAdam(m.parameters(), lr=5e-2, max_norm=10.0)  # a large step: the weights really move
    ny, cl = O.make_noisy(3, 2048, seed=5, speechlike=True), 0.5 * O.make_noisy(3, 2048, seed=6)
    nm, cirm = TO.targets(ny, cl, 2)
    loss = mse_loss()(cirm.to(dev), m(nm.unsqueeze(1).to(dev)).permute(0, 2, 3, 1))
    loss.backward()
    opt.step()
    tc1, ref1 = both()
    assert rel_max(ref1.cpu(), ref0.cpu()) > 1e-2          # the update changed the model
    assert rel_max(tc1.cpu(), ref1.cpu()) < 5e-5            # and the packed image was rebuilt from the new weights


def test_fused_lstm_forward_step_matches_float64_cell(dev):
    """fsn_debug_lstm_fwd_step (tg::lstm_fwd_step_kernel, the per-step kernel of the training forward): one nn.LSTM step
    against a float64 cell - folded input (tf32 / fp16 operands), hoisted projection already in G, first step without
    h / c, row counts off the 128-row tile, the compile-time (384, 512) and run-time (64) hidden sizes.  Tolerance:
    11-bit operand rounding of K <= 1024 products plus the MUFU activations."""
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    torch.manual_seed(11)
    cases = [  # R, H, K0, half, fold, first
        (200, 384, 32, 0, True, False), (200, 384, 32, 1, True, False), (333, 384, 384, 1, True, False),
        (64, 512, 512, 1, True, False), (130, 512, 0, 1, False, False), (130, 512, 0, 0, False, False),
        (100, 64, 16, 1, True, False), (100, 64, 16, 0, True, True), (257, 384, 32, 1, True, True),
    ]
    for (R, H, K0, half, fold, first) in cases:
        k = 1.0 / H ** 0.5
        w_hh = (torch.rand(4 * H, H, device=dev) * 2 - 1) * k
        w_ih = (torch.rand(4 * H, max(K0, 1), device=dev) * 2 - 1) * k
        b_ih, b_hh = (torch.rand(4 * H, device=dev) * 2 - 1) * k, (torch.rand(4 * H, device=dev) * 2 - 1) * k
        hp, cp = torch.rand(R, H, device=dev) * 2 - 1, torch.randn(R, H, device=dev)
        x = torch.randn(R, max(K0, 1), device=dev)
        P = torch.randn(R, 4 * H, device=dev)
        pad = 8  # rows past R must stay untouched
        G = torch.full((R + pad, 4 * H), 7.0, device=dev)
        if not fold:
            G[:R] = P
        C_out, H_out = torch.full((R + pad, H), 7.0, device=dev), torch.full((R + pad, H), 7.0, device=dev)
        scratch = torch.empty(2 * (2 * R * H + 4 * H * (H + K0) + R * K0) + 4096, dtype=torch.uint8, device=dev)
        _lib.check(lib.fsn_debug_lstm_fwd_step(None if first else hp.data_ptr(), w_hh.data_ptr(), x.data_ptr() if fold else None,
                                               w_ih.data_ptr() if fold else None, K0, G.data_ptr(), b_ih.data_ptr(),
                                               b_hh.data_ptr(), None if first else cp.data_ptr(), C_out.data_ptr(),
                                               H_out.data_ptr(), R, H, half, scratch.data_ptr(), scratch.numel(), st))
        z = (x.double() @ w_ih.double().T if fold else P.double()) + b_ih.double() + b_hh.double()
        if not first:
            z = z + hp.double() @ w_hh.double().T
        i, f, g, o = z[:, :H].sigmoid(), z[:, H:2 * H].sigmoid(), z[:, 2 * H:3 * H].tanh(), z[:, 3 * H:].sigmoid()
        c = i * g if first else f * cp.double() + i * g
        h = o * c.tanh()
        ref_g = torch.cat([i, f, g, o], dim=1)
        case = (R, H, K0, half, fold, first)
        assert (G[:R].double() - ref_g).abs().max().item() < 2e-3, case
        assert (C_out[:R].double() - c).abs().max().item() < 4e-3, case
        assert (H_out[:R].double() - h).abs().max().item() < 4e-3, case
        assert bool((G[R:] == 7.0).all()) and bool((C_out[R:] == 7.0).all()) and bool((H_out[R:] == 7.0).all()), case
