"""GPU: the tensor-core LSTM layer / Linear layer of the full-band stacks (fsn_lstm_rec_tc.cu: hoisted tf32 GEMM +
persistent wgmma recurrence) against float64 torch on the CPU (audio_zen/model/module/sequence_model.py:52-58,117).
x3 = compensated arithmetic (fp32 error class), single pass = fp16/tf32 operands (~1e-3)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _layer(dev, R, T, K, H, x3, seed=0):
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(seed)
    k = 1.0 / H ** 0.5
    w = [(torch.rand(*s, generator=g) * 2 - 1) * k for s in ((4 * H, K), (4 * H, H), (4 * H,), (4 * H,))]
    x = torch.randn(R, T, K, generator=g)
    lstm = torch.nn.LSTM(K, H, batch_first=True).double()
    with torch.no_grad():
        for p, v in zip((lstm.weight_ih_l0, lstm.weight_hh_l0, lstm.bias_ih_l0, lstm.bias_hh_l0), w):
            p.copy_(v)
        ref = lstm(x.double())[0]
    n = lib.fsn_debug_lstm_tc_workspace_bytes(R, T, K, H, x3)
    ws = torch.empty(n, dtype=torch.uint8, device=dev)
    d = [t.to(dev).contiguous() for t in w + [x]]
    outs = []
    for _ in range(2):
        out = torch.full((R, T, H), float("nan"), device=dev)
        _lib.check(lib.fsn_debug_lstm_layer_tc(*[t.data_ptr() for t in d], R, T, K, H, x3, out.data_ptr(), ws.data_ptr(), n,
                                               torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        outs.append(out.cpu())
    assert torch.equal(outs[0], outs[1]), "run-to-run difference"  # fixed-order arithmetic, no atomics in the data path
    return float((outs[0].double() - ref).abs().max())


@pytest.mark.parametrize("R,T,K,H", [(2, 26, 64, 384), (3, 253, 384, 257), (256, 60, 257, 512), (300, 12, 128, 512),
                                     (1, 9, 33, 64), (130, 5, 100, 200)])
def test_lstm_layer_tc_matches_float64(dev, R, T, K, H):
    """Rows beyond one 128-row group, partial groups, partial unit slices (H % 8 != 0), odd strides, launch chunking."""
    e3, e1 = _layer(dev, R, T, K, H, 1), _layer(dev, R, T, K, H, 0)
    print(f"lstm_layer_tc R={R} T={T} K={K} H={H}: max-abs error x3 {e3:.1e}, single pass {e1:.1e}")
    assert e3 < 5e-6 and e1 < 3e-3


@pytest.mark.parametrize("rows,K,N,act", [(52, 257, 64, 1), (506, 512, 514, 0), (64768, 512, 257, 1), (1000, 257, 2048, 0)])
def test_linear_tc_matches_float64(dev, rows, K, N, act):
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(rows + K + N)
    x, W, b = torch.randn(rows, K, generator=g), torch.randn(N, K, generator=g) / K ** 0.5, torch.randn(N, generator=g)
    ref = x.double() @ W.double().T + b.double()
    if act:
        ref = ref.clamp_min(0)
    Hm = max(8, (N + 3) // 4)
    for x3, tol in ((1, 5e-6), (0, 3e-3)):
        n = lib.fsn_debug_lstm_tc_workspace_bytes(rows, 1, K, Hm, x3)
        ws = torch.empty(n, dtype=torch.uint8, device=dev)
        out = torch.full((rows, N), float("nan"), device=dev)
        xd, Wd, bd = x.to(dev), W.to(dev), b.to(dev)
        _lib.check(lib.fsn_debug_linear_tc(xd.data_ptr(), rows, K, Wd.data_ptr(), bd.data_ptr(), N, act, x3, out.data_ptr(),
                                           ws.data_ptr(), n, torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        e = (out.cpu().double() - ref)
        assert float(e.norm() / ref.norm()) < tol, (x3, float(e.norm() / ref.norm()))


def test_unsupported_hidden_size_is_reported(dev):
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    z = torch.zeros(16, device=dev)
    with pytest.raises(NotImplementedError):
        _lib.check(lib.fsn_debug_lstm_layer_tc(z.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(), 1, 2, 4, 8,
                                               1, z.data_ptr(), z.data_ptr(), 64, torch.cuda.current_stream().cuda_stream))
