"""The LSTM layer shared by the three training steps (fsn_train.cu: layer_forward, layer_bwd_transpose_weights, stack_bwd,
layer_weight_grads) through its unit-test hook `fsn_debug_lstm_train`, against torch.nn.LSTM(K0, H, num_layers=n) in
float64 under autograd.  The loss is  sum(h_top * dh_top) + sum((h_top W_fc^T) * dout),  so one backward gives h_top,
dx and all 4n gradients.

Every case runs in fp32 and in tf32_tc, and checks:
  * end to end: rel-L2 and max-abs / max(1, max|ref|) of h_top, dx and every gradient against float64;
  * per GEMM, from the kernel's own operands (the hook's trace of H and dG): dW_ih = dG^T X, dW_hh = dG[1:]^T H[:-1],
    dx = dG_0 W_ih recomputed in float64 (tf32-truncated operands where the GEMM runs on the tensor cores), and
    b_ih = b_hh = column sums of dG.  These catch a dropped k block or a shifted step that the end-to-end bound hides;
  * every output element is written (outputs start as NaN) and guard floats (7.0) past each output stay untouched;
  * two runs give the same bits, and a row that repeats row 0's sequence gives row 0's h_top and dx bits;
  * a tf32_tc run whose layers fall back to the fp32 kernels gives the fp32 run's bits.

Worst errors measured on an H100 80GB HBM3 at a 700 W power limit (inputs are seeded and every kernel is
deterministic, so the numbers repeat), over all cases; a tf32_tc request whose layers run the fp32 kernels counts as
fp32:

                                  fp32       tf32_tc
    end to end, up to 4 layers    1.4e-6     3.0e-3   (depth4, dx)
    end to end, 8 layers          5.9e-7     6.2e-3
    per GEMM                      1.4e-6     1.4e-5   (6 144-row dW without split-K)
    bias column sums              1.8e-7     3.2e-7

TOL sits about 4x above these.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

PRECISIONS = ("fp32", "tf32_tc")
TOL = {  # effective precision of the layers -> bound (module docstring); "e2e_deep": stacks of more than 4 layers
    "fp32": {"e2e": 5.5e-6, "e2e_deep": 5.5e-6, "gemm": 5.5e-6, "bias": 8e-7},
    "tf32_tc": {"e2e": 1.4e-2, "e2e_deep": 2.5e-2, "gemm": 6e-5, "bias": 1.3e-6},
}
GUARD = 64  # 7.0 floats past every output

# name -> (n_layers, R, T, K0, H, top gradient, O, dx, weight scale), and the branch it reaches
CASES = {
    "simt_gates_odd_k0": (2, 3, 7, 33, 24, "both", 2, True, 1.0),    # SIMT step kernel with gate saving, sgemm BPTT
    "h257_fp32_rule": (2, 5, 4, 20, 257, "dh", 0, True, 1.0),        # tf32_layer: H % 4 != 0 -> fp32 kernels
    "one_step_one_row": (1, 1, 1, 32, 64, "dh", 0, True, 1.0),       # T = 1: dW_hh memset, first step only
    "r31_second_dg_copy": (2, 31, 6, 20, 64, "dh", 0, True, 1.0),    # R % 32 != 0; fold without / with the fp16 input
    "r32_kblock_offset": (2, 32, 6, 20, 64, "dh", 0, False, 1.0),    # R % 32 == 0: dW_hh by a k-block offset
    "h384_two_row_tiles": (3, 129, 5, 257, 384, "fc", 1, False, 1.0),  # HT = 384, hoisted SIMT projection (K0 odd)
    "h512_wide_input": (2, 64, 4, 1024, 512, "dh", 0, False, 1.0),   # HT = 512, K0 > 512: hoisted tgemm, plain cell
    "depth4": (4, 3, 9, 33, 96, "both", 1, True, 1.0),               # both dh_mid buffers, both parities; generic HT
    "depth8": (8, 2, 4, 16, 32, "dh", 0, True, 1.0),
    "h36_unfused": (2, 4, 5, 24, 36, "fc", 2, True, 1.0),            # H % 32 != 0: per-step tgemm + cell kernel
    "split_k_tf32": (1, 160, 64, 40, 64, "dh", 0, False, 1.0),       # 10 240 rows: split-K, several colsum slabs
    "split_k_sgemm": (1, 96, 64, 40, 64, "dh", 0, False, 1.0),       # 6 144 rows: sgemm split-K + reduce
    "three_row_tiles": (2, 300, 3, 33, 128, "dh", 0, True, 1.0),     # dx tgemm with an odd ldc
    "saturating": (2, 8, 10, 24, 64, "both", 2, True, 4.0),          # gate derivatives near 0
}


def _trunc(x):
    return (x.view(torch.int32) & ~0x1FFF).view(torch.float32)


def _inputs(name):
    n, R, T, K0, H, top, O, dx, scale = CASES[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    k = 1.0 / H ** 0.5

    def u(*shape):
        return (torch.rand(*shape, generator=g) * 2 - 1) * k

    w = []
    for l in range(n):
        kin = K0 if l == 0 else H
        w.append([u(4 * H, kin) * scale, u(4 * H, H) * scale, u(4 * H) * scale, u(4 * H) * scale])
    x = torch.randn(T, R, K0, generator=g)
    dh = torch.randn(T, R, H, generator=g) if top in ("dh", "both") else None
    dout = torch.randn(T, R, O, generator=g) if O else None
    fc_w = u(O, H) if O else None
    for t in (x, dh, dout):  # the last row repeats row 0's sequence
        if t is not None:
            t[:, R - 1] = t[:, 0]
    return w, x, dh, dout, fc_w


def _reference(name, w, x, dh, dout, fc_w):
    n, R, T, K0, H = CASES[name][:5]
    lstm = torch.nn.LSTM(K0, H, num_layers=n).double()
    with torch.no_grad():
        for l in range(n):
            for p, v in zip(("weight_ih", "weight_hh", "bias_ih", "bias_hh"), w[l]):
                getattr(lstm, f"{p}_l{l}").copy_(v.double())
    xd = x.double().requires_grad_(True)
    h, _ = lstm(xd)
    loss = 0
    if dh is not None:
        loss = loss + (h * dh.double()).sum()
    if dout is not None:
        loss = loss + ((h @ fc_w.double().T) * dout.double()).sum()
    loss.backward()
    grads = [[getattr(lstm, f"{p}_l{l}").grad for p in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")] for l in range(n)]
    return h.detach(), xd.grad, grads


def _out(numel, dev):
    buf = torch.full((numel + GUARD,), float("nan"), device=dev)
    buf[numel:] = 7.0
    return buf


def run_hook(name, prec, w, x, dh, dout, fc_w, dev):
    """One fsn_debug_lstm_train call; checks that every output element was written and no guard float was touched."""
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    n, R, T, K0, H, top, O, want_dx, _ = CASES[name]
    wd = [[t.to(dev) for t in lw] for lw in w]
    xd = x.to(dev)
    dhd = dh.to(dev) if dh is not None else None
    doutd, fcd = (dout.to(dev), fc_w.to(dev)) if O else (None, None)
    layers = (_lib.LstmLayer * n)(*[_lib.LstmLayer(*[t.data_ptr() for t in lw]) for lw in wd])
    sizes = {"h_top": T * R * H, "trace": n * 5 * T * R * H}
    if want_dx:
        sizes["dx"] = T * R * K0
    for l in range(n):
        kin = K0 if l == 0 else H
        sizes.update({f"w_ih{l}": 4 * H * kin, f"w_hh{l}": 4 * H * H, f"b_ih{l}": 4 * H, f"b_hh{l}": 4 * H})
    bufs = {k: _out(v, dev) for k, v in sizes.items()}
    grads = (_lib.LstmGrads * n)(*[_lib.LstmGrads(*[bufs[f"{p}{l}"].data_ptr() for p in ("w_ih", "w_hh", "b_ih", "b_hh")])
                                   for l in range(n)])
    nbytes = lib.fsn_debug_lstm_train_workspace_bytes(n, R, T, K0, H, _lib.PREC[prec])
    ws = torch.empty(_lib.check_workspace(nbytes), dtype=torch.uint8, device=dev)
    _lib.check(lib.fsn_debug_lstm_train(layers, n, R, T, K0, H, _lib.PREC[prec], xd.data_ptr(), _lib.ptr(dhd), _lib.ptr(doutd),
                                        _lib.ptr(fcd), O, bufs["h_top"].data_ptr(), _lib.ptr(bufs.get("dx")), grads,
                                        bufs["trace"].data_ptr(), ws.data_ptr(), nbytes,
                                        torch.cuda.current_stream(dev).cuda_stream))
    torch.cuda.synchronize(dev)
    out = {}
    for k, b in bufs.items():
        b = b.cpu()
        assert bool((b[sizes[k]:] == 7.0).all()), (name, prec, k, "guard overwritten")
        assert bool(torch.isfinite(b[:sizes[k]]).all()), (name, prec, k, "element not written")
        out[k] = b[:sizes[k]]
    return out


def _err(got, ref):
    got, ref = got.double().reshape(ref.shape), ref.double()
    rl2 = ((got - ref).norm() / max(ref.norm().item(), 1e-30)).item()
    mabs = ((got - ref).abs().max() / max(1.0, ref.abs().max().item())).item()
    return max(rl2, mabs)


def measure(name, prec, dev):
    """Runs one case; asserts the bit-level properties and returns the worst error of each kind (module docstring)."""
    n, R, T, K0, H, top, O, want_dx, _ = CASES[name]
    w, x, dh, dout, fc_w = _inputs(name)
    got = run_hook(name, prec, w, x, dh, dout, fc_w, dev)
    again = run_hook(name, prec, w, x, dh, dout, fc_w, dev)
    for k in got:
        assert torch.equal(got[k].view(torch.int32), again[k].view(torch.int32)), (name, prec, k, "two runs differ")
    tc = prec == "tf32_tc" and H % 4 == 0  # the layers on the tensor cores: forward, BPTT and weight gradients alike
    if prec == "tf32_tc" and not tc:  # every layer on the fp32 kernels: the fp32 run, bit for bit
        f32 = run_hook(name, "fp32", w, x, dh, dout, fc_w, dev)
        for k in got:
            assert torch.equal(got[k].view(torch.int32), f32[k].view(torch.int32)), (name, k, "differs from the fp32 run")
    h_top = got["h_top"].view(T, R, H)
    if R > 1:  # row R-1 repeats row 0
        assert torch.equal(h_top[:, 0].view(torch.int32), h_top[:, R - 1].view(torch.int32)), (name, prec, "h_top rows")
        if want_dx:
            dxv = got["dx"].view(T, R, K0)
            assert torch.equal(dxv[:, 0].view(torch.int32), dxv[:, R - 1].view(torch.int32)), (name, prec, "dx rows")

    ref_h, ref_dx, ref_g = _reference(name, w, x, dh, dout, fc_w)
    e2e = {"h_top": _err(got["h_top"], ref_h)}
    if want_dx:
        e2e["dx"] = _err(got["dx"], ref_dx)
    for l in range(n):
        for p, r in zip(("w_ih", "w_hh", "b_ih", "b_hh"), ref_g[l]):
            e2e[f"{p}{l}"] = _err(got[f"{p}{l}"], r)

    # per GEMM, from the kernel's own operands
    def op(t, on):
        return (_trunc(t) if on else t).double()

    def rel(a, r):
        return ((a.double() - r).abs().max() / max(r.abs().max().item(), 1e-30)).item()

    gemm, bias = {}, {}
    tr = got["trace"].view(n, 5 * T * R * H)
    Hs = [tr[l, :T * R * H].view(T * R, H) for l in range(n)]
    dG = [tr[l, T * R * H:].view(T * R, 4 * H) for l in range(n)]
    for l in range(n):
        X = x.reshape(T * R, K0) if l == 0 else Hs[l - 1]
        kin = X.shape[1]
        gemm[f"w_ih{l}"] = rel(got[f"w_ih{l}"].view(4 * H, kin), op(dG[l], tc).T @ op(X, tc))
        g_hh = got[f"w_hh{l}"].view(4 * H, H)
        if T > 1:
            gemm[f"w_hh{l}"] = rel(g_hh, op(dG[l][R:], tc).T @ op(Hs[l][:-R], tc))
        else:
            assert bool((g_hh == 0).all()), (name, prec, l, "dW_hh of one step must be zero")
        assert torch.equal(got[f"b_ih{l}"].view(torch.int32), got[f"b_hh{l}"].view(torch.int32)), (name, prec, l, "b_ih != b_hh")
        d = dG[l].double()
        bias[f"b{l}"] = ((got[f"b_ih{l}"].double() - d.sum(0)).abs() / d.abs().sum(0).clamp_min(1e-30)).max().item()
    if want_dx:  # dx of each step from the same dG: the BPTT GEMM of layer 0 (tensor cores when the layer is)
        gemm["dx"] = rel(got["dx"].view(T * R, K0), op(dG[0], tc) @ op(w[0][0], tc))
    return {"e2e": e2e, "gemm": gemm, "bias": bias, "eff": "tf32_tc" if tc else "fp32"}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("prec", PRECISIONS)
def test_lstm_stack_matches_float64(dev, prec, name):
    m = measure(name, prec, dev)
    tol = dict(TOL[m["eff"]])
    if CASES[name][0] > 4:
        tol["e2e"] = tol["e2e_deep"]
    for kind in ("e2e", "gemm", "bias"):
        worst = max(m[kind].items(), key=lambda kv: kv[1]) if m[kind] else ("-", 0.0)
        assert worst[1] < tol[kind], (name, prec, kind, worst, m[kind])
