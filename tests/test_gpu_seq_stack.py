"""The SequenceModel every inference forward runs its clip-major LSTM stacks through (seq_stack_forward, fsn_fullband.cu;
audio_zen/model/module/sequence_model.py:106-125) through its unit-test hook `fsn_debug_seq_stack`, against one float64
torch.nn.LSTM (or nn.GRU) per layer on the CPU, the layer-0 input scaled per clip (scale[r]) or per step and clip
(scale[t*R + r], the cumulative norm), then the Linear and its activation.

Each case asserts the path the hook reports, computed here from the device's SM count and opt-in shared memory:
  tc          lstm_layer_tc per layer (tf32 GEMM + wgmma recurrence; x3 or single pass) and linear_tc
  persistent  layers 0-1 on fb_lstm_kernel (weights in shared memory, one grid barrier per step), the rest per step
  step2       layers 0-1 as two per-step launches per step (lstm_step2_launch), the rest per step
  one_layer   one layer on the per-step kernel
and checks:
  * max-abs error / max(1, max|ref|) against float64, within the bound of its arithmetic (TOL);
  * every output element written (out starts as NaN) and the guard floats past out untouched;
  * two runs give the same bits;
  * batch invariance: a row that repeats another row's sequence (and scale) gives that row's bits, including a copy in
    another 64-row tile and one across the persistent kernel's 256-row chunks; a call with R = 1 on that row alone
    gives the same bits on the same path.

Worst errors measured on an H100 80GB HBM3 at a 700 W power limit (132 SMs, 227 KB opt-in shared memory; seeded
inputs, deterministic kernels, so the numbers repeat):

    fp32 kernels (persistent, step2, one_layer)   1.2e-6   (saturating_stepwise; 4.1e-7 without saturated gates)
    tensor cores, x3                              2.1e-6   (tc_x3)
    tensor cores, single pass                     3.0e-4   (tc_single_zero_copy)

TOL sits about 4x above these.
"""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

PATHS = {0: "tc", 1: "persistent", 2: "step2", 3: "one_layer"}  # FSN_SEQ_PATH_*
ACTS = {"none": 0, "relu": 1, "tanh": 2, "relu6": 3}
TOL = {"fp32": 5e-6, "x3": 8.5e-6, "single": 1.2e-3}
GUARD = 64  # 7.0 floats past out
PERSISTENT_RING_BYTES = 5 * 256 * 20 * 4  # fb_lstm_kernel's A-tile ring; weights take (K0 + 2 H0 + H1) * 64 B next to it


def _case(n, H, R, Tp, K0, O, act, gru=False, step_scale=False, scale=True, tc=False, x3=False, force=False, wgain=1.0,
          xgain=1.0, fc_gain=1.0):
    return dict(n=n, H=H, R=R, Tp=Tp, K0=K0, O=O, act=act, gru=gru, step_scale=step_scale, scale=scale, tc=tc, x3=x3,
                force=force, wgain=wgain, xgain=xgain, fc_gain=fc_gain)


def _kmax(d):
    """largest K0 for which a 512/512 stack still fits the persistent kernel's shared memory"""
    return (d["optin"] - PERSISTENT_RING_BYTES) // 64 - 3 * 512


# H and K0 may depend on the device (d: sms, optin).  Relu6 cases scale the Linear so that outputs pass 6.
CASES = {
    "fullsubnet": _case(2, 512, 3, 40, 257, 257, "relu"),                      # upc 4, per-clip scale
    "row_chunks": _case(2, 64, 513, 5, 33, 40, "tanh"),                        # three 256-row launches
    "h40_scalar_loader": _case(2, 40, 37, 9, 17, 17, "relu6", fc_gain=30.0),   # H % 16 != 0, upc 1
    "uneven_layers": _case(2, (384, 257), 5, 12, 64, 64, "relu"),              # fast_fullsubnet encoder, idle units
    "upc_remainder": _case(2, lambda d: 2 * d["sms"] + 1, 4, 6, 24, 16, "none"),  # upc 3, short last CTA
    "tp1": _case(2, 96, 6, 1, 20, 12, "tanh"),                                 # one- and two-phase wavefront
    "tp2": _case(2, 96, 6, 2, 20, 12, "relu"),
    "smem_fits": _case(2, 512, 2, 4, _kmax, 8, "none"),
    "smem_over": _case(2, 512, 2, 4, lambda d: _kmax(d) + 1, 8, "none"),
    "sm_fits": _case(2, lambda d: 4 * d["sms"], 2, 5, 32, 8, "tanh"),
    "sm_over": _case(2, lambda d: 4 * d["sms"] + 8, 2, 5, 32, 8, "tanh"),
    "fullsubnet_forced_stepwise": _case(2, 512, 3, 40, 257, 257, "relu", force=True),
    "one_layer": _case(1, 512, 3, 20, 257, 514, "none"),                       # fullband_baseline, num_layers 1
    "fbb_three_layers": _case(3, 512, 2, 16, 257, 514, "relu"),                # persistent + one per-step layer
    # hall ping-pong of both parities; deeper stacks take larger weights so that the input still reaches the output
    "depth4": _case(4, 48, 5, 7, 20, 10, "tanh", wgain=2.0),
    "depth8_cum": _case(8, 32, 3, 6, 16, 6, "none", step_scale=True, wgain=3.0),
    "cum_norm": _case(2, 512, 3, 24, 257, 257, "relu", step_scale=True),       # row_scale = scale + t*R
    "cum_norm_tc": _case(2, 512, 3, 24, 257, 257, "relu", step_scale=True, tc=True, x3=True),  # split_tf32 scale_B = R
    "gru_one_layer": _case(1, 48, 5, 10, 24, 24, "tanh", gru=True),
    "gru_two_layers": _case(2, 48, 70, 10, 24, 20, "relu6", gru=True, fc_gain=30.0),  # two 64-row tiles
    "tc_x3": _case(2, 512, 300, 6, 257, 257, "relu", tc=True, x3=True),        # copied operand, recurrence row chunks
    "tc_single_zero_copy": _case(2, 512, 4, 16, 256, 514, "none", scale=False, tc=True),
    "tc_uneven_x3": _case(2, (384, 257), 5, 12, 64, 64, "relu", tc=True, x3=True),  # fast_fullsubnet encoder
    "tc_decoder_single": _case(2, 512, 4, 12, 128, 514, "none", tc=True),      # fast_fullsubnet decoder
    "saturating": _case(2, 64, 6, 12, 32, 16, "tanh", wgain=4.0, xgain=20.0),  # sigmoid / tanh saturation
    "saturating_stepwise": _case(2, 64, 70, 12, 32, 16, "tanh", force=True, wgain=4.0, xgain=20.0),
}
BOUNDARIES = (("smem_fits", "smem_over"), ("sm_fits", "sm_over"))


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def dims(dev):
    p = torch.cuda.get_device_properties(dev)
    return {"sms": p.multi_processor_count, "optin": p.shared_memory_per_block_optin}


def resolve(name, d):
    c = dict(CASES[name])
    H = c["H"](d) if callable(c["H"]) else c["H"]
    c["H"] = tuple(H) if isinstance(H, tuple) else (H,) * c["n"]
    c["K0"] = c["K0"](d) if callable(c["K0"]) else c["K0"]
    return c


def expected_path(c, d):
    if c["tc"] and not c["force"]:
        return "tc"
    if c["n"] == 1:
        return "one_layer"
    H0, H1 = c["H"][:2]
    fits = (c["K0"] + 2 * H0 + H1) * 64 + PERSISTENT_RING_BYTES <= d["optin"] and math.ceil(max(H0, H1) / 4) <= d["sms"]
    return "persistent" if fits and not (c["gru"] or c["step_scale"] or c["force"]) else "step2"


def copies(R):
    """(row, row it repeats): the last row, one in another 64-row tile, one across the persistent kernel's 256-row chunks"""
    pairs = [(R - 1, 0)] if R > 1 else []
    if R > 66:
        pairs.append((65, 1))
    if R > 300:
        pairs.append((300, 2))
    return pairs


def make_inputs(name, c):
    n, Hs, R, Tp, K0, O = c["n"], c["H"], c["R"], c["Tp"], c["K0"], c["O"]
    g = torch.Generator().manual_seed(sum(map(ord, name)))

    def u(k, *shape):
        return (torch.rand(*shape, generator=g) * 2 - 1) * k

    G = 3 if c["gru"] else 4
    w, kin = [], K0
    for H in Hs:
        k = 1.0 / H ** 0.5
        w.append([u(k, G * H, kin) * c["wgain"], u(k, G * H, H) * c["wgain"], u(k, G * H) * c["wgain"], u(k, G * H) * c["wgain"]])
        kin = H
    k = 1.0 / Hs[-1] ** 0.5
    fc_w, fc_b = u(k, O, Hs[-1]) * c["fc_gain"], u(k, O) * c["fc_gain"]
    mag = torch.exp(1.2 * torch.randn(R, Tp, K0, generator=g))  # nonnegative, heavy-tailed, like a magnitude
    for dst, src in copies(R):
        mag[dst] = mag[src]
    scale = None
    if c["scale"]:
        frame = mag.double().mean(2)  # [R, Tp]
        if c["step_scale"]:  # causal running mean (cumulative_laplace_norm), time-major [Tp, R]
            run = frame.cumsum(1) / torch.arange(1, Tp + 1, dtype=torch.float64)
            scale = (1.0 / (run + 1e-5)).T.contiguous()
        else:
            scale = 1.0 / (frame.mean(1) + 1e-5)
        scale = (scale * c["xgain"]).float()
    return w, mag, scale, fc_w, fc_b


def reference(c, w, mag, scale, fc_w, fc_b):
    x = mag.double()
    if scale is not None:
        x = x * (scale.double().T[:, :, None] if c["step_scale"] else scale.double()[:, None, None])
    kin = c["K0"]
    with torch.no_grad():
        for H, lw in zip(c["H"], w):
            mod = (torch.nn.GRU if c["gru"] else torch.nn.LSTM)(kin, H, batch_first=True).double()
            for p, v in zip((mod.weight_ih_l0, mod.weight_hh_l0, mod.bias_ih_l0, mod.bias_hh_l0), lw):
                p.copy_(v.double())
            x = mod(x)[0]
            kin = H
        y = x @ fc_w.double().T + fc_b.double()
    act = c["act"]
    if act == "relu":
        y = y.clamp_min(0)
    elif act == "tanh":
        y = torch.tanh(y)
    elif act == "relu6":
        y = y.clamp(0, 6)
    return y


def run_hook(c, w, mag, scale, fc_w, fc_b, dev):
    """One fsn_debug_seq_stack call -> (out [R, Tp, O] on the CPU, path); every element written, guard untouched."""
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    n, R, Tp, K0, O = c["n"], mag.shape[0], c["Tp"], c["K0"], c["O"]
    wd = [[t.to(dev).contiguous() for t in lw] for lw in w]
    layers = (_lib.LstmLayer * n)(*[_lib.LstmLayer(*[t.data_ptr() for t in lw]) for lw in wd])
    Hs = (C.c_int * n)(*c["H"])
    xd, fcw, fcb = mag.to(dev).contiguous(), fc_w.to(dev), fc_b.to(dev)
    sd = scale.to(dev).contiguous() if scale is not None else None
    flags = [int(c["gru"]), int(c["step_scale"]), int(c["tc"]), int(c["x3"])]
    nbytes = _lib.check_workspace(lib.fsn_debug_seq_stack_workspace_bytes(n, Hs, R, Tp, K0, *flags, O))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    numel = R * Tp * O
    out = torch.full((numel + GUARD,), float("nan"), device=dev)
    out[numel:] = 7.0
    path = C.c_int(-1)
    _lib.check(lib.fsn_debug_seq_stack(layers, n, Hs, R, Tp, K0, *flags, int(c["force"]), xd.data_ptr(), _lib.ptr(sd),
                                       fcw.data_ptr(), fcb.data_ptr(), O, ACTS[c["act"]], out.data_ptr(), ws.data_ptr(), nbytes,
                                       C.byref(path), torch.cuda.current_stream(dev).cuda_stream))
    torch.cuda.synchronize(dev)
    out = out.cpu()
    assert bool((out[numel:] == 7.0).all()), "guard overwritten"
    assert bool(torch.isfinite(out[:numel]).all()), "element not written"
    return out[:numel].view(R, Tp, O), PATHS[path.value]


def _bits(t):
    return t.contiguous().view(torch.int32)


def test_cases_cover_every_path(dims):
    """Every path is asserted by some case, and each boundary pair has one case on each side of its rule."""
    paths = {name: expected_path(resolve(name, dims), dims) for name in CASES}
    assert set(paths.values()) == set(PATHS.values()), paths
    for a, b in BOUNDARIES:
        assert (paths[a], paths[b]) == ("persistent", "step2"), (a, b, paths[a], paths[b])


@pytest.mark.parametrize("name", list(CASES))
def test_seq_stack_matches_float64(dev, dims, name):
    c = resolve(name, dims)
    assert c["K0"] > 0, (name, "no K0 fits the persistent kernel on this device")
    want = expected_path(c, dims)
    w, mag, scale, fc_w, fc_b = make_inputs(name, c)
    got, path = run_hook(c, w, mag, scale, fc_w, fc_b, dev)
    assert path == want, (name, path, want)
    again, _ = run_hook(c, w, mag, scale, fc_w, fc_b, dev)
    assert torch.equal(_bits(got), _bits(again)), (name, "two runs differ")
    for dst, src in copies(c["R"]):
        assert torch.equal(_bits(got[dst]), _bits(got[src])), (name, dst, src, "a repeated row differs")
        one = None if scale is None else (scale[:, src:src + 1] if c["step_scale"] else scale[src:src + 1])
        alone, p1 = run_hook(c, w, mag[src:src + 1], one, fc_w, fc_b, dev)
        assert p1 == path and torch.equal(_bits(alone[0]), _bits(got[src])), (name, src, "differs when run alone")
    ref = reference(c, w, mag, scale, fc_w, fc_b)
    diff = (got.double() - ref).abs()
    err = diff.max().item() / max(1.0, ref.abs().max().item())
    kind = ("x3" if c["x3"] else "single") if path == "tc" else "fp32"
    i, Tp, O = int(diff.argmax()), c["Tp"], c["O"]
    r, t, o = i // (Tp * O), (i // O) % Tp, i % O  # row, step, output of the worst element
    print(f"seq_stack {name}: path {path}, H {c['H']}, K0 {c['K0']}, max-abs error {err:.2e} at row {r} step {t} out {o}")
    assert err < TOL[kind], (name, path, kind, err, (r, t, o))
