"""The CTA-pair split of the sub-band tensor-core LSTM stack (`sb_lstm_tc_kernel<X3>`, fsn_subband_tc.cu): CTA `half`
of a pair owns hidden units [H/2 half, H/2 (half + 1)) of the same 32 rows and receives the other half's h over DSMEM;
half 1 sends its Linear sums to half 0.  Checked against the float64 statement of test_gpu_subband_tc.py, with its
tolerances, where its matrix cannot reach:

* starved halves: the output is made by one half's units only, and those are driven only by the h that the OTHER
  half sends across (a dropped, stale or misplaced exchange, or a lost Linear partial, changes the output);
* the headline length: H = 384, F = 257, 253 steps, 2 clips (514 rows: 17 pairs, the last one partly padded), every
  row, so that every barrier phase of the exchange wraps many times; clusters of 1, 2 and 4 pairs give the same bits.
"""
import numpy as np
import pytest
import torch

from test_gpu_subband_tc import TOLERANCES, _case, _inputs, _launch, _row_map, _weights, gather, stack


def _run(dev, c, w, configs):
    """Every config of `configs` [(cluster, stages)] in both arithmetics: identical bits across configs, error of all
    rows against float64 within the module tolerances.  Returns {x3: error}."""
    Ksb = (2 * c["Ns"] + 1) + (2 * c["Nf"] + 1)
    assert w["weight_ih_l0"].shape[1] == Ksb
    seed = sum(map(ord, c["name"]))
    magT, fbT, inv2, unit, _ = _inputs(c, seed)
    _, Fsub, _, _ = _row_map(c["B"], c["F"], c["G"])
    rows = np.arange(c["B"] * Fsub)
    x = gather(magT.double(), fbT.double(), inv2.double(), None, c["Ns"], c["Nf"], c["G"], c["steps"], c["shrink"],
               rows)
    ref = stack(x, {k: v.double() for k, v in w.items()}, c["act"], c["la"])  # [R, fc_out, T]
    wd = {k: v.to(dev).contiguous() for k, v in w.items()}
    d_in = [None if t is None else t.to(dev).contiguous() for t in (magT, fbT, inv2, unit)]
    scale = max(1.0, float(ref.abs().max()))
    errs = {}
    for x3 in (1, 0):
        outs = [_launch(dev, c, wd, d_in, x3, st, cl) for cl, st in configs]
        for (cl, st), o in zip(configs, outs):
            assert torch.equal(o, outs[0]), f"{c['name']}: cluster {cl}, stages {st} differ from {configs[0]}"
        r = torch.as_tensor(rows)
        got = outs[0][r // Fsub, :c["fc_out"], r % Fsub].double()
        err = float((got - ref).abs().max()) / scale
        print(f"{c['name']} {'x3' if x3 else 'single pass'}: error {err:.2e} (scale {scale:.3g}, {len(rows)} rows)")
        assert err < TOLERANCES[(x3, c["H"])], (c["name"], x3, err)
        errs[x3] = err
    return errs


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 384])
@pytest.mark.parametrize("starved", [0, 1])
def test_starved_half_is_driven_by_the_peer(dev, H, starved):
    """The Linear weights of half `starved`'s units are zero, and so are the recurrent and layer-1 input columns that
    read the other half's units.  The output is then made by the other half's units alone, and their only input
    besides x_t is the h that half `starved` sends across.  Both the exchange of h0 and h1 and the Linear sums of
    half 1 (when it is the driven half) are on the path of every output."""
    c = _case(f"starve{starved}_h{H}", H=H, B=3, F=33, G=2, steps=12, la=2, Ns=15, Nf=0, act=0, weights="gain").values[0]
    w = _weights(H, 32, 2, "gain", sum(map(ord, c["name"])))
    own = slice(starved * H // 2, (starved + 1) * H // 2)  # units of the starved half
    other = slice((1 - starved) * H // 2, (2 - starved) * H // 2)
    w["fc_w"][:, own] = 0
    for name in ("weight_hh_l0", "weight_ih_l1", "weight_hh_l1"):
        w[name][:, other] = 0
    errs = _run(dev, c, w, [(1, 4), (2, 3), (4, 2)])
    assert errs[1] < TOLERANCES[(1, H)]


@pytest.mark.gpu
def test_headline_length_all_rows_every_cluster(dev):
    """H = 384, F = 257, 253 steps (4 s clips plus the look-ahead), 2 clips: 514 rows in 17 pairs, the last one with 30
    padding rows; all rows against float64 and the same bits for clusters of 1, 2 and 4 pairs."""
    c = _case("headline", H=384, B=2, F=257, G=1, steps=253, la=2, Ns=15, Nf=0, act=0).values[0]
    w = _weights(384, 32, 2, "std", sum(map(ord, c["name"])))
    _run(dev, c, w, [(1, 4), (2, 4), (4, 4), (2, 3)])
