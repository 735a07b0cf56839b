"""Diagnostic (GPU): compare the tensor-core sub-band path against the fp32 path on a tiny case."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from fullsubnet_b200.fullsubnet.model import Model
from fullsubnet_b200.acoustics.feature import stft
from oracle import fullsubnet_oracle as O

dev = torch.device("cuda:0")
B, L = int(sys.argv[1]) if len(sys.argv) > 1 else 1, int(sys.argv[2]) if len(sys.argv) > 2 else 2000
sd = O.make_state_dict(0)
y = O.make_noisy(B, L, seed=5, speechlike=True).to(dev)
outs = {}
for prec in ("fp32", "f16_tc"):
    m = Model(**dict(O.DEFAULT_MODEL_ARGS, num_groups_in_drop_band=1), precision=prec)
    m.load_state_dict(sd); m = m.to(dev).eval()
    mag = stft(y, 512, 256, 512)[0]
    with torch.no_grad():
        outs[prec] = m(mag.unsqueeze(1)).cpu().numpy()
    torch.cuda.synchronize()
    print(prec, "done", outs[prec].shape, float(np.abs(outs[prec]).max()), flush=True)
a, b = outs["fp32"], outs["f16_tc"]
print("max rel", np.abs(a - b).max() / np.abs(a).max(), "nan", np.isnan(b).sum())
err = np.abs(a - b) / np.abs(a).max()
print("err by t:", np.round(err.max(axis=(0, 1, 2)), 5))
print("err by f (first 40):", np.round(err.max(axis=(0, 1, 3))[:40], 5))
print("err by o:", err.max(axis=(0, 2, 3)))
print("ref[0,0,:4,:4]\n", a[0, 0, :4, :4], "\ntc\n", b[0, 0, :4, :4])
