"""TEST INFRASTRUCTURE ONLY.  Fixtures of ``norm_type="forgetting_norm"`` (audio_zen/model/base_model.py:102-151) from the
UNMODIFIED upstream code in ``/root/reference`` on CPU, same recipes as make_golden_long.py / make_golden_train.py /
make_golden_fbb_wav.py:

  forgetting.npz          the reference's BaseModel.forgetting_norm on [3,1,17,200] and [2,5,7,196] inputs (both sides
                          of the t = 192 switch); two training steps of the small fullsubnet at the recipe crop (5 clips,
                          T = 193 frames, so T' = 195 crosses 192; drop_band G = 2); fullband_baseline (F = 33, n_fft 64)
                          wav -> wav through Inferencer.full_band_crm_mask, one clip at a time, for three clip lengths
  model_forget_{wa,wb}.npz  fullsubnet inference (full size), 1 clip of 51456 samples (T = 202, T' = 204), weight sets
                          W-a and W-b (|cRM| up to the 9.9 clip); the input is regenerated from its seed (fingerprint)

Run:  python oracle/make_golden_forgetting.py
"""
from __future__ import annotations

import importlib.util
import os
import sys
from functools import partial

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

FULL_LEN = 51456          # T = 202 at hop 256
TRAIN_LEN = 6144          # T = 193 at hop 32: the recipe crop's frame count
FBB_LENGTHS = (6500, 5100, 6211)  # T = 204, 160, 195 at hop 32
NORM = "forgetting_norm"


def main():
    from make_golden import REF, import_reference
    from make_golden_fbb_wav import reference as fbb_reference
    from make_golden_long import fingerprint
    from make_golden_train import SMALL, reference_step
    from oracle import fullband_baseline_oracle as BO
    from oracle import fullsubnet_oracle as O
    feature, mask, Model, Inferencer = import_reference()
    from audio_zen.model.base_model import BaseModel
    out_dir = os.path.join(ROOT, "tests", "golden")
    torch.set_num_threads(8)
    res = {}

    # ---------------------------------------------------------------- the norm alone
    g = torch.Generator().manual_seed(61)
    for tag, shape in (("n1", (3, 1, 17, 200)), ("n2", (2, 5, 7, 196))):
        x = torch.rand(*shape, generator=g) * 3.0 + 0.01
        res[tag + "_x"], res[tag + "_y"] = x.numpy(), BaseModel.forgetting_norm(x).numpy()

    # ---------------------------------------------------------------- two training steps, small fullsubnet
    args = dict(SMALL, norm_type=NORM)
    sd = O.make_state_dict(seed=7, args=args, sb_fc_gain=8.0)
    noisy = O.make_noisy(5, TRAIN_LEN, seed=71, speechlike=True)
    clean = 0.5 * O.make_noisy(5, TRAIN_LEN, seed=72, speechlike=True)
    r = reference_step(feature, mask, Model, args, sd, noisy, clean, 64, 32)
    print("train: loss", r["loss0"], r["loss1"], "gnorm", r["gnorm0"], r["gnorm1"], "crm", r["crm"].shape)
    res.update({"train_noisy": noisy.numpy(), "train_clean": clean.numpy(), "train_crm": r["crm"],
                "train_loss": np.array([r["loss0"], r["loss1"]]), "train_gnorm": np.array([r["gnorm0"], r["gnorm1"]])})
    res.update({"train_grad." + k: v for k, v in r["grads"].items()})
    res.update({"train_p1." + k: v for k, v in r["params1"].items()})

    # ---------------------------------------------------------------- fullband_baseline wav -> wav, three lengths
    spec = importlib.util.spec_from_file_location(
        "fbb_model", os.path.join(REF, "recipes", "dns_interspeech_2020", "fullband_baseline", "model.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    fargs = dict(BO.DEFAULT_FBB_ARGS, num_freqs=33, hidden_size=32, output_activate_function="ReLU", norm_type=NORM)
    y, wav, crm = fbb_reference(fargs, 1.0, dict(n_fft=64, lengths=FBB_LENGTHS), feature, mod, Inferencer, O, BO)
    res.update({"fbb_y": y, "fbb_lengths": np.asarray(FBB_LENGTHS, np.int32), "fbb_wav": wav, "fbb_crm": crm})
    print("fbb crm max", float(np.abs(crm).max()), "wav max", float(np.abs(wav).max()))
    out = os.path.join(out_dir, "forgetting.npz")
    np.savez_compressed(out, **res)
    print(out, os.path.getsize(out))

    # ---------------------------------------------------------------- fullsubnet inference, W-a and W-b
    full = dict(O.DEFAULT_MODEL_ARGS, norm_type=NORM)
    y = O.make_noisy(1, FULL_LEN, seed=73, speechlike=True)
    for tag, gain in (("wa", 1.0), ("wb", 220.0)):
        model = Model(**full).eval()
        model.load_state_dict(O.make_state_dict(seed=0, args=full, sb_fc_gain=gain), strict=True)
        inf = Inferencer.__new__(Inferencer)
        inf.model, inf.device = model, torch.device("cpu")
        inf.torch_stft = partial(feature.stft, n_fft=512, hop_length=256, win_length=512)
        inf.torch_istft = partial(feature.istft, n_fft=512, hop_length=256, win_length=512)
        with torch.no_grad():
            crm = model(feature.stft(y, 512, 256, 512)[0].unsqueeze(1))
            wav = inf.full_band_crm_mask(y, {})
        print(tag, "crm", tuple(crm.shape), "range", float(crm.min()), float(crm.max()), "wav max", float(np.abs(wav).max()))
        out = os.path.join(out_dir, f"model_forget_{tag}.npz")
        np.savez_compressed(out, y_fp=fingerprint(y), crm=crm.numpy(), wav=wav[None])
        print(out, os.path.getsize(out))


if __name__ == "__main__":
    main()
