"""Generate tests/golden/convnext.npz from the UNMODIFIED reference ConvNext denoiser, imported by file path (only possible
where the reference checkout is present; the vectors are committed).  Run:  python tests/golden/make_golden_convnext.py

What is loaded from the reference:
  fish_diffusion/modules/convnext.py        its one package import, `fish_diffusion.modules.wavenet`, is served by the
                                            file-loaded reference wavenet.py (DiffusionEmbedding)
  archs/diffsinger/diffusions/*.py          through oracle/ref_loader.py, whose stub registry gets ConvNext registered as
                                            "ConvNextDenoiser"
Weights are oracle.convnext.make_convnext_weights (gamma re-randomised); every random draw of the reference sampler is
served from a recorded numpy stream so the same numbers can be injected into the CUDA path.
"""
import importlib.util
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden import RecordedRandom  # noqa: E402
from oracle import convnext as ocnx  # noqa: E402
from oracle.ref_loader import load_reference  # noqa: E402

# the small configuration of the golden cases: dilations 1, 2, 4, 8 (halo 24 against T = 40)
SMALL = dict(mel_channels=16, dim=32, mlp_factor=4, condition_dim=16, num_layers=4, dilation_cycle=4)
SEED = 61


def load_convnext(ref):
    fd = types.ModuleType("fish_diffusion")
    mods = types.ModuleType("fish_diffusion.modules")
    fd.modules, mods.wavenet = mods, ref.wavenet
    for name, mod in (("fish_diffusion", fd), ("fish_diffusion.modules", mods),
                      ("fish_diffusion.modules.wavenet", ref.wavenet)):
        sys.modules.setdefault(name, mod)
    path = os.path.join(ref.root, "fish_diffusion", "modules", "convnext.py")
    spec = importlib.util.spec_from_file_location("ref_convnext", path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules["ref_convnext"] = mod
    spec.loader.exec_module(mod)
    sys.modules["refdiff.builder"].DENOISERS.register_module(name="ConvNextDenoiser", module=mod.ConvNext)
    return mod


def inventory(net):
    return json.dumps([[k, list(v.shape)] for k, v in net.state_dict().items()])


def small_net(cnx, sd):
    cfg = {k: v for k, v in SMALL.items() if k != "dilation_cycle"}
    net = cnx.ConvNext(**cfg, dilation_cycle=SMALL["dilation_cycle"])
    net.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    return net.eval()


def main():
    ref = load_reference(with_mel=False)
    cnx = load_convnext(ref)
    out = {}
    torch.manual_seed(0)
    out["inv_default"] = np.array(inventory(cnx.ConvNext()))
    out["inv_small"] = np.array(inventory(cnx.ConvNext(**{k: v for k, v in SMALL.items()})))
    out["config_small"] = np.array(json.dumps(SMALL))
    sd = ocnx.make_convnext_weights(SEED, **{k: v for k, v in SMALL.items() if k != "dilation_cycle"})
    for k, v in sd.items():
        out["w/" + k] = v
    net = small_net(cnx, sd)

    M, E = SMALL["mel_channels"], SMALL["condition_dim"]
    B, T = 2, 40
    rng = np.random.RandomState(62)
    x = rng.randn(B, M, T).astype(np.float32)
    cond = rng.randn(B, E, T).astype(np.float32)
    out["x"], out["cond"] = x, cond
    xm = np.stack([np.arange(T) >= n for n in (40, 29)])
    cm = np.stack([np.arange(T) >= n for n in (33, 21)])
    out["x_masks"], out["cond_masks"] = xm, cm
    steps = {"stepsB_int": np.array([3, 871], dtype=np.int64), "stepsB_float": np.array([17.5, 990.0], np.float32),
             "steps1_int": np.array([500], dtype=np.int64), "steps1_float": np.array([250.25], np.float32)}
    cases = {name: dict(steps=s) for name, s in steps.items()}
    cases["masked"] = dict(steps=steps["stepsB_int"], x_masks=xm, cond_masks=cm)
    cases["cond_masked_only"] = dict(steps=steps["stepsB_int"], cond_masks=cm)
    cases["x_masked_only"] = dict(steps=steps["steps1_float"], x_masks=xm)
    with torch.no_grad():
        for name, c in cases.items():
            kw = {k: torch.from_numpy(c[k]) for k in ("x_masks", "cond_masks") if k in c}
            y = net(torch.from_numpy(x), torch.from_numpy(c["steps"]), torch.from_numpy(cond), **kw)
            out[f"case_{name}_steps"] = c["steps"]
            out[f"case_{name}_out"] = y.numpy()
        y4 = net(torch.from_numpy(x)[:, None], torch.from_numpy(steps["stepsB_int"]), torch.from_numpy(cond))
        assert y4.dim() == 4
        out["case_4d_out"] = y4.numpy()

    # sampler trajectories through the reference GaussianDiffusion with the reference ConvNext as its denoiser
    feats = rng.randn(B, T, E).astype(np.float32)
    out["samp_features"] = feats
    for pred in ("naive", "plms", "unipc"):
        diff = ref.diffusion.GaussianDiffusion(
            denoiser=dict(type="ConvNextDenoiser", **SMALL), mel_channels=M, noise_schedule="linear", timesteps=1000,
            max_beta=0.01, noise_loss="smoothed-l1", sampler_interval=100, spec_min=[-5.0], spec_max=[0.0],
            noise_predictor=pred)
        diff.denoise_fn.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
        diff.eval()
        with RecordedRandom(2000) as rr, torch.no_grad():
            y = diff(torch.from_numpy(feats), sampler_interval=100, noise_predictor=pred)
        key = f"samp_{pred}"
        out[key + "_mel"] = y.numpy()
        for j, (kind, a) in enumerate(rr.log):
            out[key + f"_noise{j}"] = a
        out[key + "_nnoise"] = np.array(len(rr.log))
    path = os.path.join(HERE, "convnext.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {os.path.getsize(path)} bytes, {len(out)} arrays")


if __name__ == "__main__":
    main()
