"""ConvNext denoiser on the H100: the 100-evaluation DDPM sampler at B = 32, T = 4000 with the default ConvNext (dim 512,
mlp_factor 4, 20 layers) against the default WaveNet at the same shape, f16 and f16x1, alternated in one process so that
all numbers come from one session; then CUDA-event times of the three per-layer kernels of the ConvNext block (dwln,
pwconv1 + GELU, pwconv2 + residual) at the same shape.  Weights are synthetic and seeded (ConvNext gamma re-randomised
log-uniform over [1e-2, 1]).  Prints one JSON line.

  python tools/bench_convnext.py [--B 32] [--T 4000] [--reps 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from fish_diffusion_b200 import DIFFUSIONS  # noqa: E402
from fish_diffusion_b200 import _native as N  # noqa: E402
from oracle import convnext as ocnx, wavenet as ownet  # noqa: E402

HBM_BPS = 3.35e12        # H100 SXM data sheet
DENSE_FLOPS = 989e12     # H100 SXM data sheet, dense FP16 / BF16
CNX = dict(mel_channels=128, dim=512, mlp_factor=4, condition_dim=256, num_layers=20, dilation_cycle=4)
WN = dict(mel_channels=128, d_encoder=256, residual_channels=512, residual_layers=20, use_linear_bias=True,
          dilation_cycle=4)


def counts(cfg):
    """Algorithmic FLOPs per position (multiply-add = 2) and HBM bytes per position of one ConvNext evaluation, from
    shapes; f16 split planes are 4 bytes per element."""
    M, C, E, L = cfg["mel_channels"], cfg["dim"], cfg["condition_dim"], cfg["num_layers"]
    H = C * cfg["mlp_factor"]
    dwln = 2 * 7 * C + 8 * C                                   # depthwise taps + LayerNorm
    layer = {"dwln": dwln, "pwconv1": 2 * C * H, "pwconv2": 2 * H * C}
    per_eval = 2 * M * C + L * sum(layer.values()) + 2 * C * C + 2 * C * M
    per_call = 2 * E * H + 2 * H * C + L * 2 * C * C           # conditioner MLP + the L condition projections
    layer_bytes = {"dwln": 3 * 4 * C,                          # x planes + projection in, planes out
                   "pwconv1": 4 * C + 4 * H,                   # LN planes in, GELU planes out
                   "pwconv2": 4 * H + 2 * 4 * C}               # GELU planes + residual in, residual out
    return layer, per_eval, per_call, layer_bytes


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        return f"unknown ({ex!r})"


def sampler(kind, precision, dev):
    if kind == "convnext":
        den = dict(type="ConvNextDenoiser", precision=precision, **CNX)
        sd = ocnx.make_convnext_weights(5, **{k: v for k, v in CNX.items() if k != "dilation_cycle"})
    else:
        den = dict(type="WaveNetDenoiser", precision=precision, **WN)
        sd = ownet.make_wavenet_weights(5, **{k: v for k, v in WN.items() if k != "dilation_cycle"})
    diff = DIFFUSIONS.build(dict(type="GaussianDiffusion", denoiser=den, mel_channels=128, noise_schedule="linear",
                                 timesteps=1000, max_beta=0.01, sampler_interval=10, spec_min=[-5.0], spec_max=[0.0],
                                 noise_predictor="naive"))
    diff.denoise_fn.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    return diff.to(dev).eval()


def time_call(fn, reps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    fn()
    ev[0].record()
    for _ in range(reps):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / reps


def kernel_times(diff, B, T, dev, reps=20):
    """ms per launch of dwln (per dilation of the cycle), pwconv1 and pwconv2 at layer l's weights"""
    net = diff.denoise_fn
    pk = net._packed(dev)
    ws = net._workspace(dev, B, T)
    C, H = net.dim, net.hidden
    prec, mma, be = N.prec_code(net.precision), pk["mma"], pk["backend"]
    g = torch.Generator(device=dev).manual_seed(3)
    N.split_nwc(torch.randn(B, T, C, device=dev, generator=g), prec, out=ws["xr"])
    N.split_nwc(torch.randn(B, T, C, device=dev, generator=g), prec, out=ws["a"])
    N.split_nwc(torch.randn(B, T, H, device=dev, generator=g) * 0.1, prec, out=ws["h"])
    p = torch.randn(B, T, C, device=dev, generator=g)
    sv = torch.randn(1, C, device=dev, generator=g)
    st = N.stream_ptr(dev)
    out = {}
    dw = []
    for l in range(4):
        def run(l=l):
            N.check(N.lib().fd_convnext_dwln_fwd(
                N.ptr(ws["xr"]), N.ptr(p), N.ptr(sv), 0, None, N.ptr(pk["dw_w"][l]), N.ptr(pk["dw_b"][l]),
                N.ptr(pk["ln_w"][l]), N.ptr(pk["ln_b"][l]), N.ptr(ws["a"]), B, T, C, pk["dil"][l], prec, st), "dwln")
        dw.append(time_call(run, reps))
    out["dwln"] = float(np.mean(dw))
    out["dwln_by_dilation"] = {str(pk["dil"][l]): dw[l] for l in range(4)}
    out["pwconv1"] = time_call(lambda: N.conv_cl(
        ws["a"], pk["w_pw1"][0], B, T, C, H, [0], bias=pk["b_pw1"][0], out_planes=ws["h"],
        w_inv_scale=pk["inv"]["pw10"], act=N.ACT_GELU, prec=mma, backend=be), reps)
    out["pwconv2"] = time_call(lambda: N.conv_cl(
        ws["h"], pk["w_pw2"][0], B, T, H, C, [0], bias=pk["b_pw2"][0], res_planes=ws["xr"], out_planes=ws["xr"],
        w_inv_scale=pk["inv"]["pw20"], prec=mma, backend=be), reps)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--T", type=int, default=4000)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_convnext needs a CUDA device: nothing is measured without one")
    dev = torch.device("cuda:0")
    B, T = a.B, a.T
    g = torch.Generator().manual_seed(1)
    feats = torch.randn(B, T, 256, generator=g).to(dev)
    runs = {(k, p): sampler(k, p, dev) for p in ("f16", "f16x1") for k in ("convnext", "wavenet")}
    evals = 100
    res = {k: [] for k in runs}
    for k, d in runs.items():                      # warm-up: workspace, packs, graph capture
        d(feats, seed=1)
    torch.cuda.synchronize()
    for _ in range(a.reps):
        for k, d in runs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            d(feats, seed=1)
            torch.cuda.synchronize()
            res[k].append(time.perf_counter() - t0)
    layer, per_eval, per_call, layer_bytes = counts(CNX)
    pos = B * T
    out = {"metric": "convnext_ddpm100_sampler", "B": B, "T": T, "evaluations": evals, "card": card(),
           "flop_per_position_per_eval": per_eval, "flop_per_eval": per_eval * pos,
           "flop_per_position_per_call_once": per_call, "bytes_per_position_per_layer": layer_bytes,
           "hbm_bytes_per_eval": (sum(layer_bytes.values()) * CNX["num_layers"]) * pos,
           "hoisted_projection_bytes": 4 * CNX["num_layers"] * CNX["dim"] * pos, "samplers": {}, "kernels": {}}
    for (k, p), ts in res.items():
        best = min(ts)
        out["samplers"][f"{k}/{p}"] = {"s_per_call": best, "all_s": ts, "ms_per_eval": 1e3 * best / evals,
                                       "mel_frames_per_s": pos / best}
    for p in ("f16", "f16x1"):
        kt = kernel_times(runs[("convnext", p)], B, T, dev)
        products = 1 if p.endswith("x1") else 3
        ent = {"ms": kt}
        ent["dwln_hbm_share"] = layer_bytes["dwln"] * pos / HBM_BPS / (kt["dwln"] * 1e-3)
        for gk in ("pwconv1", "pwconv2"):
            ent[f"{gk}_tensor_share"] = products * layer[gk] * pos / DENSE_FLOPS / (kt[gk] * 1e-3)
            ent[f"{gk}_hbm_share"] = layer_bytes[gk] * pos / HBM_BPS / (kt[gk] * 1e-3)
        ent["share_note"] = (f"tensor share counts the {products} tensor-core product(s) per multiply-add over the "
                             "989 TFLOP/s dense data-sheet rate; HBM share over 3.35 TB/s")
        out["kernels"][p] = ent
    print(json.dumps(out))


if __name__ == "__main__":
    main()
