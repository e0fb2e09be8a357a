"""Times the resampling kernel (fd_resample_fwd) with CUDA events and sets it against its two bounds.

    python tools/bench_resample.py [--launches 50] [--warmup 5]

Workloads: a batch of B = 32 clips of 46 s (the flagship batch of bench.py) at the DAW <-> model rates and at the model
-> content-encoder rate, and one 3 s clip, the frame of the TCP service.  For each, one JSON line with
  ms            time per call (events around `launches` back-to-back calls after `warmup`)
  GBps, hbm     algorithmic bytes 4 * (n_in + n_out) * B over time, and as a share of 3.35 TB/s (H100 SXM data sheet)
  TFLOPs, fp32  2 * FMAs over time (FMAs = sum over outputs of the taps of their phase), share of 67 TFLOP/s (data sheet)
  bound         which of the two takes longer at data-sheet rates, and the time it would take
and the card's name and power limit as nvidia-smi reports them.  Needs a CUDA device; there is no CPU path."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fish_diffusion_b200 import resample, resample_length          # noqa: E402
from fish_diffusion_b200.mel import resample_bank                  # noqa: E402

HBM_BPS, FP32_FLOPS = 3.35e12, 67e12
WORKLOADS = [("batch 48k->44.1k", 32, 46.0, 48000, 44100), ("batch 44.1k->48k", 32, 46.0, 44100, 48000),
             ("batch 44.1k->16k", 32, 46.0, 44100, 16000), ("tcp frame 48k->44.1k", 1, 3.0, 48000, 44100)]


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi failed"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_resample needs a CUDA device")
    dev = torch.device("cuda:0")
    card = gpu_info()
    for name, B, secs, sr_in, sr_out in WORKLOADS:
        n_in = int(secs * sr_in)
        n_out = resample_length(n_in, sr_in, sr_out)
        x = torch.rand((B, n_in), device=dev) * 2 - 1
        _, _, count, (O, P, W, taps) = resample_bank(sr_in, sr_out, dev)
        cnt = count.cpu().to(torch.int64)
        fmas = B * (int(cnt.sum()) * (n_out // P) + int(cnt[:n_out % P].sum()))
        nbytes = 4 * (n_in + n_out) * B
        for _ in range(a.warmup):
            resample(x, sr_in, sr_out)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.launches):
            resample(x, sr_in, sr_out)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / a.launches
        t_mem, t_flop = nbytes / HBM_BPS * 1e3, 2 * fmas / FP32_FLOPS * 1e3
        print(json.dumps({
            "workload": name, "B": B, "n_in": n_in, "n_out": n_out, "O": O, "P": P, "taps_per_output": round(fmas / (B * n_out), 1),
            "launches": a.launches, "ms": round(ms, 4),
            "GBps": round(nbytes / ms / 1e6, 1), "hbm_share": round(nbytes / ms / 1e-3 / HBM_BPS, 4),
            "TFLOPs": round(2 * fmas / ms / 1e9, 2), "fp32_share": round(2 * fmas / ms / 1e-3 / FP32_FLOPS, 4),
            "bound": "fp32" if t_flop > t_mem else "hbm", "bound_ms": round(max(t_flop, t_mem), 4),
            "share_of_bound": round(max(t_flop, t_mem) / ms, 4), "gpu": card}), flush=True)


if __name__ == "__main__":
    main()
