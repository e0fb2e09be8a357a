"""Per-launch device time of the two WaveNet tap-GEMMs (GEMM1 = GATE, GEMM2 = RES_SKIP) at the headline sampler shape
(B=32, T=4000, C=512, E=256, f16), with the shared-memory traffic the tiling implies.

    python tools/prof_wavenet_gemm.py [--single] [--hoisted] [--reps N]

Every dilation 1, 2, 4, 8 runs `reps` middle-layer blocks through fd_wavenet_block_fwd; each tap-GEMM launch is timed
by its own CUDA-event pair (N.prof_enable / N.prof_collect).  Bytes per launch come from the ping-pong tiling of
fd_tapgemm_tc.cu: 64-row position tiles x 256-column tiles, NPL operand planes each.  "staged" is what the TMA unit
writes into shared memory (every CTA holds its own A box and the whole W box per 64 rows); "L2 read" is what it reads
from L2 (the two CTAs of a cluster pair each fetch half of the W box and multicast it, so W is read once per 128 rows).
--single repeats the run in single-product mode (one hi*hi product, one plane staged).
--hoisted also times the sampler's path: the conditioner projection of all layers computed once per call
(fd_wavenet_cond_proj, L linear tap-GEMMs with K = E; each launch timed) and GEMM1 over the three conv taps only
(K = 3C) with the projection added in its epilogue, through fd_wavenet_fwd of a WaveNet with L = 4 layers
(dilations 1, 2, 4, 8).  TFLOP/s are those of the K each launch actually sums."""
import argparse
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, T, C, E = 32, 4000, 512, 256
BLOCK_M, BLOCK_N = 64, 256
DILATIONS = (1, 2, 4, 8)


def staged_bytes(k_total, npl):
    """-> (bytes written into shared memory per launch, bytes read from L2 per launch); independent of BLOCK_K."""
    m_tiles = B * math.ceil(T / BLOCK_M)
    m_tiles += m_tiles % 2                     # an odd tile count leaves a pair half that still stages its W half
    tiles = m_tiles * (2 * C // BLOCK_N)
    a = BLOCK_M * k_total * 2 * npl
    w = BLOCK_N * k_total * 2 * npl
    return tiles * (a + w), tiles * (a + w / 2)


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else f"nvidia-smi failed: {r.stderr}"


def run(N, torch, single, reps):
    dev = torch.device("cuda", 0)
    pc = N.PREC_F16
    mma = pc | (N.PREC_SINGLE if single else 0)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(B, T, C, device=dev, generator=g)
    cond = torch.randn(B, T, E, device=dev, generator=g)
    w1 = torch.randn(2 * C, 3 * C + E, device=dev, generator=g) * math.sqrt(2.0 / (3 * C))
    w2 = torch.randn(2 * C, C, device=dev, generator=g) * math.sqrt(2.0 / C)
    gb = torch.randn(3, 2 * C, device=dev, generator=g) * 0.1
    b2 = torch.randn(2 * C, device=dev, generator=g) * 0.1
    s1, s2 = N.pow2_scale(w1), N.pow2_scale(w2)
    w1p, w2p = N.pack_weight(w1, pc, s1), N.pack_weight(w2, pc, s2)
    xp, cp = N.split_nwc(x, pc), N.split_nwc(cond, pc)
    del x, cond
    z = torch.zeros((2, B, T, C), dtype=torch.int16, device=dev)
    skip = torch.zeros((B, T, C), dtype=torch.float32, device=dev)
    skp = torch.zeros((2, B, T, C), dtype=torch.int16, device=dev)
    st = N.stream_ptr(dev)

    def block(dil):
        # flags 0: a middle layer (reads and writes the fp32 skip accumulator, updates the residual planes)
        N.check(N.lib().fd_wavenet_block_fwd(
            N.ptr(xp), N.ptr(cp), N.ptr(z), N.ptr(w1p), N.ptr(w2p), N.ptr(gb[0]), N.ptr(gb[1]), N.ptr(gb[2]), 0,
            N.ptr(b2), N.ptr(skip), N.ptr(skp), 1.0, B, T, C, E, dil, 256, 1.0 / s1, 1.0 / s2, 0, mma, N.BACKEND_TC,
            st), "fd_wavenet_block_fwd")

    for dil in DILATIONS:          # warm-up: module load, tensor maps, clocks
        for _ in range(5):
            block(dil)
    torch.cuda.synchronize()
    N.prof_enable(True)
    for dil in DILATIONS:
        for _ in range(reps):
            block(dil)
    prof, overflow = N.prof_collect()
    N.prof_enable(False)
    assert not overflow, "per-launch event buffer overflowed: lower --reps"

    npl = 1 if single else 2
    mode = "single product (hi*hi)" if single else "three products (lo*hi + hi*lo + hi*hi)"
    print(f"== {mode}, B={B} T={T} C={C} E={E}, dilations {DILATIONS} x {reps} blocks")
    for name, key, k_total in (("GEMM1 gate", "gate/tc", 3 * C + E), ("GEMM2 res_skip", "res_skip/tc", C)):
        ms_sum, n = prof[key]
        ms = ms_sum / n
        alg = 2.0 * B * T * (2 * C) * k_total
        products = 1 if single else 3
        staged, l2 = staged_bytes(k_total, npl)
        print(f"{name:15s} {ms:7.3f} ms/launch over {n} launches ({ms_sum / 1e3:.2f} s) | "
              f"{alg / ms / 1e9:6.1f} TFLOP/s alg, {products}x issued = "
              f"{products * alg / ms / 1e9:6.1f} TFLOP/s | smem staged {staged / 1e9:5.2f} GB/launch "
              f"({staged / ms / 1e9:5.2f} TB/s into shared memory), L2 read {l2 / 1e9:5.2f} GB "
              f"({l2 / ms / 1e9:5.2f} TB/s)", flush=True)


def run_hoisted(N, torch, single, reps):
    from fish_diffusion_b200 import WaveNet, synthetic
    dev = torch.device("cuda", 0)
    M, L = 128, len(DILATIONS)
    prec = "f16x1" if single else "f16"
    cfg = dict(mel_channels=M, d_encoder=E, residual_channels=C, residual_layers=L, use_linear_bias=True)
    net = WaveNet(**cfg, dilation_cycle=L, precision=prec, backend="tc").to(dev).eval()
    net.load_state_dict({k: torch.from_numpy(v) for k, v in synthetic.wavenet_weights(0, **cfg).items()})
    net.use_graph = False
    pc = N.prec_code(prec)
    g = torch.Generator(device=dev).manual_seed(0)
    xp = N.split_nwc(torch.randn(B, T, M, device=dev, generator=g), pc)
    cp = N.split_nwc(torch.randn(B, T, E, device=dev, generator=g), pc)
    proj = torch.empty(net.cond_proj_shape(B, T), device=dev)
    steps = torch.tensor([500.0], device=dev)
    for _ in range(3):
        net.cond_projection(cp, proj)
        net.forward_cl(xp, steps, cp, cond_proj=proj)
    torch.cuda.synchronize()
    N.prof_enable(True)
    for _ in range(reps):
        net.cond_projection(cp, proj)
    proj_prof, overflow = N.prof_collect()
    for _ in range(reps):
        net.forward_cl(xp, steps, cp, cond_proj=proj)
    fwd_prof, overflow2 = N.prof_collect()
    N.prof_enable(False)
    assert not (overflow or overflow2), "per-launch event buffer overflowed: lower --reps"

    products = 1 if single else 3
    mode = "single product (hi*hi)" if single else "three products (lo*hi + hi*lo + hi*hi)"
    print(f"== hoisted conditioner projection, {mode}, B={B} T={T} C={C} E={E}, dilations {DILATIONS} x {reps} calls")
    proj_bytes = B * T * 2 * C * 4
    rows = (("cond_proj linear", proj_prof["linear/tc"], E, "written"),
            ("GEMM1 gate 3-seg", fwd_prof["gate/tc"], 3 * C, "read"))
    for name, (ms_sum, n), k, how in rows:
        ms = ms_sum / n
        alg = 2.0 * B * T * (2 * C) * k
        print(f"{name:17s} {ms:7.3f} ms/launch over {n} launches | {alg / ms / 1e9:6.1f} TFLOP/s alg (K={k}), "
              f"{products}x issued = {products * alg / ms / 1e9:6.1f} TFLOP/s | fp32 projection {how} "
              f"{proj_bytes / 1e9:5.2f} GB/launch ({proj_bytes / ms / 1e6:6.1f} GB/s)", flush=True)
    ms_sum, n = fwd_prof["res_skip/tc"]
    print(f"{'GEMM2 res_skip':17s} {ms_sum / n:7.3f} ms/launch over {n} launches", flush=True)
    ms_sum, n = proj_prof["linear/tc"]
    print(f"projection per sampler call of the 20-layer net: 20 x {ms_sum / n:.3f} = {20 * ms_sum / n:.2f} ms", flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--single", action="store_true", help="also run in single-product mode")
    ap.add_argument("--hoisted", action="store_true",
                    help="also time the projection hoisted out of GEMM1 (fd_wavenet_cond_proj + three-segment GATE)")
    ap.add_argument("--reps", type=int, default=200, help="blocks per dilation in the timed window")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    ge.build()
    from fish_diffusion_b200 import _native as N
    assert torch.cuda.is_available(), "prof_wavenet_gemm.py needs a CUDA device"
    print(f"gpu: {gpu_info()} (name, power limit, max SM clock)")
    run(N, torch, False, args.reps)
    if args.hoisted:
        run_hoisted(N, torch, False, args.reps)
    if args.single:
        run(N, torch, True, args.reps)
        if args.hoisted:
            run_hoisted(N, torch, True, args.reps)


if __name__ == "__main__":
    main()
