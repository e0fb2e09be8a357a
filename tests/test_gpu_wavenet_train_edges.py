"""The WaveNet training path end to end at its edges: `WaveNet` in grad mode (WaveNetTrainFn: native forward, one
fd_wavenet_block_bwd per block, the step MLP and diffusion projections under torch autograd) against torch.autograd of
the float64 restatement of the whole forward (wavenet_block_ref.wavenet_forward, pinned to the oracle by
test_wavenet_block_ref_cpu.py).  Every parameter gradient, d_x and d_cond are compared, so wavenet_train.py's
post-processing -- the packed -> reference permutation, 1/sqrt2 on gw2's residual rows, the rank-one step-vector term,
gb2, and the step-vector gradient d_d = cs_dx - cs_x_next/sqrt2 that reaches the MLP -- is pinned against first
principles rather than against a restatement of itself.

Dilation cycle 4 over 4 layers at T = 5 and T = 1: dilations 4 and 8 reach or pass T, where every side tap reads only
zero padding.  Per-item steps with B >= 5, masks, a tensor-core, a SIMT-only and a bf16 configuration.

Tolerances: rel-L2 per gradient and, for the conv weights, max|err| per tap in units of the whole gradient's RMS (a tap
whose reference gradient is exactly zero -- the side taps when dil >= T -- is judged by that max alone); each bar at
most 4x the largest value measured on an H100 80GB HBM3 over the configurations (in the comment).
"""
import numpy as np
import pytest
import torch

from fish_diffusion_b200 import WaveNet
from gpu_util import dev
from oracle import wavenet as ownet
from region_check import F64, check_parts
from wavenet_block_ref import wavenet_forward

pytestmark = pytest.mark.gpu

# (name, C, E, M, precision, backend, B, per-item steps, masks)
CONFIGS = [
    ("tc-f16-item-masks", 128, 64, 64, "f16", "tc", 5, True, True),
    ("simt-c80-f16-item-masks", 80, 40, 24, "f16", "simt", 6, True, True),
    ("tc-bf16-shared", 128, 64, 64, "bf16", "tc", 5, False, False),
]
L, CYCLE = 4, 4

# (rel-L2, max) bars: eps is the forward output, "grad" every parameter gradient, d_x and d_cond
TOL = {
    ("eps", "f16"): (1e-5, 6.5e-5),       # measured 2.7e-6 / 1.6e-5
    ("grad", "f16"): (2.8e-5, 9e-4),      # measured 7.2e-6 / 2.3e-4
    ("eps", "bf16"): (4.4e-5, 1.5e-4),    # measured 1.1e-5 / 3.9e-5
    ("grad", "bf16"): (7e-5, 2.7e-3),     # measured 1.8e-5 / 7.0e-4
}


@pytest.mark.parametrize("T", [5, 1])
@pytest.mark.parametrize("cfg", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_train_gradients_vs_float64_autograd(cfg, T):
    name, C, E, M, prec, backend, B, per_item, masks = cfg
    d0 = dev()
    seed = sum(map(ord, name)) + T
    sd = ownet.make_wavenet_weights(seed, mel_channels=M, d_encoder=E, residual_channels=C, residual_layers=L,
                                    use_linear_bias=True)
    rng = np.random.RandomState(seed)
    x_np, c_np, w_np = rng.randn(B, M, T), rng.randn(B, E, T), rng.randn(B, M, T)
    steps_np = rng.randint(0, 1000, size=B if per_item else 1).astype(np.float64)
    xm = cm = None
    if masks:
        xm, cm = rng.rand(B, T) < 0.3, rng.rand(B, T) < 0.3
        xm[0], cm[0] = False, False                   # one item keeps every row
    tb = lambda a: None if a is None else torch.from_numpy(a).to(d0)

    net = WaveNet(mel_channels=M, d_encoder=E, residual_channels=C, residual_layers=L, use_linear_bias=True,
                  dilation_cycle=CYCLE, precision=prec, backend=backend).to(d0)
    net.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    t32 = lambda a: torch.from_numpy(a.astype(np.float32)).to(d0)
    x, cond = t32(x_np).requires_grad_(True), t32(c_np).requires_grad_(True)
    y = net(x, t32(steps_np), cond, x_masks=tb(xm), cond_masks=tb(cm))
    (y * t32(w_np)).sum().backward()
    torch.cuda.synchronize()

    t64 = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float64)).to(d0)
    p64 = {k: t64(v).requires_grad_(True) for k, v in sd.items()}
    x64, c64 = t64(x_np).requires_grad_(True), t64(c_np).requires_grad_(True)
    y64 = wavenet_forward(p64, x64, t64(steps_np), c64, x_masks=tb(xm), cond_masks=tb(cm), dilation_cycle=CYCLE)
    (y64 * t64(w_np)).sum().backward()

    print(f"\n[{name} T={T}] dilations {[2 ** (i % CYCLE) for i in range(L)]}")
    tol = lambda k: TOL[(k, prec)]
    bad = check_parts("eps", y.detach().to(F64), y64.detach(), {}, tol("eps"))
    bad += check_parts("d_x", x.grad.to(F64), x64.grad, {}, tol("grad"))
    bad += check_parts("d_cond", cond.grad.to(F64), c64.grad, {}, tol("grad"))
    taps = {"tap-dil": (..., 0), "tap0": (..., 1), "tap+dil": (..., 2)}
    for k, p in net.named_parameters():
        assert p.grad is not None, k
        parts = taps if k.endswith("conv_layer.conv.weight") else {}
        bad += check_parts(k, p.grad.to(F64), p64[k].grad, parts, tol("grad"), exact_zero=False)
    assert not bad, "; ".join(bad)
