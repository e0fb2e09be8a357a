"""The transposed GATE: the sampler's GEMM1 (three conv taps, conditioner projection hoisted into the epilogue, three
products) with 64 packed W1 rows on the wgmma M side and BLOCK_T = 200 or 240 time steps on the N side, one staged
activation tile per channel block read by all three taps at row offsets 0, d, 2d of a 64 B-swizzled tile.

Checked through whole WaveNet evaluations on the hoisted path (L = 4 layers: dilations 1, 2, 4, 8 as in the model, and
3, 5, 6, 7, so that the taps' row offsets j d cover every row of the 8-row swizzle atom), against float64 and against
the SIMT twin on the same path:
  * T a multiple of BLOCK_T, not a multiple, T < BLOCK_T, T < 2d; odd and even time-tile counts; both widths;
  * C = 128 (gate tile 128) / 256 / 512, B > 1 with one step vector and with one per item, f16 and bf16;
  * placement: an item's output is bit-identical whatever batch position it occupies;
  * the same evaluation with the projection inside the K loop (the other GATE orientation) agrees to the f16 level.
"""
import zlib

import pytest
import torch

from conftest import rel_l2
from fish_diffusion_b200 import WaveNet
from fish_diffusion_b200 import _native as N
from oracle import wavenet as ownet

pytestmark = pytest.mark.gpu

TOL = {"f16": 2e-5, "bf16": 3e-4}      # those of tests/test_gpu_cond_proj.py


def _dev():
    return torch.device("cuda:0")


def _net(seed, C, prec, backend, M=64, E=256, L=4):
    sd = ownet.make_wavenet_weights(seed, mel_channels=M, d_encoder=E, residual_channels=C, residual_layers=L)
    net = WaveNet(mel_channels=M, d_encoder=E, residual_channels=C, residual_layers=L, use_linear_bias=True,
                  dilation_cycle=4, precision=prec, backend=backend).to(_dev())
    net.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    net.use_graph = False
    return sd, net.eval()


def _eval(net, x, steps, cond, hoist=True):
    pc = N.prec_code(net.precision)
    cond_planes, x_planes = N.split_nwc(cond, pc), N.split_nwc(x, pc)
    proj = None
    if hoist:
        B, T = x.shape[:2]
        proj = net.cond_projection(cond_planes, torch.empty(net.cond_proj_shape(B, T), device=_dev()))
    eps = net.forward_cl(x_planes, steps, cond_planes, cond_proj=proj)
    torch.cuda.synchronize()
    return eps.clone()


# (C, B, T, Bs, precision); BLOCK_T is the width that pads T least (200 on ties with more padding at 240)
CASES = [
    (512, 2, 400, 1, "f16"),      # 2 tiles of 200, T a multiple of BLOCK_T
    (512, 3, 590, 3, "bf16"),     # 3 tiles of 200 (odd), ragged, per-item steps
    (512, 2, 430, 1, "f16"),      # 2 tiles of 240, ragged
    (256, 3, 77, 3, "f16"),       # T < BLOCK_T
    (256, 2, 13, 1, "bf16"),      # T < 2d for d = 8
    (128, 5, 5, 5, "f16"),        # T < d for d = 8, gate tile 128
    (128, 3, 700, 1, "bf16"),     # 3 tiles of 240 (odd), gate tile 128
]


def _check(case, dils, monkeypatch):
    C, B, T, Bs, prec = case
    seed = zlib.crc32(repr((case, dils)).encode()) & 0xFFFF
    sd, net = _net(seed, C, prec, "tc")
    _, twin = _net(seed, C, prec, "simt")
    for m in (net, twin):
        for blk, dil in zip(m.residual_layers, dils):
            blk.dilation = dil
    # the oracle takes its dilations from the layer index
    block = ownet.residual_block
    monkeypatch.setattr(ownet, "residual_block", lambda sd_, prefix, x_, c_, s_, _dil:
                        block(sd_, prefix, x_, c_, s_, dils[int(prefix.split(".")[1])]))
    g = torch.Generator().manual_seed(seed)
    x, cond = torch.randn(B, T, 64, generator=g), torch.randn(B, T, 256, generator=g)
    steps = torch.tensor([990.0, 17.0, 503.25, 40.0, 3.0][:Bs])
    ref = ownet.wavenet_forward(sd, x.transpose(1, 2).numpy(), steps.numpy(), cond.transpose(1, 2).numpy()
                                ).transpose(0, 2, 1)
    d = _dev()
    got = _eval(net, x.to(d), steps.to(d), cond.to(d)).cpu().numpy()
    simt = _eval(twin, x.to(d), steps.to(d), cond.to(d)).cpu().numpy()
    fused = _eval(net, x.to(d), steps.to(d), cond.to(d), hoist=False).cpu().numpy()
    e64, es, ef = rel_l2(got, ref), rel_l2(got, simt), rel_l2(got, fused)
    print(f"gate_t[{case}, d={dils}] rel-L2 vs float64 {e64:.2e}, vs simt {es:.2e}, vs projection in the K loop {ef:.2e}")
    assert e64 < TOL[prec] and es < TOL[prec] and ef < TOL[prec]


@pytest.mark.parametrize("case", CASES, ids=[f"c{c[0]}-B{c[1]}-T{c[2]}-Bs{c[3]}-{c[4]}" for c in CASES])
def test_transposed_gate_vs_float64_and_simt(case, monkeypatch):
    _check(case, (1, 2, 4, 8), monkeypatch)


# dilations 3, 5, 6, 7: tap row offsets 3, 5, 6, 7, 10, 12, 14 (with 1, 2, 4, 8 above: every residue modulo 8)
ODD = [(512, 2, 590, 1, "f16"), (256, 3, 13, 3, "bf16")]


@pytest.mark.parametrize("case", ODD, ids=[f"c{c[0]}-B{c[1]}-T{c[2]}-Bs{c[3]}-{c[4]}" for c in ODD])
def test_transposed_gate_other_row_offsets(case, monkeypatch):
    _check(case, (3, 5, 6, 7), monkeypatch)


def test_transposed_gate_item_bits_independent_of_placement():
    """T = 590: three time tiles per item, so an item's tiles meet other pairs and warpgroups at each position."""
    C, B, T = 512, 4, 590
    _, net = _net(77, C, "f16", "tc")
    g = torch.Generator().manual_seed(77)
    x, cond = torch.randn(B, T, 64, generator=g).to(_dev()), torch.randn(B, T, 256, generator=g).to(_dev())
    steps = torch.tensor([990.0, 17.0, 503.25, 40.0], device=_dev())
    batch = _eval(net, x, steps, cond)
    rev = _eval(net, x.flip(0), steps.flip(0), cond.flip(0))
    for j in range(B):
        alone = _eval(net, x[j:j + 1], steps[j:j + 1], cond[j:j + 1])
        assert torch.equal(alone[0], batch[j]), f"item {j} differs between B=1 and batch position {j}"
        assert torch.equal(alone[0], rev[B - 1 - j]), f"item {j} differs between B=1 and batch position {B - 1 - j}"
