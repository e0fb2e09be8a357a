"""The WaveNet block GEMMs (GATE and RES_SKIP) on their ping-pong schedule: 64-row tiles, taken in turn by the two consumer
warpgroups of a CTA, CTAs in pairs that share each W tile (DESIGN.md section 1.1).

  * float64 parity (test_gpu_wavenet_block._run_block) at shapes that stress the schedule: odd 64-row tile counts (the
    second CTA of the last pair has no tile), T < 64 and T not a multiple of 64, pairs whose two tiles belong to two
    items, grids smaller than the SM count, per-item gate bias, at every column-tile width (C = 128, 192, 256, 512);
  * placement: one item's outputs are bit-identical whether it runs alone or at any position of a batch, i.e. the
    CTA, pair half and warpgroup a tile lands on do not change its bits.
"""
import math
import zlib

import pytest
import torch

from fish_diffusion_b200 import _native as N
from gpu_util import dev
from test_gpu_wavenet_block import _run_block
from wavenet_block_ref import gate_bias_tables, gate_perm

pytestmark = pytest.mark.gpu

# (name, C, E, gate_tile, precision, B, T, dil, flags, per_item_bias, train), as in test_gpu_wavenet_block.FWD;
# "tiles" = B * ceil(T / 64)
PP = [
    ("pp-c512-f16-B3-T130-d8-mid", 512, 256, 256, "f16", 3, 130, 8, 0, True, False),              # 9 tiles, pairs across items
    ("pp-c512-bf16x1-B1-T192-d64-first", 512, 256, 256, "bf16x1", 1, 192, 64, 1, True, False),    # 3 tiles
    ("pp-c512-f16-B7-T960-d16-mid-train", 512, 256, 256, "f16", 7, 960, 16, 0, True, True),       # 105 tiles, turns
    ("pp-c256-f16-B3-T40-d4-last-train", 256, 64, 256, "f16", 3, 40, 4, 2, True, True),           # T < 64, 3 tiles
    ("pp-c256-bf16-B2-T64-d1-single", 256, 64, 256, "bf16", 2, 64, 1, 3, True, False),            # one tile per item
    ("pp-c192-bf16-B2-T130-d2-mid", 192, 64, 128, "bf16", 2, 130, 2, 0, True, False),             # GATE 128 / RES 64 wide
    ("pp-c192-f16x1-B3-T77-d8-first", 192, 64, 128, "f16x1", 3, 77, 8, 1, True, False),
    ("pp-c128-f16x1-B5-T63-d1-mid", 128, 64, 128, "f16x1", 5, 63, 1, 0, True, False),             # T < 64, 5 tiles
    ("pp-c128-bf16-B3-T200-d64-last-train", 128, 64, 128, "bf16", 3, 200, 64, 2, True, True),     # 12 tiles, ragged
]


@pytest.mark.parametrize("case", PP, ids=[c[0] for c in PP])
def test_pingpong_block_vs_float64(case):
    _run_block(case, "tc")


def _block_inputs(C, E, gt, pc, B, T, seed):
    d0 = dev()
    g = torch.Generator(device=d0)
    g.manual_seed(seed)

    def rn(*shape, scale=1.0):
        return torch.randn(*shape, generator=g, device=d0, dtype=torch.float32) * scale

    w_conv = rn(2 * C, C, 3, scale=math.sqrt(2.0 / (3 * C)))
    w_cond = rn(2 * C, E, scale=math.sqrt(2.0 / E))
    b_sum = rn(2 * C, scale=0.1)
    w_out = rn(2 * C, C, scale=math.sqrt(2.0 / C))
    b_out = rn(2 * C, scale=0.1)
    d = rn(B, C, scale=0.5)
    perm = gate_perm(C, gt).to(d0)
    w1p = torch.cat([w_conv[:, :, 0], w_conv[:, :, 1], w_conv[:, :, 2], w_cond], dim=1)[perm].contiguous()
    s1, s2 = N.pow2_scale(w1p), N.pow2_scale(w_out)
    w1, w2 = N.pack_weight(w1p, pc, s1), N.pack_weight(w_out, pc, s2)
    dt = torch.float16 if pc == N.PREC_F16 else torch.bfloat16
    w1v = (w1[0].view(dt).double() + w1[1].view(dt).double()) / s1
    gb = [t.to(torch.float32).contiguous() for t in gate_bias_tables(d.double(), w1v, b_sum[perm].double())]
    return dict(w1=w1, w2=w2, s1=s1, s2=s2, gb=gb, b_out=b_out, x=rn(B, T, C), cond=rn(B, T, E), skip=rn(B, T, C))


def _run_items(inp, items, C, E, gt, prec, T, dil):
    """one middle-layer block over the items `items` of `inp` -> (z planes, x planes, skip) [*, len(items), ...]"""
    pc, mma = N.prec_code(prec), N.mma_code(prec)
    d0 = dev()
    idx = torch.tensor(items, device=d0)
    B = len(items)
    x_planes = N.split_nwc(inp["x"][idx].contiguous(), pc)
    cond_planes = N.split_nwc(inp["cond"][idx].contiguous(), pc)
    gb = [t[idx].contiguous() for t in inp["gb"]]
    skip = inp["skip"][idx].contiguous()
    z = torch.zeros((2, B, T, C), dtype=torch.int16, device=d0)
    skip_planes = torch.zeros((2, B, T, C), dtype=torch.int16, device=d0)
    N.check(N.lib().fd_wavenet_block_fwd(
        N.ptr(x_planes), N.ptr(cond_planes), N.ptr(z), N.ptr(inp["w1"]), N.ptr(inp["w2"]), N.ptr(gb[0]),
        N.ptr(gb[1]), N.ptr(gb[2]), 2 * C, N.ptr(inp["b_out"]), N.ptr(skip), N.ptr(skip_planes), 1.0, B, T, C, E,
        dil, gt, 1.0 / inp["s1"], 1.0 / inp["s2"], 0, mma, N.BACKEND_TC, N.stream_ptr(d0)), "fd_wavenet_block_fwd")
    torch.cuda.synchronize()
    return z, x_planes, skip


# (name, C, E, gate_tile, precision, T, dil): 3 tiles per item, so an item's tiles start at a different pair half and
# warpgroup at each batch position
PLACE = [
    ("place-c512-f16-T130-d8", 512, 256, 256, "f16", 130, 8),
    ("place-c192-bf16x1-T130-d2", 192, 64, 128, "bf16x1", 130, 2),
]


@pytest.mark.parametrize("case", PLACE, ids=[c[0] for c in PLACE])
def test_pingpong_item_bits_independent_of_placement(case):
    name, C, E, gt, prec, T, dil = case
    B = 5
    inp = _block_inputs(C, E, gt, N.prec_code(prec), B, T, zlib.crc32(name.encode()))
    batch = _run_items(inp, list(range(B)), C, E, gt, prec, T, dil)
    rev = _run_items(inp, list(range(B))[::-1], C, E, gt, prec, T, dil)
    for j in range(B):
        alone = _run_items(inp, [j], C, E, gt, prec, T, dil)
        for what, a, bt, rv in zip(("z", "x", "skip"), alone, batch, rev):
            a0 = a[:, 0] if what != "skip" else a[0]
            got = bt[:, j] if what != "skip" else bt[j]
            got_rev = rv[:, B - 1 - j] if what != "skip" else rv[B - 1 - j]
            assert torch.equal(a0, got), f"item {j}: {what} differs between B=1 and batch position {j}"
            assert torch.equal(a0, got_rev), f"item {j}: {what} differs between B=1 and batch position {B - 1 - j}"
