"""GPU parity of the WaveNet block backward against float64 (tests/wavenet_block_ref.py, whose closed forms are pinned to
autograd by test_wavenet_block_ref_cpu.py):

  * fd_wavenet_block_bwd, every raw output (dy, column / edge sums, gw2, gw1, dx planes and fp32 copy, d_cond,
    cs_dx), on both back ends, with the weights packed by fd_wavenet_pack_layers as training packs them,
  * fd_wavenet_pack_layers' forward and transposed packs, bit for bit against fd_pack_weight of the restated matrices,
  * the elementwise and reduction kernels of the training step (fd_colsum, fd_relu_bwd, fd_reduce_batch) at ragged
    shapes.

Each stage is judged on the operands the kernel read (its own planes, its own dy), so an error is pinned to the stage
that made it; one end-to-end comparison per case follows the reference's dy instead.  Inputs have the magnitudes of a
trained block (pre-activations of std 2, residual stream 1) and the incoming gradients carry S = 2^8 with inv_S = 2^-8:
a missing or doubled inv_S is a factor of 256.  Every output is prefilled with a sentinel (0x7FFF is a NaN in f16 and
bf16 planes, NaN in fp32) and every accumulated output with random values, so unwritten rows, columns or halves and an
overwrite instead of an accumulation show up.  Errors are reported per row region (first / last `dil` rows, last
128-row tile, interior) for [B, T, n] outputs, per column segment (tap -dil, tap 0, tap +dil, cond) for gw1 and per row
half for gw2.

Tolerances: (rel-L2, max|err| / RMS) bars, each at most 4x the largest value measured on an H100 80GB HBM3 over the
cases and back ends it covers; the measured value is written next to it.
"""
import ctypes
import math
import zlib

import pytest
import torch

from fish_diffusion_b200 import _native as N
from fish_diffusion_b200.wavenet import _gate_half
from gpu_util import dev
from region_check import F64, Regions, check_parts, pf64
from wavenet_block_ref import (block_bwd, bwd_col_sums, bwd_d_cond, bwd_dx, bwd_dz, bwd_gw1, bwd_gw2, gate_bwd,
                               gate_perm, gate_z)

pytestmark = pytest.mark.gpu

S = 2.0 ** 8
INV_S = 2.0 ** -8
SENTINEL = 0x7FFF
INV_SQRT2_F32 = 0.70710678118654752440

# (rel-L2, max) bars per quantity and precision class, each <= 4x the worst value measured over the cases and back ends
# that use it (in the comment).  Stage bars are on the kernel's own operands (dy: the reference's dz, which the fused
# epilogue never stores); *_e2e follow the reference's dy.
# Single product multiplies hi planes, whose products are exact in fp32: only the accumulation is left.
TOL = {
    # f16 (three products on 22-bit planes)
    ("dy", "f16"): (1.2e-5, 2.5e-4),      # measured 3.2e-6 / 6.8e-5
    ("cs", "f16"): (8e-7, 5e-6),          # measured 2.2e-7 / 1.4e-6
    ("gw2", "f16"): (1.6e-5, 8e-5),       # measured 4.3e-6 / 2.1e-5
    ("gw1", "f16"): (2.5e-5, 1.8e-4),     # measured 6.3e-6 / 4.6e-5
    ("dx", "f16"): (3e-5, 1.8e-4),        # measured 7.9e-6 / 4.6e-5 (planes and fp32 copy)
    ("d_cond", "f16"): (1.2e-5, 9e-5),    # measured 3.4e-6 / 2.4e-5
    ("cs_dx", "f16"): (9e-7, 5e-6),       # measured 2.3e-7 / 1.3e-6
    ("dy_e2e", "f16"): (1.2e-5, 2.5e-4),  # measured 3.2e-6 / 6.8e-5
    ("gw1_e2e", "f16"): (3.5e-5, 2.5e-4),  # measured 8.8e-6 / 6.4e-5
    ("dx_e2e", "f16"): (3.5e-5, 2.4e-4),  # measured 9.7e-6 / 6.0e-5
    # bf16 (three products on 16-bit planes)
    ("dy", "bf16"): (1.6e-5, 3.8e-4),     # measured 4.1e-6 / 9.7e-5
    ("cs", "bf16"): (1e-5, 6.5e-5),       # measured 2.7e-6 / 1.9e-5
    ("gw2", "bf16"): (4e-5, 2.5e-4),      # measured 1.1e-5 / 6.4e-5
    ("gw1", "bf16"): (4e-5, 2.7e-4),      # measured 1.1e-5 / 6.8e-5
    ("dx", "bf16"): (2.5e-5, 2e-4),       # measured 6.6e-6 / 5.2e-5
    ("d_cond", "bf16"): (1.2e-5, 8e-5),   # measured 3.2e-6 / 2.0e-5
    ("cs_dx", "bf16"): (4.8e-7, 2.8e-6),  # measured 1.2e-7 / 7.1e-7
    ("dy_e2e", "bf16"): (1.6e-5, 3.8e-4),  # measured 4.1e-6 / 9.7e-5
    ("gw1_e2e", "bf16"): (4.5e-5, 2.8e-4),  # measured 1.2e-5 / 7.2e-5
    ("dx_e2e", "bf16"): (3.4e-5, 2.4e-4),  # measured 8.5e-6 / 6.0e-5
    # single product, on the hi-plane values
    ("dy", "f16x1"): (4e-6, 7.5e-5),      # measured 1.1e-6 / 2.0e-5
    ("cs", "f16x1"): (8.5e-7, 5e-6),      # measured 2.2e-7 / 1.3e-6
    ("gw2", "f16x1"): (3.7e-6, 2.9e-5),   # measured 9.4e-7 / 7.4e-6
    ("gw1", "f16x1"): (3.8e-6, 3.7e-5),   # measured 9.5e-7 / 9.3e-6
    ("dx", "f16x1"): (2.5e-6, 1.5e-5),    # measured 6.4e-7 / 3.9e-6
    ("d_cond", "f16x1"): (4.7e-6, 3e-5),  # measured 1.2e-6 / 7.6e-6
    ("cs_dx", "f16x1"): (8.5e-7, 3.8e-6),  # measured 2.2e-7 / 9.6e-7
    ("dy", "bf16x1"): (9e-6, 8.5e-5),     # measured 2.4e-6 / 2.2e-5
    ("cs", "bf16x1"): (9e-6, 8.5e-5),     # measured 2.4e-6 / 2.3e-5
    ("gw2", "bf16x1"): (2.4e-8, 1e-6),    # measured 6.0e-9 / 2.6e-7 (T = 1 only)
    ("gw1", "bf16x1"): (5e-8, 3e-6),      # measured 1.3e-8 / 7.6e-7 (T = 1 only)
    ("dx", "bf16x1"): (9.5e-6, 5.4e-5),   # measured 2.4e-6 / 1.4e-5
    ("d_cond", "bf16x1"): (6e-7, 2.9e-6),  # measured 1.5e-7 / 7.4e-7
    ("cs_dx", "bf16x1"): (2.6e-7, 1.5e-6),  # measured 6.7e-8 / 4.0e-7
    # the reduction kernels alone
    ("k_colsum", "f16"): (8.5e-7, 9e-6),  # measured 2.2e-7 / 2.4e-6
    ("k_reduce", "f32"): (2.6e-7, 1.2e-6),  # measured 6.7e-8 / 3.1e-7
}


def _randn(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g, device=dev(), dtype=torch.float32) * scale


def pack_layers(conv_w, cond_w, out_w, s1, s2, pc, half, bwd=True):
    """fd_wavenet_pack_layers over L layers of raw parameters (conv [2C,C,3], conditioner [2C,E,1], output projection
    [2C,C,1]) at prescales s1 / s2 -> dict of the packs ([L, ...] each)."""
    L = len(conv_w)
    C, E = conv_w[0].shape[1], cond_w[0].shape[1]
    d0 = conv_w[0].device
    i16 = dict(dtype=torch.int16, device=d0)
    tab = torch.tensor([[t.data_ptr() for t in grp] for grp in (conv_w, cond_w, out_w)], dtype=torch.int64).to(d0)
    scales = torch.tensor(list(s1) + list(s2), dtype=torch.float32, device=d0)
    KT = 3 * C + E
    pk = {"w1p_f32": torch.empty((L, 2 * C, KT), dtype=torch.float32, device=d0),
          "w1": torch.empty((L, 2, 2 * C, KT), **i16), "w2": torch.empty((L, 2, 2 * C, C), **i16),
          "w1t": torch.empty((L, 2, C, 6 * C), **i16) if bwd else None,
          "wct": torch.empty((L, 2, E, 2 * C), **i16) if bwd else None,
          "w2t": torch.empty((L, 2, C, 2 * C), **i16) if bwd else None}
    N.check(N.lib().fd_wavenet_pack_layers(N.ptr(tab[0]), N.ptr(tab[1]), N.ptr(tab[2]), N.ptr(scales),
                                           *[N.ptr(pk[k]) for k in ("w1p_f32", "w1", "w2", "w1t", "wct", "w2t")],
                                           L, C, E, half, pc, N.stream_ptr(d0)), "fd_wavenet_pack_layers")
    return pk


# ---------------------------------------------------------------------------------------------- fd_wavenet_block_bwd
# (name, C, E, gate_tile, precision, B, T, dil, top layer, dx_f32 + d_cond given, splits1 / splits2)
#   splits: an int, "B" (one item per split) or None (N.wgrad_splits, as training chooses them)
BWD = [
    ("c512-f16-B2-T1000-d8-mid", 512, 256, 256, "f16", 2, 1000, 8, False, True, "B"),
    ("c512-bf16-B5-T77-d64-top-s2", 512, 256, 256, "bf16", 5, 77, 64, True, False, 2),          # 3 + 2 items
    ("c512-f16x1-B3-T50-d64-mid-s1", 512, 256, 256, "f16x1", 3, 50, 64, False, True, 1),         # dil >= T
    ("c192-f16-B7-T50-d64-mid-s3", 192, 64, 128, "f16", 7, 50, 64, False, True, 3),              # 3 + 3 + 1 items
    ("c192-bf16x1-B2-T1-d64-top", 192, 64, 128, "bf16x1", 2, 1, 64, True, False, "B"),
    ("c192-bf16-B3-T1000-d8-top-s1", 192, 64, 128, "bf16", 3, 1000, 8, True, True, 1),
    ("c128-f16x1-B3-T77-d64-mid", 128, 64, 256, "f16x1", 3, 77, 64, False, True, "B"),           # T < 2 dil
    ("c128-bf16-B5-T1000-d8-mid-s2", 128, 64, 256, "bf16", 5, 1000, 8, False, False, 2),
    ("c128-f16-B2-T1-d8-mid", 128, 64, 256, "f16", 2, 1, 8, False, False, 1),
    # SIMT-only width (C, E not multiples of 64; gate tile 32)
    ("c80-f16-B2-T77-d64-mid", 80, 40, 32, "f16", 2, 77, 64, False, True, "B"),
    ("c80-bf16-B5-T50-d64-top-s2", 80, 40, 32, "bf16", 5, 50, 64, True, False, 2),
    ("c80-f16x1-B7-T1000-d8-mid-s3", 80, 40, 32, "f16x1", 7, 1000, 8, False, True, 3),
    ("c80-bf16x1-B2-T1-d8-top", 80, 40, 32, "bf16x1", 2, 1, 8, True, True, 1),
]
# production shape: wgrad_splits gives splits1 = 11 (three items each, two in the last)
BWD_PROD = ("c512-f16-B32-T600-d8-mid-prod", 512, 256, 256, "f16", 32, 600, 8, False, True, None)


def _run_block_bwd(case, backend):
    name, C, E, gt, prec, B, T, dil, top, outs, splits = case
    pc, mma, bk = N.prec_code(prec), N.mma_code(prec), N.backend_code(backend)
    single = prec.endswith("x1")
    KT = 3 * C + E
    d0 = dev()
    g = torch.Generator(device=d0)
    g.manual_seed(zlib.crc32(name.encode()))
    i16 = dict(dtype=torch.int16, device=d0)
    f32 = dict(dtype=torch.float32, device=d0)

    # weights, packed as training packs them (L = 1)
    w_conv = _randn(g, 2 * C, C, 3, scale=math.sqrt(2.0 / (3 * C)))
    w_cond = _randn(g, 2 * C, E, 1, scale=math.sqrt(2.0 / E))
    w_out = _randn(g, 2 * C, C, 1, scale=math.sqrt(2.0 / C))
    s1 = N.pow2_scale(torch.cat([w_conv.flatten(), w_cond.flatten()]))
    s2 = N.pow2_scale(w_out)
    pk = pack_layers([w_conv], [w_cond], [w_out], [s1], [s2], pc, gt // 2)
    w1t, wct, w2t = pk["w1t"][0], pk["wct"][0], pk["w2t"][0]

    # saved activations and incoming gradients (S-scaled)
    x = N.split_nwc(_randn(g, B, T, C), pc)
    cond = N.split_nwc(_randn(g, B, T, E), pc)
    y_f32 = _randn(g, B, T, 2 * C, scale=2.0)
    y = N.split_nwc(y_f32, pc)
    z = N.split_nwc(gate_z(y_f32.to(F64), C, gt).to(torch.float32), pc)
    dskip = N.split_nwc(_randn(g, B, T, C, scale=S), pc)
    dxn = None if top else N.split_nwc(_randn(g, B, T, C, scale=S), pc)

    # outputs: sentinels; accumulated outputs prefilled with random values
    nan = float("nan")
    dy = torch.full((2, B, T, 2 * C), SENTINEL, **i16)
    dx = torch.full((2, B, T, C), SENTINEL, **i16)
    dx_f32 = torch.full((B, T, C), nan, **f32) if outs else None
    d_cond0 = _randn(g, B, T, E)
    d_cond = d_cond0.clone() if outs else None
    gw1 = torch.full((2 * C, KT), nan, **f32)
    gw2 = torch.full((2 * C, C), nan, **f32)
    cs_dy0, cs_edge0, cs_dx0 = _randn(g, B, 2 * C), _randn(g, 2, B, 2 * C), _randn(g, B, C)
    cs_dy, cs_edge, cs_dx = cs_dy0.clone(), cs_edge0.clone(), cs_dx0.clone()
    if splits is None:
        splits1, splits2 = N.wgrad_splits(2 * C, KT, B, T), N.wgrad_splits(2 * C, C, B, T)
    else:
        splits1 = splits2 = B if splits == "B" else splits
    part1 = torch.full((splits1, 2 * C, KT), nan, **f32)
    part2 = torch.full((splits2, 2 * C, C), nan, **f32)

    bd = N.WaveNetBwdDesc()
    bd.x_planes, bd.y_planes, bd.z_planes, bd.cond_planes = N.ptr(x), N.ptr(y), N.ptr(z), N.ptr(cond)
    bd.dx_next, bd.dskip = N.ptr(dxn), N.ptr(dskip)
    bd.w2t, bd.w1t, bd.wct = N.ptr(w2t), N.ptr(w1t), N.ptr(wct)
    bd.w2t_inv, bd.w1t_inv, bd.wct_inv = 1.0 / s2, 1.0 / s1, 1.0 / s1
    bd.dx_out, bd.dx_f32, bd.d_cond, bd.gw1, bd.gw2 = N.ptr(dx), N.ptr(dx_f32), N.ptr(d_cond), N.ptr(gw1), N.ptr(gw2)
    bd.cs_dy, bd.cs_edge, bd.cs_dx, bd.dy = N.ptr(cs_dy), N.ptr(cs_edge), N.ptr(cs_dx), N.ptr(dy)
    bd.part1, bd.part2, bd.splits1, bd.splits2 = N.ptr(part1), N.ptr(part2), splits1, splits2
    bd.B, bd.T, bd.C, bd.E, bd.dilation, bd.gate_tile = B, T, C, E, dil, gt
    bd.inv_S, bd.prec, bd.backend = INV_S, mma, bk
    N.check(N.lib().fd_wavenet_block_bwd(ctypes.byref(bd), N.stream_ptr(d0)), "fd_wavenet_block_bwd")
    torch.cuda.synchronize()

    # ---- operands as the kernels read them: single product multiplies the hi planes, epilogues read full values
    op = lambda t, s=1.0: None if t is None else pf64(t, pc, single) / s
    xv, cv, zv, dskv, dxnv = op(x), op(cond), op(z), op(dskip), op(dxn)
    yv = pf64(y, pc)
    dxn_full = None if top else pf64(dxn, pc)
    w2tv = op(w2t, s2)                                                   # [C, 2C], 1/sqrt2 on the residual half
    w1t_v, wct_v = op(w1t, s1), op(wct, s1)                              # [C, 6C], [E, 2C]
    w1p_v = torch.cat([w1t_v[:, j * 2 * C:(j + 1) * 2 * C].T for j in range(3)] + [wct_v.T], dim=1)   # [2C, KT]
    dy_k, dy_op = pf64(dy, pc), op(dy)
    dx_k = pf64(dx, pc)

    print(f"\n[{name} {backend}] splits {splits1}/{splits2}")
    bad = []

    def tol(k):
        return TOL[(k, prec)]

    def regions(what, got, ref, key=None):
        r = Regions(T, dil, d0)
        r.add(got, ref)
        return r.check(what, tol(key or what))

    def sums(what, got, ref):
        return check_parts(what, got, ref, {}, tol("cs"))

    bad += regions("dy", dy_k, gate_bwd(bwd_dz(dxnv, dskv, w2tv), yv, gt))     # GATE_BWD epilogue of the dz GEMM
    cs_ref, ce_ref = bwd_col_sums(dy_k, dil, INV_S)
    bad += sums("cs_dy", (cs_dy - cs_dy0).to(F64), cs_ref)
    bad += sums("cs_edge_lo", (cs_edge[0] - cs_edge0[0]).to(F64), ce_ref[0])
    bad += sums("cs_edge_hi", (cs_edge[1] - cs_edge0[1]).to(F64), ce_ref[1])
    if top:
        assert bool((gw2[:C] == 0).all()), "top layer: the residual half of gw2 must be exactly 0"
    bad += check_parts("gw2", gw2.to(F64), bwd_gw2(dxnv, dskv, zv, INV_S), {"res": slice(0, C), "skip": slice(C, None)},
                       tol("gw2"))
    gw1_ref = bwd_gw1(dy_op, xv, cv, dil, INV_S)
    segs = {"tap-dil": (slice(None), slice(0, C)), "tap0": (slice(None), slice(C, 2 * C)),
            "tap+dil": (slice(None), slice(2 * C, 3 * C)), "cond": (slice(None), slice(3 * C, None))}
    bad += check_parts("gw1", gw1.to(F64), gw1_ref, segs, tol("gw1"))
    dx_ref = bwd_dx(dy_op, w1p_v, dxn_full, dil)
    bad += regions("dx", dx_k, dx_ref)
    if outs:
        bad += regions("dx_f32", dx_f32.to(F64), dx_ref, key="dx")
        bad += regions("d_cond", (d_cond - d_cond0).to(F64), bwd_d_cond(dy_op, w1p_v, INV_S))
    bad += sums("cs_dx", (cs_dx - cs_dx0).to(F64), dx_k.sum(1) * INV_S)
    if not single:
        # end to end: every stage on the reference's dy
        ref = block_bwd(xv, cv, yv, zv, dxn_full, dskv, w1p_v, w2tv, gt, dil, INV_S)
        bad += regions("dy_e2e", dy_k, ref["dy"])
        bad += check_parts("gw1_e2e", gw1.to(F64), ref["gw1"], segs, tol("gw1_e2e"))
        bad += regions("dx_e2e", dx_k, ref["dx"])
    assert not bad, "; ".join(bad)


def _bwd_params():
    out = []
    for c in BWD:
        tc_ok = c[1] % 64 == 0 and c[2] % 64 == 0
        out += [pytest.param(c, b, id=f"{c[0]}-{b}") for b in (("tc", "simt") if tc_ok else ("simt",))]
    return out


@pytest.mark.parametrize("case,backend", _bwd_params())
def test_block_bwd_vs_float64(case, backend):
    _run_block_bwd(case, backend)


def test_block_bwd_production_splits_vs_float64():
    """C=512, B=32, T=600 on the tensor cores with the weight-gradient splits training uses: 11 partials of 3 items,
    the last of 2."""
    C, E, B, T = BWD_PROD[1], BWD_PROD[2], BWD_PROD[5], BWD_PROD[6]
    assert N.wgrad_splits(2 * C, 3 * C + E, B, T) == 11 and -(-B // 11) == 3
    _run_block_bwd(BWD_PROD, "tc")


# ---------------------------------------------------------------------------------------------- fd_wavenet_pack_layers
@pytest.mark.parametrize("prec", ["f16", "bf16"])
@pytest.mark.parametrize("C,E", [(512, 256), (192, 64), (80, 40)])
def test_pack_layers_bitwise(C, E, prec):
    """Forward packs, the fp32 copy and the transposed packs of L = 3 layers (each at its own power-of-two scales)
    equal fd_pack_weight of the restated fp32 matrices bit for bit: w1t [C][6C] = the three [2C, C] taps transposed
    side by side, wct [E][2C] = the conditioner block transposed, w2t [C][2C] = W2^T with 1/sqrt2 on the residual half
    ((w s) / sqrt2 = (w / sqrt2) s exactly: s is a power of two)."""
    L, pc, half = 3, N.prec_code(prec), _gate_half(C)
    d0 = dev()
    g = torch.Generator(device=d0)
    g.manual_seed(C * 7 + E + pc)
    conv = [_randn(g, 2 * C, C, 3, scale=0.05 * 8 ** l) for l in range(L)]
    cond = [_randn(g, 2 * C, E, 1, scale=0.1 * 8 ** l) for l in range(L)]
    out = [_randn(g, 2 * C, C, 1, scale=0.07 / 8 ** l) for l in range(L)]
    s1 = [N.pow2_scale(torch.cat([conv[l].flatten(), cond[l].flatten()])) for l in range(L)]
    s2 = [N.pow2_scale(out[l]) for l in range(L)]
    assert len(set(s1)) == L and len(set(s2)) == L
    pk = pack_layers(conv, cond, out, s1, s2, pc, half)
    torch.cuda.synchronize()
    perm = gate_perm(C, 2 * half).to(d0)
    r = torch.tensor(INV_SQRT2_F32, dtype=torch.float32, device=d0)
    for l in range(L):
        w1p = torch.cat([conv[l][:, :, 0], conv[l][:, :, 1], conv[l][:, :, 2], cond[l][:, :, 0]], dim=1)[perm]
        w2 = out[l][:, :, 0]
        want = {"w1p_f32": w1p, "w1": N.pack_weight(w1p, pc, s1[l]), "w2": N.pack_weight(w2, pc, s2[l]),
                "w1t": N.pack_weight(torch.cat([w1p[:, j * C:(j + 1) * C].T for j in range(3)], dim=1), pc, s1[l]),
                "wct": N.pack_weight(w1p[:, 3 * C:].T, pc, s1[l]),
                "w2t": N.pack_weight(torch.cat([w2[:C].T * r, w2[C:].T], dim=1), pc, s2[l])}
        for k, v in want.items():
            assert torch.equal(pk[k][l], v), f"layer {l}: {k} differs from the restated pack"


def test_pack_layers_refuses_partial_transposed_packs():
    """The transposed packs come all or none: a call with some of them is refused before any launch."""
    C, E = 128, 64
    d0 = dev()
    conv, cond, out = (torch.zeros(2 * C, C, 3, device=d0), torch.zeros(2 * C, E, 1, device=d0),
                       torch.zeros(2 * C, C, 1, device=d0))
    tab = torch.tensor([[conv.data_ptr()], [cond.data_ptr()], [out.data_ptr()]], dtype=torch.int64).to(d0)
    scales = torch.ones(2, device=d0)
    w1p = torch.empty((2 * C, 3 * C + E), device=d0)
    w1 = torch.full((2, 2 * C, 3 * C + E), SENTINEL, dtype=torch.int16, device=d0)
    w2 = torch.full((2, 2 * C, C), SENTINEL, dtype=torch.int16, device=d0)
    w1t = torch.empty((2, C, 6 * C), dtype=torch.int16, device=d0)
    wct = torch.empty((2, E, 2 * C), dtype=torch.int16, device=d0)
    w2t = torch.empty((2, C, 2 * C), dtype=torch.int16, device=d0)
    lib = N.lib()
    for t1, tc, t2 in ((w1t, None, None), (None, wct, w2t), (w1t, wct, None)):
        rc = lib.fd_wavenet_pack_layers(N.ptr(tab[0]), N.ptr(tab[1]), N.ptr(tab[2]), N.ptr(scales), N.ptr(w1p),
                                        N.ptr(w1), N.ptr(w2), N.ptr(t1), N.ptr(tc), N.ptr(t2), 1, C, E, 128,
                                        N.PREC_F16, N.stream_ptr(d0))
        assert rc != 0 and "all or none" in N.last_error(), N.last_error()
    torch.cuda.synchronize()
    assert bool((w1 == SENTINEL).all()) and bool((w2 == SENTINEL).all()), "a refused call launched"


# ---------------------------------------------------------------------------- elementwise and reduction kernels
@pytest.mark.parametrize("src", ["planes", "f32"])
@pytest.mark.parametrize("B,T,Nn", [(3, 300, 200), (2, 1, 64), (1, 129, 1000)])
def test_colsum_kernel_vs_float64(B, T, Nn, src):
    """fd_colsum: per-item column sums accumulated into the output (prefilled), T and N not multiples of 128."""
    d0 = dev()
    g = torch.Generator(device=d0)
    g.manual_seed(B * T + Nn)
    a = _randn(g, B, T, Nn, scale=S)
    pl = N.split_nwc(a, N.PREC_F16)
    v = pf64(pl, N.PREC_F16) if src == "planes" else a.to(F64)
    out0 = _randn(g, B, Nn)
    out = out0.clone()
    N.check(N.lib().fd_colsum(N.ptr(pl if src == "planes" else None), N.ptr(a if src == "f32" else None), N.ptr(out),
                              B, T, Nn, INV_S, N.PREC_F16, N.stream_ptr(d0)), "fd_colsum")
    torch.cuda.synchronize()
    print(f"\n[colsum B={B} T={T} N={Nn} {src}]")
    bad = check_parts("colsum", (out - out0).to(F64), v.sum(1) * INV_S, {}, TOL[("k_colsum", "f16")])
    assert not bad, "; ".join(bad)


@pytest.mark.parametrize("prec", ["f16", "bf16"])
def test_relu_bwd_kernel_bitwise(prec):
    """fd_relu_bwd: planes of grad * scale where the activation is > 0, exactly 0 where it is 0, -0 or negative; equal
    bit for bit to the split of that fp32 value."""
    pc = N.prec_code(prec)
    d0 = dev()
    g = torch.Generator(device=d0)
    g.manual_seed(11 + pc)
    n = 4 * 1037
    a = _randn(g, 1, 1, n)
    kind = torch.randint(0, 4, (n,), generator=g, device=d0)
    a[0, 0, kind == 0] = 0.0
    a[0, 0, kind == 1] = -0.0
    act = N.split_nwc(a, pc)
    grad = _randn(g, n, scale=S)
    out = torch.full((2, n), SENTINEL, dtype=torch.int16, device=d0)
    N.check(N.lib().fd_relu_bwd(N.ptr(grad), N.ptr(act), N.ptr(out), n, 0.5, pc, N.stream_ptr(d0)), "fd_relu_bwd")
    torch.cuda.synchronize()
    keep = pf64(act, pc)[0, 0] > 0
    assert int((~keep).sum()) > n // 3
    want = N.split_nwc(torch.where(keep, grad * 0.5, torch.zeros_like(grad)).view(1, 1, n), pc).view(2, n)
    assert torch.equal(out, want)
    assert bool((out[:, ~keep] == 0).all()), "masked entries must be +0 in both planes"


@pytest.mark.parametrize("B,n", [(1, 1000), (5, 777), (11, 256 * 3 + 5)])
def test_reduce_batch_kernel_vs_float64(B, n):
    """fd_reduce_batch: scale * sum over B partials, B = 1 and n not a multiple of the 256-thread block."""
    d0 = dev()
    g = torch.Generator(device=d0)
    g.manual_seed(B * n)
    part = _randn(g, B, n, scale=S)
    out = torch.full((n,), float("nan"), dtype=torch.float32, device=d0)
    N.check(N.lib().fd_reduce_batch(N.ptr(part), N.ptr(out), B, n, INV_S, N.stream_ptr(d0)), "fd_reduce_batch")
    torch.cuda.synchronize()
    if B == 1:
        assert torch.equal(out, part[0] * INV_S)
    print(f"\n[reduce_batch B={B} n={n}]")
    bad = check_parts("reduce", out.to(F64), part.to(F64).sum(0) * INV_S, {}, TOL[("k_reduce", "f32")])
    assert not bad, "; ".join(bad)
