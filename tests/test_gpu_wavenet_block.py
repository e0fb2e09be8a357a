"""GPU parity of the WaveNet block GEMMs against a float64 restatement of the block (tests/wavenet_block_ref.py, pinned
to the oracle by test_wavenet_block_ref_cpu.py):

  * GEMM1 + GATE epilogue (dilated conv + conditioner + per-item or shared gate bias with its zero-padding
    corrections, z = sigmoid * tanh, pre-activations y in packed order when training),
  * GEMM2 + RES_SKIP epilogue (x' = (x + r)/sqrt2, skip accumulation, last-layer skip planes * skip_scale),
  * the dz GEMM + GATE_BWD epilogue of the backward (dy, column sums and edge sums) on both back ends,
  * the gate-bias tables (fd_wavenet_gate_bias / _from_d).

Every reference runs on the exact operand values the kernel read (split planes, fp32 bias tables), in torch float64
on the GPU.  GEMM2 is judged on the kernel's own z, so each GEMM is checked in isolation; one end-to-end comparison
follows the reference's z instead.  Errors are reported per row region -- the first / last `dil` rows (edge
corrections), the last (ragged) 128-row tile, and the interior -- since a one-row error vanishes in a whole-tensor
rel-L2.  "max" is max|err| in units of the whole tensor's RMS.

Tolerances: f16 planes carry 22-bit values and bf16 planes 16-bit ones (2.4e-7 / 7.6e-6 relative per stored value);
the GEMMs accumulate in fp32 on the tensor cores (truncating adds over K = 3C+E up to 1792); fd_sigmoid / fd_tanh use
__expf (a few ulp).  So ~1e-6..1e-5 (f16) and ~1e-5..1e-4 (bf16).  The measured value (H100 80GB HBM3) of each bar is
written next to it; no bar is more than 4x the largest value measured across the cases it covers.
"""
import math
import zlib

import pytest
import torch

from fish_diffusion_b200 import _native as N
from gpu_util import dev
from region_check import F64, Regions, pf64
from wavenet_block_ref import gate_bias_tables, gate_bwd, gate_perm, gate_pre_packed, gate_z, res_skip

pytestmark = pytest.mark.gpu

SKIP_SCALE = 1.0 / math.sqrt(20.0)

# (rel-L2, max) bars per quantity and precision class, each <= 4x the worst value measured over the cases and back ends
# that use it (in the comment).  The tensor-core back end is the worse one: its fp32 accumulation truncates, and over
# K = 3C+E = 1792 (C=512) that gives ~5e-6 rel-L2 whatever the plane precision; the SIMT twin stays below 1e-6 in f16.
TOL = {
    # f16 (three products on 22-bit planes)
    ("y", "f16"): (1.5e-5, 1e-4),         # measured 4.6e-6 / 2.8e-5
    ("z", "f16"): (1.5e-5, 2.5e-4),        # measured 5.0e-6 / 8.5e-5
    ("x", "f16"): (3e-6, 3e-5),            # measured 1.0e-6 / 8.7e-6
    ("skip", "f16"): (5e-6, 4e-5),         # measured 1.8e-6 / 1.1e-5
    ("x_e2e", "f16"): (1e-5, 6e-5),        # measured 3.2e-6 / 2.0e-5
    ("skip_e2e", "f16"): (1e-5, 6e-5),     # measured 3.3e-6 / 1.9e-5
    # bf16 (three products on 16-bit planes)
    ("y", "bf16"): (1.5e-5, 1.5e-4),       # measured 5.6e-6 / 4.5e-5
    ("z", "bf16"): (2e-5, 2e-4),           # measured 6.4e-6 / 6.8e-5
    ("x", "bf16"): (1e-5, 1e-4),           # measured 3.0e-6 / 3.5e-5
    ("skip", "bf16"): (1.2e-5, 1e-4),      # measured 4.0e-6 / 3.0e-5
    ("x_e2e", "bf16"): (1.5e-5, 1.2e-4),   # measured 4.8e-6 / 3.6e-5
    ("skip_e2e", "bf16"): (2e-5, 1.2e-4),  # measured 6.7e-6 / 3.5e-5
    # single product, on the hi-plane values
    ("z", "f16x1"): (5e-6, 5e-5),          # measured 1.7e-6 / 1.7e-5
    ("x", "f16x1"): (6e-7, 5e-6),          # measured 2.1e-7 / 1.5e-6
    ("skip", "f16x1"): (1.2e-6, 8e-6),     # measured 3.8e-7 / 2.5e-6
    ("y", "bf16x1"): (8e-6, 1e-4),         # measured 2.8e-6 / 3.4e-5
    ("z", "bf16x1"): (8e-6, 6e-5),         # measured 2.6e-6 / 1.9e-5
    ("x", "bf16x1"): (8e-6, 6e-5),         # measured 2.6e-6 / 1.8e-5
    ("skip", "bf16x1"): (8e-6, 8e-5),      # measured 2.5e-6 / 2.8e-5
    # gate backward: dz (same GEMM, linear epilogue), dy, column / edge sums
    ("dz", "f16"): (1e-5, 8e-5),           # measured 3.6e-6 / 2.5e-5
    ("dy", "f16"): (1e-5, 3e-4),           # measured 3.6e-6 / 9.2e-5
    ("cs", "f16"): (1e-5, 8e-5),           # measured 3.7e-6 / 2.9e-5
    ("dz", "bf16"): (1e-5, 8e-5),          # measured 3.2e-6 / 2.1e-5
    ("dy", "bf16"): (1.2e-5, 4e-4),        # measured 4.1e-6 / 1.2e-4
    ("cs", "bf16"): (1e-5, 1.2e-4),        # measured 3.3e-6 / 4.1e-5
    ("dz", "bf16x1"): (1.5e-6, 1.2e-5),    # measured 4.8e-7 / 3.4e-6
    ("dy", "bf16x1"): (8e-6, 2.5e-4),      # measured 2.6e-6 / 7.1e-5
    ("cs", "bf16x1"): (1.6e-6, 1.5e-5),    # measured 5.4e-7 / 4.1e-6
}
# single product against the FULL plane values: the half-precision rounding of both operands must show
# (lower bound: it really is one product) and stay at that level (upper bound)
X1_DEV = {"f16x1": (5e-5, 1e-3), "bf16x1": (5e-4, 8e-3)}   # measured 3.8e-4..4.0e-4 / 3.1e-3


def rel_l2(a, b):
    return float(torch.linalg.vector_norm(a - b) / max(float(torch.linalg.vector_norm(b)), 1e-300))


def _randn(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g, device=dev(), dtype=torch.float32) * scale


# ---------------------------------------------------------------------------------------------- forward block
# (name, C, E, gate_tile, precision, B, T, dil, flags, per_item_bias, train)
#   flags: 1 first layer (skip written), 0 middle (skip accumulated), 2 last (skip planes * skip_scale), 3 single layer
FWD = [
    ("c512-f16-T77-d64-first", 512, 256, 256, "f16", 2, 77, 64, 1, False, False),          # T < 2 dil
    ("c512-bf16-T129-d8-mid-train", 512, 256, 256, "bf16", 3, 129, 8, 0, True, True),
    ("c512-f16x1-T128-d1-last", 512, 256, 256, "f16x1", 2, 128, 1, 2, False, False),
    ("c512-bf16x1-T1000-d64-single-train", 512, 256, 256, "bf16x1", 2, 1000, 64, 3, True, True),
    ("c512-f16-T1000-d200-last-train", 512, 256, 256, "f16", 2, 1000, 200, 2, True, True),
    ("c256-f16-T1000-d8-last-train", 256, 64, 256, "f16", 2, 1000, 8, 2, True, True),
    ("c256-bf16-T1-d1-first", 256, 64, 256, "bf16", 3, 1, 1, 1, False, False),              # dil >= T
    ("c256-f16x1-T129-d64-mid", 256, 64, 256, "f16x1", 2, 129, 64, 0, True, False),
    ("c128-f16-T77-d100-mid", 128, 64, 128, "f16", 2, 77, 100, 0, True, False),            # dil > T
    ("c128-bf16-T129-d64-single-train", 128, 64, 128, "bf16", 2, 129, 64, 3, False, True),
    ("c128-bf16x1-T77-d8-first-train", 128, 64, 128, "bf16x1", 2, 77, 8, 1, True, True),
    ("c192-f16-T129-d64-mid-train", 192, 64, 128, "f16", 2, 129, 64, 0, True, True),
    ("c192-bf16-T1000-d1-last", 192, 64, 128, "bf16", 2, 1000, 1, 2, False, False),
    ("c192-f16x1-T77-d8-first", 192, 64, 128, "f16x1", 3, 77, 8, 1, False, False),
]
# the persistent multi-tile loop: training shape with per-item gate bias (~8 tiles per CTA), sampler shape (~31).
# The per-item bias vectors are re-staged only when a CTA's next tile has another (item, column tile) key; with one or
# two gate column tiles (C=128 / 256) a CTA meets the same columns of another item back to back, which a key that
# ignored the item would get wrong (with four, at C=512 on 132 SMs, consecutive tiles always change columns).
FWD_LARGE = [
    ("c512-f16-B32-T1000-d8-mid-train-item", 512, 256, 256, "f16", 32, 1000, 8, 0, True, True),
    ("c512-f16-B32-T4000-d64-mid-shared", 512, 256, 256, "f16", 32, 4000, 64, 0, False, False),
    ("c256-bf16-B32-T1000-d64-last-train-item", 256, 64, 256, "bf16", 32, 1000, 64, 2, True, True),
    ("c128-f16-B20-T1000-d2-first-item", 128, 64, 256, "f16", 20, 1000, 2, 1, True, False),
]


def _run_block(case, backend):
    name, C, E, gt, prec, B, T, dil, flags, per_item, train = case
    pc, mma, bk = N.prec_code(prec), N.mma_code(prec), N.backend_code(backend)
    single = prec.endswith("x1")
    d0 = dev()
    g = torch.Generator(device=d0)
    g.manual_seed(zlib.crc32(name.encode()))
    i16 = dict(dtype=torch.int16, device=d0)
    # inputs (magnitudes of a trained block: pre-activations of std ~2, residual stream ~1)
    w_conv = _randn(g, 2 * C, C, 3, scale=math.sqrt(2.0 / (3 * C)))
    w_cond = _randn(g, 2 * C, E, scale=math.sqrt(2.0 / E))
    b_sum = _randn(g, 2 * C, scale=0.1)
    w_out = _randn(g, 2 * C, C, scale=math.sqrt(2.0 / C))
    b_out = _randn(g, 2 * C, scale=0.1)
    Bd = B if per_item else 1
    d = _randn(g, Bd, C, scale=0.5)
    x = _randn(g, B, T, C)
    cond = _randn(g, B, T, E)
    skip_prev = _randn(g, B, T, C)

    perm = gate_perm(C, gt).to(d0)
    w1p_f32 = torch.cat([w_conv[:, :, 0], w_conv[:, :, 1], w_conv[:, :, 2], w_cond], dim=1)[perm].contiguous()
    s1, s2 = N.pow2_scale(w1p_f32), N.pow2_scale(w_out)
    w1 = N.pack_weight(w1p_f32, pc, s1)
    w2 = N.pack_weight(w_out, pc, s2)
    x_planes, cond_planes = N.split_nwc(x, pc), N.split_nwc(cond, pc)
    w1v, w2v = pf64(w1, pc) / s1, pf64(w2, pc) / s2
    # gate-bias tables from the packed weights the kernel multiplies with, in float64, stored as float32
    gb = [t.to(torch.float32).contiguous() for t in gate_bias_tables(d.to(F64), w1v, b_sum[perm].to(F64))]

    x_in = x_planes.clone()
    z_planes = torch.zeros((2, B, T, C), **i16)
    skip_f32 = skip_prev.clone() if not flags & 1 else torch.full((B, T, C), 1e3, dtype=torch.float32, device=d0)
    skip_planes = torch.zeros((2, B, T, C), **i16)
    x_out = torch.full((2, B, T, C), 0x1234, **i16) if train else None
    y_planes = torch.zeros((2, B, T, 2 * C), **i16) if train else None
    args = (N.ptr(w1), N.ptr(w2), N.ptr(gb[0]), N.ptr(gb[1]), N.ptr(gb[2]), 2 * C if per_item else 0,
            N.ptr(b_out), N.ptr(skip_f32), N.ptr(skip_planes), SKIP_SCALE, B, T, C, E, dil, gt, 1.0 / s1, 1.0 / s2,
            flags, mma, bk, N.stream_ptr(d0))
    lib = N.lib()
    if train:
        N.check(lib.fd_wavenet_block_fwd_train(N.ptr(x_planes), N.ptr(x_out), N.ptr(cond_planes), N.ptr(z_planes),
                                               N.ptr(y_planes), *args), "fd_wavenet_block_fwd_train")
    else:
        N.check(lib.fd_wavenet_block_fwd(N.ptr(x_planes), N.ptr(cond_planes), N.ptr(z_planes), *args),
                "fd_wavenet_block_fwd")
    torch.cuda.synchronize()

    # ---- bit-exact bookkeeping
    last = bool(flags & 2)
    if train:
        assert torch.equal(x_planes, x_in), "training forward changed its input residual planes"
        x_new = x_out
        if last:
            assert bool((x_out == 0x1234).all()), "last layer wrote the residual output"
    else:
        x_new = x_planes
        if last:
            assert torch.equal(x_planes, x_in), "last layer changed the residual planes"

    # ---- float64 references, item chunk by item chunk.  Single product: the GEMM operands are the hi planes (the
    #      epilogues still read x and the bias tables at full precision); a second GEMM1 reference on the full values
    #      shows the reduced arithmetic.  The end-to-end check needs z at full precision, so it runs for three products.
    keys = ["z", "x", "skip"] + ([] if single else ["x_e2e", "skip_e2e"]) + (["y"] if train else [])
    reg = {k: Regions(T, dil, d0) for k in keys}
    full_z = Regions(T, dil, d0)
    b_out64 = b_out.to(F64)
    cb = max(1, 32000 // T)
    for b0 in range(0, B, cb):
        sl = slice(b0, min(B, b0 + cb))
        gbs = [t[sl if per_item else slice(0, 1)].to(F64) for t in gb]
        x_full = pf64(x_in[:, sl], pc)
        z_got = pf64(z_planes[:, sl], pc)
        y_ref = gate_pre_packed(pf64(x_in[:, sl], pc, single), pf64(cond_planes[:, sl], pc, single),
                                (pf64(w1, pc, True) / s1) if single else w1v, *gbs, dil)
        if train:
            reg["y"].add(pf64(y_planes[:, sl], pc), y_ref)
        z_ref = gate_z(y_ref, C, gt)
        del y_ref
        reg["z"].add(z_got, z_ref)
        if single:
            full_z.add(z_got, gate_z(gate_pre_packed(x_full, pf64(cond_planes[:, sl], pc), w1v, *gbs, dil), C, gt))
        # GEMM2 on the kernel's own z (as the kernel read it), and end to end on the reference's z
        w2u = (pf64(w2, pc, True) / s2) if single else w2v
        for tag, zz in (("", pf64(z_planes[:, sl], pc, single)),) + ((("_e2e", z_ref),) if not single else ()):
            xr, sk = res_skip(x_full, zz, w2u, b_out64)
            if not flags & 1:
                sk = sk + skip_prev[sl].to(F64)
            if last:
                reg["skip" + tag].add(pf64(skip_planes[:, sl], pc), sk * SKIP_SCALE)
            else:
                reg["skip" + tag].add(skip_f32[sl].to(F64), sk)
                reg["x" + tag].add(pf64(x_new[:, sl], pc), xr)
    print(f"\n[{name} {backend}]")
    bad = []
    for k in keys:
        if reg[k].n_all:
            bad += reg[k].check(k, TOL[(k, prec)])
    if single:
        # it really is the reduced arithmetic: against the full values the deviation is the half-precision level
        dev_full = math.sqrt(full_z.se["all"] / full_z.sr["all"])
        lo, hi_ = X1_DEV[prec]
        print(f"  z vs full-value reference: {dev_full:.2e} (expected in [{lo:.0e}, {hi_:.0e}])")
        if not lo < dev_full < hi_:
            bad.append(f"z vs full-value reference {dev_full:.2e} outside [{lo:.0e}, {hi_:.0e}]")
    assert not bad, "; ".join(bad)


@pytest.mark.parametrize("backend", ["tc", "simt"])
@pytest.mark.parametrize("case", FWD, ids=[c[0] for c in FWD])
def test_block_forward_vs_float64(case, backend):
    _run_block(case, backend)


@pytest.mark.parametrize("case", FWD_LARGE, ids=[c[0] for c in FWD_LARGE])
def test_block_forward_multi_tile_vs_float64(case):
    _run_block(case, "tc")


# ---------------------------------------------------------------------------------------------- gate backward
# (name, C, gate_tile, precision, B, T, dil, two_segments)  --  gate_dil = min(dil, T) as fd_wavenet_block_bwd passes
BWD = [
    ("c80-f16-T77-d8-two", 80, 32, "f16", 3, 77, 8, True),                 # SIMT only (C not a multiple of 64)
    ("c96-f16-T100-d17-two", 96, 32, "f16", 3, 100, 17, True),             # SIMT only: 2C = 192, 17-step edges
    ("c128-bf16-T1-d8-one", 128, 256, "bf16", 3, 1, 8, False),             # T = 1: every row is in both edges
    ("c192-f16-T129-d0-two", 192, 128, "f16", 2, 129, 0, True),            # gate_dil = 0: no edge rows
    ("c128-f16-T77-d8-two", 128, 256, "f16", 2, 77, 8, True),
    ("c128-bf16-T129-d200-one", 128, 256, "bf16", 3, 129, 200, False),     # gate_dil = T
    ("c192-f16-T200-d64-one", 192, 128, "f16", 2, 200, 64, False),
    ("c192-bf16-T129-d1-two", 192, 128, "bf16", 2, 129, 1, True),
    ("c512-f16-T1000-d64-two", 512, 256, "f16", 2, 1000, 64, True),
    ("c512-f16-T300-d200-one", 512, 256, "f16", 2, 300, 200, False),       # ragged T < 2 dil over three row tiles
    ("c512-bf16-T77-d64-one", 512, 256, "bf16", 2, 77, 64, False),         # T < 2 dil
    ("c512-bf16x1-T300-d4-one", 512, 256, "bf16x1", 2, 300, 4, False),
    ("c512-f16-B32-T1000-d8-two", 512, 256, "f16", 32, 1000, 8, True),     # ~8 tiles per CTA
    ("c512-bf16-B32-T1000-d2-one", 512, 256, "bf16", 32, 1000, 2, False),
]


def _gate_bwd_params():
    return [pytest.param(c, b, id=f"{c[0]}-{b}") for c in BWD
            for b in (("tc", "simt") if c[1] % 64 == 0 else ("simt",))]


@pytest.mark.parametrize("case,backend", _gate_bwd_params())
def test_gate_bwd_epilogue_vs_float64(case, backend):
    name, C, gt, prec, B, T, dil, two = case
    pc, mma = N.prec_code(prec), N.mma_code(prec)
    hi = prec.endswith("x1")
    d0 = dev()
    g = torch.Generator(device=d0)
    g.manual_seed(zlib.crc32(name.encode()))
    i16 = dict(dtype=torch.int16, device=d0)
    w_out = _randn(g, 2 * C, C, scale=math.sqrt(1.0 / C))
    dxn = N.split_nwc(_randn(g, B, T, C), pc)
    dsk = N.split_nwc(_randn(g, B, T, C), pc)
    y = N.split_nwc(_randn(g, B, T, 2 * C, scale=2.0), pc)
    w2t_f32 = w_out.t().contiguous()                     # [C, 2C]: K = [dx_next | d_skip]
    s = N.pow2_scale(w2t_f32)
    w2t = N.pack_weight(w2t_f32, pc, s)
    gd = min(dil, T)
    inv_S = 0.25
    cs0 = _randn(g, B, 2 * C)
    ce0 = _randn(g, 2, B, 2 * C)
    cs, ce = cs0.clone(), ce0.clone()
    dy = torch.zeros((2, B, T, 2 * C), **i16)
    dz = torch.empty((B, T, C), dtype=torch.float32, device=d0)
    if two:
        kw = dict(src1=dsk, C1=C, w_kshift=0)
        segs, src0 = [(0, 0, 0, C), (1, 0, 0, C)], dxn
    else:
        kw = dict(w_kshift=C)                             # the last layer: d_skip against the skip half of W2^T
        segs, src0 = [(0, 0, 0, C)], dsk
    common = dict(w_inv_scale=1.0 / s, prec=mma, backend=N.backend_code(backend), **kw)
    N.gemm_cl(src0, C, w2t, C, 2 * C, B, T, segs, out_f32=dz, **common)
    N.gemm_cl(src0, C, w2t, C, 2 * C, B, T, segs, out_planes=dy, gate_y=y, gate_tile=gt, gate_dil=gd, gate_cs=cs,
              gate_cs_edge=ce, gate_cs_scale=inv_S, **common)
    torch.cuda.synchronize()

    wv = pf64(w2t, pc, hi) / s
    dz_ref = pf64(dsk, pc, hi) @ wv[:, C:].T
    if two:
        dz_ref += pf64(dxn, pc, hi) @ wv[:, :C].T
    dy_ref = gate_bwd(dz_ref, pf64(y, pc), gt)   # the epilogue reads y at full plane precision in every mode
    print(f"\n[{name} {backend}]")
    bad = []
    for what, got, ref in (("dz", dz.to(F64), dz_ref), ("dy", pf64(dy, pc), dy_ref)):
        r = Regions(T, gd, d0)
        r.add(got, ref)
        bad += r.check(what, TOL[(what, prec)])
    sums = {"cs": (cs, cs0, dy_ref.sum(1)),
            "cs_edge_lo": (ce[0], ce0[0], dy_ref[:, :gd].sum(1)),
            "cs_edge_hi": (ce[1], ce0[1], dy_ref[:, T - gd:].sum(1))}
    rtol, mtol = TOL[("cs", prec)]
    for what, (got, pre, ref) in sums.items():
        if what != "cs" and gd == 0:
            assert torch.equal(got, pre), f"{what}: gate_dil = 0 changed the edge sums"
            continue
        inc, ref = got.to(F64) - pre.to(F64), ref * inv_S     # the prefill must be accumulated into, not overwritten
        rel = rel_l2(inc, ref)
        mx = float((inc - ref).abs().max()) / float(ref.pow(2).mean().sqrt())
        print(f"  {what}: {rel:.2e}/{mx:.2e}")
        if not (rel < rtol and mx < mtol):
            bad.append(f"{what}: rel-L2 {rel:.2e} (bar {rtol:.1e}), max {mx:.2e} (bar {mtol:.1e})")
    assert not bad, "; ".join(bad)


# ---------------------------------------------------------------------------------------------- gate-bias tables
@pytest.mark.parametrize("from_d", [False, True])
@pytest.mark.parametrize("Bs", [1, 4])
@pytest.mark.parametrize("C,E", [(128, 64), (512, 256)])
def test_gate_bias_tables_vs_float64(C, E, Bs, from_d):
    L, KT = 3, 3 * C + E
    d0 = dev()
    g = torch.Generator(device=d0)
    g.manual_seed(C * 10 + Bs)
    w1p = _randn(g, L, 2 * C, KT, scale=math.sqrt(2.0 / (3 * C)))
    bias_sum = _randn(g, L, 2 * C, scale=0.1)
    st = N.stream_ptr(d0)
    gb = torch.full((3, L, Bs, 2 * C), 7.0, dtype=torch.float32, device=d0)
    if from_d:
        d = _randn(g, Bs, L, C)
        N.check(N.lib().fd_wavenet_gate_bias_from_d(N.ptr(d), N.ptr(w1p), N.ptr(bias_sum), N.ptr(gb[0]), N.ptr(gb[1]),
                                                    N.ptr(gb[2]), L, Bs, C, KT, st), "fd_wavenet_gate_bias_from_d")
        d64 = d.to(F64)
    else:
        s = _randn(g, Bs, C)
        wd = _randn(g, L, C, C, scale=math.sqrt(1.0 / C))
        bd = _randn(g, L, C, scale=0.1)
        ws = torch.empty((Bs * L * C,), dtype=torch.float32, device=d0)
        N.check(N.lib().fd_wavenet_gate_bias(N.ptr(s), N.ptr(wd), N.ptr(bd), N.ptr(w1p), N.ptr(bias_sum), N.ptr(gb[0]),
                                             N.ptr(gb[1]), N.ptr(gb[2]), N.ptr(ws), L, Bs, C, KT, st),
                "fd_wavenet_gate_bias")
        d64 = torch.einsum("bk,lck->blc", s.to(F64), wd.to(F64)) + bd.to(F64)
    torch.cuda.synchronize()
    worst = 0.0
    for l in range(L):
        ref = gate_bias_tables(d64[:, l], w1p[l].to(F64), bias_sum[l].to(F64))
        for i in range(3):
            worst = max(worst, rel_l2(gb[i, l].to(F64), ref[i]))
    print(f"\ngate bias C={C} Bs={Bs} from_d={from_d}: worst rel-L2 {worst:.2e}")
    assert worst < 5e-7, worst            # fp32 dot products of length C; measured 1.5e-7
