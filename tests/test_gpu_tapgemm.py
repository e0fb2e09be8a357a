"""GPU parity: the tap-GEMM kernels (wgmma and SIMT twin) through the C ABI against a float64 restatement on the
exact operand values (read back from the split planes)."""
import numpy as np
import pytest
import torch

from conftest import rel_l2
from fish_diffusion_b200 import _native as N
from gpu_util import dev, planes_to_f64, tap_gemm_ref

pytestmark = pytest.mark.gpu

CASES = [
    # B, T,   Ci,  N,   shifts
    (2, 300, 64, 128, [-2, 0, 2]),
    (1, 128, 128, 512, [0]),
    (3, 77, 64, 64, [-3, -1, 0, 1, 3]),
    (2, 257, 128, 256, [-8, 0, 8]),
    (1, 500, 32, 32, [-1, 0, 1]),
    (1, 500, 16, 16, [-5, -4, -3, -2, -1, 0, 1, 2, 3, 4, 5]),
    (2, 130, 64, 2048, [-1, 0, 1]),
    (1, 40, 512, 128, [0]),
]


@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("prec", ["f16", "bf16"])
@pytest.mark.parametrize("case", CASES)
def test_linear_tapgemm(case, prec, backend):
    B, T, Ci, Nn, shifts = case
    pc, bk = N.prec_code(prec), N.backend_code(backend)
    if bk == N.BACKEND_TC and not N.tc_supported_linear(Nn, Ci, len(shifts)):
        pytest.skip("no tensor-core instantiation")
    rng = np.random.RandomState(hash((B, T, Ci, Nn)) % (2 ** 31))
    a = torch.from_numpy(rng.randn(B, T, Ci).astype(np.float32)).to(dev())
    w = torch.from_numpy((rng.randn(Nn, len(shifts) * Ci) / np.sqrt(Ci * len(shifts))).astype(np.float32)).to(dev())
    bias = torch.from_numpy(rng.randn(Nn).astype(np.float32)).to(dev())
    res = torch.from_numpy(rng.randn(B, T, Nn).astype(np.float32)).to(dev())
    mask = torch.zeros((B, T), dtype=torch.uint8, device=dev())
    mask[0, T // 2:] = 1
    ap = N.split_nwc(a, pc)
    s = N.pow2_scale(w)
    wp = N.pack_weight(w, pc, s)
    out = torch.full((B, T, Nn), 7.0, dtype=torch.float32, device=dev())
    outp = torch.zeros((2, B, T, Nn), dtype=torch.int16, device=dev())
    N.conv_cl(ap, wp, B, T, Ci, Nn, shifts, bias=bias, res_f32=res, row_mask=mask, out_f32=out, out_planes=outp,
              w_inv_scale=1.0 / s, post_scale=0.5, planes_scale=2.0, act=N.ACT_LRELU, act_slope=0.1, prec=pc,
              backend=bk)
    torch.cuda.synchronize()
    ref = (tap_gemm_ref(planes_to_f64(ap, pc), planes_to_f64(wp, pc) / s, shifts, bias.cpu().numpy().astype(np.float64))
           + res.cpu().numpy()) * 0.5
    ref[mask.cpu().numpy().astype(bool)] = 0
    got = out.cpu().numpy()
    tol = 2e-6 if prec == "f16" else 5e-5
    assert rel_l2(got, ref) < tol, (rel_l2(got, ref), np.abs(got - ref).max())
    pl = ref * 2.0
    pl = np.where(pl > 0, pl, pl * 0.1)
    assert rel_l2(planes_to_f64(outp, pc), pl) < (2e-6 if prec == "f16" else 2e-5)


@pytest.mark.parametrize("backend", ["simt", "tc"])
def test_accumulate_and_addend(backend):
    B, T, Ci, Nn, shifts = 2, 200, 64, 128, [-1, 0, 1]
    pc, bk = N.PREC_F16, N.backend_code(backend)
    rng = np.random.RandomState(3)
    a = torch.from_numpy(rng.randn(B, T, Ci).astype(np.float32)).to(dev())
    w = torch.from_numpy((rng.randn(Nn, 3 * Ci) * 0.05).astype(np.float32)).to(dev())
    add = torch.from_numpy(rng.randn(B, T, Nn).astype(np.float32)).to(dev())
    prev = torch.from_numpy(rng.randn(B, T, Nn).astype(np.float32)).to(dev())
    ap, s = N.split_nwc(a, pc), N.pow2_scale(w)
    wp = N.pack_weight(w, pc, s)
    out = prev.clone()
    N.conv_cl(ap, wp, B, T, Ci, Nn, shifts, addend=add, out_f32=out, out_accum=True, w_inv_scale=1.0 / s, prec=pc,
              backend=bk)
    torch.cuda.synchronize()
    ref = tap_gemm_ref(planes_to_f64(ap, pc), planes_to_f64(wp, pc) / s, shifts) + add.cpu().numpy() + prev.cpu().numpy()
    assert rel_l2(out.cpu().numpy(), ref) < 2e-6


# every LINEAR operand in one launch, at channel counts that give the wgmma kernel 128-, 32- and 16-column tiles
@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("act", ["relu", "lrelu"])
@pytest.mark.parametrize("prec", ["f16", "bf16"])
@pytest.mark.parametrize("Ci,Nn", [(64, 128), (32, 32), (16, 16)])
def test_linear_all_operands(Ci, Nn, prec, act, backend):
    B, T, shifts = 3, 203, [-1, 0, 1]
    pc, bk = N.prec_code(prec), N.backend_code(backend)
    assert bk != N.BACKEND_TC or N.tc_supported_linear(Nn, Ci, len(shifts))
    act_code, slope = (N.ACT_RELU, 0.0) if act == "relu" else (N.ACT_LRELU, 0.2)
    rng = np.random.RandomState(Ci + Nn)
    d = dev()
    t32 = lambda *shape: torch.from_numpy(rng.randn(*shape).astype(np.float32)).to(d)
    a, w = t32(B, T, Ci), t32(Nn, 3 * Ci) / np.sqrt(3 * Ci)
    bias, add, res, resp, prev = t32(B, Nn), t32(B, T, Nn), t32(B, T, Nn), t32(B, T, Nn), t32(B, T, Nn)
    mask = torch.zeros((B, T), dtype=torch.uint8, device=d)
    mask[1, T // 3:] = 1
    mask[2, ::7] = 1
    ap, rp, s = N.split_nwc(a, pc), N.split_nwc(resp, pc), N.pow2_scale(w)
    wp = N.pack_weight(w, pc, s)
    out = prev.clone()
    outp = torch.zeros((2, B, T, Nn), dtype=torch.int16, device=d)
    N.gemm_cl(ap, Ci, wp, Nn, 3 * Ci, B, T, [(0, sh, 0, Ci) for sh in shifts], bias=bias, bias_per_item=True,
              addend=add, res_f32=res, res_planes=rp, res_scale=0.75, row_mask=mask, out_f32=out, out_planes=outp,
              w_inv_scale=1.0 / s, post_scale=0.5, planes_scale=2.0, act=act_code, act_slope=slope, out_accum=True,
              prec=pc, backend=bk)
    torch.cuda.synchronize()
    f64 = lambda x: x.cpu().numpy().astype(np.float64)
    y = (tap_gemm_ref(planes_to_f64(ap, pc), planes_to_f64(wp, pc) / s, shifts) + f64(bias)[:, None, :] + f64(add)
         + f64(res) + 0.75 * planes_to_f64(rp, pc)) * 0.5 + f64(prev)
    y[mask.cpu().numpy().astype(bool)] = 0
    got = out.cpu().numpy()
    assert rel_l2(got, y) < (2e-6 if prec == "f16" else 5e-5), (rel_l2(got, y), np.abs(got - y).max())
    pl = np.where(y > 0, 2.0 * y, 2.0 * slope * y)
    assert rel_l2(planes_to_f64(outp, pc), pl) < (2e-6 if prec == "f16" else 2e-5)


def test_tc_matches_simt_full_width_block():
    """One WaveNet residual block at the real width (C=512, E=256), wgmma vs SIMT twin on identical planes."""
    import math
    B, T, C, E = 2, 1000, 512, 256
    pc = N.PREC_F16
    rng = np.random.RandomState(9)
    d = dev()
    x = torch.from_numpy(rng.randn(B, T, C).astype(np.float32)).to(d)
    cond = torch.from_numpy(rng.randn(B, T, E).astype(np.float32)).to(d)
    w1 = torch.from_numpy((rng.randn(2 * C, 3 * C + E) * math.sqrt(2.0 / (3 * C))).astype(np.float32)).to(d)
    w2 = torch.from_numpy((rng.randn(2 * C, C) * math.sqrt(2.0 / C)).astype(np.float32)).to(d)
    gb = torch.from_numpy((rng.randn(3, 2 * C) * 0.1).astype(np.float32)).to(d)
    b2 = torch.from_numpy((rng.randn(2 * C) * 0.1).astype(np.float32)).to(d)
    s1, s2 = N.pow2_scale(w1), N.pow2_scale(w2)
    w1p, w2p = N.pack_weight(w1, pc, s1), N.pack_weight(w2, pc, s2)
    cp = N.split_nwc(cond, pc)
    outs = {}
    for name, bk in (("simt", N.BACKEND_SIMT), ("tc", N.BACKEND_TC)):
        xp = N.split_nwc(x, pc)
        z = torch.zeros((2, B, T, C), dtype=torch.int16, device=d)
        skip = torch.zeros((B, T, C), dtype=torch.float32, device=d)
        skp = torch.zeros((2, B, T, C), dtype=torch.int16, device=d)
        for flags in (1, 0):
            N.check(N.lib().fd_wavenet_block_fwd(
                N.ptr(xp), N.ptr(cp), N.ptr(z), N.ptr(w1p), N.ptr(w2p), N.ptr(gb[0]), N.ptr(gb[1]), N.ptr(gb[2]), 0,
                N.ptr(b2), N.ptr(skip), N.ptr(skp), 1.0, B, T, C, E, 2, 256, 1.0 / s1, 1.0 / s2, flags, pc, bk,
                N.stream_ptr(d)), "block")
        torch.cuda.synchronize()
        outs[name] = (planes_to_f64(xp, pc), skip.cpu().numpy().astype(np.float64), planes_to_f64(z, pc))
    for i, what in enumerate(("x", "skip", "z")):
        e = rel_l2(outs["tc"][i], outs["simt"][i])
        assert e < 2e-5, (what, e)   # tensor-core fp32 accumulation truncates (not IEEE round-to-nearest)
