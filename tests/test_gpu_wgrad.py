"""GPU parity of the weight-gradient GEMM (fd_wgrad_cl, read straight from channels-last planes: wgmma with MN-major
operands, and its SIMT twin) against float64 on the exact plane values."""
import numpy as np
import pytest
import torch

from conftest import rel_l2
from fish_diffusion_b200 import _native as N
from gpu_util import dev, planes_to_f64

pytestmark = pytest.mark.gpu


def hi_to_f64(planes, pc):
    p = planes[0].cpu()
    return p.view(torch.float16 if pc == N.PREC_F16 else torch.bfloat16).to(torch.float64).numpy()


def shifted(a, s):
    """a [B,T,C] -> a[b, t+s, c] with zeros outside [0,T)"""
    B, T, C = a.shape
    out = np.zeros_like(a)
    lo, hi = max(0, -s), min(T, T - s)
    if hi > lo:
        out[:, lo:hi] = a[:, lo + s:hi + s]
    return out


CASES = [
    # B, T, row channel counts, row segs (src, coff, width), col channel counts, col segs (src, shift, coff, width)
    (3, 200, [128], [(0, 0, 128)], [64, 64], [(0, -2, 0, 64), (0, 0, 0, 64), (0, 2, 0, 64), (1, 0, 0, 64)]),
    (2, 77, [64], [(0, 0, 64)], [128], [(0, 0, 0, 128)]),
    (4, 130, [128, 128], [(0, 0, 128), (1, 0, 128)], [192], [(0, 0, 0, 192)]),
    (2, 1000, [256], [(0, 0, 256)], [128, 256], [(0, -64, 0, 128), (0, 0, 0, 128), (0, 64, 0, 128), (1, 0, 0, 256)]),
    (5, 64, [192], [(0, 64, 128)], [320], [(0, 3, 64, 256)]),
]
# segments that are not multiples of 64 channels: the SIMT twin only (widths 16 / 32, segments at channel offset 8,
# several row and column tiles of 64 with ragged last tiles)
SIMT_CASES = [
    (2, 150, [16], [(0, 0, 16)], [32, 16], [(0, -3, 0, 32), (0, 0, 0, 32), (0, 3, 0, 32), (1, 0, 0, 16)]),
    (3, 77, [48, 32], [(0, 8, 32), (1, 0, 32)], [40], [(0, 5, 8, 32)]),
    (2, 300, [96], [(0, 0, 96)], [72], [(0, -2, 8, 56), (0, 1, 0, 16)]),
]
BACKEND_CASES = ([pytest.param(c, "tc", id=f"case{i}") for i, c in enumerate(CASES)] +
                 [pytest.param(c, "simt", id=f"simt-case{i}") for i, c in enumerate(CASES + SIMT_CASES)])
# rel-L2 bars (largest measured over all cases and split counts, H100 80GB HBM3 at 700 W).  tc: fp32 tensor-core
# accumulation over K = B*T up to 2000 terms (measured 7.0e-6 f16, 7.2e-6 bf16, 2.4e-6 f16x1).  simt: fp32 FFMA over
# the same K (measured 7.9e-7 in f16, bf16 and f16x1).
TOL = {("tc", N.PREC_F16): 2e-5, ("tc", N.PREC_BF16): 5e-5, ("simt", N.PREC_F16): 3e-6, ("simt", N.PREC_BF16): 3e-6}


@pytest.mark.parametrize("prec", ["f16", "bf16", "f16x1"])
@pytest.mark.parametrize("splits", [None, 1])
@pytest.mark.parametrize("case,backend", BACKEND_CASES)
def test_wgrad_direct_vs_float64(case, backend, prec, splits):
    B, T, rowC, row_segs, colC, col_segs = case
    pc, mma = N.prec_code(prec), N.mma_code(prec)
    rng = np.random.RandomState(B * 1000 + T)
    rows = [N.split_nwc(torch.from_numpy(rng.randn(B, T, c).astype(np.float32)).to(dev()), pc) for c in rowC]
    cols = [N.split_nwc(torch.from_numpy(rng.randn(B, T, c).astype(np.float32)).to(dev()), pc) for c in colC]
    out = N.wgrad_cl(rows, cols, row_segs, col_segs, B, T, scale=0.25, prec=mma, splits=splits,
                     backend=N.backend_code(backend))
    torch.cuda.synchronize()
    conv = hi_to_f64 if prec.endswith("x1") else planes_to_f64
    r64 = [conv(p, pc) for p in rows]
    c64 = [conv(p, pc) for p in cols]
    Rm = np.concatenate([r64[s][:, :, co:co + w] for s, co, w in row_segs], axis=2)
    Cm = np.concatenate([shifted(c64[s], sh)[:, :, co:co + w] for s, sh, co, w in col_segs], axis=2)
    ref = 0.25 * np.einsum("btr,btc->rc", Rm, Cm)
    got = out.cpu().numpy()
    assert got.shape == ref.shape
    e = rel_l2(got, ref)
    print(f"wgrad[{backend},{prec},B={B},T={T}] rel-L2 {e:.2e}")
    assert e < TOL[backend, pc], (e, np.abs(got - ref).max())
