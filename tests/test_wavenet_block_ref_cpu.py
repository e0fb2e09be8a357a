"""CPU tests behind test_gpu_wavenet_block.py: its float64 block restatement equals the oracle's ResidualBlock, and the
tensor-core launcher refuses a gate-backward GEMM whose 32-bit epilogue offsets would wrap."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import wavenet as ownet
from wavenet_block_ref import (gate_bias_tables, gate_perm, gate_pre_direct, gate_pre_packed, gate_z, pack_w1,
                               res_skip)


@pytest.mark.parametrize("T,dil", [(9, 1), (9, 3), (9, 5), (9, 9), (9, 12), (1, 1), (4, 2)])
@pytest.mark.parametrize("per_item", [False, True])
def test_block_restatement_matches_oracle(T, dil, per_item):
    """Both forms (first principles; gb tables + packed column order) against oracle.wavenet.residual_block, including
    T < 2*dil (both edge corrections on one row) and dil >= T (both side taps outside the sequence everywhere)."""
    B, C, E, gate_tile = 2, 16, 8, 16          # two gate tiles of 8 gates + 8 filters
    rng = np.random.RandomState(T * 100 + dil + (7 if per_item else 0))
    r = lambda *s: rng.randn(*s)
    pre = "residual_layers.0."
    sd = {pre + "conv_layer.conv.weight": r(2 * C, C, 3) * 0.3, pre + "conv_layer.conv.bias": r(2 * C) * 0.1,
          pre + "diffusion_projection.linear.weight": r(C, C) * 0.3, pre + "diffusion_projection.linear.bias": r(C) * 0.1,
          pre + "conditioner_projection.conv.weight": r(2 * C, E, 1) * 0.3,
          pre + "conditioner_projection.conv.bias": r(2 * C) * 0.1,
          pre + "output_projection.conv.weight": r(2 * C, C, 1) * 0.3, pre + "output_projection.conv.bias": r(2 * C) * 0.1}
    x, cond = r(B, C, T), r(B, E, T)
    step = r(B if per_item else 1, C)
    x_ref, skip_ref = ownet.residual_block(sd, pre, x, cond, np.broadcast_to(step, (B, C)), dil)

    t64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64))
    g = lambda k: t64(sd[pre + k])
    d = t64(step) @ g("diffusion_projection.linear.weight").T + g("diffusion_projection.linear.bias")
    xc, cc = t64(x).transpose(1, 2), t64(cond).transpose(1, 2)
    w_conv, w_cond = g("conv_layer.conv.weight"), g("conditioner_projection.conv.weight")[:, :, 0]
    b_conv, b_cond = g("conv_layer.conv.bias"), g("conditioner_projection.conv.bias")
    w_out, b_out = g("output_projection.conv.weight")[:, :, 0], g("output_projection.conv.bias")

    y_nat = gate_pre_direct(xc, cc, d, w_conv, b_conv, w_cond, b_cond, dil)
    perm = gate_perm(C, gate_tile)
    w1p = pack_w1(w_conv, w_cond, perm)
    y_pk = gate_pre_packed(xc, cc, w1p, *gate_bias_tables(d, w1p, (b_conv + b_cond)[perm]), dil)
    assert torch.equal(perm.sort().values, torch.arange(2 * C))
    np.testing.assert_allclose(y_pk.numpy(), y_nat[..., perm].numpy(), rtol=0, atol=1e-12)
    for z in (gate_z(y_nat, C), gate_z(y_pk, C, gate_tile)):
        x_new, skip = res_skip(xc, z, w_out, b_out)
        np.testing.assert_allclose(x_new.transpose(1, 2).numpy(), x_ref, rtol=0, atol=1e-12)
        np.testing.assert_allclose(skip.transpose(1, 2).numpy(), skip_ref, rtol=0, atol=1e-12)


@pytest.mark.skipif(torch.cuda.is_available(), reason="host-side check only: nothing may launch on these fake pointers")
def test_gate_bwd_offset_guard():
    """GATE_BWD's epilogue offsets reach B*T*2C (dy / y planes are 2C wide) while n_total = C: a problem with
    2^31 <= B*T*C < 2^32 must be refused before any launch."""
    from fish_diffusion_b200 import _native as N
    C, B, T = 512, 1, (1 << 31) // 512 + 64          # B*T*C just above 2^31, B*T*2C above 2^32
    assert (1 << 31) <= B * T * C < (1 << 32) <= B * T * 2 * C
    d = N.GemmDesc()
    fake = 1 << 40                                   # never dereferenced: the launcher must stop before the launch
    d.src[0], d.src_C[0] = fake, C
    d.src[1], d.src_C[1] = fake, C
    d.w, d.n_total, d.k_total = fake, C, 2 * C
    d.B, d.T, d.num_seg = B, T, 2
    d.seg_src[0], d.seg_klen[0], d.seg_src[1], d.seg_klen[1] = 0, C, 1, C
    d.out_planes, d.gate_y, d.gate_tile, d.gate_dil = fake, fake, 256, 8
    d.w_inv_scale, d.res_scale, d.post_scale, d.planes_scale = 1.0, 1.0, 1.0, 1.0
    d.prec, d.backend = N.PREC_F16, N.BACKEND_TC
    rc = N.lib().fd_gemm_cl_fwd(ctypes.byref(d), None)
    assert rc != 0
    assert "exceeds the 32-bit element offsets" in N.last_error(), N.last_error()
