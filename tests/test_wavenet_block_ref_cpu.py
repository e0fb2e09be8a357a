"""CPU tests behind test_gpu_wavenet_block.py, test_gpu_wavenet_block_bwd.py and test_gpu_wavenet_train_edges.py: the
float64 block restatement equals the oracle's ResidualBlock, the closed forms of the block backward equal the autograd
of that restatement, the whole-WaveNet restatement equals the oracle's, the tensor-core launcher refuses a
gate-backward GEMM whose 32-bit epilogue offsets would wrap, and fd_gemm_cl_fwd refuses a gate tile that does not tile
the 2C-wide dy / y rows."""
import ctypes
import math

import numpy as np
import pytest
import torch

from fish_diffusion_b200.wavenet_train import _add_step_vector_term
from oracle import wavenet as ownet
from wavenet_block_ref import (block_bwd, gate_bias_tables, gate_perm, gate_pre_direct, gate_pre_packed, gate_z,
                               pack_w1, pack_w2t, res_skip, wavenet_forward)


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


@pytest.mark.parametrize("T,dil", [(9, 1), (9, 3), (9, 5), (9, 9), (9, 12), (1, 1), (1, 4), (6, 4)])
@pytest.mark.parametrize("top", [False, True])
def test_block_backward_closed_forms_match_autograd(T, dil, top):
    """Every raw output of fd_wavenet_block_bwd as restated by block_bwd equals torch.autograd of the packed forward
    (gate_pre_packed -> gate_z -> res_skip) for the loss <x_new, dx_next> + <skip, dskip>, on S-scaled incoming
    gradients, including T < 2*dil, dil >= T and T = 1, for a top layer (no residual gradient) and a middle one.
    A second pass takes the gate-bias tables from d and W1 and pins the caller's post-processing: the rank-one
    step-vector term of wavenet_train._add_step_vector_term, the step-vector gradient cs_dx - colsum(dx_next)/sqrt2
    and the bias gradient cs_dy."""
    B, C, E, gt = 2, 16, 8, 16
    S = 2.0 ** 8
    inv_S = 1.0 / S
    g = torch.Generator().manual_seed(T * 100 + dil + (50 if top else 0))
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g, dtype=torch.float64) * scale)
    x, cond = r(B, T, C), r(B, T, E)
    w_conv, w_cond = r(2 * C, C, 3, scale=0.3), r(2 * C, E, scale=0.3)
    perm = gate_perm(C, gt)
    w1p0 = pack_w1(w_conv, w_cond, perm)
    bias_p, d = r(2 * C, scale=0.1), r(B, C, scale=0.5)
    w_out0, b_out = r(2 * C, C, scale=0.3), r(2 * C, scale=0.1)
    dskip = r(B, T, C, scale=S)
    dx_next = None if top else r(B, T, C, scale=S)

    def forward(xl, condl, w1pl, w_outl, gb):
        y = gate_pre_packed(xl, condl, w1pl, *gb, dil)
        y.retain_grad()
        z = gate_z(y, C, gt)
        z.retain_grad()
        x_new, skip = res_skip(xl, z, w_outl, b_out)
        loss = (skip * dskip).sum() + (0.0 if top else (x_new * dx_next).sum())
        loss.backward()
        return y, z

    # raw outputs: gate-bias tables held fixed (the step-vector term is the caller's)
    leaf = lambda t: t.clone().requires_grad_(True)
    xl, condl, w1pl, w_outl = leaf(x), leaf(cond), leaf(w1p0), leaf(w_out0)
    gb = [leaf(t) for t in gate_bias_tables(d, w1p0, bias_p)]
    y, z = forward(xl, condl, w1pl, w_outl, gb)
    ref = block_bwd(x, cond, y.detach(), z.detach(), dx_next, dskip, w1p0, pack_w2t(w_out0), gt, dil, inv_S)
    gw2 = w_outl.grad * inv_S
    gw2[:C] *= math.sqrt(2.0)                      # the closed form leaves the residual rows' 1/sqrt2 to the caller
    auto = dict(dz=z.grad, dy=y.grad, cs_dy=gb[0].grad * inv_S,
                cs_edge=-torch.stack([gb[1].grad, gb[2].grad]) * inv_S, gw2=gw2, gw1=w1pl.grad * inv_S, dx=xl.grad,
                d_cond=condl.grad * inv_S, cs_dx=xl.grad.sum(1) * inv_S)
    for k, a in auto.items():
        assert ref[k].shape == a.shape, k
        np.testing.assert_allclose(ref[k].numpy(), a.numpy(), rtol=1e-12, atol=1e-12 * float(a.abs().max()) + 1e-300,
                                   err_msg=k)
    if top:
        assert not bool(ref["gw2"][:C].any())

    # with the tables made from d: W1 gets the rank-one step-vector term, d its gradient, the biases cs_dy
    xl, condl, w1pl, w_outl, dl, bl = leaf(x), leaf(cond), leaf(w1p0), leaf(w_out0), leaf(d), leaf(bias_p)
    forward(xl, condl, w1pl, w_outl, gate_bias_tables(dl, w1pl, bl))
    gw1 = ref["gw1"][None].clone()
    _add_step_vector_term(gw1, ref["cs_dy"][None], ref["cs_edge"][None], d[None], B, C)
    np.testing.assert_allclose(gw1[0].numpy(), (w1pl.grad * inv_S).numpy(), rtol=1e-12, atol=1e-12)
    d_d = ref["cs_dx"] - (0.0 if top else dx_next.sum(1) * inv_S / math.sqrt(2.0))
    np.testing.assert_allclose(d_d.numpy(), (dl.grad * inv_S).numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(ref["cs_dy"].sum(0).numpy(), (bl.grad * inv_S).numpy(), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("T,per_item,masks,bias", [(5, True, True, True), (1, False, False, False),
                                                   (9, True, False, True), (5, False, True, False)])
def test_wavenet_restatement_matches_oracle(T, per_item, masks, bias):
    """wavenet_block_ref.wavenet_forward (float64 torch; its autograd is the reference of
    test_gpu_wavenet_train_edges.py) equals oracle.wavenet.wavenet_forward: dilation cycle 4 over 5 layers, so that
    dilations 4 and 8 reach or pass T, per-item or shared steps, masks, with and without the linear biases."""
    B, M, E, C, L = 3, 8, 6, 16, 5
    sd = ownet.make_wavenet_weights(T * 10 + int(per_item), mel_channels=M, d_encoder=E, residual_channels=C,
                                    residual_layers=L, use_linear_bias=bias)
    rng = np.random.RandomState(T)
    x, cond = rng.randn(B, M, T), rng.randn(B, E, T)
    steps = rng.randint(0, 1000, size=B if per_item else 1).astype(np.float64)
    xm = cm = None
    if masks:
        xm, cm = rng.rand(B, T) < 0.3, rng.rand(B, T) < 0.3
    ref = ownet.wavenet_forward(sd, x, steps, cond, x_masks=xm, cond_masks=cm, dilation_cycle=4)
    t64 = lambda a: None if a is None else torch.from_numpy(np.asarray(a, dtype=np.float64))
    tb = lambda a: None if a is None else torch.from_numpy(a)
    got = wavenet_forward({k: t64(v) for k, v in sd.items()}, t64(x), t64(steps), t64(cond), x_masks=tb(xm),
                          cond_masks=tb(cm), dilation_cycle=4)
    np.testing.assert_allclose(got.numpy(), ref, rtol=0, atol=1e-12 * float(np.abs(ref).max()))


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


@pytest.mark.skipif(torch.cuda.is_available(), reason="host-side check only: nothing may launch on these fake pointers")
@pytest.mark.parametrize("backend", ["tc", "simt"])
@pytest.mark.parametrize("C,gate_tile", [(192, 256), (80, 64), (128, 12)])
def test_gate_bwd_gate_tile_guard(C, gate_tile, backend):
    """The GATE_BWD epilogue reads y and writes dy at the packed gate column pg of a 4-column group and at pg + half:
    a gate tile whose half does not divide n_total = C (C=192 with 256: pg + half runs to 2C + 64), or that is not a
    multiple of 8, would reach past the 2C-wide rows and must be refused on either back end before any launch."""
    from fish_diffusion_b200 import _native as N
    B, T = 2, 16
    d = N.GemmDesc()
    fake = 1 << 40                                   # never dereferenced: the entry point must stop before the launch
    d.src[0], d.src_C[0] = fake, C
    d.w, d.n_total, d.k_total = fake, C, 2 * C
    d.B, d.T, d.num_seg = B, T, 1
    d.seg_src[0], d.seg_klen[0] = 0, C
    d.out_planes, d.gate_y, d.gate_tile, d.gate_dil = fake, fake, gate_tile, 8
    d.w_inv_scale, d.res_scale, d.post_scale, d.planes_scale = 1.0, 1.0, 1.0, 1.0
    d.prec, d.backend = N.PREC_F16, N.backend_code(backend)
    rc = N.lib().fd_gemm_cl_fwd(ctypes.byref(d), None)
    assert rc != 0
    assert "needs out_planes and a gate tile" in N.last_error(), N.last_error()
