"""Training path of the native WaveNet: forward that keeps what the backward needs, and a hand-derived backward
built from the same tap-GEMM kernels (reference: autograd through fish_diffusion/modules/wavenet.py:106-120,194-236
inside GaussianDiffusion.p_losses, diffusion.py:129-151).

Per residual block the backward is 5 GEMM launches (2x the forward FLOPs), issued by ONE native call
(fd_wavenet_block_bwd) on either back end:
  dz      = [dx_next/sqrt2 | d_skip] . W2                        data gradient of the output projection (K = 2C); its
                                                                 epilogue turns dz into dy (gate backward) and the
                                                                 column sums of dy, so dz is never stored
  dW2     = [dx_next/sqrt2 ; d_skip]^T . z                       weight gradient (K = time)
  dW1     = dy^T . [x(t-d)+d ; x(t)+d ; x(t+d)+d ; cond]         weight gradient of conv taps + conditioner, one GEMM
  dx      = sum_tap dy(t -/+ d) . W1_tap + dx_next/sqrt2         data gradient of the dilated conv (K = 6C)
  dcond  += dy . Wc
Weight gradients read both operands straight from the channels-last planes (fd_wgrad_cl: MN-major operands on the
tensor cores, which take segments of 64 channels; the SIMT twin takes any multiple of 8, so it serves the SIMT back end
and narrow channel counts); the step vector d_l added to x inside the conv is a rank-one term added afterwards
(_add_step_vector_term).  With `net.grad_sync` set (train.GradSync) every finished bucket of layers is handed to an
NCCL all-reduce from inside the loop, overlapping the backward of the layers below.  The tiny step-embedding MLP /
diffusion projections stay under torch autograd (they act on [B or 1, C] vectors); their output d enters the block
through the gate-bias tables and its gradient is a column sum of dx.
"""
from __future__ import annotations

import ctypes
import math

import torch

from . import _native as N


def _backend_for(pref, n_total, k_seg, num_seg):
    if pref == N.BACKEND_TC and N.tc_supported_linear(n_total, k_seg, num_seg):
        return N.BACKEND_TC
    return N.BACKEND_SIMT


def _bwd_packs(net, pk, device):
    """Transposed packed weights of the data-gradient GEMMs (made by the same batched pack launches as the forward
    packs when the forward ran with gradients enabled; see WaveNet._packed)."""
    if pk.get("_bwd") is None:
        pk = net._packed(device, want_bwd=True)
    return pk["_bwd"]


def _add_step_vector_term(gw1, cs_dy, cs_edge, dl, Bs, C):
    """gw1 [n,2C,KT] += rank-one term of the conv input x + d_l (zero padded): sum_t dy[t,r] * d[c] over the steps where
    tap j reads inside [0,T) = (column sums of dy minus their first / last `dil` edge sums) (x) d_l."""
    n = gw1.shape[0]
    wj = torch.stack([cs_dy - cs_edge[:, 0], cs_dy, cs_dy - cs_edge[:, 1]], dim=1)        # [n,3,B,2C]
    if Bs > 1:
        corr = torch.einsum("ljbr,lbc->lrjc", wj, dl)
    else:
        corr = torch.einsum("ljr,lc->lrjc", wj.sum(2), dl[:, 0])
    gw1[:, :, :3 * C] += corr.reshape(n, 2 * C, 3 * C)


class WaveNetTrainFn(torch.autograd.Function):
    """eps_cl = f(x_cl [B,T,M], cond_cl [B,T,E], d [Bs,L,C], *conv weights);  see WaveNet.train_param_list().
    `masks` = (x_mask, cond_mask) uint8 [B,T] or None each, the reference's masked_fill points (wavenet.py:217-221,
    233-234): masked rows of relu(input_projection(x)), of the conditioner and of the output are zero; in the backward
    that is a zeroed d_eps row, the ReLU mask of the (exactly zero) head rows, and zeroed d_cond rows."""

    @staticmethod
    def forward(ctx, net, masks, x_cl, cond_cl, d, *weights):
        dev = x_cl.device
        N.require_cuda(x_cl, "x")
        B, T, M = x_cl.shape
        C, E, L = net.residual_channels, net.d_encoder, net.n_layers
        Bs = d.shape[0]
        pk = net._packed(dev, want_bwd=True)        # packs are re-made whenever a parameter version changes
        prec, mma, backend = pk["prec"], pk["mma"], pk["backend"]
        lib, st = N.lib(), N.stream_ptr(dev)
        i16 = dict(dtype=torch.int16, device=dev)
        f32 = dict(dtype=torch.float32, device=dev)

        x_mask, cond_mask = masks if masks is not None else (None, None)
        x_planes = N.split_nwc(x_cl.detach().to(torch.float32), prec)
        cond_planes = N.split_nwc(cond_cl.detach().to(torch.float32), prec, mask=cond_mask)
        d = d.detach().to(torch.float32).contiguous()
        gb = torch.empty((3, L, Bs, 2 * C), **f32)
        N.check(lib.fd_wavenet_gate_bias_from_d(N.ptr(d), N.ptr(pk["w1p_f32"]), N.ptr(pk["bias_sum"]), N.ptr(gb[0]),
                                                N.ptr(gb[1]), N.ptr(gb[2]), L, Bs, C, 3 * C + E, st),
                "fd_wavenet_gate_bias_from_d")
        xs = torch.empty((L + 1, 2, B, T, C), **i16)      # residual stream entering each layer (x_L is unused)
        ys = torch.empty((L, 2, B, T, 2 * C), **i16)      # gate/filter pre-activations (packed order)
        zs = torch.empty((L, 2, B, T, C), **i16)          # gated activations (operand of the W2 weight gradient)
        skip_f32 = torch.empty((B, T, C), **f32)
        s_planes = torch.empty((2, B, T, C), **i16)
        h_planes = torch.empty((2, B, T, C), **i16)
        eps = torch.empty((B, T, M), **f32)
        N.conv_cl(x_planes, pk["w_in"], B, T, M, C, [0], bias=pk["b_in"], row_mask=x_mask, out_planes=xs[0],
                  w_inv_scale=pk["w_in_inv"], act=N.ACT_RELU, prec=mma, backend=backend)
        gb_stride = 2 * C if Bs > 1 else 0
        for l in range(L):
            flags = (1 if l == 0 else 0) | (2 if l == L - 1 else 0)
            N.check(lib.fd_wavenet_block_fwd_train(
                N.ptr(xs[l]), N.ptr(xs[l + 1]), N.ptr(cond_planes), N.ptr(zs[l]), N.ptr(ys[l]), N.ptr(pk["w1"][l]),
                N.ptr(pk["w2"][l]), N.ptr(gb[0, l]), N.ptr(gb[1, l]), N.ptr(gb[2, l]), gb_stride, N.ptr(pk["b2"][l]),
                N.ptr(skip_f32), N.ptr(s_planes), 1.0 / math.sqrt(L), B, T, C, E, pk["dil"][l], pk["gate_tile"],
                pk["w1_inv"][l], pk["w2_inv"][l], flags, mma, backend, st), "fd_wavenet_block_fwd_train")
        N.conv_cl(s_planes, pk["w_skip"], B, T, C, C, [0], bias=pk["b_skip"], out_planes=h_planes,
                  w_inv_scale=pk["w_skip_inv"], act=N.ACT_RELU, prec=mma, backend=backend)
        N.conv_cl(h_planes, pk["w_out"], B, T, C, M, [0], bias=pk["b_out"], row_mask=x_mask, out_f32=eps,
                  w_inv_scale=pk["w_out_inv"], prec=mma, backend=backend)
        ctx.net = net
        # the packs used here are captured: a parameter update between forward and backward must not change the
        # weights the gradients are taken at (ADVICE r1); the version key lets backward say so instead of mixing
        ctx.saved = dict(x_planes=x_planes, cond_planes=cond_planes, d=d, xs=xs, ys=ys, zs=zs, s_planes=s_planes,
                         h_planes=h_planes, shape=(B, T, M, Bs), x_mask=x_mask, cond_mask=cond_mask,
                         pack_key=net._pack_key)
        ctx.need_cond = cond_cl.requires_grad
        ctx.need_x = x_cl.requires_grad
        return eps

    @staticmethod
    def backward(ctx, d_eps):
        net, sv = ctx.net, ctx.saved
        if sv is None:
            raise RuntimeError("WaveNetTrainFn: backward ran twice (retain_graph is not supported: the saved "
                               "activations -- ~3 GB per 20k positions -- are released after the first backward)")
        B, T, M, Bs = sv["shape"]
        C, E, L = net.residual_channels, net.d_encoder, net.n_layers
        dev = d_eps.device
        pk = net._packed(dev, want_bwd=True)
        if net._pack_key != sv["pack_key"]:
            raise RuntimeError("WaveNetTrainFn: a parameter of the denoiser changed between forward and backward "
                               "(optimizer / EMA step or load_state_dict in between); run backward first")
        bw = _bwd_packs(net, pk, dev)
        prec, mma, pref = pk["prec"], pk["mma"], pk["backend"]
        perm, gate_tile = pk["perm"], pk["gate_tile"]
        lib, st = N.lib(), N.stream_ptr(dev)
        i16 = dict(dtype=torch.int16, device=dev)
        f32 = dict(dtype=torch.float32, device=dev)
        inv_sqrt2, inv_sqrtL = 1.0 / math.sqrt(2.0), 1.0 / math.sqrt(L)
        rows = B * T
        KT = 3 * C + E

        # Gradient scaling: loss gradients are ~1/numel (1e-6 and below at training shapes), under the fp16 plane
        # range.  The whole backward chain therefore runs on S * gradient with S a power of two that puts
        # max|d_eps| into [1024, 2048) (32x of head room to the fp16 maximum for the channel sums of the chain, while the lo
        # planes of gradients 1000x smaller than the maximum stay out of the fp16 subnormals); every quantity that leaves the chain (weight / bias / conditioner / step-vector
        # gradients) is multiplied by 1/S exactly.  `net.grad_scale` (a float) skips the one host sync per backward.
        if getattr(net, "grad_scale", None):
            S = float(net.grad_scale)
        else:
            amax = float(d_eps.detach().abs().max())
            S = 1.0 if amax == 0.0 or not math.isfinite(amax) else 2.0 ** math.floor(math.log2(2048.0 / amax))
        inv_S = 1.0 / S

        # ---------------------------------------------------------------- helpers
        def colsum(planes=None, f32t=None, Nn=0):
            # gradients stored in planes are S-scaled; fp32 inputs are not
            out = torch.zeros((B, Nn), **f32)
            N.check(lib.fd_colsum(N.ptr(planes), N.ptr(f32t), N.ptr(out), B, T, Nn, inv_S if planes is not None else 1.0,
                                  prec, st), "fd_colsum")
            return out

        def dgrad(src0, C0, w, w_inv, n_total, k_total, segs, **kw):
            N.gemm_cl(src0, C0, w, n_total, k_total, B, T, segs, w_inv_scale=w_inv, prec=mma,
                      backend=_backend_for(pref, n_total, segs[0][3], len(segs)), **kw)

        def wgrad(row_src, R, col_src, Cc):
            """sum_{b,t} rows[b,t,r] * cols[b,t,c] / S -> fp32 [R, Cc], read straight from the channels-last planes"""
            row_segs, col_segs = [(0, 0, R)], [(0, 0, 0, Cc)]
            backend = N.BACKEND_TC if pref == N.BACKEND_TC and N.wgrad_supported(row_segs, col_segs) else N.BACKEND_SIMT
            return N.wgrad_cl([row_src], [col_src], row_segs, col_segs, B, T, scale=inv_S, prec=mma, backend=backend)

        grads = {}

        # ---------------------------------------------------------------- tail (wavenet.py:229-231)
        de = d_eps.detach().to(torch.float32).contiguous()
        if sv["x_mask"] is not None:
            de = de.masked_fill(sv["x_mask"].bool()[:, :, None], 0.0)
        de_planes = N.split_nwc(de, prec, scale=S)
        grads["output_projection.w"] = wgrad(de_planes, M, sv["h_planes"], C)                   # [M, C]
        grads["output_projection.b"] = colsum(f32t=de, Nn=M).sum(0)
        dh_raw = torch.empty((B, T, C), **f32)
        dgrad(de_planes, M, bw["wot"], bw["wot_inv"], C, M, [(0, 0, 0, M)], out_f32=dh_raw)
        dh_planes = torch.empty((2, B, T, C), **i16)
        N.check(lib.fd_relu_bwd(N.ptr(dh_raw), N.ptr(sv["h_planes"]), N.ptr(dh_planes), rows * C, 1.0, prec, st),
                "fd_relu_bwd")
        grads["skip_projection.w"] = wgrad(dh_planes, C, sv["s_planes"], C)
        grads["skip_projection.b"] = colsum(planes=dh_planes, Nn=C).sum(0)
        dskip_planes = torch.empty((2, B, T, C), **i16)                           # d(skip_l) = ds / sqrt(L), every layer
        dgrad(dh_planes, C, bw["wst"], bw["wst_inv"], C, C, [(0, 0, 0, C)], out_planes=dskip_planes,
              planes_scale=inv_sqrtL)
        cs_skip = colsum(planes=dskip_planes, Nn=C)                              # [B, C]
        d_cond = torch.zeros((B, T, E), **f32) if ctx.need_cond else None

        # ---------------------------------------------------------------- residual blocks, last to first
        # One native call per block (fd_wavenet_block_bwd); per-layer column sums land in [L, ...] arrays and are turned
        # into bias / step-vector gradients for all layers at once after the loop.
        cs_dy = torch.zeros((L, B, 2 * C), **f32)                            # column sums of dy per item
        cs_edge = torch.zeros((L, 2, B, 2 * C), **f32)                       # ... over the first / last `dil` steps
        cs_x = torch.zeros((L + 1, B, C), **f32)                             # colsum of d(x_l); row L stays zero
        gw1_all = torch.empty((L, 2 * C, KT), **f32)                         # packed row order, un-permuted at the end
        gw2_all = torch.empty((L, 2 * C, C), **f32)
        dx0 = torch.empty((B, T, C), **f32)       # fp32 copy of d(x_0), written by the layer-0 data gradient
        dy = torch.empty((2, B, T, 2 * C), **i16)
        dx_bufs = [torch.empty((2, B, T, C), **i16) for _ in range(2)]
        sync = getattr(net, "grad_sync", None)   # overlapped gradient all-reduce (train.GradSync)
        net._synced_in_backward = sync is not None
        splits1, splits2 = N.wgrad_splits(2 * C, KT, B, T), N.wgrad_splits(2 * C, C, B, T)
        part1 = torch.empty((splits1, 2 * C, KT), **f32)
        part2 = torch.empty((splits2, 2 * C, C), **f32)
        bd = N.WaveNetBwdDesc()
        bd.cond_planes, bd.dskip = N.ptr(sv["cond_planes"]), N.ptr(dskip_planes)
        bd.d_cond, bd.dy = N.ptr(d_cond), N.ptr(dy)
        bd.part1, bd.part2, bd.splits1, bd.splits2 = N.ptr(part1), N.ptr(part2), splits1, splits2
        bd.B, bd.T, bd.C, bd.E, bd.gate_tile = B, T, C, E, gate_tile
        bd.inv_S, bd.prec = inv_S, mma
        bd.backend = N.BACKEND_TC if pref == N.BACKEND_TC and C % 64 == 0 and E % 64 == 0 else N.BACKEND_SIMT
        dl_all = sv["d"].transpose(0, 1)                                       # [L,Bs,C]
        bucket = sync.bucket_layers if sync is not None else L
        dx_next = None            # planes of d(x_{l+1}); None above the last layer (its residual output is unused)
        for l in reversed(range(L)):
            dx_l = dx_bufs[l & 1]
            bd.x_planes, bd.y_planes, bd.z_planes = N.ptr(sv["xs"][l]), N.ptr(sv["ys"][l]), N.ptr(sv["zs"][l])
            bd.dx_next = N.ptr(dx_next)
            bd.w2t, bd.w1t, bd.wct = N.ptr(bw["w2t"][l]), N.ptr(bw["w1t"][l]), N.ptr(bw["wct"][l])
            bd.w2t_inv, bd.w1t_inv, bd.wct_inv = bw["w2t_inv"][l], bw["w1t_inv"][l], bw["wct_inv"][l]
            bd.dx_out, bd.dx_f32 = N.ptr(dx_l), N.ptr(dx0 if l == 0 else None)
            bd.gw1, bd.gw2 = N.ptr(gw1_all[l]), N.ptr(gw2_all[l])
            bd.cs_dy, bd.cs_edge, bd.cs_dx = N.ptr(cs_dy[l]), N.ptr(cs_edge[l]), N.ptr(cs_x[l])
            bd.dilation = pk["dil"][l]
            N.check(lib.fd_wavenet_block_bwd(ctypes.byref(bd), st), "fd_wavenet_block_bwd")
            dx_next = dx_l
            if sync is not None and (l % bucket == 0):
                # layers [l, hi) are final: add their rank-one step-vector term (it depends on this rank's d) and
                # start the all-reduce of the bucket; it overlaps the backward of the layers below
                hi = min(L, l + bucket)
                _add_step_vector_term(gw1_all[l:hi], cs_dy[l:hi], cs_edge[l:hi], dl_all[l:hi], Bs, C)
                sync.reduce_async(gw1_all[l:hi], gw2_all[l:hi])
        d_d = cs_x[:L] - cs_x[1:] * inv_sqrt2                                  # [L,B,C] gradient wrt the step vectors d_l
        d_d = d_d.transpose(0, 1) if Bs > 1 else d_d.sum(1, keepdim=True).transpose(0, 1)
        d_d = d_d.contiguous()
        gb2_all = torch.cat([cs_x[1:].sum(1) * inv_sqrt2, cs_skip.sum(0).expand(L, C)], dim=1)   # [L,2C]
        gb1_all = cs_dy.sum(1)
        # conv input is x + d_l (zero padded): sum_t dy[t,r] * d[c] over the steps where tap j reads inside [0,T)
        if sync is None:
            _add_step_vector_term(gw1_all, cs_dy, cs_edge, dl_all, Bs, C)
        else:
            sync.wait()            # every bucket reduced before the gradients are laid out for autograd
        gw2_all[:, :C] *= inv_sqrt2
        for l in range(L):
            grads[f"l{l}.w2"], grads[f"l{l}.b2"] = gw2_all[l], gb2_all[l]

        # packed -> reference layouts for all layers at once
        gw1_o = torch.empty_like(gw1_all)
        gw1_o[:, perm] = gw1_all
        gb1_o = torch.empty_like(gb1_all)
        gb1_o[:, perm] = gb1_all
        for l in range(L):
            grads[f"l{l}.w1"] = gw1_o[l, :, :3 * C].reshape(2 * C, 3, C).permute(0, 2, 1)
            grads[f"l{l}.wc"] = gw1_o[l, :, 3 * C:]
            grads[f"l{l}.b1"] = gb1_o[l]

        # ---------------------------------------------------------------- head (wavenet.py:211-212)
        # dx_next now is d(x_0) where x_0 = relu(input_projection(x)): mask with x_0 > 0
        dx0m = torch.empty((2, B, T, C), **i16)
        N.check(lib.fd_relu_bwd(N.ptr(dx0), N.ptr(sv["xs"][0]), N.ptr(dx0m), rows * C, 1.0, prec, st), "fd_relu_bwd")
        grads["input_projection.w"] = wgrad(dx0m, C, sv["x_planes"], M)
        grads["input_projection.b"] = colsum(planes=dx0m, Nn=C).sum(0)
        d_x = None
        if ctx.need_x:     # d(x) = d(x_0 masked by the ReLU) . W_in   (wavenet.py:211)
            d_x = torch.empty((B, T, M), **f32)
            dgrad(dx0m, C, bw["wit"], bw["wit_inv"] * inv_S, M, C, [(0, 0, 0, C)], out_f32=d_x)
        if d_cond is not None and sv["cond_mask"] is not None:
            d_cond = d_cond.masked_fill(sv["cond_mask"].bool()[:, :, None], 0.0)

        out = [None, None, d_x, d_cond, d_d]
        for kind, key in net.train_param_keys():
            gr = grads[key]
            if kind == "w1x1":
                gr = gr[:, :, None]
            out.append(gr)
        ctx.saved = None
        return tuple(out)
