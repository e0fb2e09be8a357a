"""H100-native NSF-HiFiGAN vocoder: drop-in for the reference
``fish_diffusion/modules/vocoders/nsf_hifigan/{models.py:Generator, nsf_hifigan.py:NsfHifiGAN}``.

Same parameter names / checkpoint formats (weight-norm ``weight_g``/``weight_v`` pairs or folded ``weight``), same
``spec2wav`` / ``wav2spec`` / ``model(mel, f0)`` contracts (SURVEY.md section 8b), registered as
``VOCODERS["NsfHifiGAN"]``.  Everything runs channels-last on sm_90a kernels:
  f0 -> exact-phase harmonic source (fd_sinegen_fwd) -> 1-channel source convs (fd_source_conv_fwd)
  mel -> conv_pre -> per stage { polyphase ConvTranspose1d tap-GEMM (+ source addend) -> 3 x ResBlock1 chains of
  dilated-conv tap-GEMMs with fused LeakyReLU / residual / MRF accumulation } -> conv_post + tanh.
"""
from __future__ import annotations

import json
import os
from pathlib import Path
from typing import Optional

import numpy as np
import torch
from torch import nn
from torch.nn import Conv1d, ConvTranspose1d
from torch.nn.utils import remove_weight_norm, weight_norm

from . import _native as N
from .mel import PitchAdjustableMelSpectrogram, dynamic_range_compression
from .registry import VOCODERS
from .resample import resample

LRELU_SLOPE = 0.1


class AttrDict(dict):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.__dict__ = self


def init_weights(m, mean=0.0, std=0.01):
    if m.__class__.__name__.find("Conv") != -1:
        m.weight.data.normal_(mean, std)


def get_padding(kernel_size, dilation=1):
    return int((kernel_size * dilation - dilation) / 2)


def _effective_weight(conv) -> torch.Tensor:
    """Folded weight of a (possibly weight-normed) conv: w = g * v / ||v|| (models.py:440-448)."""
    if hasattr(conv, "weight_g"):
        return torch._weight_norm(conv.weight_v, conv.weight_g, 0)
    return conv.weight


class ResBlock1(nn.Module):
    """Parameter holder (models.py:27-116)."""

    def __init__(self, h, channels, kernel_size=3, dilation=(1, 3, 5)):
        super().__init__()
        self.h, self.kernel_size, self.dilation = h, kernel_size, tuple(dilation)
        self.convs1 = nn.ModuleList([
            weight_norm(Conv1d(channels, channels, kernel_size, 1, dilation=d, padding=get_padding(kernel_size, d)))
            for d in dilation])
        self.convs1.apply(init_weights)
        self.convs2 = nn.ModuleList([
            weight_norm(Conv1d(channels, channels, kernel_size, 1, dilation=1, padding=get_padding(kernel_size, 1)))
            for _ in dilation])
        self.convs2.apply(init_weights)

    def remove_weight_norm(self):
        for l in list(self.convs1) + list(self.convs2):
            remove_weight_norm(l)


class ResBlock2(nn.Module):
    """Parameter holder (models.py:119-158)."""

    def __init__(self, h, channels, kernel_size=3, dilation=(1, 3)):
        super().__init__()
        self.h, self.kernel_size, self.dilation = h, kernel_size, tuple(dilation)
        self.convs = nn.ModuleList([
            weight_norm(Conv1d(channels, channels, kernel_size, 1, dilation=d, padding=get_padding(kernel_size, d)))
            for d in dilation])
        self.convs.apply(init_weights)

    def remove_weight_norm(self):
        for l in self.convs:
            remove_weight_norm(l)


class SineGen(nn.Module):
    """Hyper-parameter holder (models.py:161-199); computed inside fd_sinegen_fwd."""

    def __init__(self, samp_rate, harmonic_num=0, sine_amp=0.1, noise_std=0.003, voiced_threshold=0,
                 flag_for_pulse=False):
        super().__init__()
        self.sine_amp, self.noise_std, self.harmonic_num = sine_amp, noise_std, harmonic_num
        self.dim = harmonic_num + 1
        self.sampling_rate, self.voiced_threshold, self.flag_for_pulse = samp_rate, voiced_threshold, flag_for_pulse


class SourceModuleHnNSF(nn.Module):
    """Parameter holder (models.py:297-335)."""

    def __init__(self, sampling_rate, harmonic_num=0, sine_amp=0.1, add_noise_std=0.003, voiced_threshod=0):
        super().__init__()
        self.sine_amp, self.noise_std = sine_amp, add_noise_std
        self.l_sin_gen = SineGen(sampling_rate, harmonic_num, sine_amp, add_noise_std, voiced_threshod)
        self.l_linear = torch.nn.Linear(harmonic_num + 1, 1)
        self.l_tanh = torch.nn.Tanh()


def fold_conv_weight(w: torch.Tensor, d: int, F: int):
    """'same'-padded Conv1d weight w [Co, Ci, K] with dilation d, on the time-folded view [T, C] == [T/F, F*C]:
    returns (W' [F*Co, S*F*Ci], row shifts [S]) of the equivalent tap-GEMM over folded rows,
        y'[r, fo*Co + n] = sum_s sum_{fi,c} W'[fo*Co + n, (s, fi, c)] * x'[r + shift_s, fi*Ci + c].
    Folded row r holds time steps F*r + f, so output sub-step fo reads input time F*r + fo + off_j = F*(r + s) + fi with
    s = floor((fo + off_j) / F), fi = (fo + off_j) mod F.  Zero padding carries over because item lengths are
    multiples of F (rows outside [0, T/F) are whole groups of out-of-range steps)."""
    Co, Ci, K = w.shape
    offs = [(j - (K - 1) // 2) * d for j in range(K)]
    srows = sorted({(fo + o) // F for fo in range(F) for o in offs})
    Wf = torch.zeros((F, Co, len(srows), F, Ci), dtype=w.dtype, device=w.device)
    for fo in range(F):
        for j, o in enumerate(offs):
            Wf[fo, :, srows.index((fo + o) // F), (fo + o) % F, :] = w[:, :, j]
    return Wf.reshape(F * Co, len(srows) * F * Ci).contiguous(), srows


class Generator(nn.Module):
    """NSF-HiFiGAN generator (models.py:353-448) on sm_90a kernels.  `h` is the JSON config (AttrDict)."""

    def __init__(self, h, precision="f16", backend="auto"):
        super().__init__()
        if not isinstance(h, AttrDict):
            h = AttrDict(h)
        self.h = h
        self.num_kernels = len(h.resblock_kernel_sizes)
        self.num_upsamples = len(h.upsample_rates)
        self.m_source = SourceModuleHnNSF(sampling_rate=h.sampling_rate, harmonic_num=8)
        self.noise_convs = nn.ModuleList()
        self.conv_pre = weight_norm(Conv1d(h.num_mels, h.upsample_initial_channel, 7, 1, padding=3))
        resblock = ResBlock1 if h.resblock == "1" else ResBlock2
        self.ups = nn.ModuleList()
        for i, (u, k) in enumerate(zip(h.upsample_rates, h.upsample_kernel_sizes)):
            c_cur = h.upsample_initial_channel // (2 ** (i + 1))
            self.ups.append(weight_norm(ConvTranspose1d(h.upsample_initial_channel // (2 ** i), c_cur, k, u,
                                                        padding=(k - u) // 2)))
            if i + 1 < len(h.upsample_rates):
                stride_f0 = int(np.prod(h.upsample_rates[i + 1:]))
                self.noise_convs.append(Conv1d(1, c_cur, kernel_size=stride_f0 * 2, stride=stride_f0,
                                               padding=stride_f0 // 2))
            else:
                self.noise_convs.append(Conv1d(1, c_cur, kernel_size=1))
        self.resblocks = nn.ModuleList()
        for i in range(len(self.ups)):
            ch = h.upsample_initial_channel // (2 ** (i + 1))
            for k, d in zip(h.resblock_kernel_sizes, h.resblock_dilation_sizes):
                self.resblocks.append(resblock(h, ch, k, d))
        self.conv_post = weight_norm(Conv1d(ch, 1, 7, 1, padding=3))
        self.ups.apply(init_weights)
        self.conv_post.apply(init_weights)
        self.precision = precision
        self.backend = os.environ.get("FD_BACKEND", backend)
        # fused ResBlock pairs (csrc/fd_respair_tc.cu): c1 -> lrelu -> c2 -> +x in one kernel, residual stream kept
        # as split planes only.  FD_VOC_FUSED=0 selects the conv-by-conv path (the SIMT back end always uses it).
        self.fused = os.environ.get("FD_VOC_FUSED", "1") != "0"
        self._pack = None
        self._pack_key = None

    def remove_weight_norm(self):
        for l in self.ups:
            remove_weight_norm(l)
        for l in self.resblocks:
            l.remove_weight_norm()
        remove_weight_norm(self.conv_pre)
        remove_weight_norm(self.conv_post)

    # ------------------------------------------------------------------------------------ packing
    def _backend_for(self, n_total, k_seg, num_seg):
        if self.backend != "auto":
            return N.backend_code(self.backend)
        return N.BACKEND_TC if N.tc_supported_linear(n_total, k_seg, num_seg) else N.BACKEND_SIMT

    @staticmethod
    def _fold_factor(Ci, Co, K, d):
        """Time-folding factor of a narrow square conv (1 = keep).  A [T, C] tensor with C = 16 / 32 / 64 is the same
        memory as [T/F, F*C]; on that view the conv is a block-Toeplitz tap-GEMM with 128 input and output columns and
        far fewer taps.  Narrow tiles are bound by TMA row rate (32-byte rows) and by the tensor core's poor efficiency
        at N = 16..64, so trading zero blocks in the weights (tensor pipe is idle there) for 256-byte rows and N = 128
        wins: always at C = 16, for dilation-1 convs at C = 32, for the 11-tap dilation-1 convs at C = 64."""
        if Ci != Co:
            return 1
        if Ci == 16:
            return 8
        if Ci == 32 and d == 1:
            return 4
        if Ci == 64 and d == 1 and K >= 11:
            return 2
        return 1

    def _pack_conv(self, conv, prec, device):
        """Conv1d(Ci->Co, K, dilation d, 'same' padding) -> tap-GEMM weights [Co][K*Ci] + row shifts."""
        w = _effective_weight(conv).detach().to(device=device, dtype=torch.float32)
        Co, Ci, K = w.shape
        d = conv.dilation[0]
        w2 = w.permute(0, 2, 1).reshape(Co, K * Ci).contiguous()
        s = N.pow2_scale(w2)
        bias = conv.bias.detach().to(device=device, dtype=torch.float32).contiguous()
        offs = [(j - (K - 1) // 2) * d for j in range(K)]
        pc = dict(w=N.pack_weight(w2, prec, s), inv=1.0 / s, Ci=Ci, N=Co, shifts=offs, bias=bias, K=K, d=d,
                  backend=self._backend_for(Co, Ci, K))
        F = self._fold_factor(Ci, Co, K, d)
        if F > 1 and pc["backend"] == N.BACKEND_TC:
            wf, srows = fold_conv_weight(w, d, F)
            if len(srows) <= 16 and self._backend_for(F * Co, F * Ci, len(srows)) == N.BACKEND_TC:
                pc["fold"] = dict(F=F, w=N.pack_weight(wf, prec, s), inv=1.0 / s, Ci=F * Ci, N=F * Co, shifts=srows,
                                  bias=bias.repeat(F).contiguous(), backend=N.BACKEND_TC)
        return pc

    def _pack_conv_folded_pair(self, conv, prec, device, F=2):
        """Pack for the fused pair kernel on the time-folded view [T/F, F*C] (C = 16 -> 32): the conv becomes a
        dilation-1 conv with K' = 2*max|row shift|+1 taps of (F*C x F*C) blocks (zero blocks where a shift does not
        occur).  32-byte rows are what bounds the C = 16 stage (TMA row rate); 64-byte rows and a quarter of the tiles
        cost 3x the tensor-core work, which is idle there."""
        w = _effective_weight(conv).detach().to(device=device, dtype=torch.float32)
        Co, Ci, K = w.shape
        d = conv.dilation[0]
        wf, srows = fold_conv_weight(w, d, F)                       # [F*Co, S*F*Ci], sorted row shifts
        hmax = max(abs(srows[0]), abs(srows[-1]))
        Kp = 2 * hmax + 1
        W = torch.zeros((F * Co, Kp, F * Ci), dtype=torch.float32, device=device)
        wf3 = wf.reshape(F * Co, len(srows), F * Ci)
        for j, sr in enumerate(srows):
            W[:, sr + hmax, :] = wf3[:, j, :]
        w2 = W.reshape(F * Co, Kp * F * Ci).contiguous()
        s = N.pow2_scale(w2)
        bias = conv.bias.detach().to(device=device, dtype=torch.float32).repeat(F).contiguous()
        # which (tap, 16-input-channel slice) blocks hold weights: most of a folded dilated kernel is zero blocks, which
        # the fused kernel neither loads nor multiplies (fd_respair_desc.kmask1/2)
        kmask = 0
        if (F * Ci) % 16 == 0 and Kp * (F * Ci // 16) <= 64:
            nz = (W.reshape(F * Co, Kp, F * Ci // 16, 16) != 0).any(dim=3).any(dim=0).reshape(-1).tolist()
            kmask = sum(1 << i for i, b in enumerate(nz) if b)
        return dict(w=N.pack_weight(w2, prec, s), inv=1.0 / s, K=Kp, d=1, bias=bias, F=F, C=F * Co, kmask=kmask)

    def _pack_convt(self, conv, prec, device):
        """ConvTranspose1d(Ci->Co, k, stride u, padding p) as a polyphase tap-GEMM: output row q of width u*Co
        holds output samples q*u + r;  W'[(r,co)][(delta,ci)] = w[ci,co, r + p - delta*u] when that tap exists."""
        w = _effective_weight(conv).detach().to(device=device, dtype=torch.float32)   # [Ci, Co, k]
        Ci, Co, k = w.shape
        u, p = conv.stride[0], conv.padding[0]
        dmin = -((k - 1 - p) // u)            # smallest delta with r + p - delta*u <= k-1 for r = 0
        dmax = (u - 1 + p) // u
        deltas = list(range(dmin, dmax + 1))
        W = torch.zeros((u, Co, len(deltas), Ci), dtype=torch.float32, device=device)
        for r in range(u):
            for j, dl in enumerate(deltas):
                kk = r + p - dl * u
                if 0 <= kk < k:
                    W[r, :, j, :] = w[:, :, kk].t()
        w2 = W.reshape(u * Co, len(deltas) * Ci).contiguous()
        s = N.pow2_scale(w2)
        bias = conv.bias.detach().to(device=device, dtype=torch.float32).repeat(u).contiguous()
        return dict(w=N.pack_weight(w2, prec, s), inv=1.0 / s, Ci=Ci, N=u * Co, Co=Co, u=u, shifts=deltas, bias=bias,
                    backend=self._backend_for(u * Co, Ci, len(deltas)))

    def _packed(self, device):
        key = (str(device), self.precision, tuple(p._version for p in self.parameters()),
               tuple(p.data_ptr() for p in self.parameters()))
        if self._pack is not None and self._pack_key == key:
            return self._pack
        prec = N.prec_code(self.precision)
        f32 = lambda t: t.detach().to(device=device, dtype=torch.float32).contiguous()
        pk = {"prec": prec, "mma": N.mma_code(self.precision), "pre": self._pack_conv(self.conv_pre, prec, device), "ups": [], "src": [], "res": []}
        for i, up in enumerate(self.ups):
            pk["ups"].append(self._pack_convt(up, prec, device))
            nc = self.noise_convs[i]
            pk["src"].append(dict(w_t=f32(nc.weight[:, 0, :].t()), bias=f32(nc.bias), k=nc.kernel_size[0],
                                  s=nc.stride[0], p=nc.padding[0], C=nc.out_channels))
        for rb in self.resblocks:
            if isinstance(rb, ResBlock1):
                ent = dict(kind=1, c1=[self._pack_conv(c, prec, device) for c in rb.convs1],
                           c2=[self._pack_conv(c, prec, device) for c in rb.convs2])
                if rb.convs1[0].in_channels == 16 and self.fused and self.backend != "simt":
                    ent["c1f"] = [self._pack_conv_folded_pair(c, prec, device) for c in rb.convs1]
                    ent["c2f"] = [self._pack_conv_folded_pair(c, prec, device) for c in rb.convs2]
                pk["res"].append(ent)
            else:
                pk["res"].append(dict(kind=2, c=[self._pack_conv(c, prec, device) for c in rb.convs]))
        post = _effective_weight(self.conv_post).detach().to(device=device, dtype=torch.float32)   # [1, C, 7]
        pk["post_w"] = post[0].t().contiguous()      # [k][C]
        pk["post_b"] = f32(self.conv_post.bias)
        pk["post_k"] = post.shape[2]
        pk["lin_w"] = f32(self.m_source.l_linear.weight).reshape(-1)
        pk["lin_b"] = f32(self.m_source.l_linear.bias).reshape(-1)
        self._pack, self._pack_key = pk, key
        return pk

    # ------------------------------------------------------------------------------------ forward
    def _conv(self, pc, in_planes, B, T, **kw):
        fold = pc.get("fold")
        if fold is not None and T % fold["F"] == 0:      # same memory viewed as [T/F, F*C] (see _fold_factor)
            pc, T = fold, T // fold["F"]
        N.conv_cl(in_planes, pc["w"], B, T, pc["Ci"], pc["N"], pc["shifts"], bias=pc["bias"], w_inv_scale=pc["inv"],
                  prec=self._pack["mma"], backend=pc["backend"], **kw)

    def _stage_fused(self, pk, i, Co) -> bool:
        """All three ResBlocks of stage i can run as fused pairs (tensor-core back end, ResBlock1, supported shapes)."""
        if not self.fused or self.backend == "simt":
            return False
        nk = self.num_kernels
        for j in range(nk):
            rb = pk["res"][i * nk + j]
            if rb["kind"] != 1:
                return False
            for c1, c2 in zip(rb["c1"], rb["c2"]):
                if c1["backend"] != N.BACKEND_TC or not N.respair_supported(Co, c1["K"], c1["d"], c2["K"]) or c2["d"] != 1:
                    return False
        return True

    def _stage_fused_run(self, pk, i, PA, B, Lo, Co, out_slope):
        """MRF stage (models.py:426-432) on fused pairs.  PA = planes of lrelu(x, 0.1).  Each ResBlock chain runs pair
        by pair on plane buffers (4 B/element in, 4 B/element out); one elementwise pass over the three chain outputs
        makes the next stage's input lrelu(sum / num_kernels)."""
        nk = self.num_kernels
        mma = pk["mma"]
        tmp = [torch.empty_like(PA), torch.empty_like(PA)]
        outs = []
        folded = all("c1f" in pk["res"][i * nk + j] for j in range(nk)) and Lo % 2 == 0 and all(
            N.respair_supported(2 * Co, a["K"], 1, b["K"]) for j in range(nk)
            for a, b in zip(pk["res"][i * nk + j].get("c1f", []), pk["res"][i * nk + j].get("c2f", [])))
        if folded:                       # same memory viewed as [Lo/2, 2*Co] (see _pack_conv_folded_pair)
            Lo, Co = Lo // 2, 2 * Co
        for j in range(nk):
            rb = pk["res"][i * nk + j]
            n = len(rb["c1"])
            src = PA
            for m in range(n):
                c1, c2 = (rb["c1f"][m], rb["c2f"][m]) if folded else (rb["c1"][m], rb["c2"][m])
                dst = tmp[m % 2] if m < n - 1 else torch.empty_like(PA)
                N.respair(src, c1["w"], c2["w"], c1["bias"], c2["bias"], B, Lo, Co, c1["K"], c1["d"], c2["K"],
                          out_planes=dst, w1_inv_scale=c1["inv"], w2_inv_scale=c2["inv"], in_slope=LRELU_SLOPE,
                          out_slope=LRELU_SLOPE, prec=mma, kmask1=c1.get("kmask", 0), kmask2=c2.get("kmask", 0))
                src = dst
            outs.append(src)
        nxt = tmp[0]
        N.mrf_finish(outs, nxt, in_slope=LRELU_SLOPE, scale=1.0 / nk, out_slope=out_slope, prec=pk["prec"])
        return nxt

    @torch.no_grad()
    def source(self, f0, S_hop, rand_ini=None, sine_noise=None, seed=None):
        """f0 [B,T] -> harmonic excitation [B, T*hop] (models.py:411-415).  rand_ini [B,9] / sine_noise [B,S,9] may
        be injected (parity tests); otherwise they are drawn (rand_ini from torch's generator, noise by Philox)."""
        pk = self._packed(f0.device)
        B, T = f0.shape
        dev = f0.device
        H = self.m_source.l_sin_gen.dim
        if rand_ini is None:
            rand_ini = torch.rand(B, H, device=dev)
        rand_ini = rand_ini.to(device=dev, dtype=torch.float32).clone()
        rand_ini[:, 0] = 0                                          # models.py:213
        S = T * S_hop
        lib = N.lib()
        ws = torch.empty((int(lib.fd_sinegen_ws_bytes(B, S)),), dtype=torch.uint8, device=dev)
        har = torch.empty((B, S), dtype=torch.float32, device=dev)
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        sg = self.m_source.l_sin_gen
        N.check(lib.fd_sinegen_fwd(N.ptr(f0.to(torch.float32).contiguous()), N.ptr(pk["lin_w"]), N.ptr(pk["lin_b"]),
                                   N.ptr(rand_ini.contiguous()),
                                   N.ptr(None if sine_noise is None else sine_noise.to(torch.float32).contiguous()),
                                   N.ptr(har), N.ptr(ws), B, T, S_hop, H, float(sg.sampling_rate), float(sg.sine_amp),
                                   float(sg.noise_std), seed, N.stream_ptr(dev)), "fd_sinegen_fwd")
        return har

    def _check_source_lengths(self, T):
        """fd_source_conv_fwd writes (S + 2p - k) / s + 1 rows of noise_convs[i](har) and stage i adds them to its
        T * prod(rates[:i+1]) rows.  With an odd stride s (upsample rates 3 or 5 after stage i) that is one row short,
        which the reference refuses with a shape error: refuse it too, before anything is launched."""
        S = T * int(np.prod(self.h.upsample_rates))
        L = T
        for i, (u, nc) in enumerate(zip(self.h.upsample_rates, self.noise_convs)):
            L *= u
            k, s, p = nc.kernel_size[0], nc.stride[0], nc.padding[0]
            n = (S + 2 * p - k) // s + 1
            if n != L:
                raise ValueError(f"noise_convs[{i}] (kernel {k}, stride {s}, padding {p}) gives {n} rows of the "
                                 f"{S}-sample excitation for a stage of {L} rows")

    @torch.no_grad()
    def forward(self, x, f0, rand_ini=None, sine_noise=None, seed=None):
        """x mel [B,M,T], f0 [B,T] or [B,1,T] -> wav [B,1,T*hop] (models.py:407-438)."""
        self._check_source_lengths(x.shape[-1])
        N.require_cuda(x, "mel")
        if f0.ndim == 3:
            f0 = f0[:, 0]
        dev = x.device
        pk = self._packed(dev)
        prec = pk["prec"]
        B, M, T = x.shape
        hop = int(np.prod(self.h.upsample_rates))
        har = self.source(f0, hop, rand_ini=rand_ini, sine_noise=sine_noise, seed=seed)
        S = T * hop
        lib = N.lib()
        st = N.stream_ptr(dev)
        i16 = dict(dtype=torch.int16, device=dev)
        f32 = dict(dtype=torch.float32, device=dev)

        mel_planes = N.split_ncw(x.to(torch.float32), prec)
        C0 = self.h.upsample_initial_channel
        cur = torch.empty((2, B, T, C0), **i16)          # lrelu(conv_pre(mel)) : input of ups[0]
        self._conv(pk["pre"], mel_planes, B, T, out_planes=cur, act=N.ACT_LRELU, act_slope=LRELU_SLOPE)
        L = T
        nk = self.num_kernels
        for i in range(self.num_upsamples):
            up, src = pk["ups"][i], pk["src"][i]
            u, Co = up["u"], up["Co"]
            Lo = L * u
            # excitation branch: noise_convs[i](har_source) -> fp32 [B, Lo, Co]
            xs_src = torch.empty((B, Lo, Co), **f32)
            N.check(lib.fd_source_conv_fwd(N.ptr(har), N.ptr(src["w_t"]), N.ptr(src["bias"]), N.ptr(xs_src), B, S, Co,
                                           src["k"], src["s"], src["p"], st), "fd_source_conv_fwd")
            # x = ups[i](lrelu(x)) + x_source  -> X (fp32 master) and PA = lrelu(X) planes
            PA = torch.empty((2, B, Lo, Co), **i16)
            last_stage = i == self.num_upsamples - 1
            if self._stage_fused(pk, i, Co):     # the residual stream lives in the planes only: no fp32 master
                self._conv(up, cur, B, L, addend=xs_src, out_planes=PA, act=N.ACT_LRELU, act_slope=LRELU_SLOPE)
                del xs_src
                cur = self._stage_fused_run(pk, i, PA, B, Lo, Co, 0.01 if last_stage else LRELU_SLOPE)
                L = Lo
                del PA
                continue
            X = torch.empty((B, Lo, Co), **f32)
            self._conv(up, cur, B, L, addend=xs_src, out_f32=X, out_planes=PA, act=N.ACT_LRELU, act_slope=LRELU_SLOPE)
            del xs_src
            XS = torch.empty((B, Lo, Co), **f32)
            nxt = torch.empty((2, B, Lo, Co), **i16)      # lrelu(xs / nk): next stage input (slope 0.01 at the end)
            PB = torch.empty((2, B, Lo, Co), **i16)
            PC = torch.empty((2, B, Lo, Co), **i16)
            Xj = torch.empty((B, Lo, Co), **f32)
            out_slope = 0.01 if last_stage else LRELU_SLOPE   # models.py:434 uses the default slope (SURVEY D9)
            for j in range(nk):
                rb = pk["res"][i * nk + j]
                final_kw = dict(out_f32=XS, out_accum=j > 0)
                if j == nk - 1:
                    final_kw.update(out_planes=nxt, planes_scale=1.0 / nk, act=N.ACT_LRELU, act_slope=out_slope)
                if rb["kind"] == 1:
                    n = len(rb["c1"])
                    for m in range(n):
                        inp = PA if m == 0 else PC
                        res = X if m == 0 else Xj
                        self._conv(rb["c1"][m], inp, B, Lo, out_planes=PB, act=N.ACT_LRELU, act_slope=LRELU_SLOPE)
                        if m < n - 1:
                            self._conv(rb["c2"][m], PB, B, Lo, res_f32=res, out_f32=Xj, out_planes=PC,
                                       act=N.ACT_LRELU, act_slope=LRELU_SLOPE)
                        else:
                            self._conv(rb["c2"][m], PB, B, Lo, res_f32=res, **final_kw)
                else:
                    # ResBlock2 (models.py:150-155) with the reference's aliasing: its LeakyReLU is IN PLACE, so the residual
                    # that is added is lrelu(x) (not x), and the stage input shared by the three blocks (models.py:426-430)
                    # has been LeakyReLU'd once more for every block that ran before: block j sees u_j = lrelu^(j+1)(x).
                    # Everything therefore lives in plane tensors: conv input = residual = planes of the lrelu'd value.
                    n = len(rb["c"])
                    if j == 0:
                        U = PA                                    # planes of lrelu(x)
                    else:
                        U2 = torch.empty_like(PA)                 # one more LeakyReLU on the shared stage input
                        N.mrf_finish([U], U2, in_slope=1.0, scale=1.0, out_slope=LRELU_SLOPE, prec=pk["prec"])
                        U = U2
                    inp = U
                    for m in range(n):
                        if m < n - 1:
                            self._conv(rb["c"][m], inp, B, Lo, res_planes=inp, out_planes=PC, act=N.ACT_LRELU,
                                       act_slope=LRELU_SLOPE)
                            inp = PC
                            PC = torch.empty_like(PC)
                        else:
                            self._conv(rb["c"][m], inp, B, Lo, res_planes=inp, **final_kw)
            cur, L = nxt, Lo
            del X, PA, XS, PB, PC, Xj
        wav = torch.empty((B, 1, S), **f32)
        N.check(lib.fd_conv_post_fwd(N.ptr(cur), N.ptr(pk["post_w"]), N.ptr(pk["post_b"]), N.ptr(wav), B, S,
                                     cur.shape[3], pk["post_k"], prec, st), "fd_conv_post_fwd")
        return wav


try:  # pragma: no cover - lightning is absent from the build image
    import pytorch_lightning as pl
    _Base = pl.LightningModule
except Exception:  # noqa: BLE001
    _Base = nn.Module


@VOCODERS.register_module(name="NsfHifiGAN", force=True)
class NsfHifiGAN(_Base):
    """Wrapper with the reference constructor / methods (nsf_hifigan.py:16-107).  Extension: `checkpoint_path`
    may be None when `config` (dict) is given -- a randomly initialised generator for synthetic benchmarks."""

    def __init__(self, checkpoint_path: Optional[str] = "checkpoints/nsf_hifigan/model",
                 config_file: Optional[str] = None, use_natural_log: bool = True, config: Optional[dict] = None,
                 precision: str = "f16", backend: str = "auto", **kwargs):
        super().__init__()
        if config is None:
            if config_file is None:
                config_file = Path(checkpoint_path).parent / "config.json"
            with open(config_file) as f:
                config = json.loads(f.read())
        self.h = AttrDict(config)
        self.model = Generator(self.h, precision=precision, backend=backend)
        self.use_natural_log = use_natural_log
        if checkpoint_path is not None:
            cp_dict = torch.load(checkpoint_path, map_location="cpu")
            if "state_dict" not in cp_dict:
                self.model.load_state_dict(cp_dict["generator"])
            else:
                self.model.load_state_dict({k.replace("generator.", ""): v for k, v in cp_dict["state_dict"].items()
                                            if k.startswith("generator.")})
        self.model.eval()
        self.model.remove_weight_norm()
        self.mel_transform = PitchAdjustableMelSpectrogram(
            sample_rate=self.h.sampling_rate, n_fft=self.h.n_fft, win_length=self.h.win_size,
            hop_length=self.h.hop_size, f_min=self.h.fmin, f_max=self.h.fmax, n_mels=self.h.num_mels,
            precision=precision, backend=backend)
        if "mel_channels" in kwargs:
            kwargs["num_mels"] = kwargs.pop("mel_channels")
        for k, v in kwargs.items():
            if getattr(self.h, k, None) != v:
                raise ValueError(f"Incorrect value for {k}: {v}")

    if _Base is nn.Module:
        def freeze(self):
            for p in self.parameters():
                p.requires_grad = False
            self.eval()

    @property
    def device(self):
        return next(self.model.parameters()).device

    @torch.no_grad()
    def spec2wav(self, mel, f0, key_shift=0):
        c = mel[None]
        if key_shift is not None and key_shift != 0:
            f0 *= 2 ** (key_shift / 12)          # in place, like the reference (nsf_hifigan.py:76-77)
        if self.use_natural_log is False:
            c = 2.30259 * c
        f0 = f0[None].to(c.dtype)
        return self.model(c, f0).view(-1)

    @torch.no_grad()
    def wav2spec(self, wav_torch, sr=None, key_shift=0, speed=1.0):
        if sr is None:
            sr = self.h.sampling_rate
        if sr != self.h.sampling_rate:
            wav_torch = resample(wav_torch, sr, self.h.sampling_rate)   # on the device (librosa.resample in the reference)
        mel_torch = self.mel_transform(wav_torch, key_shift=key_shift, speed=speed)[0]
        mel_torch = dynamic_range_compression(mel_torch)
        if self.use_natural_log is False:
            mel_torch = 0.434294 * mel_torch
        return mel_torch
