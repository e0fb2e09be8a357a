"""H100-native ConvNext denoiser: drop-in for the reference ``ConvNext`` of ``fish_diffusion/modules/convnext.py``.

Same constructor arguments, same ``state_dict`` keys and the same ``forward`` contract as the reference class
(convnext.py:155-261), registered as ``DENOISERS["ConvNextDenoiser"]``.  Inference only; the arithmetic runs in the
hand-written sm_90a kernels of libfishdiff_b200.so, there is no PyTorch/CPU fallback.

Data flow of one call (all activations channels-last split planes, see csrc/fd_common.cuh):
  step vectors (step MLP + all L diffusion_step_projections, 4 small launches) -> head GEMM (input_projection + GELU
  + mask) -> L x [dwln: mask(x + step + condition) -> depthwise k=7 conv -> LayerNorm | pwconv1 + GELU | pwconv2
  * gamma + residual + mask, in place] -> tail GEMMs (Conv1x1 + GELU, Conv1x1 + mask).
The condition (conditioner MLP, masked, then each layer's condition_projection) is computed once per sampler call by
cond_projection, or inside the call when none is given.
"""
from __future__ import annotations

import ctypes
import math
import os

import torch
from torch import nn

from . import _native as N
from .graphs import run_cached
from .registry import DENOISERS
from .wavenet import DiffusionEmbedding


class ConvNeXtBlock(nn.Module):
    """Parameter holder for one block (convnext.py:12-53), reference key names, shapes and initialisation
    (gamma = 1e-6); computed by fd_convnext_dwln_fwd and two LINEAR tap-GEMMs."""

    def __init__(self, dim, intermediate_dim, dilation=1, layer_scale_init_value=1e-6):
        super().__init__()
        self.dilation = dilation
        self.dwconv = nn.Conv1d(dim, dim, kernel_size=7, groups=dim, dilation=dilation, padding=3 * dilation)
        self.norm = nn.LayerNorm(dim, eps=1e-6)
        self.pwconv1 = nn.Linear(dim, intermediate_dim)
        self.act = nn.GELU()
        self.pwconv2 = nn.Linear(intermediate_dim, dim)
        self.gamma = nn.Parameter(layer_scale_init_value * torch.ones(dim), requires_grad=True)
        self.diffusion_step_projection = nn.Conv1d(dim, dim, 1)
        self.condition_projection = nn.Conv1d(dim, dim, 1)


class ConvNext(nn.Module):
    """ConvNext denoiser (reference convnext.py:155-261) on sm_90a kernels.

    Extra keyword arguments (not in the reference, defaults keep reference configs working), as for the WaveNet:
      precision: "f16" / "bf16" split planes with three tensor-core products, "f16x1" / "bf16x1" one product
      backend:   "auto" (wgmma where every GEMM shape has a tensor-core instantiation, else the SIMT twin), "tc", "simt"
    cross_attention=True (interleaved nn.TransformerDecoderLayer blocks) is not implemented and raises.
    gradient_checkpointing is accepted and has no effect: there is no training path.
    """

    def __init__(self, mel_channels=128, dim=512, mlp_factor=4, condition_dim=256, num_layers=20, dilation_cycle=4,
                 gradient_checkpointing=False, cross_attention=False, cross_every_n_layers=5, precision="f16",
                 backend="auto"):
        super().__init__()
        if cross_attention:
            raise NotImplementedError("fish_diffusion_b200.ConvNext: cross_attention=True (the interleaved "
                                      "TransformerDecoderLayer blocks) is not implemented")
        if num_layers > 64:
            raise ValueError("fd_convnext_fwd supports up to 64 layers")
        self.mel_channels, self.dim, self.hidden, self.condition_dim = mel_channels, dim, dim * mlp_factor, condition_dim
        self.n_layers = num_layers
        self.input_projection = nn.Conv1d(mel_channels, dim, 1)
        self.diffusion_embedding = nn.Sequential(
            DiffusionEmbedding(dim), nn.Linear(dim, dim * mlp_factor), nn.GELU(), nn.Linear(dim * mlp_factor, dim))
        self.conditioner_projection = nn.Sequential(
            nn.Conv1d(condition_dim, dim * mlp_factor, 1), nn.GELU(), nn.Conv1d(dim * mlp_factor, dim, 1))
        self.residual_layers = nn.ModuleList([
            ConvNeXtBlock(dim, dim * mlp_factor, dilation=2 ** (i % dilation_cycle)) for i in range(num_layers)])
        self.output_projection = nn.Sequential(
            nn.Conv1d(dim, dim, kernel_size=1), nn.GELU(), nn.Conv1d(dim, mel_channels, kernel_size=1))
        self.gradient_checkpointing = gradient_checkpointing
        self.cross_attention = cross_attention

        self.precision = precision
        self.backend = os.environ.get("FD_BACKEND", backend)
        self._pack = None
        self._pack_key = None
        self._ws = {}
        self._graphs = {}
        # CUDA-graph replay of repeated evaluations on the same buffers (the sampler loop); FD_GRAPH=0 disables it
        self.use_graph = os.environ.get("FD_GRAPH", "1") != "0"

    # ------------------------------------------------------------------------------------ packing
    def _gemm_shapes(self):
        """(N, K) of every GEMM of a call"""
        C, H, E, M = self.dim, self.hidden, self.condition_dim, self.mel_channels
        return [(C, M), (H, E), (C, H), (C, C), (H, C), (M, C)]

    def _resolve_backend(self) -> int:
        if self.backend != "auto":
            return N.backend_code(self.backend)
        ok = all(N.tc_supported_linear(n, k, 1) for n, k in self._gemm_shapes())
        return N.BACKEND_TC if ok else N.BACKEND_SIMT

    def _packed(self, device):
        """Packed weights for `device`, rebuilt whenever a parameter changed (version counters).  Every GEMM weight is
        prescaled by a power of two (max |w| * s in [32, 64), undone by the kernels' acc_scale); gamma is folded into
        pwconv2's rows and bias first."""
        key = (str(device), self.precision, tuple(p._version for p in self.parameters()),
               tuple(p.data_ptr() for p in self.parameters()))
        if self._pack is not None and self._pack_key == key:
            return self._pack
        prec = N.prec_code(self.precision)
        L = self.n_layers
        f32 = lambda t: t.detach().to(device=device, dtype=torch.float32)
        blocks = list(self.residual_layers)
        gamma = [f32(b.gamma) for b in blocks]
        mats = {"in": f32(self.input_projection.weight)[:, :, 0],
                "c1": f32(self.conditioner_projection[0].weight)[:, :, 0],
                "c2": f32(self.conditioner_projection[2].weight)[:, :, 0],
                "o1": f32(self.output_projection[0].weight)[:, :, 0],
                "o2": f32(self.output_projection[2].weight)[:, :, 0]}
        for l, b in enumerate(blocks):
            mats[f"cp{l}"] = f32(b.condition_projection.weight)[:, :, 0]
            mats[f"pw1{l}"] = f32(b.pwconv1.weight)
            mats[f"pw2{l}"] = gamma[l][:, None] * f32(b.pwconv2.weight)
        names = list(mats)
        amax = torch.stack(torch._foreach_norm([mats[k] for k in names], float("inf"))).tolist()

        def p2(m):
            return 1.0 if m == 0.0 or m != m else float(2.0 ** math.floor(math.log2(64.0 / m)))

        scale = {k: p2(m) for k, m in zip(names, amax)}
        packed = {k: N.pack_weight(w, prec, scale[k]) for k, w in mats.items()}
        pk = {"mma": N.mma_code(self.precision), "backend": self._resolve_backend(),
              "inv": {k: 1.0 / v for k, v in scale.items()}, "dil": [b.dilation for b in blocks]}
        for k in ("in", "c1", "c2", "o1", "o2"):
            pk["w_" + k] = packed[k]
        pk["w_cp"] = torch.stack([packed[f"cp{l}"] for l in range(L)]).contiguous()
        pk["w_pw1"] = torch.stack([packed[f"pw1{l}"] for l in range(L)]).contiguous()
        pk["w_pw2"] = torch.stack([packed[f"pw2{l}"] for l in range(L)]).contiguous()
        pk["b_in"] = f32(self.input_projection.bias).contiguous()
        pk["b_c1"] = f32(self.conditioner_projection[0].bias).contiguous()
        pk["b_c2"] = f32(self.conditioner_projection[2].bias).contiguous()
        pk["b_o1"] = f32(self.output_projection[0].bias).contiguous()
        pk["b_o2"] = f32(self.output_projection[2].bias).contiguous()
        emb = self.diffusion_embedding
        pk["emb_w0"], pk["emb_b0"] = f32(emb[1].weight).contiguous(), f32(emb[1].bias).contiguous()
        pk["emb_w1"], pk["emb_b1"] = f32(emb[3].weight).contiguous(), f32(emb[3].bias).contiguous()
        pk["w_step"] = torch.cat([f32(b.diffusion_step_projection.weight)[:, :, 0] for b in blocks]).contiguous()
        pk["b_step"] = torch.cat([f32(b.diffusion_step_projection.bias) + f32(b.condition_projection.bias)
                                  for b in blocks]).contiguous()
        pk["dw_w"] = torch.stack([f32(b.dwconv.weight)[:, 0, :] for b in blocks]).contiguous()
        pk["dw_b"] = torch.stack([f32(b.dwconv.bias) for b in blocks]).contiguous()
        pk["ln_w"] = torch.stack([f32(b.norm.weight) for b in blocks]).contiguous()
        pk["ln_b"] = torch.stack([f32(b.norm.bias) for b in blocks]).contiguous()
        pk["b_pw1"] = torch.stack([f32(b.pwconv1.bias) for b in blocks]).contiguous()
        pk["b_pw2"] = torch.stack([gamma[l] * f32(b.pwconv2.bias) for l, b in enumerate(blocks)]).contiguous()
        self._pack, self._pack_key = pk, key
        return pk

    def _workspace(self, device, B, T):
        """Activation planes and scratch of a [B, T] call; the step buffers are sized for per-item steps (Bs = B)."""
        key = (str(device), B, T)
        ws = self._ws.get(key)
        if ws is None:
            C, H, L = self.dim, self.hidden, self.n_layers
            i16 = dict(dtype=torch.int16, device=device)
            f32 = dict(dtype=torch.float32, device=device)
            ws = {"xr": torch.empty((2, B, T, C), **i16), "a": torch.empty((2, B, T, C), **i16),
                  "h": torch.empty((2, B, T, H), **i16), "cpl": torch.empty((2, B, T, C), **i16),
                  "p": torch.empty((B, T, C), **f32), "s": torch.empty((B, C), **f32),
                  "sv": torch.empty((B, L * C), **f32), "mlp_ws": torch.empty((B * (C + H),), **f32),
                  "steps": torch.empty((B,), **f32)}
            self._ws = {key: ws}   # keep one shape resident
            self._graphs = {}      # captured evaluations reference the old workspace
        return ws

    def _desc(self, pk, ws, B, T, Bs):
        d = N.ConvNextFwdDesc()
        inv = pk["inv"]
        d.w_in, d.b_in, d.w_in_inv = N.ptr(pk["w_in"]), N.ptr(pk["b_in"]), inv["in"]
        d.emb_w0, d.emb_b0, d.emb_w1, d.emb_b1 = (N.ptr(pk["emb_w0"]), N.ptr(pk["emb_b0"]), N.ptr(pk["emb_w1"]),
                                                  N.ptr(pk["emb_b1"]))
        d.w_step, d.b_step = N.ptr(pk["w_step"]), N.ptr(pk["b_step"])
        d.w_c1, d.b_c1, d.w_c1_inv = N.ptr(pk["w_c1"]), N.ptr(pk["b_c1"]), inv["c1"]
        d.w_c2, d.b_c2, d.w_c2_inv = N.ptr(pk["w_c2"]), N.ptr(pk["b_c2"]), inv["c2"]
        d.w_cp, d.dw_w, d.dw_b, d.ln_w, d.ln_b = (N.ptr(pk["w_cp"]), N.ptr(pk["dw_w"]), N.ptr(pk["dw_b"]),
                                                  N.ptr(pk["ln_w"]), N.ptr(pk["ln_b"]))
        d.w_pw1, d.b_pw1, d.w_pw2, d.b_pw2 = N.ptr(pk["w_pw1"]), N.ptr(pk["b_pw1"]), N.ptr(pk["w_pw2"]), N.ptr(pk["b_pw2"])
        d.w_o1, d.b_o1, d.w_o1_inv = N.ptr(pk["w_o1"]), N.ptr(pk["b_o1"]), inv["o1"]
        d.w_o2, d.b_o2, d.w_o2_inv = N.ptr(pk["w_o2"]), N.ptr(pk["b_o2"]), inv["o2"]
        for l in range(self.n_layers):
            d.w_cp_inv[l], d.w_pw1_inv[l], d.w_pw2_inv[l] = inv[f"cp{l}"], inv[f"pw1{l}"], inv[f"pw2{l}"]
            d.dilation[l] = pk["dil"][l]
        d.xr, d.a, d.h, d.cpl, d.p = N.ptr(ws["xr"]), N.ptr(ws["a"]), N.ptr(ws["h"]), N.ptr(ws["cpl"]), N.ptr(ws["p"])
        d.s, d.sv, d.mlp_ws = N.ptr(ws["s"]), N.ptr(ws["sv"]), N.ptr(ws["mlp_ws"])
        d.B, d.T, d.M, d.C, d.H, d.E, d.L, d.Bs = (B, T, self.mel_channels, self.dim, self.hidden, self.condition_dim,
                                                   self.n_layers, Bs)
        d.prec, d.backend = pk["mma"], pk["backend"]
        return d

    @staticmethod
    def _u8(mask, dev):
        return None if mask is None else mask.to(device=dev, dtype=torch.uint8).contiguous()

    # ------------------------------------------------------------------------------------ native forward
    def cond_proj_shape(self, B, T):
        """Shape of the buffer cond_projection fills: [L, B, T, C] fp32 (L * 4C bytes per position)."""
        return (self.n_layers, B, T, self.dim)

    @torch.no_grad()
    def cond_projection(self, cond_planes, out, cond_mask=None):
        """conditioner_projection(conditioner) masked by cond_mask (convnext.py:234, 239-240), then every layer's
        condition_projection without its bias (:73), for cond_planes [2,B,T,E], into the caller-owned fp32 buffer
        `out` (cond_proj_shape): fd_convnext_cond_proj.  forward_cl(..., cond_proj=out) then skips that work; a
        sampler computes it once per call, since all its evaluations share the conditioner.  Returns `out`."""
        dev = cond_planes.device
        N.require_cuda(cond_planes, "cond_planes")
        _, B, T, E = cond_planes.shape
        if E != self.condition_dim or tuple(out.shape) != self.cond_proj_shape(B, T) or out.dtype != torch.float32 \
                or not out.is_contiguous() or out.device != dev:
            raise ValueError(f"cond_projection: out must be contiguous float32 {self.cond_proj_shape(B, T)} on {dev}")
        pk = self._packed(dev)
        d = self._desc(pk, self._workspace(dev, B, T), B, T, 1)
        cmask = self._u8(cond_mask, dev)
        d.cond_planes, d.cond_mask, d.cond_proj = N.ptr(cond_planes), N.ptr(cmask), N.ptr(out)
        N.check(N.lib().fd_convnext_cond_proj(ctypes.byref(d), N.stream_ptr(dev)), "fd_convnext_cond_proj")
        return out

    @torch.no_grad()
    def forward_cl(self, x_planes, steps, cond_planes, x_mask=None, out=None, cond_proj=None, cond_mask=None):
        """Channels-last entry used by the fused sampler.

        x_planes [2,B,T,M] int16 split planes, steps float32 [1] or [B] (device), cond_planes [2,B,T,E],
        x_mask / cond_mask uint8/bool [B,T] or None (True = masked).  cond_proj: what cond_projection made of these
        cond_planes and cond_mask under the current weights, or None (the call then runs the conditioner MLP, masked
        by cond_mask, and each layer's condition projection itself).  Returns eps fp32 [B,T,M]."""
        dev = x_planes.device
        N.require_cuda(x_planes, "x_planes")
        _, B, T, M = x_planes.shape
        if M != self.mel_channels or tuple(cond_planes.shape) != (2, B, T, self.condition_dim):
            raise ValueError(f"x_planes / cond_planes do not match mel_channels={self.mel_channels}, "
                             f"condition_dim={self.condition_dim}")
        if cond_proj is not None and (tuple(cond_proj.shape) != self.cond_proj_shape(B, T) or
                                      cond_proj.dtype != torch.float32 or not cond_proj.is_contiguous()):
            raise ValueError(f"cond_proj must be contiguous float32 {self.cond_proj_shape(B, T)}")
        pk = self._packed(dev)
        steps = steps.to(device=dev, dtype=torch.float32).reshape(-1).contiguous()
        Bs = steps.numel()
        if Bs not in (1, B):
            raise ValueError(f"diffusion_step must have 1 or B={B} entries, got {Bs}")
        ws = self._workspace(dev, B, T)
        x_mask, cond_mask = self._u8(x_mask, dev), self._u8(cond_mask, dev)
        if out is None:
            out = torch.empty((B, T, M), dtype=torch.float32, device=dev)
        steps_buf = ws["steps"][:Bs]
        steps_buf.copy_(steps, non_blocking=True)
        d = self._desc(pk, ws, B, T, Bs)
        d.x_planes, d.cond_planes, d.steps, d.out = N.ptr(x_planes), N.ptr(cond_planes), N.ptr(steps_buf), N.ptr(out)
        d.x_mask, d.cond_mask, d.cond_proj = N.ptr(x_mask), N.ptr(cond_mask), N.ptr(cond_proj)
        lib = N.lib()
        key = (x_planes.data_ptr(), cond_planes.data_ptr(), out.data_ptr(), 0 if x_mask is None else x_mask.data_ptr(),
               0 if cond_mask is None else cond_mask.data_ptr(), 0 if cond_proj is None else cond_proj.data_ptr(),
               B, T, Bs, self._pack_key, id(ws))
        run_cached(self._graphs, key, (x_planes, cond_planes, out, x_mask, cond_mask, cond_proj, pk),
                   lambda: N.check(lib.fd_convnext_fwd(ctypes.byref(d), N.stream_ptr(dev)), "fd_convnext_fwd"), dev,
                   self.use_graph)
        return out

    def forward_train_cl(self, *args, **kwargs):
        raise NotImplementedError("fish_diffusion_b200.ConvNext is inference only: training (backward) of the ConvNext "
                                  "denoiser is not implemented; run it under torch.no_grad()")

    def forward(self, x, diffusion_step, conditioner, x_masks=None, cond_masks=None):
        """Reference contract (convnext.py:208-261): x [B,M,T] (or [B,1,M,T]), diffusion_step [B] or [1] (int64 or
        float), conditioner [B,E,T], masks [B,T] bool -> [B,M,T] (4-D in -> 4-D out).  Inference only."""
        if torch.is_grad_enabled() and (x.requires_grad or conditioner.requires_grad or
                                        any(p.requires_grad for p in self.parameters())):
            self.forward_train_cl()
        use_4_dim = x.dim() == 4
        if use_4_dim:
            x = x[:, 0]
        assert x.dim() == 3, f"mel must be 3 dim tensor, but got {x.dim()}"
        N.require_cuda(x, "x")
        prec = N.prec_code(self.precision)
        B, M, T = x.shape
        x_planes = N.split_ncw(x.to(torch.float32), prec)
        cond_planes = N.split_ncw(conditioner.to(torch.float32), prec)
        eps = self.forward_cl(x_planes, diffusion_step.to(torch.float32), cond_planes, x_mask=x_masks,
                              cond_mask=cond_masks)
        out = torch.empty((B, M, T), dtype=torch.float32, device=x.device)
        N.check(N.lib().fd_transpose_nwc_to_ncw(N.ptr(eps), N.ptr(out), B, T, M, N.stream_ptr(x.device)),
                "fd_transpose_nwc_to_ncw")
        return out[:, None] if use_4_dim else out


DENOISERS.register_module(name="ConvNextDenoiser", module=ConvNext, force=True)
