"""The conditioner projection computed once per sampler call (fd_wavenet_cond_proj) instead of inside every GEMM1 launch.

With `cond_proj`, fd_wavenet_fwd runs each layer's GEMM1 over the three conv taps only and adds the layer's projection
(fp32, packed column order) in the gate epilogue.  Checked here:
  * a whole WaveNet evaluation on the hoisted path against the float64 oracle and against the fused path, on both back
    ends, at C = 128 / 256 / 512, E = 256, dilations 1..8, T < 64 and ragged T, odd B and odd tile counts, Bs = 1 and
    Bs = B, x / cond masks, f16 / bf16 / f16x1;
  * placement: one item's eps is bit-identical whether it runs alone or at any position of a batch;
  * the sampler: no stale projection across calls (new features, new weights) through the same workspace and graphs,
    and the fused fallback when the projection does not fit or the GEMMs run one product;
  * argument checks of fd_wavenet_cond_proj (no GPU needed: they refuse before any launch).
"""
import ctypes
import zlib

import numpy as np
import pytest
import torch

from conftest import rel_l2
from fish_diffusion_b200 import DIFFUSIONS, WaveNet
from fish_diffusion_b200 import _native as N
from oracle import wavenet as ownet

gpu = pytest.mark.gpu

# relative L2 bounds of tests/test_gpu_wavenet.py (f16 / bf16) and tests/test_gpu_single_product.py (f16x1)
TOL = {"f16": 2e-5, "bf16": 3e-4, "f16x1": 2e-3}


def _dev():
    return torch.device("cuda:0")


def _weights(seed, M, E, C, L):
    return ownet.make_wavenet_weights(seed, mel_channels=M, d_encoder=E, residual_channels=C, residual_layers=L)


def _net(sd, M, E, C, L, prec, backend):
    net = WaveNet(mel_channels=M, d_encoder=E, residual_channels=C, residual_layers=L, use_linear_bias=True,
                  dilation_cycle=4, precision=prec, backend=backend).to(_dev())
    net.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    net.use_graph = False
    return net.eval()


def _eval(net, x, steps, cond, x_mask=None, cond_mask=None, hoist=True):
    """x [B,T,M], cond [B,T,E] fp32 device, masks bool [B,T] -> eps [B,T,M] (fd_wavenet_fwd, hoisted or fused)"""
    pc = N.prec_code(net.precision)
    cm = None if cond_mask is None else cond_mask.to(torch.uint8).contiguous()
    cond_planes = N.split_nwc(cond, pc, mask=cm)
    x_planes = N.split_nwc(x, pc)
    proj = None
    if hoist:
        B, T = x.shape[:2]
        proj = net.cond_projection(cond_planes, torch.empty(net.cond_proj_shape(B, T), device=_dev()))
    eps = net.forward_cl(x_planes, steps, cond_planes, x_mask=x_mask, cond_proj=proj)
    torch.cuda.synchronize()
    return eps.clone()


# (C, E, M, L, B, T, Bs, precision, masks); L = 4 with dilation cycle 4: dilations 1, 2, 4, 8.  Row tiles of the
# ping-pong GEMMs = B * ceil(T / 64)
CASES = [
    (128, 256, 64, 4, 3, 40, 3, "f16", False),       # T < 64, 3 tiles, per-item steps
    (128, 256, 64, 4, 3, 130, 1, "bf16", True),      # ragged T, 9 tiles, masks
    (256, 256, 64, 4, 5, 77, 5, "f16x1", True),      # 10 tiles over odd B
    (256, 256, 128, 4, 1, 200, 1, "f16", False),     # 4 tiles, B = 1
    (512, 256, 128, 4, 3, 130, 1, "f16", True),      # the headline width, 9 tiles
    (512, 256, 128, 4, 1, 192, 1, "bf16", False),    # 3 tiles
    (512, 256, 128, 4, 3, 63, 3, "f16x1", False),    # T < 64
]


@gpu
@pytest.mark.parametrize("backend", ["tc", "simt"])
@pytest.mark.parametrize("case", CASES, ids=[f"c{c[0]}-B{c[4]}-T{c[5]}-Bs{c[6]}-{c[7]}{'-mask' if c[8] else ''}"
                                             for c in CASES])
def test_hoisted_forward_vs_float64_and_fused(case, backend):
    C, E, M, L, B, T, Bs, prec, masked = case
    seed = zlib.crc32(repr(case).encode()) & 0xFFFF
    sd = _weights(seed, M, E, C, L)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, M, generator=g)
    cond = torch.randn(B, T, E, generator=g)
    steps = torch.tensor([990.0, 17.0, 503.25, 40.0, 3.0][:Bs])
    xm = cm = None
    if masked:
        lens = [T - 7 * (i + 1) for i in range(B)]
        xm = torch.stack([torch.arange(T) >= n for n in lens])
        cm = xm
    ref = ownet.wavenet_forward(sd, x.transpose(1, 2).numpy(), steps.numpy(), cond.transpose(1, 2).numpy(),
                                x_masks=None if xm is None else xm.numpy(), cond_masks=None if cm is None else cm.numpy(),
                                dilation_cycle=4).transpose(0, 2, 1)
    net = _net(sd, M, E, C, L, prec, backend)
    d = _dev()
    args = (x.to(d), steps.to(d), cond.to(d), None if xm is None else xm.to(d), None if cm is None else cm.to(d))
    hoisted = _eval(net, *args, hoist=True).cpu().numpy()
    fused = _eval(net, *args, hoist=False).cpu().numpy()
    e64, ef = rel_l2(hoisted, ref), rel_l2(hoisted, fused)
    print(f"cond_proj[{case},{backend}] rel-L2 vs float64 {e64:.2e} (fused {rel_l2(fused, ref):.2e}), vs fused {ef:.2e}")
    assert e64 < TOL[prec] and ef < TOL[prec]
    if masked:
        for i in range(B):
            assert np.all(hoisted[i, T - 7 * (i + 1):] == 0)


@gpu
@pytest.mark.parametrize("prec", ["f16", "bf16x1"])
def test_hoisted_item_bits_independent_of_placement(prec):
    """3 row tiles per item (T = 130): an item's tiles start at a different pair half and warpgroup at each batch
    position, and its rows at a different place in the projection buffer."""
    C, E, M, L, B, T = 512, 256, 128, 4, 5, 130
    net = _net(_weights(31, M, E, C, L), M, E, C, L, prec, "tc")
    g = torch.Generator().manual_seed(31)
    x, cond = torch.randn(B, T, M, generator=g).to(_dev()), torch.randn(B, T, E, generator=g).to(_dev())
    steps = torch.tensor([990.0, 17.0, 503.25, 40.0, 3.0], device=_dev())
    batch = _eval(net, x, steps, cond)
    rev = _eval(net, x.flip(0), steps.flip(0), cond.flip(0))
    for j in range(B):
        alone = _eval(net, x[j:j + 1], steps[j:j + 1], cond[j:j + 1])
        assert torch.equal(alone[0], batch[j]), f"item {j} differs between B=1 and batch position {j}"
        assert torch.equal(alone[0], rev[B - 1 - j]), f"item {j} differs between B=1 and batch position {B - 1 - j}"


# ------------------------------------------------------------------ sampler
SCFG = dict(mel_channels=64, d_encoder=256, residual_channels=128, residual_layers=4, use_linear_bias=True,
            dilation_cycle=4)


def _diffusion(seed):
    d = DIFFUSIONS.build(dict(type="GaussianDiffusion", denoiser=dict(type="WaveNetDenoiser", backend="tc", **SCFG),
                              mel_channels=64, noise_schedule="linear", timesteps=1000, max_beta=0.01,
                              sampler_interval=100, spec_min=[-5.0], spec_max=[0.0], noise_predictor="naive"))
    d = d.to(_dev()).eval()
    d.denoise_fn.load_state_dict({k: torch.from_numpy(v) for k, v in _weights(seed, 64, 256, 128, 4).items()})
    return d


def _feats(seed, B=3, T=130):
    return torch.randn(B, T, 256, generator=torch.Generator().manual_seed(seed)).to(_dev())


@gpu
@pytest.mark.parametrize("pred", ["naive", "unipc", "plms"])
def test_sampler_has_no_stale_projection(pred):
    """Consecutive calls on one module reuse the sampler workspace (projection buffer included) and replay the
    denoiser's captured graphs; each call must still equal a fresh module's, after new features and after new weights."""
    diff = _diffusion(41)
    f1, f2 = _feats(1), _feats(2)
    a = diff(f1, noise_predictor=pred, seed=5)
    assert diff._sws.get("cond_proj") is not None                       # the hoisted path ran
    buf = diff._sws["cond_proj"].data_ptr()
    b = diff(f2, noise_predictor=pred, seed=5)
    assert diff._sws["cond_proj"].data_ptr() == buf
    if pred != "plms":      # PLMS hands every evaluation a fresh eps tensor, so its evaluations run eagerly
        assert any(e["graph"] is not None for e in diff.denoise_fn._graphs.values())
    assert torch.equal(a, _diffusion(41)(f1, noise_predictor=pred, seed=5))
    assert torch.equal(b, _diffusion(41)(f2, noise_predictor=pred, seed=5))
    assert not torch.equal(a, b)
    diff.denoise_fn.load_state_dict({k: torch.from_numpy(v) for k, v in _weights(42, 64, 256, 128, 4).items()})
    c = diff(f2, noise_predictor=pred, seed=5)
    assert torch.equal(c, _diffusion(42)(f2, noise_predictor=pred, seed=5))
    assert not torch.equal(b, c)


@gpu
def test_sampler_falls_back_to_fused_gemm1_when_projection_does_not_fit(monkeypatch):
    from fish_diffusion_b200 import diffusion as D
    f = _feats(3)
    hoisted_diff = _diffusion(43)
    hoisted = hoisted_diff(f, seed=9)
    assert hoisted_diff._sws.get("cond_proj") is not None
    monkeypatch.setattr(D, "hoist_cond_proj", lambda denoiser, B, T, device: False)
    fused_diff = _diffusion(43)
    fused = fused_diff(f, seed=9)
    assert fused_diff._sws.get("cond_proj") is None
    e = rel_l2(fused.cpu().numpy(), hoisted.cpu().numpy())
    print(f"sampler hoisted vs fused rel-L2 {e:.2e}")
    assert e < TOL["f16"]


@gpu
def test_single_product_sampler_keeps_fused_gemm1():
    diff = _diffusion(44)
    diff.denoise_fn.precision = "f16x1"
    diff(_feats(4), seed=9)
    assert diff._sws.get("cond_proj") is None


@gpu
def test_hoisting_rule():
    """three products and at most a quarter of the card's total memory (L * 8C bytes per position)"""
    from fish_diffusion_b200.diffusion import hoist_cond_proj
    net = WaveNet(mel_channels=64, d_encoder=256, residual_channels=128, residual_layers=4)
    per_pos = 4 * 8 * 128
    fit = torch.cuda.mem_get_info(_dev())[1] // 4 // per_pos          # positions that fit
    assert hoist_cond_proj(net, 1, fit, _dev()) and not hoist_cond_proj(net, 1, fit + 1, _dev())
    for prec, hoisted in (("bf16", True), ("f16x1", False), ("bf16x1", False)):
        net.precision = prec
        assert hoist_cond_proj(net, 3, 130, _dev()) == hoisted


# ------------------------------------------------------------------ argument checks (no launch)
def _desc(**kw):
    d = N.WaveNetFwdDesc()
    d.cond_planes, d.cond_proj, d.w1, d.w1_lstride = 4096, 8192, 16384, 1024
    d.B, d.T, d.C, d.E, d.L = 2, 100, 512, 256, 20
    d.prec, d.backend = N.PREC_F16, N.BACKEND_TC
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("bad,msg", [
    (dict(cond_proj=None), "required"),
    (dict(cond_planes=None), "required"),
    (dict(w1=None), "required"),
    (dict(L=0), "out of range"),
    (dict(L=65), "out of range"),
    (dict(B=0), "bad shape"),
    (dict(C=500), "multiples of 8"),
    (dict(E=12), "multiples of 8"),
    (dict(B=1024, T=4096), "32-bit"),                 # B*T*2C = 2^32
])
def test_cond_proj_refuses_bad_arguments(bad, msg):
    lib = N.lib()
    rc = lib.fd_wavenet_cond_proj(ctypes.byref(_desc(**bad)), None)
    assert rc != 0 and msg in N.last_error()
    assert lib.fd_wavenet_cond_proj(None, None) != 0 and "null descriptor" in N.last_error()
