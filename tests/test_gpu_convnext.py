"""The ConvNext denoiser on the H100, against float64 and against the reference's own outputs (tests/golden/convnext.npz).

  * fd_convnext_dwln_fwd alone against a float64 restatement on the exact plane values: dilations 1..64, T = 1, T below
    the halo, ragged T over many tiles, masks, shared and per-item steps, C = 512 / 1024 and a width no tensor-core GEMM
    takes;
  * the GELU activation of the LINEAR epilogue on both back ends against float64, and tc against SIMT;
  * the whole forward at the default configuration (several row tiles) against the oracle, hoisted and not;
  * every golden case and sampler trajectory of the reference;
  * no stale projection or graph across sampler calls; an item's output does not depend on its batch position.
Bounds: the WaveNet's (tests/test_gpu_cond_proj.py TOL): rel-L2 2e-5 (f16), 3e-4 (bf16), 2e-3 (f16x1).
"""
import json

import numpy as np
import pytest
import torch

from conftest import rel_l2
from fish_diffusion_b200 import DIFFUSIONS, ConvNext
from fish_diffusion_b200 import _native as N
from oracle import convnext as ocnx

pytestmark = pytest.mark.gpu

TOL = {"f16": 2e-5, "bf16": 3e-4, "f16x1": 2e-3}


def dev():
    return torch.device("cuda:0")


def T_(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def planes_value(planes, prec):
    """exact float64 values of split planes [2, ...] (int16 storage)"""
    u = planes.cpu().numpy().view(np.uint16)
    if prec == N.PREC_F16:
        f = u.view(np.float16).astype(np.float64)
    else:
        f = (u.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    return f[0] + f[1]


# ------------------------------------------------------------------ block front alone
def dwln_ref(x, p, s, mask, w, b, lw, lb, dil):
    """float64: x / p [B,T,C], s [B or 1, C], mask [B,T] bool or None"""
    u = x + s[:, None, :] + p
    if mask is not None:
        u = np.where(mask[:, :, None], 0.0, u)
    v = ocnx.dwconv(u.transpose(0, 2, 1), w[:, None, :], b, dil).transpose(0, 2, 1)
    return ocnx.layer_norm(v, lw, lb)


DW_CASES = [  # (C, B, T, dilation, Bs, masked, precision)
    (512, 2, 1, 1, 2, False, "f16"),          # T = 1
    (512, 3, 10, 4, 1, True, "f16"),          # T below the halo (12)
    (512, 2, 77, 1, 2, True, "bf16"),         # ragged T, 5 tiles
    (512, 2, 130, 2, 1, False, "f16"),
    (512, 1, 301, 8, 1, True, "f16"),
    (512, 2, 200, 16, 2, False, "f16"),       # stp = tile height: seven disjoint windows
    (512, 2, 450, 64, 1, True, "bf16"),
    (1024, 2, 100, 4, 2, True, "f16"),        # the widest supported C
    (48, 3, 95, 2, 3, True, "f16"),           # a width without a tensor-core GEMM, partial channel chunk
    (208, 1, 33, 64, 1, False, "f16"),        # dilation past T: only the centre tap sees data
]


@pytest.mark.parametrize("case", DW_CASES, ids=[f"C{c[0]}-B{c[1]}-T{c[2]}-d{c[3]}-Bs{c[4]}{'-mask' if c[5] else ''}-{c[6]}"
                                                for c in DW_CASES])
def test_dwln_vs_float64(case):
    C, B, T, dil, Bs, masked, prec_name = case
    prec = N.prec_code(prec_name)
    rng = np.random.RandomState(C + T + dil)
    x = rng.randn(B, T, C).astype(np.float32)
    p = rng.randn(B, T, C).astype(np.float32)
    s = rng.randn(Bs, C).astype(np.float32)
    w = (rng.randn(C, 7) * 0.4).astype(np.float32)
    b, lw, lb = [(rng.randn(C) * 0.3 + o).astype(np.float32) for o in (0.0, 1.0, 0.0)]
    mask = np.stack([np.arange(T) >= max(1, T - 5 * i - 3) for i in range(B)]) if masked else None
    xp = N.split_nwc(T_(x), prec)
    out = torch.empty_like(xp)
    m = None if mask is None else T_(mask.astype(np.uint8))
    tw, tb, tlw, tlb, ts, tp = T_(w), T_(b), T_(lw), T_(lb), T_(s), T_(p)
    N.check(N.lib().fd_convnext_dwln_fwd(N.ptr(xp), N.ptr(tp), N.ptr(ts), C if Bs > 1 else 0, N.ptr(m), N.ptr(tw),
                                         N.ptr(tb), N.ptr(tlw), N.ptr(tlb), N.ptr(out), B, T, C, dil, prec,
                                         N.stream_ptr(dev())), "fd_convnext_dwln_fwd")
    torch.cuda.synchronize()
    ref = dwln_ref(planes_value(xp, prec), p.astype(np.float64), s.astype(np.float64), mask, w.astype(np.float64),
                   b.astype(np.float64), lw.astype(np.float64), lb.astype(np.float64), dil)
    got = planes_value(out, prec)
    e = rel_l2(got, ref)
    print(f"dwln[{case}] rel-L2 vs float64 {e:.2e}")
    assert e < TOL[prec_name]


# ------------------------------------------------------------------ GELU epilogue
@pytest.mark.parametrize("n_out", [512, 48])
@pytest.mark.parametrize("prec_name", ["f16", "bf16"])
def test_gelu_linear_epilogue_both_back_ends(n_out, prec_name):
    prec = N.prec_code(prec_name)
    B, T, K = 2, 150, 256
    rng = np.random.RandomState(n_out)
    x = rng.randn(B, T, K).astype(np.float32)
    w = (rng.randn(n_out, K) / 8).astype(np.float32)
    b = rng.randn(n_out).astype(np.float32)
    xp = N.split_nwc(T_(x), prec)
    wp = N.pack_weight(T_(w), prec, 32.0)
    ref = ocnx.gelu(planes_value(xp, prec) @ w.astype(np.float64).T + b)
    got = {}
    backends = ["tc", "simt"] if N.tc_supported_linear(n_out, K, 1) else ["simt"]
    for be in backends:
        out = torch.empty((2, B, T, n_out), dtype=torch.int16, device=dev())
        N.gemm_cl(xp, K, wp, n_out, K, B, T, [(0, 0, 0, K)], bias=T_(b), out_planes=out, w_inv_scale=1 / 32.0,
                  act=N.ACT_GELU, prec=prec, backend=N.backend_code(be))
        torch.cuda.synchronize()
        got[be] = planes_value(out, prec)
        e = rel_l2(got[be], ref)
        print(f"gelu epilogue[{be},{prec_name},N={n_out}] rel-L2 vs float64 {e:.2e}")
        assert e < TOL[prec_name]
    if len(got) == 2:
        assert rel_l2(got["tc"], got["simt"]) < TOL[prec_name]


# ------------------------------------------------------------------ whole forward at the default configuration
DEFAULT = dict(mel_channels=128, dim=512, mlp_factor=4, condition_dim=256, num_layers=20)
_sd_cache = {}


def _default_weights():
    if "sd" not in _sd_cache:
        _sd_cache["sd"] = ocnx.make_convnext_weights(71, **DEFAULT)
    return _sd_cache["sd"]


def _net(sd, cfg, precision="f16", backend="auto", graph=False):
    net = ConvNext(**cfg, precision=precision, backend=backend).to(dev())
    net.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    net.use_graph = graph
    return net.eval()


def _eval(net, x, steps, cond, x_mask=None, cond_mask=None, hoist=True):
    """x [B,T,M], cond [B,T,E] fp32 device -> eps [B,T,M] through forward_cl (hoisted projection or not)"""
    pc = N.prec_code(net.precision)
    cond_planes = N.split_nwc(cond, pc)
    x_planes = N.split_nwc(x, pc)
    proj = None
    if hoist:
        B, T = x.shape[:2]
        proj = net.cond_projection(cond_planes, torch.empty(net.cond_proj_shape(B, T), device=dev()),
                                   cond_mask=cond_mask)
    eps = net.forward_cl(x_planes, steps, cond_planes, x_mask=x_mask, cond_proj=proj, cond_mask=cond_mask)
    torch.cuda.synchronize()
    return eps.clone()


@pytest.mark.parametrize("precision,Bs,masked", [("f16", 1, True), ("bf16", 2, False), ("f16x1", 2, True)])
def test_default_forward_vs_oracle_hoisted_and_not(precision, Bs, masked):
    """B*T = 2 * 300: 10 row tiles of 64 in the ping-pong GEMMs, 38 dwln tiles; dilations 1, 2, 4, 8."""
    sd = _default_weights()
    B, T, M, E = 2, 300, 128, 256
    g = torch.Generator().manual_seed(72)
    x, cond = torch.randn(B, T, M, generator=g), torch.randn(B, T, E, generator=g)
    steps = torch.tensor([990.0, 17.0][:Bs])
    xm = cm = None
    if masked:
        xm = torch.stack([torch.arange(T) >= n for n in (300, 251)])
        cm = torch.stack([torch.arange(T) >= n for n in (280, 240)])
    ref = ocnx.convnext_forward(sd, x.transpose(1, 2).numpy(), steps.numpy(), cond.transpose(1, 2).numpy(),
                                x_masks=None if xm is None else xm.numpy(),
                                cond_masks=None if cm is None else cm.numpy()).transpose(0, 2, 1)
    net = _net(sd, DEFAULT, precision)
    assert net._resolve_backend() == N.BACKEND_TC
    d = lambda t: None if t is None else t.to(dev())
    args = (x.to(dev()), steps.to(dev()), cond.to(dev()), d(xm), d(cm))
    hoisted = _eval(net, *args, hoist=True).cpu().numpy()
    fused = _eval(net, *args, hoist=False).cpu().numpy()
    e64, ef = rel_l2(hoisted, ref), rel_l2(hoisted, fused)
    print(f"convnext default[{precision},Bs={Bs},mask={masked}] rel-L2 vs float64 {e64:.2e} "
          f"(not hoisted {rel_l2(fused, ref):.2e}), hoisted vs not {ef:.2e}")
    assert e64 < TOL[precision] and rel_l2(fused, ref) < TOL[precision] and ef < TOL[precision]
    if masked:
        assert np.all(hoisted[1, 251:] == 0)


def test_default_forward_simt_back_end_vs_oracle():
    sd = _default_weights()
    B, T = 1, 70
    g = torch.Generator().manual_seed(73)
    x, cond = torch.randn(B, 128, T, generator=g), torch.randn(B, 256, T, generator=g)
    ref = ocnx.convnext_forward(sd, x.numpy(), np.array([321]), cond.numpy())
    net = _net(sd, DEFAULT, "f16", backend="simt")
    with torch.no_grad():
        y = net(x.to(dev()), torch.tensor([321], device=dev()), cond.to(dev()))
    e = rel_l2(y.cpu().numpy(), ref)
    print(f"convnext default[simt] rel-L2 vs float64 {e:.2e}")
    assert e < TOL["f16"]


# ------------------------------------------------------------------ golden cases of the reference
def _golden_net(g, precision="f16", backend="auto"):
    cfg = json.loads(str(g["config_small"]))
    sd = {k[2:]: v for k, v in g.items() if k.startswith("w/")}
    return _net(sd, cfg, precision, backend)


@pytest.mark.parametrize("backend", ["auto", "simt"])
@pytest.mark.parametrize("case", ["stepsB_int", "stepsB_float", "steps1_int", "steps1_float", "masked",
                                  "cond_masked_only", "x_masked_only", "4d"])
def test_forward_vs_reference_golden(golden, case, backend):
    g = golden("convnext")
    net = _golden_net(g, backend=backend)
    steps = g["case_stepsB_int_steps"] if case == "4d" else g[f"case_{case}_steps"]
    x = g["x"][:, None] if case == "4d" else g["x"]
    kw = {}
    if case in ("masked", "x_masked_only"):
        kw["x_masks"] = T_(g["x_masks"])
    if case in ("masked", "cond_masked_only"):
        kw["cond_masks"] = T_(g["cond_masks"])
    with torch.no_grad():
        y = net(T_(x), T_(steps), T_(g["cond"]), **kw).cpu().numpy()
    ref = g[f"case_{case}_out"]
    assert y.shape == ref.shape
    e = rel_l2(y, ref)
    print(f"convnext golden[{case},{backend}] rel-L2 vs reference {e:.2e}")
    assert e < TOL["f16"]
    if "x_masks" in kw:
        assert np.all(y[1, ..., 29:] == 0)


def _golden_diffusion(g, pred, backend="auto"):
    cfg = json.loads(str(g["config_small"]))
    diff = DIFFUSIONS.build(dict(type="GaussianDiffusion", denoiser=dict(type="ConvNextDenoiser", backend=backend, **cfg),
                                 mel_channels=cfg["mel_channels"], noise_schedule="linear", timesteps=1000,
                                 max_beta=0.01, noise_loss="smoothed-l1", sampler_interval=100, spec_min=[-5.0],
                                 spec_max=[0.0], noise_predictor=pred)).to(dev())
    diff.denoise_fn.load_state_dict({k[2:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("w/")})
    return diff.eval()


@pytest.mark.parametrize("pred", ["naive", "plms", "unipc"])
def test_sampler_vs_reference_golden(golden, pred):
    g = golden("convnext")
    key = f"samp_{pred}"
    noises = [T_(g[key + f"_noise{j}"]) for j in range(int(g[key + "_nnoise"]))]
    diff = _golden_diffusion(g, pred)
    mel = diff(T_(g["samp_features"]), sampler_interval=100, noise_predictor=pred, x_T=noises[0],
               step_noises=noises[1:])
    assert diff._sws.get("cond_proj") is not None                       # the projection was hoisted
    e = rel_l2(mel.cpu().numpy(), g[key + "_mel"])
    print(f"convnext sampler[{pred}] rel-L2 vs reference {e:.2e}")
    assert mel.shape == g[key + "_mel"].shape
    assert e < 1e-4


def test_train_step_forward_only_under_no_grad(golden):
    g = golden("convnext")
    diff = _golden_diffusion(g, "naive")
    feats = T_(g["samp_features"])
    mel = torch.rand(2, 40, 16, device=dev()) * 5 - 5
    with torch.no_grad():
        out = diff.train_step(feats, mel, t=torch.tensor([3, 871], device=dev()))
    assert torch.isfinite(out["loss"]) and out["epsilon"].shape == (2, 40, 16)
    with pytest.raises(NotImplementedError):
        diff.train_step(feats, mel)


# ------------------------------------------------------------------ sampler state across calls, placement
SCFG = dict(mel_channels=64, dim=64, mlp_factor=4, condition_dim=64, num_layers=4)


def _diffusion(seed, pred="naive"):
    d = DIFFUSIONS.build(dict(type="GaussianDiffusion", denoiser=dict(type="ConvNextDenoiser", backend="tc", **SCFG),
                              mel_channels=64, noise_schedule="linear", timesteps=1000, max_beta=0.01,
                              sampler_interval=100, spec_min=[-5.0], spec_max=[0.0], noise_predictor=pred))
    d = d.to(dev()).eval()
    d.denoise_fn.load_state_dict({k: torch.from_numpy(v) for k, v in ocnx.make_convnext_weights(seed, **SCFG).items()})
    return d


def _feats(seed, B=3, T=130):
    return torch.randn(B, T, 64, generator=torch.Generator().manual_seed(seed)).to(dev())


@pytest.mark.parametrize("pred", ["naive", "unipc", "plms"])
def test_sampler_has_no_stale_projection(pred):
    """Consecutive calls on one module reuse the sampler workspace (projection buffer included) and replay the
    denoiser's captured graphs; each call must still equal a fresh module's, after new features and after new weights."""
    diff = _diffusion(41)
    f1, f2 = _feats(1), _feats(2)
    m = torch.zeros(3, 130, dtype=torch.bool, device=dev())
    m[1, 100:] = True
    a = diff(f1, noise_predictor=pred, seed=5, x_masks=m, cond_masks=m)
    assert diff._sws.get("cond_proj") is not None
    buf = diff._sws["cond_proj"].data_ptr()
    b = diff(f2, noise_predictor=pred, seed=5, x_masks=m, cond_masks=m)
    assert diff._sws["cond_proj"].data_ptr() == buf
    if pred != "plms":      # PLMS hands every evaluation a fresh eps tensor, so its evaluations run eagerly
        assert any(e["graph"] is not None for e in diff.denoise_fn._graphs.values())
    assert torch.equal(a, _diffusion(41)(f1, noise_predictor=pred, seed=5, x_masks=m, cond_masks=m))
    assert torch.equal(b, _diffusion(41)(f2, noise_predictor=pred, seed=5, x_masks=m, cond_masks=m))
    assert not torch.equal(a, b)
    diff.denoise_fn.load_state_dict({k: torch.from_numpy(v) for k, v in ocnx.make_convnext_weights(42, **SCFG).items()})
    c = diff(f2, noise_predictor=pred, seed=5, x_masks=m, cond_masks=m)
    assert torch.equal(c, _diffusion(42)(f2, noise_predictor=pred, seed=5, x_masks=m, cond_masks=m))
    assert not torch.equal(b, c)


@pytest.mark.parametrize("precision", ["f16", "bf16x1"])
def test_item_bits_independent_of_placement(precision):
    net = _net(ocnx.make_convnext_weights(31, **SCFG), SCFG, precision, backend="tc")
    B, T = 5, 130
    g = torch.Generator().manual_seed(31)
    x, cond = torch.randn(B, T, 64, generator=g).to(dev()), torch.randn(B, T, 64, generator=g).to(dev())
    steps = torch.tensor([990.0, 17.0, 503.25, 40.0, 3.0], device=dev())
    mask = torch.stack([torch.arange(T) >= T - 9 * i for i in range(B)]).to(dev())
    batch = _eval(net, x, steps, cond, mask, mask)
    rev = _eval(net, x.flip(0), steps.flip(0), cond.flip(0), mask.flip(0), mask.flip(0))
    for j in range(B):
        alone = _eval(net, x[j:j + 1], steps[j:j + 1], cond[j:j + 1], mask[j:j + 1], mask[j:j + 1])
        assert torch.equal(alone[0], batch[j]), f"item {j} differs between B=1 and batch position {j}"
        assert torch.equal(alone[0], rev[B - 1 - j]), f"item {j} differs between B=1 and batch position {B - 1 - j}"
