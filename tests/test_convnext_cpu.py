"""CPU tests of the ConvNext denoiser (no GPU needed): the module's parameters are the reference's (keys, shapes, a
reference-written state dict loads strictly, bare and inside GaussianDiffusion), the registry builds it, the unsupported
modes refuse loudly, and the float64 oracle the GPU tests compare against is pinned to the reference's own outputs."""
import json

import numpy as np
import pytest
import torch

from conftest import rel_l2
from fish_diffusion_b200 import DENOISERS, DIFFUSIONS, ConvNext
from fish_diffusion_b200 import _native as N
from oracle import convnext as ocnx


def _small_cfg(g):
    return json.loads(str(g["config_small"]))


def _weights(g):
    return {k[2:]: v for k, v in g.items() if k.startswith("w/")}


def _inventory(net):
    return [[k, list(v.shape)] for k, v in net.state_dict().items()]


def test_state_dict_matches_reference_inventory(golden):
    g = golden("convnext")
    default = ConvNext()
    assert _inventory(default) == json.loads(str(g["inv_default"]))
    assert len(default.state_dict()) == 274
    assert _inventory(ConvNext(**_small_cfg(g))) == json.loads(str(g["inv_small"]))
    assert abs(sum(p.numel() for p in default.parameters()) / 1e6 - 56.7) < 0.05


def test_reference_initialisation():
    net = ConvNext(mel_channels=16, dim=32, condition_dim=16, num_layers=2)
    blk = net.residual_layers[1]
    assert torch.all(blk.gamma == 1e-6) and blk.dilation == 2 and blk.dwconv.padding == (6,)
    assert torch.all(blk.norm.weight == 1) and blk.norm.eps == 1e-6


def test_golden_weights_load_strictly_bare_and_in_diffusion(golden):
    g = golden("convnext")
    cfg = _small_cfg(g)
    sd = {k: torch.from_numpy(v) for k, v in _weights(g).items()}
    ConvNext(**cfg).load_state_dict(sd, strict=True)
    diff = DIFFUSIONS.build(dict(type="GaussianDiffusion", denoiser=dict(type="ConvNextDenoiser", **cfg),
                                 mel_channels=cfg["mel_channels"], spec_min=[-5.0], spec_max=[0.0]))
    full = {k: v for k, v in diff.state_dict().items() if not k.startswith("denoise_fn.")}
    full.update({"denoise_fn." + k: v for k, v in sd.items()})
    diff.load_state_dict(full, strict=True)
    assert torch.equal(diff.denoise_fn.residual_layers[3].gamma, sd["residual_layers.3.gamma"])


def test_registry_builds_convnext():
    net = DENOISERS.build(dict(type="ConvNextDenoiser", mel_channels=16, dim=32, mlp_factor=2, condition_dim=16,
                               num_layers=3, dilation_cycle=2, gradient_checkpointing=True))
    assert isinstance(net, ConvNext) and net.hidden == 64
    assert [b.dilation for b in net.residual_layers] == [1, 2, 1]


def test_cross_attention_is_refused():
    with pytest.raises(NotImplementedError, match="cross_attention"):
        ConvNext(mel_channels=16, dim=32, condition_dim=16, num_layers=2, cross_attention=True)


def test_grad_mode_is_refused():
    net = ConvNext(mel_channels=16, dim=32, condition_dim=16, num_layers=2)
    with pytest.raises(NotImplementedError, match="inference only"):
        net(torch.zeros(1, 16, 8), torch.tensor([3]), torch.zeros(1, 16, 8))
    with pytest.raises(NotImplementedError, match="inference only"):
        net.forward_train_cl(torch.zeros(1, 8, 16), torch.tensor([3.0]), torch.zeros(1, 8, 16))


def test_cpu_tensors_raise_native_error():
    net = ConvNext(mel_channels=16, dim=32, condition_dim=16, num_layers=2)
    with torch.no_grad(), pytest.raises(N.NativeError):
        net(torch.zeros(1, 16, 8), torch.tensor([3]), torch.zeros(1, 16, 8))


@pytest.mark.parametrize("case", ["stepsB_int", "stepsB_float", "steps1_int", "steps1_float", "masked",
                                  "cond_masked_only", "x_masked_only", "4d"])
def test_oracle_matches_reference_outputs(golden, case):
    g = golden("convnext")
    cfg = _small_cfg(g)
    steps = g["case_stepsB_int_steps"] if case == "4d" else g[f"case_{case}_steps"]
    x = g["x"][:, None] if case == "4d" else g["x"]
    kw = {}
    if case in ("masked", "x_masked_only"):
        kw["x_masks"] = g["x_masks"]
    if case in ("masked", "cond_masked_only"):
        kw["cond_masks"] = g["cond_masks"]
    y = ocnx.convnext_forward(_weights(g), x, steps, g["cond"], dilation_cycle=cfg["dilation_cycle"], **kw)
    ref = g[f"case_{case}_out"]
    assert y.shape == ref.shape
    e = rel_l2(y, ref)
    print(f"oracle[{case}] rel-L2 vs reference {e:.2e}")
    assert e < 1e-5
    if "x_masks" in kw:
        assert np.all(y[1, ..., 29:] == 0)


@pytest.mark.parametrize("C,T,dil,msg", [(40, 8, 1, "multiple of 16"), (1040, 8, 1, "at most 1024"),
                                         (0, 8, 1, "multiple of 16"), (64, 8, 0, "bad shape"), (64, 0, 1, "bad shape")])
def test_dwln_refuses_unsupported_shapes(C, T, dil, msg):
    """refused with an error before any launch (no GPU needed)"""
    lib = N.lib()
    p = 1 << 20
    rc = lib.fd_convnext_dwln_fwd(p, p, p, 0, None, p, p, p, p, p, 2, T, C, dil, 0, None)
    assert rc != 0 and msg in N.last_error()
    rc = lib.fd_convnext_dwln_fwd(p, None, p, 0, None, p, p, p, p, p, 2, 8, 64, 1, 0, None)
    assert rc != 0 and "null pointer" in N.last_error()


def test_forward_refuses_bad_descriptors():
    lib = N.lib()
    assert lib.fd_convnext_fwd(None, None) != 0 and "null descriptor" in N.last_error()
    d = N.ConvNextFwdDesc()
    d.B, d.T, d.M, d.C, d.H, d.E, d.L, d.Bs = 2, 8, 16, 32, 128, 16, 65, 1
    assert lib.fd_convnext_fwd(d, None) != 0 and "out of range" in N.last_error()
    d.L, d.Bs = 4, 3
    assert lib.fd_convnext_fwd(d, None) != 0 and "must be 1 or B" in N.last_error()
    d.Bs = 1
    assert lib.fd_convnext_cond_proj(d, None) != 0 and "cond_proj is required" in N.last_error()
