"""Oracle: ConvNext denoiser (reference fish_diffusion/modules/convnext.py, cross_attention=False).  TEST INFRASTRUCTURE
ONLY.

Weights are passed as a dict of numpy arrays keyed exactly like the reference ``state_dict``, e.g.
``residual_layers.3.pwconv1.weight``.  Every stage is float64 unless `dtype` says otherwise.
"""
import math

import numpy as np
from scipy.special import erf

from .wavenet import diffusion_embedding, linear


def gelu(x):
    """nn.GELU() / F.gelu with approximate='none' (convnext.py:44, 173, 179, 203, 231): 0.5 x (1 + erf(x / sqrt 2))."""
    return 0.5 * x * (1.0 + erf(x / math.sqrt(2.0)))


def conv1x1(x, w, b=None):
    """nn.Conv1d(kernel_size=1): x [B,Ci,T], w [Co,Ci,1] -> [B,Co,T]."""
    y = np.einsum("oc,bct->bot", w[:, :, 0], x, optimize=True)
    return y if b is None else y + b[None, :, None]


def dwconv(x, w, b, dilation):
    """Depthwise nn.Conv1d(C, C, 7, groups=C, dilation=d, padding=3d) (convnext.py:32-39): x [B,C,T], w [C,1,7]."""
    B, C, T = x.shape
    pad = 3 * dilation
    xp = np.zeros((B, C, T + 2 * pad), dtype=x.dtype)
    xp[:, :, pad:pad + T] = x
    y = np.zeros_like(x)
    for j in range(7):
        y += w[None, :, 0, j, None] * xp[:, :, j * dilation:j * dilation + T]
    return y + b[None, :, None]


def layer_norm(x, w, b, eps=1e-6):
    """nn.LayerNorm(C, eps=1e-6) over the last axis (convnext.py:40): biased variance, affine."""
    mean = x.mean(-1, keepdims=True)
    var = ((x - mean) ** 2).mean(-1, keepdims=True)
    return (x - mean) / np.sqrt(var + eps) * w + b


def block(sd, prefix, x, condition, step, dilation, x_masks=None):
    """ConvNeXtBlock.forward (convnext.py:54-91).  x [B,C,T], condition [B,C,T] (already cond-masked: the block's own
    masked_fill at :68-69 repeats the one at :239-240), step [Bs,C]."""
    g = lambda k: sd[prefix + k]
    residual = x
    x = x + conv1x1(step[:, :, None], g("diffusion_step_projection.weight"), g("diffusion_step_projection.bias"))
    x = x + conv1x1(condition, g("condition_projection.weight"), g("condition_projection.bias"))
    if x_masks is not None:
        x = np.where(x_masks[:, None], 0.0, x)
    x = dwconv(x, g("dwconv.weight"), g("dwconv.bias"), dilation).transpose(0, 2, 1)   # [B,T,C]
    x = layer_norm(x, g("norm.weight"), g("norm.bias"))
    x = linear(x, g("pwconv1.weight"), g("pwconv1.bias"))
    x = gelu(x)
    x = linear(x, g("pwconv2.weight"), g("pwconv2.bias"))
    x = (g("gamma") * x).transpose(0, 2, 1)
    x = residual + x
    if x_masks is not None:
        x = np.where(x_masks[:, None], 0.0, x)
    return x


def convnext_forward(sd, x, diffusion_step, conditioner, x_masks=None, cond_masks=None, dilation_cycle=4,
                     dtype=np.float64):
    """ConvNext.forward (convnext.py:208-261).  x [B,M,T] (or [B,1,M,T]), diffusion_step [B] or [1], conditioner
    [B,E,T], masks [B,T] bool (True = masked)."""
    sd = {k: np.asarray(v, dtype=dtype) for k, v in sd.items()}
    x = np.asarray(x, dtype=dtype)
    conditioner = np.asarray(conditioner, dtype=dtype)
    use_4 = x.ndim == 4
    if use_4:
        x = x[:, 0]
    n_layers = len({k.split(".")[1] for k in sd if k.startswith("residual_layers.")})
    C = sd["input_projection.weight"].shape[0]
    x = gelu(conv1x1(x, sd["input_projection.weight"], sd["input_projection.bias"]))              # :230-231
    step = diffusion_embedding(np.asarray(diffusion_step, dtype=dtype), C, dtype)               # :233, wavenet.py:20-27
    step = linear(gelu(linear(step, sd["diffusion_embedding.1.weight"], sd["diffusion_embedding.1.bias"])),
                  sd["diffusion_embedding.3.weight"], sd["diffusion_embedding.3.bias"])
    cond = conv1x1(conditioner, sd["conditioner_projection.0.weight"], sd["conditioner_projection.0.bias"])  # :234
    cond = conv1x1(gelu(cond), sd["conditioner_projection.2.weight"], sd["conditioner_projection.2.bias"])
    if x_masks is not None:
        x = np.where(x_masks[:, None], 0.0, x)
    if cond_masks is not None:
        cond = np.where(cond_masks[:, None], 0.0, cond)
    for i in range(n_layers):
        x = block(sd, f"residual_layers.{i}.", x, cond, step, 2 ** (i % dilation_cycle), x_masks)
    x = conv1x1(x, sd["output_projection.0.weight"], sd["output_projection.0.bias"])           # :257
    x = conv1x1(gelu(x), sd["output_projection.2.weight"], sd["output_projection.2.bias"])
    if x_masks is not None:
        x = np.where(x_masks[:, None], 0.0, x)
    return x[:, None] if use_4 else x


def make_convnext_weights(seed, mel_channels=128, dim=512, mlp_factor=4, condition_dim=256, num_layers=20):
    """Seeded synthetic weights with the reference's key names and shapes.  Convs and linears follow PyTorch's default
    initialiser (uniform +-1/sqrt(fan_in)); gamma is re-randomised log-uniform over [1e-2, 1] (the reference's 1e-6 would
    make every block contribute almost nothing) and the LayerNorm affine is perturbed away from (1, 0)."""
    rng = np.random.RandomState(seed)
    M, C, H, E = mel_channels, dim, dim * mlp_factor, condition_dim
    sd = {}

    def param(name, shape, fan_in):
        a = 1.0 / math.sqrt(fan_in)
        sd[name + ".weight"] = rng.uniform(-a, a, shape).astype(np.float32)
        sd[name + ".bias"] = rng.uniform(-a, a, shape[0]).astype(np.float32)

    param("input_projection", (C, M, 1), M)
    param("diffusion_embedding.1", (H, C), C)
    param("diffusion_embedding.3", (C, H), H)
    param("conditioner_projection.0", (H, E, 1), E)
    param("conditioner_projection.2", (C, H, 1), H)
    for i in range(num_layers):
        p = f"residual_layers.{i}."
        param(p + "dwconv", (C, 1, 7), 7)
        sd[p + "norm.weight"] = (1.0 + 0.1 * rng.randn(C)).astype(np.float32)
        sd[p + "norm.bias"] = (0.1 * rng.randn(C)).astype(np.float32)
        param(p + "pwconv1", (H, C), C)
        param(p + "pwconv2", (C, H), H)
        sd[p + "gamma"] = np.exp(rng.uniform(math.log(1e-2), 0.0, C)).astype(np.float32)
        param(p + "diffusion_step_projection", (C, C, 1), C)
        param(p + "condition_projection", (C, C, 1), C)
    param("output_projection.0", (C, C, 1), C)
    param("output_projection.2", (M, C, 1), C)
    return sd
