"""Float64 restatement of one WaveNet residual block (reference ResidualBlock.forward, restated by
oracle/wavenet.py::residual_block) in the channels-last layout the kernels use.  torch float64, so that the same code
runs on the CPU (checked against the oracle in test_wavenet_block_ref_cpu.py) and on the GPU (the reference of
test_gpu_wavenet_block.py at sizes where numpy would take minutes).

Two forms of GEMM1's pre-activations:
  * `gate_pre_direct`: from first principles, u = x + d, zero-padded dilated conv with taps (t-dil, t, t+dil), plus
    Wc cond and both biases; natural column order (gates [0,C), filters [C,2C)).
  * `gate_pre_packed`: the decomposition the kernels evaluate, conv(x) + Wc cond + gb_full minus gb_lo on the rows
    t < dil and gb_hi on the rows t >= T - dil, with W1 in packed row order (per gate tile: gates, then the matching
    filters) and columns [tap -dil | tap 0 | tap +dil | cond].

The closed forms of the block backward (`bwd_*`, `block_bwd`: the raw outputs of fd_wavenet_block_bwd, pinned to the
autograd of the packed forward in test_wavenet_block_ref_cpu.py) and a float64 restatement of the whole
`WaveNet.forward` (`wavenet_forward`, pinned to oracle.wavenet.wavenet_forward) follow.
"""
import math

import torch


def gate_perm(C, gate_tile):
    """Packed column j of GEMM1 holds natural column perm[j]: tile q = gates [q*half, (q+1)*half), then the filters."""
    half = gate_tile // 2
    idx = torch.arange(C).view(C // half, half)
    return torch.cat([idx, idx + C], dim=1).reshape(-1)


def gate_cols(C, gate_tile):
    """Packed column of the gate of residual channel c (its filter sits `gate_tile // 2` columns further)."""
    half = gate_tile // 2
    c = torch.arange(C)
    return (c // half) * gate_tile + c % half


def conv_taps(u, w_taps, dil):
    """sum_j u[b, t + (j-1)*dil] @ w_taps[j].T with zeros outside [0, T).  u [B,T,Ci], w_taps: 3 matrices [N, Ci]."""
    T = u.shape[1]
    y = u @ w_taps[1].T
    if dil < T:
        y[:, dil:] += u[:, :T - dil] @ w_taps[0].T
        y[:, :T - dil] += u[:, dil:] @ w_taps[2].T
    return y


def gate_pre_direct(x, cond, d, w_conv, b_conv, w_cond, b_cond, dil):
    """x [B,T,C], cond [B,T,E], d [B or 1, C], w_conv [2C,C,3], w_cond [2C,E] -> pre-activations [B,T,2C]."""
    u = x + d[:, None, :]
    return conv_taps(u, [w_conv[:, :, j] for j in range(3)], dil) + cond @ w_cond.T + b_conv + b_cond


def pack_w1(w_conv, w_cond, perm):
    """[2C, 3C+E] in packed row order, columns [tap -dil | tap 0 | tap +dil | cond]."""
    return torch.cat([w_conv[:, :, 0], w_conv[:, :, 1], w_conv[:, :, 2], w_cond], dim=1)[perm]


def gate_bias_tables(d, w1p, bias_sum_p):
    """d [Bd, C], w1p packed [2C, 3C+E], bias_sum_p [2C] packed -> (gb_full, gb_lo, gb_hi), each [Bd, 2C]:
    gb_full = bias_sum + sum_j W1_j d, gb_lo = W1_0 d (tap t-dil), gb_hi = W1_2 d (tap t+dil)."""
    C = d.shape[1]
    lo, mid, hi = (d @ w1p[:, j * C:(j + 1) * C].T for j in range(3))
    return bias_sum_p + (lo + mid + hi), lo, hi


def gate_pre_packed(x, cond, w1p, gb_full, gb_lo, gb_hi, dil):
    """Pre-activations [B,T,2C] in packed column order; gb_* [B or 1, 2C] (packed)."""
    T, C = x.shape[1], x.shape[2]
    y = conv_taps(x, [w1p[:, j * C:(j + 1) * C] for j in range(3)], dil) + cond @ w1p[:, 3 * C:].T
    t = torch.arange(T, device=x.device)
    lo = (t < dil).to(y.dtype)[None, :, None]
    hi = (t + dil >= T).to(y.dtype)[None, :, None]
    return y + gb_full[:, None, :] - lo * gb_lo[:, None, :] - hi * gb_hi[:, None, :]


def gate_z(y, C, gate_tile=None):
    """z = sigmoid(gate) * tanh(filter) [B,T,C] from pre-activations in natural (gate_tile None) or packed order."""
    if gate_tile is None:
        g, f = y[..., :C], y[..., C:]
    else:
        pg = gate_cols(C, gate_tile).to(y.device)
        g, f = y[..., pg], y[..., pg + gate_tile // 2]
    return torch.sigmoid(g) * torch.tanh(f)


def res_skip(x, z, w_out, b_out):
    """GEMM2: o = W2 z + b2 -> (x + o_res) / sqrt(2), o_skip.  w_out [2C, C] (rows: residual, then skip)."""
    C = x.shape[2]
    o = z @ w_out.T + b_out
    return (x + o[..., :C]) / math.sqrt(2.0), o[..., C:]


def gate_bwd(dz, y, gate_tile):
    """Backward of z = sigmoid(g) tanh(f): dz [B,T,C], y packed pre-activations [B,T,2C] -> dy [B,T,2C] packed."""
    C = dz.shape[2]
    pg = gate_cols(C, gate_tile).to(y.device)
    half = gate_tile // 2
    sg, th = torch.sigmoid(y[..., pg]), torch.tanh(y[..., pg + half])
    dy = torch.empty_like(y)
    dy[..., pg] = dz * th * sg * (1.0 - sg)
    dy[..., pg + half] = dz * sg * (1.0 - th * th)
    return dy


# ------------------------------------------------------------------------------------------------ block backward
# Closed forms of the raw outputs of fd_wavenet_block_bwd, in packed order.  Gradients inside the chain (dx_next, dskip,
# dz, dy, dx) carry the caller's scale S; what leaves it (gw1, gw2, the column sums, d_cond) is multiplied by inv_S.
# w1p [2C, 3C+E] is W1 in packed row order with columns [tap -dil | tap 0 | tap +dil | cond]; w2t [C, 2C] is the
# transposed output projection with 1/sqrt2 on its residual half (columns [0, C)), as fd_wavenet_pack_layers packs it.

def shift_t(a, s):
    """a[:, t + s] with zeros outside [0, T).  a [B, T, n]."""
    T = a.shape[1]
    out = torch.zeros_like(a)
    if abs(s) < T:
        if s >= 0:
            out[:, :T - s] = a[:, s:]
        else:
            out[:, -s:] = a[:, :T + s]
    return out


def pack_w2t(w_out):
    """w_out [2C, C] (rows: residual, then skip) -> [C, 2C] = [W2_res^T / sqrt2 | W2_skip^T]."""
    C = w_out.shape[1]
    return torch.cat([w_out[:C].T / math.sqrt(2.0), w_out[C:].T], dim=1)


def bwd_dz(dx_next, dskip, w2t):
    """dz = [dx_next | dskip] . w2t^T; the skip half alone for the top layer (dx_next None)."""
    C = w2t.shape[0]
    dz = dskip @ w2t[:, C:].T
    return dz if dx_next is None else dz + dx_next @ w2t[:, :C].T


def bwd_col_sums(dy, dil, inv_S):
    """(cs_dy [B, 2C], cs_edge [2, B, 2C]): inv_S * sums of dy over all steps / the first and the last min(dil, T)."""
    e = min(dil, dy.shape[1])
    return dy.sum(1) * inv_S, torch.stack([dy[:, :e].sum(1), dy[:, dy.shape[1] - e:].sum(1)]) * inv_S


def bwd_gw2(dx_next, dskip, z, inv_S):
    """[dx_next ; dskip]^T z * inv_S -> [2C, C]; residual rows zero for the top layer.  Without the 1/sqrt2 of the
    residual rows (the caller applies it)."""
    sk = torch.einsum("btr,btc->rc", dskip, z)
    res = torch.zeros_like(sk) if dx_next is None else torch.einsum("btr,btc->rc", dx_next, z)
    return torch.cat([res, sk]) * inv_S


def bwd_gw1(dy, x, cond, dil, inv_S):
    """dy^T [shift(x, -dil) | x | shift(x, +dil) | cond] * inv_S -> [2C, 3C+E], without the rank-one step-vector term
    (the caller adds it)."""
    cols = torch.cat([shift_t(x, -dil), x, shift_t(x, dil), cond], dim=2)
    return torch.einsum("btr,btc->rc", dy, cols) * inv_S


def bwd_dx(dy, w1p, dx_next, dil):
    """dx = sum_j shift(dy, -s_j) . W1_j + dx_next / sqrt2 with tap offsets s = (-dil, 0, +dil)."""
    C = w1p.shape[0] // 2
    dx = sum(shift_t(dy, -s) @ w1p[:, j * C:(j + 1) * C] for j, s in enumerate((-dil, 0, dil)))
    return dx if dx_next is None else dx + dx_next / math.sqrt(2.0)


def bwd_d_cond(dy, w1p, inv_S):
    """Increment of d_cond: dy . Wc * inv_S -> [B, T, E]."""
    return dy @ w1p[:, 3 * (w1p.shape[0] // 2):] * inv_S


def block_bwd(x, cond, y, z, dx_next, dskip, w1p, w2t, gate_tile, dil, inv_S):
    """Every raw output of one block backward from its inputs, each stage on the previous stage's reference."""
    dz = bwd_dz(dx_next, dskip, w2t)
    dy = gate_bwd(dz, y, gate_tile)
    cs_dy, cs_edge = bwd_col_sums(dy, dil, inv_S)
    dx = bwd_dx(dy, w1p, dx_next, dil)
    return dict(dz=dz, dy=dy, cs_dy=cs_dy, cs_edge=cs_edge, gw2=bwd_gw2(dx_next, dskip, z, inv_S),
                gw1=bwd_gw1(dy, x, cond, dil, inv_S), dx=dx, d_cond=bwd_d_cond(dy, w1p, inv_S), cs_dx=dx.sum(1) * inv_S)


# ------------------------------------------------------------------------------------------------ whole WaveNet
def _conv1x1(a, p, name):
    """channels-last 1x1 conv: a [B, T, Ci] -> [B, T, Co] with `name`.conv.weight [Co, Ci, 1] and its bias."""
    return a @ p[name + ".conv.weight"][:, :, 0].T + p[name + ".conv.bias"]


def _linear(a, p, name):
    out = a @ p[name + ".linear.weight"].T
    b = p.get(name + ".linear.bias")
    return out if b is None else out + b


def step_embedding(steps, C):
    """DiffusionEmbedding (wavenet.py:20-27) in float64; its frequency table is float32, as in the reference, where
    `torch.arange(half) * -emb` is a float32 product (exponentiated in float64 and rounded to float32, as the oracle)."""
    half = C // 2
    arg = torch.arange(half, dtype=torch.float32, device=steps.device) * torch.tensor(
        -math.log(10000) / (half - 1), dtype=torch.float32)
    table = torch.exp(arg.to(torch.float64)).to(torch.float32).to(torch.float64)
    emb = steps.to(torch.float64)[:, None] * table[None]
    return torch.cat([emb.sin(), emb.cos()], dim=-1)


def wavenet_forward(p, x, steps, cond, x_masks=None, cond_masks=None, dilation_cycle=None):
    """WaveNet.forward (wavenet.py:194-236) as float64 torch, so that autograd gives the reference gradients.
    p: state-dict keys -> float64 tensors; x [B, M, T], steps [B] or [1], cond [B, E, T], masks [B, T] bool (True =
    masked) -> [B, M, T].  Channels-last inside; the blocks are gate_pre_direct / gate_z / res_skip."""
    L = len({k.split(".")[1] for k in p if k.startswith("residual_layers.")})
    C = p["input_projection.conv.weight"].shape[0]
    h = torch.relu(_conv1x1(x.transpose(1, 2), p, "input_projection"))
    s = _linear(step_embedding(steps, C), p, "mlp.0")
    s = s * torch.tanh(torch.nn.functional.softplus(s))
    s = _linear(s, p, "mlp.2")
    cc = cond.transpose(1, 2)
    if x_masks is not None:
        h = h.masked_fill(x_masks[:, :, None], 0.0)
    if cond_masks is not None:
        cc = cc.masked_fill(cond_masks[:, :, None], 0.0)
    skip = 0.0
    for i in range(L):
        pre = f"residual_layers.{i}."
        g = lambda k: p[pre + k]
        dil = 2 ** (i % dilation_cycle) if dilation_cycle else 1
        d = _linear(s, p, pre + "diffusion_projection")
        y = gate_pre_direct(h, cc, d, g("conv_layer.conv.weight"), g("conv_layer.conv.bias"),
                            g("conditioner_projection.conv.weight")[:, :, 0], g("conditioner_projection.conv.bias"), dil)
        h, sk = res_skip(h, gate_z(y, C), g("output_projection.conv.weight")[:, :, 0], g("output_projection.conv.bias"))
        skip = skip + sk
    out = torch.relu(_conv1x1(skip / math.sqrt(L), p, "skip_projection"))
    out = _conv1x1(out, p, "output_projection")
    if x_masks is not None:
        out = out.masked_fill(x_masks[:, :, None], 0.0)
    return out.transpose(1, 2)
