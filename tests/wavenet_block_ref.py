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
