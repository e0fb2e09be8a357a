"""Float64 references of the NSF-HiFiGAN generator stages, one per kernel launch of Generator.forward
(test_voc_stage_ref_cpu.py, test_gpu_voc_stages.py).

Each reference states the module-level operation -- the nn.Conv1d / ConvTranspose1d with the Generator's own weights --
in float64 torch on the CPU, never the packed tap-GEMM matrix, so a test built on them pins the packing
(`_pack_convt`, `fold_conv_weight`, `_pack_conv_folded_pair` and its kmask) together with the kernels.  Tensors are
channels-last [B, T, C] like the kernels' planes.

Every reference has a full form and a windowed form.  The windowed form computes output rows [t0, t1) of an item of
length T from `get(a, b)`, which returns input rows [a, b) with zeros outside the item (the conv zero padding), so a
window of a multi-GB tensor is judged from a few hundred rows of it."""
import torch
import torch.nn.functional as F

F64 = torch.float64
LRELU_SLOPE = 0.1
POST_SLOPE = 0.01           # F.leaky_relu's default slope before conv_post (models.py:434)


def lrelu(x, slope):
    return torch.where(x > 0, x, x * slope)


def inv_lrelu(a, slope):
    """x from a = lrelu(x, slope) (slope > 0)"""
    return torch.where(a > 0, a, a / slope)


def rows(x, a, b):
    """rows [a, b) of x [B, T, C] with zeros outside [0, T)"""
    Bn, T, C = x.shape
    out = x.new_zeros((Bn, b - a, C))
    lo, hi = max(a, 0), min(b, T)
    if hi > lo:
        out[:, lo - a:hi - a] = x[:, lo:hi]
    return out


def getter(x):
    return lambda a, b: rows(x, a, b)


def f64(t):
    return t.detach().to(device="cpu", dtype=F64)


def _ncw(x):
    return x.transpose(1, 2)


# ------------------------------------------------------------------------------------------------ 'same' Conv1d
def conv_halo(w, d):
    return (w.shape[2] - 1) // 2 * d


def conv(x, w, b, d=1, res=None, slope=None):
    """Conv1d(Ci -> Co, K, dilation d, padding (K-1)/2*d) on x [B, T, Ci], + res, then lrelu(slope) if given"""
    y = _ncw(F.conv1d(_ncw(x), w, b, padding=conv_halo(w, d), dilation=d))
    if res is not None:
        y = y + res
    return y if slope is None else lrelu(y, slope)


def conv_win(get, w, b, d, t0, t1, res=None, slope=None):
    """rows [t0, t1) of conv(x, ...); res is the residual on those rows"""
    h = conv_halo(w, d)
    y = _ncw(F.conv1d(_ncw(get(t0 - h, t1 + h)), w, b, dilation=d))
    if res is not None:
        y = y + res
    return y if slope is None else lrelu(y, slope)


def conv_pre(mel, w, b):
    """lrelu(conv_pre(mel), 0.1): the input of ups[0] (models.py:416-418)"""
    return conv(mel, w, b, 1, slope=LRELU_SLOPE)


def conv_pre_win(get, w, b, t0, t1):
    return conv_win(get, w, b, 1, t0, t1, slope=LRELU_SLOPE)


# ------------------------------------------------------------------------------------------------ ups[i]
def ups(a, w, b, u, p, addend):
    """X = ConvTranspose1d(a) + addend and lrelu(X, 0.1); a [B, L, Ci] is the (already lrelu'd) stage input,
    w [Ci, Co, k] -> [B, L*u, Co] each"""
    X = _ncw(F.conv_transpose1d(_ncw(a), w, b, stride=u, padding=p)) + addend
    return X, lrelu(X, LRELU_SLOPE)


def ups_win(get, w, b, u, p, addend, t0, t1):
    """output samples [t0, t1) of ups(); addend on those rows.  Output sample t = s*u - p + kk reads input row s through
    tap kk, so the rows s in [floor((t0 + p - k + 1) / u), floor((t1 - 1 + p) / u)] are all that contribute."""
    k = w.shape[2]
    s0, s1 = (t0 + p - (k - 1)) // u, (t1 - 1 + p) // u + 1
    full = _ncw(F.conv_transpose1d(_ncw(get(s0, s1)), w, None, stride=u))    # sample t at t - s0*u + p
    X = full[:, t0 - s0 * u + p:t1 - s0 * u + p] + b + addend
    return X, lrelu(X, LRELU_SLOPE)


# ------------------------------------------------------------------------------------------------ noise_convs[i]
def source_conv(har, w, b, s, p):
    """noise_convs[i]: Conv1d(1 -> C, k, stride s, padding p) of the excitation har [B, S] -> [B, S_out, C]"""
    return _ncw(F.conv1d(har[:, None, :], w, b, stride=s, padding=p))


def source_conv_win(get, w, b, s, p, t0, t1):
    """output rows [t0, t1); get(a, b) returns excitation samples [a, b) as [B, b - a, 1]"""
    k = w.shape[2]
    return _ncw(F.conv1d(_ncw(get(t0 * s - p, (t1 - 1) * s - p + k)), w, b, stride=s))


# ------------------------------------------------------------------------------------------------ ResBlock1 pair
def pair_halo(w1, d1, w2):
    return conv_halo(w1, d1) + conv_halo(w2, 1)


def resblock1_pair(x, w1, b1, d1, w2, b2, out_slope=None):
    """one step of ResBlock1 (models.py:103-110): x + c2(lrelu(c1(lrelu(x)))), then lrelu(out_slope) if given"""
    y = x + conv(conv(lrelu(x, LRELU_SLOPE), w1, b1, d1, slope=LRELU_SLOPE), w2, b2, 1)
    return y if out_slope is None else lrelu(y, out_slope)


def resblock1_pair_win(get, w1, b1, d1, w2, b2, t0, t1, T, out_slope=None):
    """rows [t0, t1) of resblock1_pair(); get returns rows of x.  The intermediate c1 output is zero outside the item
    (c2's own zero padding), not c1 evaluated there."""
    h2 = conv_halo(w2, 1)
    xw = get(t0 - pair_halo(w1, d1, w2), t1 + pair_halo(w1, d1, w2))
    h1 = conv_halo(w1, d1)
    mid = conv_win(getter_offset(lrelu(xw, LRELU_SLOPE), t0 - h1 - h2), w1, b1, d1, t0 - h2, t1 + h2,
                   slope=LRELU_SLOPE)
    tm = torch.arange(t0 - h2, t1 + h2)
    mid = mid * ((tm >= 0) & (tm < T)).to(F64)[None, :, None]
    y = xw[:, h1 + h2:h1 + h2 + t1 - t0] + _ncw(F.conv1d(_ncw(mid), w2, b2))
    return y if out_slope is None else lrelu(y, out_slope)


def getter_offset(xw, a0):
    """get() over a window xw whose row 0 is row a0 of the item (the window already holds the zero padding)"""
    return lambda a, b: xw[:, a - a0:b - a0]


# ------------------------------------------------------------------------------------------------ ResBlock2 step
def resblock2_step(u, w, b, d, slope=None):
    """one conv of ResBlock2 (models.py:150-155) with the reference's in-place LeakyReLU: the conv input u is already
    lrelu'd and is also the residual, u + conv(u); the in-place lrelu of the next step (slope) follows when given.
    The stage input the next block sees is lrelu(u) (oracle.nsf_hifigan.resblock2_inplace)."""
    return conv(u, w, b, d, res=u, slope=slope)


def resblock2_step_win(get, w, b, d, t0, t1, slope=None):
    return conv_win(get, w, b, d, t0, t1, res=get(t0, t1), slope=slope)


# ------------------------------------------------------------------------------------------------ MRF mean
def mrf(ins, in_slope, scale, out_slope):
    """lrelu(scale * sum_i x_i, out_slope) with x_i = inv_lrelu(ins_i, in_slope) (fd_mrf_finish): the mean of the
    num_kernels ResBlocks (models.py:426-432) and the next stage's LeakyReLU -- 0.1, or 0.01 before conv_post.
    (in_slope 1, scale 1, out_slope 0.1: the extra LeakyReLU of ResBlock2's shared stage input.)  Row-local, so the
    windowed form is the same function on a window."""
    s = sum(inv_lrelu(a, in_slope) for a in ins)
    return lrelu(s * scale, out_slope)


# ------------------------------------------------------------------------------------------------ conv_post
def conv_post(a, w, b):
    """tanh(conv_post(a)): a [B, S, C] = lrelu(x, 0.01), w [1, C, 7] -> [B, S, 1]"""
    return torch.tanh(conv(a, w, b, 1))


def conv_post_win(get, w, b, t0, t1):
    return torch.tanh(conv_win(get, w, b, 1, t0, t1))


# ------------------------------------------------------------------------------------------------ whole generator
def effective_weight(conv_mod):
    """float64 CPU weight of a (weight-normed or plain) conv module"""
    if hasattr(conv_mod, "weight_g"):
        return f64(torch._weight_norm(conv_mod.weight_v, conv_mod.weight_g, 0))
    return f64(conv_mod.weight)


def wb(conv_mod):
    return effective_weight(conv_mod), f64(conv_mod.bias)


def generator_chain(gen, mel, har):
    """Generator.forward (models.py:407-438) by chaining the stage references with the modules' weights.
    mel [B, M, T], har [B, S] (the harmonic excitation) -> dict of stage boundaries, all float64 channels-last:
      ups_in[i]  the input of ups[i] (lrelu(conv_pre(mel)) for i = 0, then lrelu of the previous stage's MRF mean),
      post_in    lrelu(last MRF mean, 0.01), the input of conv_post,
      wav        tanh(conv_post(post_in)) [B, S, 1]"""
    h = gen.h
    mel, har = _ncw(f64(mel)), f64(har)
    nk = len(h["resblock_kernel_sizes"])
    n_up = len(h["upsample_rates"])
    a = conv_pre(mel, *wb(gen.conv_pre))
    out = {"ups_in": [], "x": []}
    for i, up in enumerate(gen.ups):
        out["ups_in"].append(a)
        nc = gen.noise_convs[i]
        xs_src = source_conv(har, *wb(nc), nc.stride[0], nc.padding[0])
        X, _ = ups(a, *wb(up), up.stride[0], up.padding[0], xs_src)
        out["x"].append(X)
        xs = 0
        u = X
        for j in range(nk):
            rb = gen.resblocks[i * nk + j]
            if str(h.get("resblock", "1")) == "1":
                x = X
                for m, d in enumerate(rb.dilation):
                    x = resblock1_pair(x, *wb(rb.convs1[m]), d, *wb(rb.convs2[m]))
            else:
                u = lrelu(u, LRELU_SLOPE)               # in place on the shared stage input
                x = u
                for m, d in enumerate(rb.dilation):
                    last = m == len(rb.dilation) - 1
                    x = resblock2_step(x, *wb(rb.convs[m]), d, slope=None if last else LRELU_SLOPE)
            xs = xs + x
        a = lrelu(xs / nk, POST_SLOPE if i == n_up - 1 else LRELU_SLOPE)
    out["post_in"] = a
    out["wav"] = conv_post(a, *wb(gen.conv_post))
    return out
