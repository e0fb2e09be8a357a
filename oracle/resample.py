"""Oracle: band-limited sample-rate conversion (the reference resamples with librosa.resample at nsf_hifigan.py:96,
tools/diffusion/flask_api.py:42,53 and modules/feature_extractors/base.py:25).  TEST INFRASTRUCTURE ONLY.

librosa (pinned 0.9.1 in the reference's pdm.lock) is absent from this image.  Its default res_type "kaiser_best" is a
Kaiser-windowed sinc with 64 zero crossings, roll-off 0.9475937167399596 and beta 14.769656459379492, which resampy
tabulates at 2**9 points per zero crossing and interpolates linearly.  This oracle evaluates the same window exactly
at every tap instead (the filter torchaudio builds for `sinc_interp_kaiser` with these three parameters, which
tests/golden/resample.npz pins).  Its difference from resampy's interpolated table is *not measured*: bit parity
with librosa / resampy / soxr is unpinned.

The filter, with g = gcd(sr_in, sr_out), O = sr_in/g, P = sr_out/g, base = min(O, P) * ROLLOFF (zero crossings per
period of O input samples) and W = ceil(ZEROS * O / base):

    k(t)  = sinc(t) * I0(BETA * sqrt(1 - (t/ZEROS)^2)) / I0(BETA)      for |t| < ZEROS, 0 otherwise
    y[n]  = (base/O) * sum_m x[m] * k((m/O - n/P) * base),   m in [q*O - W, q*O + W + O),  q = n // P

x is zero outside [0, len).  The window of 2W + O input samples per period is the one a polyphase bank h[P][2W+O]
covers; for P > O its right edge lies up to (1/O - 1/P) * base short of the last zero crossing, which is part of the
definition (torchaudio truncates there too).  len(y) = ceil(len(x) * P / O).
"""
import math

import numpy as np

ZEROS = 64
ROLLOFF = 0.9475937167399596
BETA = 14.769656459379492


def ratio(sr_in, sr_out):
    """-> (O, P): input and output samples per common period."""
    sr_in, sr_out = int(sr_in), int(sr_out)
    if sr_in < 1 or sr_out < 1:
        raise ValueError("sample rates must be positive integers")
    g = math.gcd(sr_in, sr_out)
    return sr_in // g, sr_out // g


def half_width(O, P):
    return int(math.ceil(ZEROS * O / (min(O, P) * ROLLOFF)))


def out_len(n, sr_in, sr_out):
    O, P = ratio(sr_in, sr_out)
    return -((-int(n) * P) // O)


def kernel(t, beta=BETA):
    """Kaiser-windowed sinc at t zero crossings from the centre (float64 array)."""
    t = np.asarray(t, dtype=np.float64)
    inside = np.abs(t) < ZEROS
    s = np.sqrt(np.where(inside, 1.0 - (t / ZEROS) ** 2, 0.0))
    return np.where(inside, np.sinc(t) * np.i0(beta * s) / np.i0(beta), 0.0)


def resample_at(x, sr_in, sr_out, idx, beta=BETA):
    """Output samples idx (int array) of the resampled 1-D signal x, by the direct double sum."""
    x = np.asarray(x, dtype=np.float64)
    O, P = ratio(sr_in, sr_out)
    W = half_width(O, P)
    base = min(O, P) * ROLLOFF
    idx = np.asarray(idx, dtype=np.int64)
    y = np.zeros(idx.shape[0])
    if x.shape[0] == 0:
        return y
    span = np.arange(-W, W + O, dtype=np.int64)
    step = max(1, (1 << 22) // span.shape[0])
    for lo in range(0, idx.shape[0], step):
        n = idx[lo:lo + step, None]
        m = (n // P) * O + span[None, :]
        t = (m * P - n * O).astype(np.float64) / (O * P) * base          # (m/O - n/P) * base from an exact numerator
        ok = (m >= 0) & (m < x.shape[0])
        xm = np.where(ok, x[np.clip(m, 0, x.shape[0] - 1)], 0.0)
        y[lo:lo + step] = (base / O) * np.sum(xm * kernel(t, beta), axis=1)
    return y


def resample(x, sr_in, sr_out, beta=BETA):
    """x [..., n] -> float64 [..., ceil(n * P / O)]."""
    x = np.asarray(x, dtype=np.float64)
    if int(sr_in) == int(sr_out):
        return x.copy()
    n_out = out_len(x.shape[-1], sr_in, sr_out)
    flat = x.reshape(-1, x.shape[-1])
    out = np.stack([resample_at(row, sr_in, sr_out, np.arange(n_out), beta) for row in flat]) if flat.shape[0] else \
        np.zeros((0, n_out))
    return out.reshape(x.shape[:-1] + (n_out,))


def filter_bank(sr_in, sr_out):
    """The polyphase form of the same filter: h float64 [P][2W+O] with y[q*P + p] = sum_j h[p][j] * x[q*O - W + j],
    and per phase the first non-zero tap and the number of taps up to the last non-zero one (int32 [P] each).
    This is the table the product's host code must reproduce."""
    O, P = ratio(sr_in, sr_out)
    W = half_width(O, P)
    base = min(O, P) * ROLLOFF
    j = np.arange(2 * W + O, dtype=np.int64)[None, :]
    p = np.arange(P, dtype=np.int64)[:, None]
    h = (base / O) * kernel(((j - W) * P - p * O).astype(np.float64) / (O * P) * base)
    nz = h != 0.0
    first = np.argmax(nz, axis=1).astype(np.int32)
    last = (h.shape[1] - 1 - np.argmax(nz[:, ::-1], axis=1)).astype(np.int32)
    return h, first, (last - first + 1).astype(np.int32), W
