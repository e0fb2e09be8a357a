"""On-device sample-rate conversion: what the reference does with ``librosa.resample`` on the host
(nsf_hifigan.py:96, tools/diffusion/flask_api.py:42,53, modules/feature_extractors/base.py:25).

A polyphase Kaiser-windowed sinc with the parameters of librosa's default ``kaiser_best`` (mel.kaiser_sinc_bank),
evaluated by one CUDA kernel (fd_resample_fwd).  It agrees with librosa to filter-design accuracy, not bitwise.
"""
from __future__ import annotations

import torch

from . import _native as N
from .mel import resample_bank, resample_ratio


def resample_length(n, orig_sr, target_sr):
    """Number of output samples for n input samples: ceil(n * target_sr / orig_sr), librosa's and torchaudio's rule."""
    O, P = resample_ratio(orig_sr, target_sr)
    return -((-int(n) * P) // O)


@torch.no_grad()
def resample(wav, orig_sr, target_sr, lengths=None):
    """wav: CUDA float32 [N], [B, N] or [B, 1, N] -> the same rank with resample_length(N, ...) samples.
    lengths [B] (optional): valid samples per item; an item is resampled as if it ended there and its output past
    resample_length(lengths[b], ...) is zero.  Equal rates return `wav` itself."""
    N.require_cuda(wav, "wav")
    if wav.dim() not in (1, 2, 3) or (wav.dim() == 3 and wav.shape[1] != 1):
        raise ValueError(f"resample: wav must be [N], [B, N] or [B, 1, N], got {tuple(wav.shape)}")
    O, P = resample_ratio(orig_sr, target_sr)
    if O == P:
        return wav
    x = wav.to(torch.float32).reshape(-1, wav.shape[-1]).contiguous()
    if x.data_ptr() % 16:                    # a view into a larger buffer: the kernel loads 16-byte vectors
        x = x.clone()
    B, n_in = x.shape
    n_out = resample_length(n_in, orig_sr, target_sr)
    lens = None
    if lengths is not None:
        lens = torch.as_tensor(lengths, device=x.device).to(torch.int64).reshape(-1).contiguous()
        if lens.numel() != B:
            raise ValueError(f"resample: {lens.numel()} lengths for {B} items")
    bank, first, count, (O, P, W, taps) = resample_bank(orig_sr, target_sr, x.device)
    out = torch.empty((B, n_out), dtype=torch.float32, device=x.device)
    N.check(N.lib().fd_resample_fwd(N.ptr(x), N.ptr(lens), N.ptr(out), N.ptr(bank), N.ptr(first), N.ptr(count), B, n_in,
                                    n_out, O, P, W, taps, N.stream_ptr(x.device)), "fd_resample_fwd")
    return out.reshape(wav.shape[:-1] + (n_out,))
