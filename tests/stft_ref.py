"""Float64 restatement of the framed-DFT magnitude behind fd_stft_mag_eps_fwd and the mel front end of
fish_diffusion_b200/mel.py (reference pitch_adjustable_mel.py and the torchaudio MelSpectrogram of utils/audio.py).

Two forms of the magnitude spectrum:
  * `stft_mag`: from first principles -- reflect padding, the periodic Hann window (centred in n_fft when the window is
    shorter), np.fft.rfft, sqrt(re^2 + im^2 + eps) * mag_scale.  `resize_bins` then crops or zero-pads to n_fft//2 + 1
    bins as oracle/mel.py does under key shift.
  * `stft_mag_packed`: the decomposition the kernel computes.  Frame t of item b is P[b, t*hop : t*hop + kpad] of the
    padded signal P (overlapping rows, zero-weighted K padding past n_fft_new), multiplied by the DFT matrix W in the
    layout `dft_weights` builds (per 128-bin column tile: 128 re rows, then the 128 matching im rows), and the magnitude
    pairs the two halves of each tile.  torch float64, so the same code runs on the CPU and on the GPU.

`mel_spectrogram` restates torchaudio MelSpectrogram(power=1, center=True, reflect, Slaney) in float64.
Pinned by tests/test_stft_ref_cpu.py."""
import numpy as np
import torch

from oracle.mel import hann_window, slaney_mel_filterbank


def geometry(n_fft, win_length, hop_length, key_shift=0, speed=1.0):
    """(n_fft_new, win_new, hop, pad, mag_scale) as PitchAdjustableMelSpectrogram.__call__ derives them."""
    factor = 2 ** (key_shift / 12)
    n_fft_new = int(np.round(n_fft * factor))
    win_new = int(np.round(win_length * factor))
    hop = int(np.round(hop_length * speed))
    pad = int((win_new - hop) / 2)
    mag_scale = 1.0 if key_shift == 0 else win_length / win_new
    return n_fft_new, win_new, hop, pad, mag_scale


def window(n_fft_new, win_new):
    """torch.stft's window: hann_window(win_new) (periodic), centred in n_fft_new when shorter."""
    w = hann_window(win_new)
    if win_new < n_fft_new:
        left = (n_fft_new - win_new) // 2
        full = np.zeros(n_fft_new)
        full[left:left + win_new] = w
        w = full
    return w


def n_frames(n, n_fft_new, hop, pad):
    return 1 + (n + 2 * pad - n_fft_new) // hop


def stft_mag(y, n_fft_new, win_new, hop, pad, mag_scale=1.0, eps=1e-9):
    """First principles: y [B, n] -> magnitudes [B, frames, n_fft_new//2 + 1] (float64 numpy)."""
    y = np.asarray(y, dtype=np.float64)
    w = window(n_fft_new, win_new)
    frames = n_frames(y.shape[1], n_fft_new, hop, pad)
    idx = np.arange(n_fft_new)[None, :] + hop * np.arange(frames)[:, None]
    out = np.empty((y.shape[0], frames, n_fft_new // 2 + 1))
    for b in range(y.shape[0]):                       # item by item: a 30 s batch is 8 x 2583 frames of 2048
        yp = np.pad(y[b], (pad, pad), mode="reflect") if pad > 0 else y[b]
        spec = np.fft.rfft(yp[idx] * w, axis=-1)
        out[b] = np.sqrt(spec.real ** 2 + spec.imag ** 2 + eps) * mag_scale
    return out


def resize_bins(mag, n_fft):
    """Crop or zero-pad the bin axis (last) to n_fft//2 + 1, as oracle/mel.py does under key shift."""
    size = n_fft // 2 + 1
    if mag.shape[-1] < size:
        return np.concatenate([mag, np.zeros(mag.shape[:-1] + (size - mag.shape[-1],))], axis=-1)
    return mag[..., :size]


def dft_weights(n_fft, n_fft_new, win_new, dtype=np.float32):
    """Host restatement of PitchAdjustableMelSpectrogram._dft_weights before packing: W [2 NB, kpad] with, per 128-bin
    tile, rows [0,128) = window * cos, rows [128,256) = -window * sin, zero rows for bins >= min(n_fft_new, n_fft)//2+1
    and zero columns [n_fft_new, kpad).  Returns (W, NB, kpad, bins)."""
    NB = ((n_fft // 2 + 1) + 127) // 128 * 128
    kpad = (n_fft_new + 63) // 64 * 64
    bins = min(n_fft_new // 2 + 1, n_fft // 2 + 1)
    k = np.arange(bins)
    ang = 2.0 * np.pi * ((k[:, None] * np.arange(n_fft_new)[None, :]) % n_fft_new) / n_fft_new
    w = window(n_fft_new, win_new)[None]
    re, im = (np.cos(ang) * w).astype(dtype), (-np.sin(ang) * w).astype(dtype)
    W = np.zeros((2 * NB, kpad), dtype=dtype)
    for tile in range(NB // 128):
        lo, hi = tile * 128, min((tile + 1) * 128, bins)
        if hi > lo:
            W[tile * 256:tile * 256 + hi - lo, :n_fft_new] = re[lo:hi]
            W[tile * 256 + 128:tile * 256 + 128 + hi - lo, :n_fft_new] = im[lo:hi]
    return W, NB, kpad, bins


def stft_mag_packed(P, W, hop, rows, mag_scale=1.0, eps=1e-9):
    """Exact operands: P [B, L] padded signal, W [2 NB, kpad] packed DFT matrix (torch float64, same device), rows
    LongTensor of frame indices -> magnitudes [B, len(rows), NB]: frame t = P[b, t*hop : t*hop + kpad]."""
    B = P.shape[0]
    NB2, kpad = W.shape
    idx = rows.to(P.device)[:, None] * hop + torch.arange(kpad, device=P.device)[None, :]
    X = (P[:, idx] @ W.T).view(B, len(rows), NB2 // 256, 2, 128)
    re, im = X[..., 0, :], X[..., 1, :]
    return (torch.sqrt(re * re + im * im + eps) * mag_scale).reshape(B, len(rows), NB2 // 2)


def mel_spectrogram(y, sample_rate=44100, n_fft=2048, win_length=2048, hop_length=512, f_min=40, f_max=16000,
                    n_mels=128):
    """torchaudio MelSpectrogram(power=1, center=True, pad_mode="reflect", norm="slaney", mel_scale="slaney"):
    y [B, n] -> [B, n_mels, 1 + n // hop] float64."""
    mag = stft_mag(y, n_fft, win_length, hop_length, n_fft // 2, 1.0, 0.0)
    fb = slaney_mel_filterbank(sample_rate, n_fft, n_mels, f_min, f_max).astype(np.float64)
    return np.matmul(fb[None], mag.transpose(0, 2, 1))
