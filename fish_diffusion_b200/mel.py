"""On-device mel / STFT front end: drop-in for the reference ``PitchAdjustableMelSpectrogram``
(fish_diffusion/utils/pitch_adjustable_mel.py:9-96) and ``dynamic_range_compression`` (utils/audio.py:11-18).

reflect pad + split  ->  framed DFT as a wgmma tap-GEMM over overlapping frames (the Hann window is folded into
the DFT matrix, re/im rows paired per column tile, magnitude in the epilogue)  ->  mel filterbank tap-GEMM.
A length-2048 DFT by direct summation is 8.4 MFLOP per frame -- far below the tensor-core budget, and it keeps the
front end inside the one GEMM kernel of this library (no cuFFT).
"""
from __future__ import annotations

import numpy as np
import torch

from . import _native as N


def _hz_to_mel(f):
    f = np.asarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-10) / min_log_hz) / logstep, f / f_sp)


def _mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_filterbank(sr, n_fft, n_mels, fmin, fmax):
    """Slaney-style mel filterbank (what ``librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax)`` returns at the
    reference call site pitch_adjustable_mel.py:46-52).  librosa itself is used when it is importable."""
    try:  # pragma: no cover - librosa is absent from the build image
        from librosa.filters import mel as librosa_mel_fn
        return librosa_mel_fn(sr=sr, n_fft=n_fft, n_mels=n_mels, fmin=fmin, fmax=fmax).astype(np.float32)
    except Exception:  # noqa: BLE001
        pass
    n_bins = 1 + n_fft // 2
    fftfreqs = np.linspace(0, float(sr) / 2, n_bins)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(fmin), _hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fftfreqs[None, :]
    lower = -ramps[:-2] / fdiff[:-1, None]
    upper = ramps[2:] / fdiff[1:, None]
    weights = np.maximum(0, np.minimum(lower, upper))
    weights *= (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]
    return weights.astype(np.float32)


def dynamic_range_compression(x, C=1, clip_val=1e-5):
    """log(clamp(x, clip_val) * C) (audio.py:11-18) as one native kernel."""
    x = x.to(torch.float32).contiguous()
    N.require_cuda(x, "x")
    y = torch.empty_like(x)
    if C != 1:
        x = x * C
        clip_val = clip_val * C
    N.check(N.lib().fd_log_clamp(N.ptr(x), N.ptr(y), x.numel(), float(clip_val), 1.0, N.stream_ptr(x.device)),
            "fd_log_clamp")
    return y


# the parameters of librosa's default res_type "kaiser_best" (librosa 0.9.1 in the reference): a Kaiser-windowed sinc
RESAMPLE_ZEROS = 64
RESAMPLE_ROLLOFF = 0.9475937167399596
RESAMPLE_BETA = 14.769656459379492
_resample_banks = {}


def resample_ratio(orig_sr, target_sr):
    """-> (O, P): input / output samples per common period of the two integer rates."""
    if int(orig_sr) != orig_sr or int(target_sr) != target_sr or orig_sr < 1 or target_sr < 1:
        raise ValueError(f"sample rates must be positive integers, got {orig_sr!r} -> {target_sr!r}")
    g = int(np.gcd(int(orig_sr), int(target_sr)))
    return int(orig_sr) // g, int(target_sr) // g


def kaiser_sinc_bank(orig_sr, target_sr):
    """Polyphase filter bank of the resampler, float64 [P, 2W+O]: output q*P + p = sum_j h[p, j] * x[q*O - W + j].
    One exact Kaiser-windowed sinc per output phase (no interpolated table): cutoff min(rates) * rolloff / 2,
    RESAMPLE_ZEROS zero crossings each side, exactly zero from the last one on.  Also returns, per phase, the first
    non-zero tap and the number of taps up to the last non-zero one (int32 [P]), and W."""
    O, P = resample_ratio(orig_sr, target_sr)
    base = min(O, P) * RESAMPLE_ROLLOFF                   # zero crossings per period
    W = int(np.ceil(RESAMPLE_ZEROS * O / base))
    num = (np.arange(2 * W + O, dtype=np.int64)[None, :] - W) * P - np.arange(P, dtype=np.int64)[:, None] * O
    t = num.astype(np.float64) / (O * P) * base           # (input time - output time) in zero crossings
    inside = np.abs(t) < RESAMPLE_ZEROS
    win = np.i0(RESAMPLE_BETA * np.sqrt(np.where(inside, 1.0 - (t / RESAMPLE_ZEROS) ** 2, 0.0))) / np.i0(RESAMPLE_BETA)
    h = np.where(inside, np.sinc(t) * win * (base / O), 0.0)
    nz = h != 0.0
    first = np.argmax(nz, axis=1)
    count = h.shape[1] - np.argmax(nz[:, ::-1], axis=1) - first
    return h, first.astype(np.int32), count.astype(np.int32), W


def resample_bank(orig_sr, target_sr, device):
    """The arguments of fd_resample_fwd, built once per (orig_sr, target_sr, device): kaiser_sinc_bank cast to fp32 and
    laid out tap-major without the zero tails, bank[i, p] = h[p, first[p] + i] ([max count, P]); int32 first / count;
    (O, P, W, taps)."""
    key = (int(orig_sr), int(target_sr), str(device))
    if key not in _resample_banks:
        O, P = resample_ratio(orig_sr, target_sr)
        if P * (2 * RESAMPLE_ZEROS * max(O, P) / min(O, P) + O) > 1 << 26:
            raise ValueError(f"resample {orig_sr} -> {target_sr}: the rates share too small a common divisor "
                             f"(O = {O}, P = {P}); the filter bank would hold more than 2**26 taps")
        h, first, count, W = kaiser_sinc_bank(orig_sr, target_sr)
        i = np.arange(int(count.max()))[:, None]
        packed = np.where(i < count[None, :], h[np.arange(P)[None, :], np.minimum(first[None, :] + i, h.shape[1] - 1)], 0.0)
        _resample_banks[key] = (torch.from_numpy(packed.astype(np.float32)).to(device), torch.from_numpy(first).to(device),
                                torch.from_numpy(count).to(device), (O, P, W, h.shape[1]))
    return _resample_banks[key]


class PitchAdjustableMelSpectrogram:
    def __init__(self, sample_rate=44100, n_fft=2048, win_length=2048, hop_length=512, f_min=40, f_max=16000,
                 n_mels=128, center=False, precision="f16", backend="auto"):
        self.sample_rate, self.n_fft, self.win_size, self.hop_length = sample_rate, n_fft, win_length, hop_length
        self.f_min, self.f_max, self.n_mels, self.center = f_min, f_max, n_mels, center
        self.precision, self.backend = precision, backend
        self.mel_basis = {}
        self.hann_window = {}
        self._dft = {}
        self._melw = {}
        self.NB = ((n_fft // 2 + 1) + 127) // 128 * 128   # padded bin count (1152 for n_fft 2048)

    def _backend(self):
        return N.BACKEND_TC if self.backend == "auto" else N.backend_code(self.backend)

    def _dft_weights(self, n_fft_new, win_new, device, prec):
        key = (n_fft_new, win_new, str(device), prec)
        if key not in self._dft:
            kpad = (n_fft_new + 63) // 64 * 64
            bins = min(n_fft_new // 2 + 1, self.n_fft // 2 + 1)
            n = np.arange(n_fft_new)
            window = 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(win_new) / win_new)   # torch.hann_window (periodic)
            if win_new < n_fft_new:
                w = np.zeros(n_fft_new)
                left = (n_fft_new - win_new) // 2
                w[left:left + win_new] = window
                window = w
            k = np.arange(bins)
            ang = 2.0 * np.pi * ((k[:, None] * n[None, :]) % n_fft_new) / n_fft_new
            W = np.zeros((2 * self.NB, kpad), dtype=np.float32)
            re = (np.cos(ang) * window[None]).astype(np.float32)
            im = (-np.sin(ang) * window[None]).astype(np.float32)
            for tile in range(self.NB // 128):
                lo, hi = tile * 128, min((tile + 1) * 128, bins)
                if hi > lo:
                    W[tile * 256:tile * 256 + (hi - lo), :n_fft_new] = re[lo:hi]
                    W[tile * 256 + 128:tile * 256 + 128 + (hi - lo), :n_fft_new] = im[lo:hi]
            Wd = torch.from_numpy(W).to(device)
            s = N.pow2_scale(Wd)
            self._dft[key] = (N.pack_weight(Wd, prec, s), 1.0 / s, kpad, bins)
        return self._dft[key]

    def _mel_weights(self, bins, device, prec):
        key = (bins, str(device), prec)
        if key not in self._melw:
            basis_key = f"{self.f_max}_{device}"
            if basis_key not in self.mel_basis:
                mel = mel_filterbank(self.sample_rate, self.n_fft, self.n_mels, self.f_min, self.f_max)
                self.mel_basis[basis_key] = torch.from_numpy(mel).float().to(device)
            basis = self.mel_basis[basis_key]
            # rows padded to a multiple of 64 (zero rows) so that every n_mels has a tensor-core instantiation
            W = torch.zeros(((self.n_mels + 63) // 64 * 64, self.NB), dtype=torch.float32, device=device)
            W[:self.n_mels, :bins] = basis[:, :bins]   # bins beyond the (shrunk) spectrum are zero-padded by the reference
            s = N.pow2_scale(W)
            self._melw[key] = (N.pack_weight(W, prec, s), 1.0 / s)
        return self._melw[key]

    @torch.no_grad()
    def __call__(self, y, key_shift=0, speed=1.0):
        """y [B,N] float -> [B, n_mels, frames] (linear mel magnitudes), pitch_adjustable_mel.py:33-96."""
        factor = 2 ** (key_shift / 12)
        n_fft_new = int(np.round(self.n_fft * factor))
        win_new = int(np.round(self.win_size * factor))
        hop = int(np.round(self.hop_length * speed))
        pad = int((win_new - hop) / 2)
        mag_scale = 1.0 if key_shift == 0 else float(self.win_size) / float(win_new)
        return self._stft_mel(y, n_fft_new, win_new, hop, pad, mag_scale, 1e-9)

    def _stft_mel(self, y, n_fft_new, win_new, hop, pad, mag_scale, mag_eps):
        """reflect pad by `pad` -> framed DFT magnitude (window folded into the DFT matrix) -> mel filterbank."""
        N.require_cuda(y, "y")
        dev = y.device
        prec = N.prec_code(self.precision)
        y = y.to(torch.float32).contiguous()
        B, n = y.shape
        w_planes, w_inv, kpad, bins = self._dft_weights(n_fft_new, win_new, dev, prec)
        Np = n + 2 * pad
        frames = 1 + (Np - n_fft_new) // hop
        st = N.stream_ptr(dev)
        lib = N.lib()
        if hop % 8 == 0:
            # frames are overlapping rows of the padded signal: a TMA view with row stride = hop (16-byte aligned)
            need = (frames - 1) * hop + kpad          # room for the zero-weighted K padding of the last frame
            pitch = (max(Np, need) + 7) // 8 * 8
            padded = torch.zeros((2, B, pitch), dtype=torch.int16, device=dev)
            if pitch == (Np + 7) // 8 * 8:
                N.check(lib.fd_reflect_pad_split(N.ptr(y), N.ptr(padded), B, n, pad, prec, st), "fd_reflect_pad_split")
            else:
                tmp = torch.zeros((2, B, (Np + 7) // 8 * 8), dtype=torch.int16, device=dev)
                N.check(lib.fd_reflect_pad_split(N.ptr(y), N.ptr(tmp), B, n, pad, prec, st), "fd_reflect_pad_split")
                padded[:, :, :tmp.shape[2]] = tmp
            # the rows span the whole pitch (zeros past Np): under key shift the last frame's K padding can end inside
            # the 8-element tail of the padded signal (kpad - n_fft_new = 2 at -5, 18 at +5)
            np_arg = pitch
            row_stride = hop
        else:
            # arbitrary hop (time-stretch augmentation draws e.g. 512*1.1 = 563): the frames are gathered once into an
            # aligned [frames, kpad] buffer and read as non-overlapping rows
            yp = torch.nn.functional.pad(y[:, None], (pad, pad), mode="reflect")[:, 0] if pad > 0 else y
            fr = yp.unfold(-1, n_fft_new, hop)[:, :frames]                         # [B, frames, n_fft_new] view
            buf = torch.zeros((B, frames, kpad), dtype=torch.float32, device=dev)
            buf[:, :, :n_fft_new] = fr
            padded = N.split_nwc(buf, prec).reshape(2, B, frames * kpad)
            np_arg, row_stride = frames * kpad, kpad
        mag = torch.empty((2, B, frames, self.NB), dtype=torch.int16, device=dev)
        N.check(lib.fd_stft_mag_eps_fwd(N.ptr(padded), N.ptr(w_planes), N.ptr(mag), B, np_arg, kpad, row_stride, frames,
                                        self.NB, w_inv, mag_scale, mag_eps, N.mma_code(self.precision), self._backend(), st),
                "fd_stft_mag_eps_fwd")
        mw, mw_inv = self._mel_weights(bins, dev, prec)
        n_pad = mw.shape[1]
        mel_cl = torch.empty((B, frames, n_pad), dtype=torch.float32, device=dev)
        N.conv_cl(mag, mw, B, frames, self.NB, n_pad, [0], out_f32=mel_cl, w_inv_scale=mw_inv, prec=N.mma_code(self.precision),
                  backend=self._backend())
        out = torch.empty((B, n_pad, frames), dtype=torch.float32, device=dev)
        N.check(lib.fd_transpose_nwc_to_ncw(N.ptr(mel_cl), N.ptr(out), B, frames, n_pad, st),
                "fd_transpose_nwc_to_ncw")
        return out if n_pad == self.n_mels else out[:, :self.n_mels].contiguous()


class MelSpectrogram(PitchAdjustableMelSpectrogram):
    """What ``get_mel_transform`` returns: the torchaudio ``MelSpectrogram(power=1, center=True, pad_mode="reflect",
    norm="slaney", mel_scale="slaney")`` of the reference's training / validation losses (utils/audio.py:31-60) on the
    same framed-DFT + filterbank kernels.  Callable on [..., n] audio -> [..., n_mels, 1 + n // hop]."""

    def __init__(self, sample_rate=44100, n_fft=2048, win_length=2048, hop_length=512, f_min=40, f_max=16000, n_mels=128,
                 center=True, power=1.0, pad_mode="reflect", norm="slaney", mel_scale="slaney", precision="f16",
                 backend="auto"):
        if power != 1.0 or pad_mode != "reflect" or norm != "slaney" or mel_scale != "slaney" or not center:
            raise NotImplementedError("MelSpectrogram: only the reference's configuration (power=1, center=True, "
                                      "reflect padding, slaney norm / scale) is implemented")
        super().__init__(sample_rate, n_fft, win_length, hop_length, f_min, f_max, n_mels, center=True,
                         precision=precision, backend=backend)

    def to(self, *args, **kwargs):          # the reference moves the torchaudio module to the audio's device
        return self

    @torch.no_grad()
    def __call__(self, audio):
        lead = audio.shape[:-1]
        y = audio.reshape(-1, audio.shape[-1])
        out = self._stft_mel(y, self.n_fft, self.win_size, self.hop_length, self.n_fft // 2, 1.0, 0.0)
        return out.reshape(*lead, self.n_mels, out.shape[-1])


def get_mel_transform(sample_rate=44100, n_fft=2048, win_length=2048, hop_length=512, f_min=40, f_max=16000, n_mels=128,
                      center=True, power=1.0, pad_mode="reflect", norm="slaney", mel_scale="slaney", **kw):
    """utils/audio.py:31-60."""
    return MelSpectrogram(sample_rate, n_fft, win_length, hop_length, f_min, f_max, n_mels, center, power, pad_mode, norm,
                          mel_scale, **kw)


@torch.no_grad()
def get_mel_from_audio(audio, sample_rate=44100, n_fft=2048, win_length=2048, hop_length=512, f_min=40, f_max=16000,
                       n_mels=128, center=True, power=1.0, pad_mode="reflect", norm="slaney", mel_scale="slaney", **kw):
    """utils/audio.py:63-109: audio [1, n] -> log-mel [n_mels, frames]."""
    assert audio.ndim == 2, "Audio tensor must be 2D (1, n_samples)"
    assert audio.shape[0] == 1, "Audio tensor must be mono"
    tf = get_mel_transform(sample_rate, n_fft, win_length, hop_length, f_min, f_max, n_mels, center, power, pad_mode, norm,
                           mel_scale, **kw)
    return dynamic_range_compression(tf(audio))[0]
