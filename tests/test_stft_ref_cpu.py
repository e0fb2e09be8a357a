"""CPU tests behind test_gpu_stft.py: the two forms of its float64 STFT-magnitude restatement agree, the first-principles
form equals the oracle's pitch-adjustable spectrum before the filterbank, and the MelSpectrogram restatement matches the
torchaudio goldens of utils/audio.py."""
import numpy as np
import pytest
import torch

from conftest import rel_l2
from oracle import mel as omel
from stft_ref import dft_weights, geometry, mel_spectrogram, n_frames, resize_bins, stft_mag, stft_mag_packed

# (n_fft, win_length, hop_length, key_shift, speed): both shipped configs, key shift up and down (kpad != n_fft_new),
# a window shorter than n_fft, n_fft 1024 and 4096, and a hop that is not a multiple of 8
GEOMS = [(2048, 2048, 512, 0, 1.0), (2048, 2048, 256, 0, 1.0), (2048, 2048, 512, 5, 1.0), (2048, 2048, 512, -5, 1.0),
         (2048, 1024, 512, 0, 1.0), (1024, 1024, 256, 0, 1.0), (4096, 4096, 1024, 0, 1.0), (2048, 2048, 512, 0, 1.1)]


def _wav(B, n, seed):
    rng = np.random.RandomState(seed)
    t = np.arange(n) / 44100.0
    y = rng.randn(B, n) * 0.1 + 0.5 * np.sin(2 * np.pi * rng.uniform(50, 20000, (B, 1)) * t)
    return y.astype(np.float32)


@pytest.mark.parametrize("geom", GEOMS, ids=[f"n{g[0]}-w{g[1]}-h{g[2]}-ks{g[3]}-sp{g[4]}" for g in GEOMS])
def test_packed_form_matches_first_principles(geom):
    """The kernel's decomposition (overlapping padded rows x the packed float32 DFT matrix, re / im halves paired per
    tile) against np.fft.rfft, per bin in units of the frame's spectral norm."""
    n_fft, win, hop_len, ks, speed = geom
    n_fft_new, win_new, hop, pad, ms = geometry(n_fft, win, hop_len, ks, speed)
    W, NB, kpad, bins = dft_weights(n_fft, n_fft_new, win_new)
    assert W.shape == (2 * NB, kpad) and kpad % 64 == 0 and NB % 128 == 0
    B, n = 2, 6 * hop + n_fft_new
    y = _wav(B, n, n_fft + hop + ks)
    frames = n_frames(n, n_fft_new, hop, pad)
    ref = stft_mag(y, n_fft_new, win_new, hop, pad, ms)
    P = np.zeros((B, (frames - 1) * hop + kpad))          # the kernel's padded rows: zeros past the padded signal
    yp = np.pad(y.astype(np.float64), ((0, 0), (pad, pad)), mode="reflect")
    P[:, :min(P.shape[1], yp.shape[1])] = yp[:, :P.shape[1]]
    got = stft_mag_packed(torch.from_numpy(P), torch.from_numpy(W.astype(np.float64)), hop, torch.arange(frames), ms)
    got = got.numpy()
    norm = np.linalg.norm(ref, axis=-1, keepdims=True)
    err = np.abs(got[..., :bins] - ref[..., :bins]) / norm
    print(f"\n{geom}: worst frame-normalised error {err.max():.2e}")
    assert err.max() < 1e-8               # float32 rounding of window * cos / sin; measured 3.4e-9 (n_fft 1024)
    # bins past the spectrum are zero rows of W: sqrt(eps) * mag_scale exactly
    np.testing.assert_allclose(got[..., bins:], np.sqrt(1e-9) * ms, rtol=1e-12)


@pytest.mark.parametrize("geom", GEOMS, ids=[f"n{g[0]}-w{g[1]}-h{g[2]}-ks{g[3]}-sp{g[4]}" for g in GEOMS])
def test_first_principles_matches_oracle(geom):
    """stft_mag + resize_bins equals oracle.mel.pitch_adjustable_mel with an identity filterbank."""
    n_fft, win, hop_len, ks, speed = geom
    n_fft_new, win_new, hop, pad, ms = geometry(n_fft, win, hop_len, ks, speed)
    y = _wav(2, 5 * hop + n_fft_new + 37, n_fft + ks)
    size = n_fft // 2 + 1
    ref = omel.pitch_adjustable_mel(y, n_fft=n_fft, win_length=win, hop_length=hop_len, key_shift=ks, speed=speed,
                                    mel_basis=np.eye(size))
    got = resize_bins(stft_mag(y, n_fft_new, win_new, hop, pad, ms), n_fft).transpose(0, 2, 1)
    assert got.shape == ref.shape
    np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-12)


def test_mel_spectrogram_matches_torchaudio_golden(golden):
    """The float64 MelSpectrogram restatement against torchaudio's own output (r2_audio.npz)."""
    import json
    g = golden("r2_audio")
    wav = g["au_wav"]
    for tag, kw in (("default", {}), ("hop256", json.loads(str(g["au_kw_hop256"])))):
        ref = g[f"au_mel_{tag}"]
        got = mel_spectrogram(wav, **kw)
        assert got.shape == ref.shape
        e = rel_l2(got, ref)
        print(f"MelSpectrogram[{tag}] rel-L2 vs torchaudio {e:.2e}")
        assert e < 5e-5
