"""Writes tests/golden/resample.npz: float64 CPU outputs of torchaudio's Kaiser-sinc resampler at the parameters of
librosa's "kaiser_best" (64 zero crossings, roll-off 0.9475937167399596, beta 14.769656459379492) on a seeded
noise + chirp signal, for the rate pairs the package meets (DAW <-> model, model -> content encoder and back, 2x).

    python tests/golden/make_golden_resample.py

Needs torchaudio; the tests read only the .npz.
"""
import os

import numpy as np
import torch
import torchaudio

PAIRS = [(48000, 44100), (44100, 48000), (44100, 16000), (16000, 44100), (22050, 44100)]
N = 3000


def signal(seed, n, sr):
    rng = np.random.RandomState(seed)
    t = np.arange(n) / sr
    chirp = 0.5 * np.sin(2 * np.pi * (200.0 * t + 0.5 * (0.45 * sr - 200.0) / t[-1] * t ** 2))   # 200 Hz -> 0.45 sr
    return chirp + 0.25 * rng.randn(n)


def main():
    out = {"pairs": np.asarray(PAIRS, dtype=np.int64)}
    for i, (sr_in, sr_out) in enumerate(PAIRS):
        x = signal(1000 + i, N, sr_in)
        y = torchaudio.functional.resample(torch.from_numpy(x)[None], sr_in, sr_out, lowpass_filter_width=64,
                                           rolloff=0.9475937167399596, resampling_method="sinc_interp_kaiser",
                                           beta=14.769656459379492)[0]
        assert y.dtype == torch.float64
        out[f"x_{sr_in}_{sr_out}"] = x
        out[f"y_{sr_in}_{sr_out}"] = y.numpy()
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "resample.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
