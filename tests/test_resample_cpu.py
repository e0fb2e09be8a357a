"""The resampling filter on CPU: the float64 oracle (oracle/resample.py, a direct double sum) against torchaudio's
Kaiser-sinc output (tests/golden/resample.npz) and against scipy's polyphase resampler, the product's host-built filter
bank (fish_diffusion_b200.mel.kaiser_sinc_bank) against the oracle, the length rule, and what the filter does to tones."""
import numpy as np
import pytest

from fish_diffusion_b200 import mel as pmel
from fish_diffusion_b200 import resample_length
from oracle import resample as R

PAIRS = [(48000, 44100), (44100, 48000), (44100, 16000), (16000, 44100), (22050, 44100)]
MORE = PAIRS + [(44100, 88200), (8000, 44100)]


@pytest.mark.parametrize("sr_in,sr_out", PAIRS)
def test_oracle_vs_torchaudio_golden(golden, sr_in, sr_out):
    """torchaudio builds its float64 filter with two float32 roundings of its own: beta is held in a float32 tensor, and
    so is the window's normaliser I0(beta), which puts one constant gain of 1 - 1.9e-8 on every tap.  With those two
    roundings applied the oracle agrees to 1e-12 (measured 2.4e-14), which pins every tap position, the window, the
    scale, the zero padding and the length; at the stated beta it agrees to the size of that gain."""
    g = golden("resample")
    assert [sr_in, sr_out] in g["pairs"].tolist()
    x, y = g[f"x_{sr_in}_{sr_out}"], g[f"y_{sr_in}_{sr_out}"]
    assert y.dtype == np.float64 and y.shape == (R.out_len(x.shape[0], sr_in, sr_out),)
    beta32 = float(np.float32(R.BETA))
    gain = float(np.float32(np.i0(beta32))) / np.i0(beta32)
    assert np.abs(R.resample(x, sr_in, sr_out, beta=beta32) - gain * y).max() < 1e-12
    assert np.abs(R.resample(x, sr_in, sr_out) - y).max() < 5e-8          # measured 2.6e-8 on |y| <= 1.35


@pytest.mark.parametrize("sr_in,sr_out", MORE)
def test_product_bank_vs_oracle(sr_in, sr_out):
    """The bank the kernel is given, applied by the polyphase rule y[q*P + p] = sum_j h[p][j] x[q*O - W + j] over its
    stored support only, equals the oracle's direct sum; and it is the oracle's own bank."""
    h, first, count, W = pmel.kaiser_sinc_bank(sr_in, sr_out)
    O, P = R.ratio(sr_in, sr_out)
    assert (O, P) == pmel.resample_ratio(sr_in, sr_out) and W == R.half_width(O, P) and h.shape == (P, 2 * W + O)
    ho, fo, co, Wo = R.filter_bank(sr_in, sr_out)
    assert np.abs(h - ho).max() < 1e-15 and (first == fo).all() and (count == co).all() and W == Wo
    rng = np.random.RandomState(sr_in % 997)
    n = 3 * O + 517
    x = rng.uniform(-1, 1, n)
    xp = np.concatenate([np.zeros(W), x, np.zeros(W + 2 * O)])
    n_out = R.out_len(n, sr_in, sr_out)
    y = np.zeros(n_out)
    for k in range(n_out):
        q, p = divmod(k, P)
        lo = first[p]
        y[k] = h[p, lo:lo + count[p]] @ xp[q * O + lo:q * O + lo + count[p]]
    assert np.abs(y - R.resample(x, sr_in, sr_out)).max() < 1e-13


@pytest.mark.parametrize("sr_in,sr_out", MORE)
def test_support_covers_every_nonzero_tap(sr_in, sr_out):
    h, first, count, W = pmel.kaiser_sinc_bank(sr_in, sr_out)
    O, P = R.ratio(sr_in, sr_out)
    j = np.arange(h.shape[1])[None, :]
    inside = (j >= first[:, None]) & (j < (first + count)[:, None])
    assert not h[~inside].any()                                               # nothing non-zero is skipped
    assert (h[np.arange(P), first] != 0).all() and (h[np.arange(P), first + count - 1] != 0).all()   # and the range is tight
    assert (first >= 0).all() and (first + count <= h.shape[1]).all()
    assert count.max() <= 2 * R.ZEROS * O / (min(O, P) * R.ROLLOFF) + 1       # about 2 * 64 * O / min(O, P) taps per phase
    assert abs(h.sum(axis=1) - 1).max() < 2e-8                                # unit DC gain in every phase
    bank, fd, cd, dims = pmel.resample_bank(sr_in, sr_out, "cpu")             # what the kernel is handed: tap-major, no tails
    assert dims == (O, P, W, 2 * W + O) and bank.shape == (count.max(), P) and bank.dtype.is_floating_point
    assert (fd.numpy() == first).all() and (cd.numpy() == count).all()
    for p in range(0, P, max(1, P // 7)):
        assert np.array_equal(bank[:count[p], p].numpy(), h[p, first[p]:first[p] + count[p]].astype(np.float32))
        assert not bank[count[p]:, p].any()


def test_length_rule():
    rng = np.random.RandomState(3)
    from fish_diffusion_b200 import _native as N
    lib = N.lib()
    for sr_in, sr_out in MORE + [(44100, 44100), (7, 3)]:
        for n in [0, 1, 2, 159, 160, 161, 441, 44100, 2_116_800] + rng.randint(0, 3_000_000, 20).tolist():
            want = int(np.ceil(n * sr_out / sr_in))
            assert R.out_len(n, sr_in, sr_out) == want == resample_length(n, sr_in, sr_out)
            assert lib.fd_resample_out_len(n, sr_in, sr_out) == want          # host arithmetic only: runs without a device
    assert lib.fd_resample_out_len(-1, 48000, 44100) < 0 and lib.fd_resample_out_len(10, 0, 44100) < 0
    assert b"fd_resample_out_len" in lib.fd_last_error()
    with pytest.raises(ValueError):
        resample_length(10, 44100.5, 48000)


@pytest.mark.parametrize("sr_in,sr_out", [(48000, 44100), (16000, 44100), (44100, 16000)])
def test_oracle_vs_scipy_resample_poly(sr_in, sr_out):
    """scipy.signal.resample_poly given the same taps: the bank laid out as one prototype filter at the common rate,
    G[d] = h[p][j] at d = p*O - (j - W)*P (the tap that joins output n and input m has d = n*O - m*P)."""
    from scipy.signal import resample_poly
    h, _, _, W = R.filter_bank(sr_in, sr_out)
    O, P = R.ratio(sr_in, sr_out)
    D = max((P - 1) * O + W * P, (W + O - 1) * P)
    G = np.zeros(2 * D + 1)
    d = np.arange(P)[:, None] * O - (np.arange(h.shape[1])[None, :] - W) * P
    G[d + D] = h
    x = np.random.RandomState(0).randn(2000)
    y = resample_poly(x, P, O, window=G / P, padtype="constant")             # resample_poly multiplies its window by `up`
    assert np.abs(y - R.resample(x, sr_in, sr_out)).max() < 1e-13             # measured 4e-15


def _snr_db(y, ref):
    return 10 * np.log10(np.sum(ref ** 2) / np.sum((y - ref) ** 2))


@pytest.mark.parametrize("sr_in,sr_out", [(48000, 44100), (44100, 48000)])
def test_tone_survives_daw_rate_conversion(sr_in, sr_out):
    """A 1 kHz tone is the same tone at the new rate: SNR against the ideal sinusoid away from the edges (the signal is
    zero outside its span, so the first and last ~W samples ring).  Measured 159.4 dB one way, 153.6 dB there and back."""
    n, edge = 6000, 400
    x = np.sin(2 * np.pi * 1000 * np.arange(n) / sr_in)
    y = R.resample(x, sr_in, sr_out)
    ref = np.sin(2 * np.pi * 1000 * np.arange(y.shape[0]) / sr_out)
    assert _snr_db(y[edge:-edge], ref[edge:-edge]) > 150
    back = R.resample(y, sr_out, sr_in)[:n]
    assert _snr_db(back[2 * edge:-2 * edge], x[2 * edge:-2 * edge]) > 145


def test_tone_above_new_nyquist_is_rejected():
    """44.1 k -> 16 k: a tone above 8 kHz must not alias back.  Output power over input power, away from the edges:
    measured -147.9 dB at 8.5 kHz, -156.1 dB at 10 kHz, -177.8 dB at 15 kHz; a 7 kHz tone passes at +0.002 dB."""
    n, edge = 12000, 300

    def gain_db(f):
        x = np.sin(2 * np.pi * f * np.arange(n) / 44100)
        y = R.resample(x, 44100, 16000)
        return 10 * np.log10(np.mean(y[edge:-edge] ** 2) / np.mean(x ** 2))

    assert gain_db(8500.0) < -140 and gain_db(10000.0) < -150 and gain_db(15000.0) < -170
    assert abs(gain_db(7000.0)) < 0.01
