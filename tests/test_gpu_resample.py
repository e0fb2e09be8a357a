"""GPU parity of the resampling kernel (fd_resample_fwd, through the C ABI) against the float64 direct-sum oracle
(oracle/resample.py) on the float32 input values, and of the layers above it: resample(), NsfHifiGAN.wav2spec(sr=...)
and service.device_resampler behind make_http_server.

The kernel's only error is fp32: the bank rounded to fp32 and 135..373 fp32 FMAs per output in tap order.  For |x| <= 1
the bound asserted is 2e-6 max-abs; what an H100 gave is written beside TOL below."""
import http.client
import threading

import numpy as np
import pytest
import torch

from conftest import rel_l2
from fish_diffusion_b200 import NsfHifiGAN, _native as N, resample, resample_length
from fish_diffusion_b200 import service as S
from fish_diffusion_b200.mel import resample_bank
from gpu_util import dev
from oracle import mel as omel
from oracle import resample as R

pytestmark = pytest.mark.gpu

RATIOS = [(48000, 44100), (44100, 48000), (44100, 16000), (16000, 44100), (22050, 44100), (44100, 88200), (8000, 44100)]
TOL = 2e-6          # measured on an H100: worst over RATIOS 1.15e-6 (8000 -> 44100), 1.12e-6 at 44100 -> 16000, 6e-7 at 48 k <-> 44.1 k


def _signal(seed, n, sr, B=1):
    """noise + chirp, |x| <= 1, float32 [B, n]"""
    rng = np.random.RandomState(seed)
    t = np.arange(n) / sr
    chirp = 0.5 * np.sin(2 * np.pi * (100.0 * t + 0.5 * 0.4 * sr / max(t[-1], 1e-9) * t ** 2))
    return np.clip(chirp[None] + 0.2 * rng.randn(B, n), -1, 1).astype(np.float32)


def _fwd(x, sr_in, sr_out, lens=None, n_out=None, ratio=None):
    """x: float32 [B, n] numpy or CUDA tensor -> CUDA [B, n_out] straight through fd_resample_fwd."""
    xd = x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x)).to(dev())
    B, n = xd.shape
    bank, first, count, (O, P, W, taps) = resample_bank(sr_in, sr_out, xd.device)
    if ratio is not None:
        O, P = ratio
    n_out = resample_length(n, sr_in, sr_out) if n_out is None else n_out
    out = torch.full((B, n_out), float("nan"), dtype=torch.float32, device=xd.device)
    ld = None if lens is None else torch.tensor(lens, dtype=torch.int64, device=xd.device)
    N.check(N.lib().fd_resample_fwd(N.ptr(xd), N.ptr(ld), N.ptr(out), N.ptr(bank), N.ptr(first), N.ptr(count), B, n, n_out,
                                    O, P, W, taps, N.stream_ptr(xd.device)), "fd_resample_fwd")
    return out


@pytest.mark.parametrize("sr_in,sr_out", RATIOS)
def test_kernel_vs_oracle(sr_in, sr_out):
    O, P = R.ratio(sr_in, sr_out)
    n = 3 * (8192 // O) * O + 3 * O + 17 if O > 1 else 20011             # a few CTAs per item, not a multiple of O
    x = _signal(sr_in + sr_out, n, sr_in, B=2)
    got = _fwd(x, sr_in, sr_out).cpu().numpy().astype(np.float64)
    ref = R.resample(x, sr_in, sr_out)
    assert got.shape == ref.shape == (2, R.out_len(n, sr_in, sr_out))
    err = np.abs(got - ref).max()
    print(f"\n{sr_in}->{sr_out}: O={O} P={P} n={n} max |err| {err:.2e}")
    assert err < TOL


def test_ragged_batch_equals_items_alone():
    """Each item of a ragged batch equals, bit for bit, the same item run alone at its own length; past its own output
    length it is zero.  Lengths: full, shorter than W, empty, mid, not a multiple of O."""
    sr_in, sr_out, n = 48000, 44100, 6001
    x = _signal(5, n, sr_in, B=5)
    lens = [n, 17, 0, 3000, 4999]
    got = _fwd(x, sr_in, sr_out, lens=lens).cpu().numpy()
    assert np.isfinite(got).all()
    for b, ln in enumerate(lens):
        k = R.out_len(ln, sr_in, sr_out)
        assert not got[b, k:].any()
        if ln:
            alone = _fwd(x[b:b + 1, :ln], sr_in, sr_out).cpu().numpy()
            assert alone.shape == (1, k) and np.array_equal(alone[0], got[b, :k])
            assert np.abs(got[b, :k] - R.resample(x[b, :ln], sr_in, sr_out)).max() < TOL
    one = _fwd(x[:1], sr_in, sr_out, lens=[n]).cpu().numpy()                 # B = 1 with lens == no lens
    assert np.array_equal(one, _fwd(x[:1], sr_in, sr_out).cpu().numpy()) and np.array_equal(one[0], got[0])


@pytest.mark.parametrize("sr_in,sr_out,n", [(44100, 16000, 10), (44100, 16000, 1), (16000, 44100, 5), (48000, 44100, 73)])
def test_input_shorter_than_the_filter(sr_in, sr_out, n):
    x = _signal(n, n, sr_in)
    got = _fwd(x, sr_in, sr_out).cpu().numpy()
    assert np.abs(got - R.resample(x, sr_in, sr_out)).max() < TOL


@pytest.mark.parametrize("sr_in,sr_out", [(48000, 44100), (16000, 44100)])
def test_impulse_and_dc_edges(sr_in, sr_out):
    """Impulses at the first, a middle and the last sample read the bank back (every phase, both zero-padded edges);
    DC shows the ramp the zero padding makes at the edges and unit gain inside."""
    n = 2000
    x = np.zeros((4, n), dtype=np.float32)
    x[0, 0] = x[1, n // 2 + 1] = x[2, n - 1] = 1.0
    x[3] = 1.0
    got = _fwd(x, sr_in, sr_out).cpu().numpy().astype(np.float64)
    ref = R.resample(x, sr_in, sr_out)
    assert np.abs(got[:3] - ref[:3]).max() < 1e-7                           # one product per output: the fp32 bank itself
    assert np.abs(got[3] - ref[3]).max() < TOL
    assert np.abs(got[3, 300:-300] - 1).max() < 1e-6


def _sampled(n_out, rng, k=1500, edge=400):
    return np.unique(np.concatenate([np.arange(edge), np.arange(n_out - edge, n_out), rng.randint(0, n_out, k)]))


def test_long_item_and_offsets_past_2_31_bytes():
    """One item of 2.1 M samples (dozens of CTAs), then the same item as the last of a batch whose input and output
    offsets both pass 2**31 bytes: bit-identical, and both equal the oracle at sampled outputs and at the edges."""
    sr_in, sr_out, n, B = 48000, 44100, 2_100_003, 300
    n_out = resample_length(n, sr_in, sr_out)
    assert (B - 1) * n * 4 > 2 ** 31 and (B - 1) * n_out * 4 > 2 ** 31
    gen = torch.Generator(device=dev()).manual_seed(11)
    x = torch.rand((B, n), generator=gen, device=dev(), dtype=torch.float32) * 2 - 1
    last = x[B - 1:].clone()
    alone = _fwd(last, sr_in, sr_out)
    idx = _sampled(n_out, np.random.RandomState(1))
    ref = R.resample_at(last[0].cpu().numpy(), sr_in, sr_out, idx)
    err = np.abs(alone[0].cpu().numpy()[idx] - ref).max()
    print(f"\n2.1 M samples: max |err| at {idx.size} sampled outputs {err:.2e}")
    assert err < TOL
    lens = [n] * B
    lens[B - 2] = 1000                                                       # the neighbour's stale tail must not leak in
    out = _fwd(x, sr_in, sr_out, lens=lens)
    assert torch.equal(out[B - 1], alone[0])
    assert not out[B - 2, resample_length(1000, sr_in, sr_out):].any()
    mid = B // 2
    assert torch.equal(out[mid], _fwd(x[mid:mid + 1].clone(), sr_in, sr_out)[0])


def test_resample_ranks_lengths_and_identity():
    sr_in, sr_out, n = 44100, 16000, 5000
    x = torch.from_numpy(_signal(9, n, sr_in, B=3)).to(dev())
    y2 = resample(x, sr_in, sr_out)
    assert y2.shape == (3, resample_length(n, sr_in, sr_out)) and torch.equal(y2, _fwd(x, sr_in, sr_out))
    assert torch.equal(resample(x[1], sr_in, sr_out), y2[1])                 # [N]
    assert torch.equal(resample(x[:, None], sr_in, sr_out), y2[:, None])     # [B, 1, N]
    assert torch.equal(resample(x[0, 1:], sr_in, sr_out), _fwd(x[0:1, 1:].clone(), sr_in, sr_out)[0])   # unaligned view
    yl = resample(x, sr_in, sr_out, lengths=[n, 100, 2500])
    assert torch.equal(yl[0], y2[0]) and torch.equal(yl[1, :resample_length(100, sr_in, sr_out)],
                                                     resample(x[1, :100], sr_in, sr_out))
    assert not yl[1, resample_length(100, sr_in, sr_out):].any()
    assert resample(x, 44100, 44100) is x and resample(x, 48000, 96000 // 2) is x


def _vocoder():
    h = dict(resblock="1", upsample_rates=[4, 4, 2, 2], upsample_kernel_sizes=[8, 8, 4, 4], upsample_initial_channel=32,
             resblock_kernel_sizes=[3], resblock_dilation_sizes=[[1, 3, 5]], num_mels=128, hop_size=512, n_fft=2048,
             win_size=2048, fmin=40, fmax=16000, sampling_rate=44100)
    return NsfHifiGAN(checkpoint_path=None, config=h).to(dev())


def test_wav2spec_resamples_on_the_device():
    """wav2spec(wav, sr=48000) is wav2spec of the resampled signal, and stays within the mel front end's tolerance
    (tests/test_gpu_stft.py MEL_TOL, f16) of the oracle mel of the oracle-resampled signal."""
    voc = _vocoder()
    x = _signal(21, 48000, 48000)
    xd = torch.from_numpy(x).to(dev())
    got = voc.wav2spec(xd, sr=48000)
    assert got.is_cuda and torch.equal(got, voc.wav2spec(resample(xd, 48000, 44100)))
    assert torch.equal(voc.wav2spec(xd, sr=44100), voc.wav2spec(xd))          # the other branch is untouched
    ref = omel.pitch_adjustable_mel(R.resample(x, 48000, 44100))[0]
    assert got.shape == ref.shape
    lin = np.exp(got.cpu().numpy().astype(np.float64))
    rel = rel_l2(lin, np.maximum(ref, 1e-5))
    print(f"\nwav2spec(sr=48000): linear-mel rel-L2 vs oracle {rel:.2e}")
    assert rel < 2.5e-5


def test_device_resampler_through_the_http_route():
    """A 48 kHz DAW against a 44.1 kHz model: the request is resampled to the model rate, the answer back to 48 kHz."""
    seen = {}

    def frontend(audio, sr, pitch_adjust, speaker_id):
        seen["audio"], seen["sr"] = audio.copy(), sr
        return [(audio, np.zeros(1, np.float32), len(audio))]

    worker = S.BatchingWorker(lambda feats, f0s: [0.5 * f for f in feats], window_s=0.01)
    srv = S.make_http_server(worker, frontend, host="127.0.0.1", port=0, model_sr=44100, resample=S.device_resampler(dev()))
    threading.Thread(target=srv.serve_forever, daemon=True).start()
    n = 4800
    sig = _signal(2, n, 48000)[0]
    sig[-1] = 0.0                                                            # the multipart parser strips trailing CR / LF bytes
    wav = S.wav_bytes(sig, 48000)
    pcm = S.read_wav(wav)[0]                                                 # what the server decodes from 16-bit PCM
    b = "XBOUNDARYX"
    body = (f'--{b}\r\nContent-Disposition: form-data; name="sampleRate"\r\n\r\n48000\r\n'
            f'--{b}\r\nContent-Disposition: form-data; name="sample"; filename="a.wav"\r\n\r\n').encode()
    body += wav + f"\r\n--{b}--\r\n".encode()
    c = http.client.HTTPConnection("127.0.0.1", srv.server_address[1], timeout=60)
    c.request("POST", "/voiceChangeModel", body=body, headers={"Content-Type": f"multipart/form-data; boundary={b}"})
    r = c.getresponse()
    data = r.read()
    srv.shutdown()
    srv.server_close()
    worker.close()
    assert r.status == 200, data
    out, sr = S.read_wav(data)
    n_model = resample_length(n, 48000, 44100)
    assert sr == 48000 and seen["sr"] == 44100 and len(seen["audio"]) == n_model
    assert len(out) == resample_length(n_model, 44100, 48000)
    pd = torch.from_numpy(pcm).to(dev())
    assert np.array_equal(seen["audio"], resample(pd, 48000, 44100).cpu().numpy())
    want = resample(0.5 * resample(pd, 48000, 44100), 44100, 48000).cpu().numpy()
    assert np.abs(out - want).max() < 7e-5                                   # the answer is 16-bit PCM: scale 32767 out, 32768 in


def test_error_paths():
    x = torch.zeros(1, 1000)
    with pytest.raises(N.NativeError):
        resample(x, 48000, 44100)                                            # CPU tensor
    xd = x.to(dev())
    with pytest.raises(ValueError):
        resample(xd[None, None], 48000, 44100)
    with pytest.raises(N.NativeError, match="coprime"):
        _fwd(xd, 48000, 44100, ratio=(320, 294))
    with pytest.raises(N.NativeError, match="must be positive"):
        _fwd(xd, 48000, 44100, ratio=(0, 147))
    with pytest.raises(N.NativeError, match="n_out"):
        _fwd(xd, 48000, 44100, n_out=920)
    bank, first, count, (O, P, W, taps) = resample_bank(48000, 44100, xd.device)
    out = torch.empty(1, 919, device=dev())
    rc = N.lib().fd_resample_fwd(N.ptr(xd), None, N.ptr(out), N.ptr(bank), N.ptr(first), N.ptr(count), 1, 1000, 919, O, P,
                                 W, taps + 1, N.stream_ptr(xd.device))
    assert rc < 0 and "taps" in N.last_error()
    with pytest.raises(N.NativeError, match="shared memory"):
        resample(xd, 3001, 2)                                                # 4 * O + 2 * W samples do not fit a CTA
    with pytest.raises(ValueError, match="common divisor"):
        resample(xd, 44101, 48000)                                           # coprime rates: a 48000 x 44237 bank
