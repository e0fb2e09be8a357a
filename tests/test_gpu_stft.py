"""GPU parity of the mel front end against a float64 STFT (tests/stft_ref.py, pinned to the oracle and to torchaudio by
test_stft_ref_cpu.py):

  * fd_stft_mag_eps_fwd, the tap-GEMM's MAG epilogue: overlapping TMA rows of the reflect-padded signal (row stride hop
    < K), the packed DFT matrix of PitchAdjustableMelSpectrogram._dft_weights (K padded past n_fft_new under key shift),
    re / im halves paired per 128-bin column tile, sqrt(re^2 + im^2 + eps) * mag_scale;
  * fd_reflect_pad_split, fd_log_clamp (dynamic_range_compression) and fd_transpose_nwc_to_ncw;
  * end to end: PitchAdjustableMelSpectrogram against oracle.mel.pitch_adjustable_mel, get_mel_transform /
    get_mel_from_audio against the float64 MelSpectrogram restatement.

Each magnitude is compared twice: with the exact-operand reference (the padded planes and packed weights the kernel
read, in float64; hi planes alone in single-product mode), which isolates the GEMM, and with the first-principles
reference (np.fft.rfft of the float32 input), which adds the rounding of the operands to planes.  A bin's error is
divided by its frame's spectral norm (a per-bin relative error is meaningless where the spectrum is ~0) and reported
per region: first / last frame of each item, the last (ragged) 128-row tile, bins below / above the 16 kHz edge of the
shipped filterbank (bins above it get zero mel weight, so only this test sees them), and the last 128-bin column tile.
Bins past the spectrum (zero rows of the DFT matrix) and silent items must be sqrt(eps) * mag_scale to plane precision.

The measured value (H100 80GB HBM3) of each bar is written next to it; no bar is more than 4x the largest value
measured across the cases it covers.
"""
import math
import zlib

import numpy as np
import pytest
import torch

from conftest import rel_l2
from fish_diffusion_b200 import _native as N
from fish_diffusion_b200.mel import (PitchAdjustableMelSpectrogram, dynamic_range_compression, get_mel_from_audio,
                                     get_mel_transform)
from gpu_util import dev
from oracle import mel as omel
from stft_ref import geometry, mel_spectrogram, n_frames, stft_mag, stft_mag_packed

pytestmark = pytest.mark.gpu

F64 = torch.float64
SR = 44100
SENTINEL = 0x7FFF            # NaN in both f16 and bf16: a bin the kernel never wrote shows up

# (max, rel-L2) bars per reference, precision and back end, each <= 4x the worst value measured over the cases that use
# it (in the comment).  "max" is the worst bin error in units of its frame's spectral norm, over every region; "rel-L2"
# is over all frames and bins.  The tensor cores' truncating fp32 accumulation over K = 2048 dominates their error in
# f16 and bf16 alike; the SIMT twin's fp32 FFMA is several times tighter.
TOL = {
    ("exact", "f16", "tc"): (2.5e-5, 4e-5),        # measured 8.3e-6 / 1.4e-5
    ("exact", "f16", "simt"): (4e-6, 3e-6),        # measured 1.3e-6 / 9.7e-7
    ("exact", "bf16", "tc"): (2.5e-5, 4e-5),       # measured 8.3e-6 / 1.3e-5
    ("exact", "bf16", "simt"): (1e-5, 1e-5),       # measured 3.1e-6 / 2.8e-6
    ("exact", "f16x1", "tc"): (1.2e-5, 1.5e-5),    # measured 3.8e-6 / 4.4e-6
    ("exact", "f16x1", "simt"): (4e-6, 3e-6),      # measured 1.1e-6 / 7.7e-7
    ("direct", "f16", "tc"): (2.5e-5, 4e-5),       # measured 8.3e-6 / 1.4e-5
    ("direct", "f16", "simt"): (4e-6, 3e-6),       # measured 1.2e-6 / 9.7e-7
    ("direct", "bf16", "tc"): (2.5e-5, 4e-5),      # measured 8.2e-6 / 1.3e-5
    ("direct", "bf16", "simt"): (1e-5, 1.2e-5),    # measured 3.2e-6 / 3.6e-6
    ("direct", "f16x1", "tc"): (1.2e-4, 6e-4),     # measured 3.8e-5 / 2.0e-4 (half-precision operands)
    ("direct", "f16x1", "simt"): (1.2e-4, 6e-4),   # measured 3.8e-5 / 2.0e-4
}


def pf64(planes, pc, hi_only=False):
    """split planes int16 [2, ...] -> float64 hi + lo (or hi alone), on the planes' device"""
    dt = torch.float16 if pc == N.PREC_F16 else torch.bfloat16
    hi = planes[0].view(dt).to(F64)
    return hi if hi_only else hi + planes[1].view(dt).to(F64)


def plane_tol(v, pc):
    """How far a value v >= 0 stored as hi + lo planes may be from v: 16 significant bits for bf16; for f16 22 bits, or
    the subnormal spacing of the lo plane (2^-24 * 2^-1) once v is small (sqrt(1e-9) lies in the f16 subnormal range)."""
    return 2e-5 * v if pc == N.PREC_BF16 else 1e-6 * v + 2.0 ** -25


# geometry name -> (n_fft, win_length, hop_length, key_shift, center).  center: MelSpectrogram (pad n_fft//2, eps 0)
GEOM = {
    "h512": (2048, 2048, 512, 0, False),      # config_v1 (NSF-HiFiGAN 44.1 kHz)
    "h256": (2048, 2048, 256, 0, False),      # config_v1_256
    "ks+5": (2048, 2048, 512, 5, False),      # n_fft_new 2734, kpad 2752
    "ks-5": (2048, 2048, 512, -5, False),     # n_fft_new 1534, kpad 1536: bins 768..1151 are zero rows
    "w1024": (2048, 1024, 512, 0, False),     # window centred inside n_fft
    "n1024": (1024, 1024, 256, 0, False),     # NB 640
    "n4096": (4096, 4096, 1024, 0, False),    # NB 2176, K 4096
    "center": (2048, 2048, 512, 0, True),     # get_mel_transform: eps 0
}


def _geom(name):
    """-> (n_fft, n_fft_new, win_new, hop, pad, mag_scale, eps)"""
    n_fft, win, hop_len, ks, center = GEOM[name]
    if center:
        return n_fft, n_fft, win, hop_len, n_fft // 2, 1.0, 0.0
    return (n_fft,) + geometry(n_fft, win, hop_len, ks) + (1e-9,)


def _length(frames, n_fft_new, hop, pad):
    """A signal length with exactly `frames` frames (and a partial hop left over), longer than the reflect pad."""
    base = (frames - 1) * hop + n_fft_new - 2 * pad
    extra = max(hop // 3, pad + 1 - base)
    assert extra < hop and n_frames(base + extra, n_fft_new, hop, pad) == frames
    return base + extra


def _items(B, n, seed, silent=None):
    """Items of different content and loudness (noise and tones over the whole band, an order of magnitude apart);
    item `silent` is all zeros."""
    rng = np.random.RandomState(seed)
    t = np.arange(n) / SR
    y = np.empty((B, n), dtype=np.float32)
    for b in range(B):
        amp = 10.0 ** rng.uniform(-2, 0)
        tones = sum(np.sin(2 * np.pi * f * t + rng.uniform(0, 6.3)) for f in rng.uniform(40, 21000, 3)) / 3
        y[b] = amp * (0.3 * rng.randn(n) + tones)
    if silent is not None:
        y[silent] = 0.0
    return y


def _stft(y, geom, precision, backend, eps_variant=True):
    """reflect pad + split, then fd_stft_mag_eps_fwd (or fd_stft_mag_fwd) with the DFT weights mel.py packs."""
    n_fft, n_fft_new, win_new, hop, pad, ms, eps = geom
    d0 = dev()
    pc, lib, st = N.prec_code(precision), N.lib(), N.stream_ptr(d0)
    pam = PitchAdjustableMelSpectrogram(n_fft=n_fft, win_length=n_fft, precision=precision)
    w, w_inv, kpad, bins = pam._dft_weights(n_fft_new, win_new, d0, pc)
    B, n = y.shape
    Np = n + 2 * pad
    frames = n_frames(n, n_fft_new, hop, pad)
    pitch = (max(Np, (frames - 1) * hop + kpad) + 7) // 8 * 8     # room for the last frame's zero-weighted K padding
    yd = torch.from_numpy(y).to(d0)
    tmp = torch.zeros((2, B, (Np + 7) // 8 * 8), dtype=torch.int16, device=d0)
    N.check(lib.fd_reflect_pad_split(N.ptr(yd), N.ptr(tmp), B, n, pad, pc, st), "fd_reflect_pad_split")
    padded = torch.zeros((2, B, pitch), dtype=torch.int16, device=d0)
    padded[:, :, :tmp.shape[2]] = tmp
    mag = torch.full((2, B, frames, pam.NB), SENTINEL, dtype=torch.int16, device=d0)
    args = (N.ptr(padded), N.ptr(w), N.ptr(mag), B, pitch, kpad, hop, frames, pam.NB, w_inv, ms)
    tail = (N.mma_code(precision), N.backend_code(backend), st)
    if eps_variant:
        N.check(lib.fd_stft_mag_eps_fwd(*args, eps, *tail), "fd_stft_mag_eps_fwd")
    else:
        N.check(lib.fd_stft_mag_fwd(*args, *tail), "fd_stft_mag_fwd")
    torch.cuda.synchronize()
    return dict(mag=mag, padded=padded, w=w, w_inv=w_inv, kpad=kpad, bins=bins, NB=pam.NB, frames=frames)


def _regions(frames, bins, NB, n_fft):
    """(name, frame mask, bin mask) over [frames] x [bins]"""
    d0 = dev()
    t, k = torch.arange(frames, device=d0), torch.arange(bins, device=d0)
    k_edge = int(16000 * n_fft / SR) + 1          # first bin above 16 kHz: zero weight in the shipped filterbanks
    all_t, all_k = torch.ones_like(t, dtype=torch.bool), torch.ones_like(k, dtype=torch.bool)
    return [("all", all_t, all_k), ("first_frame", t == 0, all_k), ("last_frame", t == frames - 1, all_k),
            ("last_row_tile", t >= (frames - 1) // 128 * 128, all_k), ("below_16k", all_t, k < k_edge),
            ("above_16k", all_t, k >= k_edge), ("last_col_tile", all_t, k >= NB - 128)]


def _judge(what, got, ref, norm, regions, tol):
    """got / ref [B', frames, bins] float64, norm [B', frames] -> failure messages; prints the worst error per region"""
    d = got - ref
    e = d.abs() / norm[..., None]
    msgs, bad = [], []
    mtol, rtol = tol
    for name, tm, km in regions:
        if not bool(tm.any()) or not bool(km.any()):
            continue
        dm, rm = d[:, tm][:, :, km], ref[:, tm][:, :, km]
        mx = float(e[:, tm][:, :, km].max())
        rel = math.sqrt(float((dm * dm).sum()) / max(float((rm * rm).sum()), 1e-300))
        msgs.append(f"{name} {mx:.2e}/{rel:.2e}")
        # rel-L2 is barred over everything only: a region can be one bin of one frame (the Nyquist bin of n_fft 2048 is
        # the only live bin of the last column tile), whose own rel-L2 says nothing
        if not (mx < mtol and (name != "all" or rel < rtol)):
            bad.append(f"{what} {name}: max {mx:.2e} (bar {mtol:.1e}), rel-L2 {rel:.2e} (bar {rtol:.1e})")
    print(f"  {what} (max/rel-L2): " + ", ".join(msgs))
    return bad


def _check_stft(name, geom_name, precision, backend, B, frames=None, n=None, silent=None, exact_chunk=None):
    geom = _geom(geom_name)
    n_fft, n_fft_new, win_new, hop, pad, ms, eps = geom
    pc, single = N.prec_code(precision), precision.endswith("x1")
    if n is None:
        n = _length(frames, n_fft_new, hop, pad)
    y = _items(B, n, zlib.crc32(name.encode()), silent)
    r = _stft(y, geom, precision, backend)
    F, bins, NB = r["frames"], r["bins"], r["NB"]
    if frames is not None:
        assert F == frames
    got = pf64(r["mag"], pc)                                              # [B, F, NB]
    print(f"\n[{name} {backend}] B={B} n={n} frames={F} NB={NB} kpad={r['kpad']} bins={bins}")
    bad = []
    assert bool(torch.isfinite(got).all()), "NaN / inf bins (or bins never written)"

    # bins past the spectrum (zero DFT rows) and silent items: sqrt(eps) * mag_scale, exactly 0 when eps = 0
    v = math.sqrt(eps) * ms
    floor = [got[:, :, bins:].reshape(-1)] + ([got[silent].reshape(-1)] if silent is not None else [])
    worst = max(float((f - v).abs().max()) for f in floor if f.numel())
    print(f"  padding bins / silent item: worst |mag - sqrt(eps)*mag_scale| = {worst:.2e} (value {v:.3e})")
    if eps == 0.0:
        assert worst == 0.0, f"padding bins / silent item not exactly 0: {worst:.2e}"
    else:
        assert worst <= plane_tol(v, pc), f"padding bins / silent item off by {worst:.2e} from {v:.3e}"

    live = [b for b in range(B) if b != silent]
    direct = torch.from_numpy(stft_mag(y[live], n_fft_new, win_new, hop, pad, ms, eps)[..., :bins]).to(dev())
    norm = torch.linalg.vector_norm(direct, dim=-1)                      # the frame's spectral norm
    regions = _regions(F, bins, NB, n_fft)
    bad += _judge("direct", got[live][..., :bins], direct, norm, regions, TOL[("direct", precision, backend)])

    # exact operands, item by item (hi planes alone in single-product mode)
    W = pf64(r["w"], pc, single) * r["w_inv"]
    P = pf64(r["padded"], pc, single)
    exact = torch.empty_like(direct)
    rows = torch.arange(F, device=dev())
    for i, b in enumerate(live):
        exact[i] = stft_mag_packed(P[b:b + 1], W, hop, rows, ms, eps)[0, :, :bins]
    bad += _judge("exact", got[live][..., :bins], exact, norm, regions, TOL[("exact", precision, backend)])
    assert not bad, "; ".join(bad)


# (name, geometry, precision, B, frames, silent item)
CASES = [
    ("h512-f16-B1-F1", "h512", "f16", 1, 1, None),
    ("h512-bf16-B3-F127", "h512", "bf16", 3, 127, 1),
    ("h512-f16x1-B8-F128", "h512", "f16x1", 8, 128, None),
    ("h512-f16-B3-F129", "h512", "f16", 3, 129, None),
    ("h256-f16-B8-F129", "h256", "f16", 8, 129, 7),
    ("h256-bf16-B1-F128", "h256", "bf16", 1, 128, None),
    ("h256-f16x1-B3-F127", "h256", "f16x1", 3, 127, None),
    ("ks+5-f16-B3-F129", "ks+5", "f16", 3, 129, None),
    ("ks+5-bf16-B1-F127", "ks+5", "bf16", 1, 127, None),
    ("ks+5-f16x1-B8-F128", "ks+5", "f16x1", 8, 128, 4),
    ("ks-5-f16-B8-F128", "ks-5", "f16", 8, 128, 0),
    ("ks-5-bf16-B3-F129", "ks-5", "bf16", 3, 129, None),
    ("ks-5-f16x1-B1-F127", "ks-5", "f16x1", 1, 127, None),
    ("w1024-f16-B3-F127", "w1024", "f16", 3, 127, None),
    ("w1024-bf16-B8-F129", "w1024", "bf16", 8, 129, None),
    ("n1024-f16-B3-F129", "n1024", "f16", 3, 129, None),
    ("n1024-bf16-B8-F1", "n1024", "bf16", 8, 1, None),
    ("n4096-f16-B3-F129", "n4096", "f16", 3, 129, 2),
    ("n4096-bf16-B1-F128", "n4096", "bf16", 1, 128, None),
    ("center-f16-B3-F129", "center", "f16", 3, 129, 2),
    ("center-bf16-B8-F127", "center", "bf16", 8, 127, 5),
    ("center-f16x1-B3-F128", "center", "f16x1", 3, 128, None),
]


@pytest.mark.parametrize("backend", ["tc", "simt"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_stft_mag_vs_float64(case, backend):
    name, geom, prec, B, frames, silent = case
    _check_stft(name, geom, prec, backend, B, frames=frames, silent=silent)


# the persistent multi-tile loop: 8 items of 30 s at hop 512 -> 2583 frames, 21 row tiles (the last one ragged) x 9
# column tiles = 1512 tiles over the SMs, with the column tile rotating per row tile
LARGE = [("h512-f16-B8-30s", "h512", "f16", "tc"), ("h512-bf16-B8-30s", "h512", "bf16", "tc"),
         ("h512-f16-B8-30s", "h512", "f16", "simt")]


@pytest.mark.parametrize("case", LARGE, ids=[f"{c[0]}-{c[3]}" for c in LARGE])
def test_stft_mag_multi_tile_vs_float64(case):
    name, geom, prec, backend = case
    _check_stft(name, geom, prec, backend, 8, n=30 * SR, silent=3)


@pytest.mark.parametrize("backend", ["tc", "simt"])
def test_stft_items_independent(backend):
    """Item i of a batch equals the same item run alone, bit for bit (item strides, per-item row tiles)."""
    geom = _geom("ks+5")
    y = _items(3, _length(129, *[geom[i] for i in (1, 3, 4)]), 5)
    batch = _stft(y, geom, "f16", backend)["mag"]
    for i in range(3):
        alone = _stft(y[i:i + 1], geom, "f16", backend)["mag"]
        assert torch.equal(batch[:, i], alone[:, 0]), f"item {i} differs from its solo run"


@pytest.mark.parametrize("backend", ["tc", "simt"])
def test_stft_mag_fwd_is_eps_variant_at_1e9(backend):
    geom = _geom("ks+5")
    y = _items(2, _length(129, *[geom[i] for i in (1, 3, 4)]), 6, silent=1)
    a = _stft(y, geom, "f16", backend)["mag"]
    b = _stft(y, geom, "f16", backend, eps_variant=False)["mag"]
    assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------- small kernels
@pytest.mark.parametrize("B,n,pad,precision", [(2, 1000, 0, "f16"), (3, 1001, 1000, "bf16"), (3, 4099, 768, "f16"),
                                               (1, 5, 4, "bf16"), (4, 2047, 1023, "f16")])
def test_reflect_pad_split_bit_exact(B, n, pad, precision):
    """fd_reflect_pad_split against np.pad(reflect) split by fd_split_nwc (the same rounding); the pitch tail past
    n + 2 pad must be zero."""
    d0 = dev()
    pc = N.prec_code(precision)
    rng = np.random.RandomState(n + pad)
    y = (rng.randn(B, n) * 10.0 ** rng.uniform(-6, 1, (B, n))).astype(np.float32)
    Np = n + 2 * pad
    pitch = (Np + 7) // 8 * 8
    host = np.zeros((B, pitch), dtype=np.float32)
    host[:, :Np] = np.pad(y, ((0, 0), (pad, pad)), mode="reflect")
    want = N.split_nwc(torch.from_numpy(host).to(d0).view(B, pitch // 8, 8), pc).reshape(2, B, pitch)
    got = torch.full((2, B, pitch), SENTINEL, dtype=torch.int16, device=d0)
    N.check(N.lib().fd_reflect_pad_split(N.ptr(torch.from_numpy(y).to(d0)), N.ptr(got), B, n, pad, pc,
                                         N.stream_ptr(d0)), "fd_reflect_pad_split")
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    assert bool((got[:, :, Np:] == 0).all())


@pytest.mark.parametrize("pad", [10, 11])
def test_reflect_pad_split_refuses_pad_ge_n(pad):
    d0 = dev()
    y = torch.zeros((1, 10), dtype=torch.float32, device=d0)
    out = torch.zeros((2, 1, 40), dtype=torch.int16, device=d0)
    with pytest.raises(N.NativeError, match="must be smaller than N"):
        N.check(N.lib().fd_reflect_pad_split(N.ptr(y), N.ptr(out), 1, 10, pad, N.PREC_F16, N.stream_ptr(d0)),
                "fd_reflect_pad_split")


@pytest.mark.parametrize("C,clip", [(1, 1e-5), (2.5, 1e-4)])
def test_log_clamp_vs_float64(C, clip):
    """dynamic_range_compression = log(max(x, clip) * C) on values below, at and above clip, zeros and negatives, over
    n = 2 * 132*16*256 + 3 elements (not a multiple of 4; the grid-stride loop wraps twice)."""
    rng = np.random.RandomState(int(C * 10))
    n = 2 * 132 * 16 * 256 + 3
    kinds = rng.randint(0, 5, n)
    x = np.where(kinds == 0, 10.0 ** rng.uniform(-12, np.log10(clip), n),           # below clip
        np.where(kinds == 1, clip,                                                   # at clip
        np.where(kinds == 2, 10.0 ** rng.uniform(np.log10(clip), 4, n),              # above
        np.where(kinds == 3, 0.0, -rng.rand(n)))))                                   # zeros, negatives
    x = x.astype(np.float32)
    got = dynamic_range_compression(torch.from_numpy(x).to(dev()), C=C, clip_val=clip).cpu().numpy().astype(np.float64)
    ref = np.log(np.maximum(x.astype(np.float64), clip) * C)
    err = np.abs(got - ref)
    print(f"\nlog clamp C={C} clip={clip}: max |err| {err.max():.2e}, at the clip value {err[kinds != 2].max():.2e}")
    assert err.max() < 2e-6                  # logf and the float32 output, ~1 ulp of |log x| <= 11.5; measured 5.6e-7


@pytest.mark.parametrize("B,T,C", [(3, 77, 45), (2, 1, 33), (5, 129, 128), (1, 1000, 80)])
def test_transpose_nwc_to_ncw_bit_exact(B, T, C):
    d0 = dev()
    x = torch.randn((B, T, C), generator=torch.Generator().manual_seed(B * T + C)).to(d0)
    out = torch.full((B, C, T), float("nan"), dtype=torch.float32, device=d0)
    N.check(N.lib().fd_transpose_nwc_to_ncw(N.ptr(x), N.ptr(out), B, T, C, N.stream_ptr(d0)), "fd_transpose_nwc_to_ncw")
    torch.cuda.synchronize()
    assert torch.equal(out, x.transpose(1, 2))


# ---------------------------------------------------------------------------------------------- end to end
def _mel_err(got, ref):
    """got / ref [B, n_mels, frames] -> (rel-L2, worst bin error in units of its frame's mel norm)"""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    norm = np.linalg.norm(ref, axis=1, keepdims=True)
    return rel_l2(got, ref), float((np.abs(got - ref) / np.maximum(norm, 1e-30)).max())


# (name, key_shift, speed, n, extra constructor arguments, precision, backend).  n = 258 * 512 (+ 1, + 13): the last frame's
# zero-weighted K padding (kpad - n_fft_new = 2 at -5, 18 at +5) runs past the reflect-padded signal
PAM = [
    ("ks0", 0, 1.0, 3 * SR, {}, "f16", "tc"),
    ("ks+5", 5, 1.0, 258 * 512 + 13, {}, "f16", "tc"),
    ("ks-5", -5, 1.0, 258 * 512, {}, "f16", "tc"),
    ("ks-5-bf16-simt", -5, 1.0, 258 * 512 + 1, {}, "bf16", "simt"),
    ("speed0.5", 0, 0.5, 3 * SR, {}, "f16", "tc"),
    ("speed1.1", 0, 1.1, 3 * SR, {}, "f16", "tc"),            # hop 563: the gathered-frame path
    ("ks+5-speed1.1", 5, 1.1, 3 * SR, {}, "bf16", "tc"),
    ("mels80-fmax", 0, 1.0, 3 * SR, dict(n_mels=80, f_max=SR // 2), "f16", "tc"),
]
# (rel-L2, worst bin in units of its frame's mel norm) against the float64 oracle, per precision
MEL_TOL = {"f16": (2.5e-5, 2.5e-5),      # measured 9.4e-6 / 9.7e-6
           "bf16": (4e-5, 6e-5)}         # measured 1.1e-5 / 1.7e-5


@pytest.mark.parametrize("case", PAM, ids=[c[0] for c in PAM])
def test_pitch_adjustable_mel_vs_oracle(case):
    name, ks, speed, n, kw, precision, backend = case
    y = _items(4, n, zlib.crc32(name.encode()))
    pam = PitchAdjustableMelSpectrogram(precision=precision, backend=backend, **kw)
    got = pam(torch.from_numpy(y).to(dev()), key_shift=ks, speed=speed).cpu().numpy()
    ref = omel.pitch_adjustable_mel(y, key_shift=ks, speed=speed, **kw)
    assert got.shape == ref.shape
    rel, mx = _mel_err(got, ref)
    print(f"\n[{name}] mel rel-L2 {rel:.2e}, worst frame-normalised bin {mx:.2e}")
    rtol, mtol = MEL_TOL[precision]
    assert rel < rtol and mx < mtol


@pytest.mark.parametrize("hop", [512, 256])
def test_mel_transform_training_shape_vs_float64(hop):
    """get_mel_transform on the vocoder's training batch (B=8 x 16384-sample segments, [..., n] input), and
    get_mel_from_audio on one clip, against the float64 MelSpectrogram restatement."""
    y = _items(8, 16384, hop)
    tf = get_mel_transform(hop_length=hop)
    got = tf(torch.from_numpy(y).to(dev()).view(2, 4, -1)).cpu().numpy()
    ref = mel_spectrogram(y, hop_length=hop)
    assert got.shape == (2, 4) + ref.shape[1:]
    rel, mx = _mel_err(got.reshape(ref.shape), ref)
    lm = get_mel_from_audio(torch.from_numpy(y[:1]).to(dev()), hop_length=hop).cpu().numpy()
    dl = float(np.abs(lm - np.log(np.maximum(ref[0], 1e-5))).max())
    print(f"\n[hop {hop}] mel rel-L2 {rel:.2e}, worst frame-normalised bin {mx:.2e}; max |d log-mel| {dl:.2e}")
    assert rel < 2.5e-5 and mx < 2.5e-5      # measured 7.1e-6 / 6.2e-6
    assert dl < 2.5e-4                       # measured 7.6e-5 (a relative error where the mel is just above the clip)
