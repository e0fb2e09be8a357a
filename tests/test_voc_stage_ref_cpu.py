"""The float64 stage references of tests/voc_stage_ref.py: chained, they are the generator of the oracle; windowed, they
equal their full form at item starts, item ends, the middle and T = 1.  Also the host-side refusal of a noise conv whose
output length differs from the stage length."""
import json
import os

import numpy as np
import pytest
import torch

import voc_stage_ref as R
from conftest import GOLDEN
from fish_diffusion_b200 import Generator
from oracle import nsf_hifigan as ovoc

F64 = torch.float64


def _cpu_gen(h, sd):
    gen = Generator(h)
    gen.remove_weight_norm()
    res = gen.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    return gen


def _case(name, golden, golden_cfg):
    if name == "small":
        h = golden_cfg["VOC_SMALL"]
        return h, ovoc.make_generator_weights(3, h), 2, 5
    if name == "resblock2":
        g = golden("r2_voc_resblock2")
        h = json.loads(str(g["rb2_cfg"]))
        return h, {k[len("rb2_sd_"):]: v for k, v in g.items() if k.startswith("rb2_sd_")}, 2, 4
    with open(os.path.join(GOLDEN, "nsf_configs", name + ".json")) as f:
        h = json.load(f)
    return h, ovoc.make_generator_weights(4, h), 2, 2


@pytest.mark.parametrize("name", ["small", "resblock2", "config_v1_256"])
def test_stage_chain_equals_oracle_generator(golden, golden_cfg, name):
    h, sd, B, T = _case(name, golden, golden_cfg)
    hop = int(np.prod(h["upsample_rates"]))
    rng = np.random.RandomState(20)
    mel = (rng.randn(B, h["num_mels"], T) - 2.0).astype(np.float32)
    f0 = np.full((B, T), 180.0, dtype=np.float32)
    f0[:, 0] = 0
    f0[0, -1] = 0
    ri = rng.rand(B, 9).astype(np.float32)
    ri[:, 0] = 0
    nz = rng.randn(B, T * hop, 9).astype(np.float32)
    wav, har = ovoc.generator_forward(sd, h, mel, f0, ri, nz, mode="exact", return_source=True)
    out = R.generator_chain(_cpu_gen(h, sd), torch.from_numpy(mel), torch.from_numpy(har[:, 0]))
    got = out["wav"][:, :, 0].numpy()
    e = float(np.abs(got - wav[:, 0]).max())
    print(f"stage chain [{name}] vs oracle generator: max |d wav| {e:.2e}")
    assert got.shape == wav[:, 0].shape and e < 1e-12
    assert len(out["ups_in"]) == len(h["upsample_rates"])


def _windows(T, w):
    w = min(w, T)
    return sorted({(0, w), (T - w, T), ((T - w) // 2, (T - w) // 2 + w), (0, T)})


def _same(a, b):
    assert a.shape == b.shape
    assert float((a - b).abs().max()) <= 1e-12 * max(float(b.abs().max()), 1.0)


@pytest.mark.parametrize("T", [1, 6, 41])
def test_windowed_equals_full(T):
    g = torch.Generator().manual_seed(T)
    rn = lambda *s: torch.randn(*s, generator=g, dtype=F64)
    B, C = 3, 8
    x = rn(B, T, C)
    get = R.getter(x)
    for K, d in ((3, 1), (7, 3), (11, 5)):
        w, b = rn(C, C, K) / 8, rn(C)
        full = R.conv(x, w, b, d, slope=0.1)
        for t0, t1 in _windows(T, 4):
            _same(R.conv_win(get, w, b, d, t0, t1, slope=0.1), full[:, t0:t1])
        w2, b2 = rn(C, C, K) / 8, rn(C)
        full = R.resblock1_pair(x, w, b, d, w2, b2, out_slope=0.1)
        for t0, t1 in _windows(T, 4):
            _same(R.resblock1_pair_win(get, w, b, d, w2, b2, t0, t1, T, out_slope=0.1), full[:, t0:t1])
        full = R.resblock2_step(x, w, b, d, slope=0.1)
        for t0, t1 in _windows(T, 4):
            _same(R.resblock2_step_win(get, w, b, d, t0, t1, slope=0.1), full[:, t0:t1])
    w, b = rn(C, 24, 7) / 8, rn(C)
    mel = rn(B, T, 24)
    full = R.conv_pre(mel, w, b)
    for t0, t1 in _windows(T, 4):
        _same(R.conv_pre_win(R.getter(mel), w, b, t0, t1), full[:, t0:t1])
    wp, bp = rn(1, C, 7), rn(1)
    full = R.conv_post(x, wp, bp)
    for t0, t1 in _windows(T, 4):
        _same(R.conv_post_win(get, wp, bp, t0, t1), full[:, t0:t1])
    for k, u in ((16, 8), (8, 2), (4, 2), (2, 2)):
        p = (k - u) // 2
        wt, bt = rn(C, 4, k), rn(4)
        add = rn(B, T * u, 4)
        X, A = R.ups(x, wt, bt, u, p, add)
        assert X.shape == (B, T * u, 4)
        for t0, t1 in _windows(T * u, 5):
            Xw, Aw = R.ups_win(get, wt, bt, u, p, add[:, t0:t1], t0, t1)
            _same(Xw, X[:, t0:t1])
            _same(Aw, A[:, t0:t1])
    for s in (64, 8, 2, 1):
        k, p = (2 * s, s // 2) if s > 1 else (1, 0)
        har = rn(B, T * s)
        ws, bs = rn(C, 1, k), rn(C)
        full = R.source_conv(har, ws, bs, s, p)
        assert full.shape == (B, T, C)
        for t0, t1 in _windows(T, 3):
            _same(R.source_conv_win(R.getter(har[:, :, None]), ws, bs, s, p, t0, t1), full[:, t0:t1])


def test_mrf_reference_is_the_mean_of_the_resblocks():
    g = torch.Generator().manual_seed(1)
    xs = [torch.randn(2, 5, 4, generator=g, dtype=F64) for _ in range(3)]
    got = R.mrf([R.lrelu(x, 0.1) for x in xs], 0.1, 1 / 3, 0.01)
    want = R.lrelu((xs[0] + xs[1] + xs[2]) / 3, 0.01)
    _same(got, want)


@pytest.mark.parametrize("rates,ksz", [([8, 3], [16, 7]), ([4, 5, 3], [8, 9, 7])])
def test_odd_noise_conv_stride_is_refused_before_any_launch(monkeypatch, rates, ksz):
    """An odd noise-conv stride (upsample rates 3 or 5 after the first stage: stride 3, or 15 and 3 here) makes
    noise_convs[i] return one row fewer than the stage has; forward must refuse it instead of adding an uninitialised
    row.  Host-only: the native library is replaced by a stub that fails on any use, so no kernel can run."""
    from fish_diffusion_b200 import _native as N

    def no_native(*a, **k):
        raise AssertionError("native code reached")

    h = dict(resblock="1", upsample_rates=rates, upsample_kernel_sizes=ksz, upsample_initial_channel=64,
             resblock_kernel_sizes=[3], resblock_dilation_sizes=[[1, 3, 5]], num_mels=8, hop_size=int(np.prod(rates)),
             sampling_rate=44100)
    gen = Generator(h)
    monkeypatch.setattr(N, "lib", no_native)
    monkeypatch.setattr(N, "require_cuda", lambda *a, **k: None)
    with pytest.raises(ValueError, match="noise_convs"):
        gen(torch.zeros(1, 8, 4), torch.zeros(1, 4))
