"""NSF-HiFiGAN generator launch by launch against float64: every kernel launch of Generator.forward -- conv_pre, each
polyphase upsample tap-GEMM with its source addend, the strided source convs, the fused ResBlock pairs (time-folded with
kmask hints at C = 16), the conv-by-conv tap-GEMMs (time-folded by F = 2 / 4 / 8), the SIMT twin, fd_mrf_finish and
conv_post + tanh -- is judged on the operands it actually read against the module-level float64 operation of
tests/voc_stage_ref.py, with errors per row region (item edges, last tile, polyphase phase or fold sub-step, interior).
The stage boundaries are also compared with the float64 chain run from the mel, and the sequence of launches -- which
path each stage took -- is asserted.  The production shape (config_v1, B = 32 x T = 4000) is judged on windows inside the
launch hooks, including the row where a tensor's flat byte offset crosses 2^31.

Bars: at most 4x the worst value measured over every case on an H100 SXM (80 GB, 700 W power limit); the measured worst
is written beside each.  "max" is max|err| in units of the judged tensor's RMS."""
import json
import os

import numpy as np
import pytest
import torch

import voc_stage_ref as R
from conftest import GOLDEN
from fish_diffusion_b200 import Generator
from fish_diffusion_b200 import _native as N
from gpu_util import dev
from oracle import nsf_hifigan as ovoc
from region_check import Regions, pf64

pytestmark = pytest.mark.gpu

F64 = torch.float64

# (rel-L2, max/RMS) bars per launch kind and arithmetic, each with the worst measured value (H100 SXM, 700 W) beside it:
# x3 = f16 planes, three tensor-core products; bf16 = bf16 planes, three products; x1 = f16, one product over the hi
# planes; simt = f16 planes, fp32 SIMT back end.  x3 covers the production-shape windows too.  split / source / mrf /
# post are fp32 kernels whatever the GEMM arithmetic; bf16 planes store 16 bits, f16 planes 22.
TOL = {
    "x3": dict(split=(1.8e-7, 7.1e-7),     # measured 4.71e-08 / 1.78e-07
               pre=(1.2e-5, 1.1e-4),       # measured 3.24e-06 / 2.89e-05
               source=(8.5e-7, 1.1e-5),    # measured 2.13e-07 / 2.76e-06
               ups=(1.6e-5, 1.4e-4),       # measured 4.02e-06 / 3.58e-05
               conv=(4e-5, 3.4e-4),        # measured 1.02e-05 / 8.74e-05
               pair=(3.4e-5, 3e-4),        # measured 8.73e-06 / 7.52e-05
               mrf=(5.8e-7, 4.7e-6),       # measured 1.47e-07 / 1.18e-06
               post=(2.9e-6, 7.8e-5),      # measured 7.47e-07 / 1.97e-05
               chain=(1.5e-4, 1.4e-3)),    # measured 3.96e-05 / 3.68e-04
    "bf16": dict(split=(1e-5, 4.5e-5),     # measured 2.54e-06 / 1.14e-05
                 pre=(2e-5, 2.1e-4),       # measured 5.18e-06 / 5.49e-05
                 source=(7.2e-7, 7.5e-6),  # measured 1.82e-07 / 1.89e-06
                 ups=(2.3e-5, 2.3e-4),     # measured 5.92e-06 / 5.95e-05
                 conv=(4.4e-5, 3.7e-4),    # measured 1.11e-05 / 9.27e-05
                 pair=(3.7e-5, 4e-4),      # measured 9.25e-06 / 1.01e-04
                 mrf=(1.3e-5, 1.5e-4),     # measured 3.43e-06 / 3.93e-05
                 post=(1.9e-6, 1.3e-5),    # measured 4.84e-07 / 3.28e-06
                 chain=(1.5e-4, 1.3e-3)),  # measured 3.91e-05 / 3.36e-04
    "x1": dict(split=(1.5e-7, 7e-7),       # measured 3.92e-08 / 1.77e-07
               pre=(1.2e-3, 7.8e-3),       # measured 3.11e-04 / 1.96e-03
               source=(7.2e-7, 7.5e-6),    # measured 1.82e-07 / 1.89e-06
               ups=(1.3e-3, 1.1e-2),       # measured 3.47e-04 / 2.97e-03
               conv=(1.3e-3, 8.7e-3),      # measured 3.32e-04 / 2.19e-03
               pair=(4.6e-4, 3.4e-3),      # measured 1.17e-04 / 8.73e-04
               mrf=(5.9e-7, 4.7e-6),       # measured 1.48e-07 / 1.19e-06
               post=(1.2e-6, 1e-5),        # measured 3.16e-07 / 2.55e-06
               chain=(7.4e-3, 3e-2)),      # measured 1.87e-03 / 7.69e-03
    "simt": dict(split=(1.8e-7, 7.1e-7),   # measured 4.71e-08 / 1.78e-07
                 pre=(2.2e-6, 3.3e-5),     # measured 5.51e-07 / 8.32e-06
                 source=(8.5e-7, 1e-5),    # measured 2.13e-07 / 2.52e-06
                 ups=(2.4e-6, 4.1e-5),     # measured 6.22e-07 / 1.03e-05
                 conv=(3.9e-6, 6e-5),      # measured 9.86e-07 / 1.50e-05
                 mrf=(6e-8, 1.2e-7),       # measured 1.51e-08 / 3.16e-08
                 post=(3e-6, 7e-5),        # measured 7.69e-07 / 1.77e-05
                 chain=(2.1e-5, 4.2e-4)),  # measured 5.34e-06 / 1.06e-04
}


def _view(ptr, shape, dtype):
    """the tensor at a device pointer the generator handed to the native library (a view, no copy)"""
    class _Arr:
        pass
    a = _Arr()
    a.__cuda_array_interface__ = dict(shape=tuple(int(s) for s in shape), data=(int(ptr), False), version=3,
                                      typestr={torch.float32: "<f4", torch.int16: "<i2"}[dtype], strides=None)
    return torch.as_tensor(a, device=dev())


def crossing(t, C):
    """[(item, row)] where the flat byte offset of t -- planes [2, B, T, *] or fp32 [B, T, *] -- crosses 2^31, with rows
    of C channels (the same memory whether the launch saw it time-folded or not)"""
    e = (1 << 31) // t.element_size()
    if t.numel() <= e:
        return []
    per_plane = t.numel() // 2 if t.dtype == torch.int16 else t.numel()
    row = (e % per_plane) // C
    T = per_plane // C // t.shape[-3]
    return [(row // T, row % T)]


class Windows:
    """Row windows a launch is judged on: the whole of every item, or (production) item start, middle and end of a few
    items plus the 2^31-crossing rows."""

    def __init__(self, B, items=None, width=2048):
        self.B, self.items, self.width = B, items, width

    def __call__(self, T, extra=()):
        if self.items is None:
            return [(list(range(self.B)), 0, T)]
        w = min(self.width, T)
        out = [(list(self.items), t0, t0 + w) for t0 in sorted({0, (T - w) // 2, T - w})]
        for b, t in extra:
            t0 = min(max(0, t - w // 2), T - w)
            out.append(([b], t0, t0 + w))
        return out


def _rows_planes(planes, Cm, prec, items, a, b):
    """float64 CPU rows [a, b) (zeros outside the item) of planes viewed as [2, B, T, Cm]"""
    p = planes.reshape(2, planes.shape[1], -1, Cm)
    T = p.shape[2]
    out = torch.zeros((len(items), b - a, Cm), dtype=F64)
    lo, hi = max(a, 0), min(b, T)
    if hi > lo:
        out[:, lo - a:hi - a] = pf64(p[:, items, lo:hi], prec).cpu()
    return out


def _rows_f32(t, Cm, items, a, b):
    x = t.reshape(t.shape[0], -1, Cm)
    T = x.shape[1]
    out = torch.zeros((len(items), b - a, Cm), dtype=F64)
    lo, hi = max(a, 0), min(b, T)
    if hi > lo:
        out[:, lo - a:hi - a] = x[items, lo:hi].to(F64).cpu()
    return out


class Capture:
    """Launch hooks of one Generator.forward.  Each hook runs the native call, synchronizes, and judges the launch on
    the windows; it records the launch kind and path (`seq`), the failures (`bad`) and, when whole items are judged,
    the stage boundaries (`bound`)."""

    def __init__(self, gen, windows, arith):
        self.gen, self.win, self.tol = gen, windows, TOL[arith]
        self.prec = N.prec_code(gen.precision)
        self.full = windows.items is None
        self.seq, self.bad, self.bound = [], [], {"ups_in": []}
        self.idx = None

    # -------------------------------------------------------------------------------- which module a launch runs
    def _index(self):
        g, pk = self.gen, self.gen._pack
        idx = {}

        def put(pc, tag, mod):
            idx[pc["w"].data_ptr()] = (tag, mod, 1)
            if "fold" in pc:
                idx[pc["fold"]["w"].data_ptr()] = (tag, mod, pc["fold"]["F"])

        put(pk["pre"], "pre", g.conv_pre)
        for i, pc in enumerate(pk["ups"]):
            idx[pc["w"].data_ptr()] = (f"ups{i}", g.ups[i], 1)
        for r, ent in enumerate(pk["res"]):
            rb = g.resblocks[r]
            if ent["kind"] == 1:
                for m in range(len(rb.convs1)):
                    put(ent["c1"][m], f"res{r}.c1.{m}", rb.convs1[m])
                    put(ent["c2"][m], f"res{r}.c2.{m}", rb.convs2[m])
                    pair = (rb.convs1[m], rb.convs2[m])
                    idx[("pair", ent["c1"][m]["w"].data_ptr())] = (f"res{r}.pair{m}", pair, 1)
                    if "c1f" in ent:
                        idx[("pair", ent["c1f"][m]["w"].data_ptr())] = (f"res{r}.pair{m}", pair, ent["c1f"][m]["F"])
            else:
                for m in range(len(rb.convs)):
                    put(ent["c"][m], f"res{r}.c.{m}", rb.convs[m])
        for i, s in enumerate(pk["src"]):
            idx[("src", s["w_t"].data_ptr())] = i
        self.idx = idx

    def _judge(self, what, kind, reg, pairs):
        """pairs: iterable of (got, ref, t0) over the windows"""
        for got, ref, t0 in pairs:
            assert got.shape == ref.shape, (what, got.shape, ref.shape)
            reg.add(got, ref, t0)
        self.bad += reg.check(what, self.tol[kind])

    # -------------------------------------------------------------------------------- hooks
    def split_ncw(self, orig, x, prec, mask=None, out=None):
        out = orig(x, prec, mask=mask, out=out)
        torch.cuda.synchronize()
        B, C, T = x.shape
        self.seq.append(("split",))
        reg = Regions(T, 1, "cpu")
        self._judge("split_ncw(mel)", "split", reg,
                    ((_rows_planes(out, C, prec, it, t0, t1), x[it, :, t0:t1].transpose(1, 2).to(F64).cpu(), t0)
                     for it, t0, t1 in self.win(T)))
        return out

    def conv_cl(self, orig, in_planes, w_planes, B, T, Cin, Nn, shifts, **kw):
        if self.idx is None:
            self._index()
        tag, mod, F = self.idx[w_planes.data_ptr()]
        be = "tc" if kw.get("backend", N.BACKEND_TC) == N.BACKEND_TC else "simt"
        slope = kw.get("act_slope") if kw.get("act", N.ACT_NONE) == N.ACT_LRELU else None
        ps = kw.get("planes_scale", 1.0)
        self.seq.append(("conv", tag, F, be) + ((round(slope, 6),) if ps != 1.0 else ()))
        w, b = R.wb(mod)
        out_f32, out_planes, addend, resb = kw.get("out_f32"), kw.get("out_planes"), kw.get("addend"), kw.get("res_planes")
        if tag.startswith("ups"):
            u, p, Ci, Co = mod.stride[0], mod.padding[0], mod.in_channels, mod.out_channels
            assert F == 1 and Cin == Ci and Nn == u * Co
            Tt, d = T * u, None
        else:
            Ci, Co, d = mod.in_channels, mod.out_channels, mod.dilation[0]
            assert Cin == F * Ci and Nn == F * Co
            Tt = T * F
        wins = self.win(Tt, crossing(out_planes if out_planes is not None else out_f32, Co))
        # the epilogue may write where it reads (res_f32 is out_f32 in a ResBlock1 chain; out_accum): take those rows first
        res_f32, acc = kw.get("res_f32"), kw["out_f32"] if kw.get("out_accum") else None
        pre = [(None if res_f32 is None else _rows_f32(res_f32, Co, it, t0, t1),
                None if acc is None else _rows_f32(acc, Co, it, t0, t1)) for it, t0, t1 in wins]
        orig(in_planes, w_planes, B, T, Cin, Nn, shifts, **kw)
        torch.cuda.synchronize()
        get = lambda it: lambda a, c: _rows_planes(in_planes, Ci, self.prec, it, a, c)
        pairs_f, pairs_p = [], []
        for (it, t0, t1), (r32, a32) in zip(wins, pre):
            if d is None:
                y, _ = R.ups_win(get(it), w, b, u, p, _rows_f32(addend, Co, it, t0, t1), t0, t1)
            else:
                y = R.conv_win(get(it), w, b, d, t0, t1)
                for extra in (None if addend is None else _rows_f32(addend, Co, it, t0, t1), r32, a32,
                              None if resb is None else _rows_planes(resb, Co, self.prec, it, t0, t1)):
                    if extra is not None:
                        y = y + extra
            if out_f32 is not None:
                pairs_f.append((_rows_f32(out_f32, Co, it, t0, t1), y, t0))
            if out_planes is not None:
                v = y * ps
                pairs_p.append((_rows_planes(out_planes, Co, self.prec, it, t0, t1),
                                v if slope is None else R.lrelu(v, slope), t0))
        if d is None:
            kind, reg = "ups", lambda: Regions(Tt, mod.kernel_size[0], "cpu", tile=128 * u, phase=u)
            if self.full:
                self.bound["ups_in"].append(_rows_planes(in_planes, Ci, self.prec, list(range(B)), 0, T))
        else:
            kind = "pre" if tag == "pre" else "conv"
            reg = lambda: Regions(Tt, R.conv_halo(w, d), "cpu", tile=128 * F, phase=F, phase_name="f")
        if pairs_p:
            self._judge(f"{tag} F={F} [{be}] planes", kind, reg(), pairs_p)
        if pairs_f:
            self._judge(f"{tag} F={F} [{be}] fp32", kind, reg(), pairs_f)

    def respair(self, orig, in_planes, w1, w2, b1, b2, B, T, C, k1, d1, k2, **kw):
        if self.idx is None:
            self._index()
        orig(in_planes, w1, w2, b1, b2, B, T, C, k1, d1, k2, **kw)
        torch.cuda.synchronize()
        out = kw["out_planes"]
        assert out.data_ptr() != in_planes.data_ptr()
        tag, (c1, c2), F = self.idx[("pair", w1.data_ptr())]
        km1, km2 = kw.get("kmask1", 0), kw.get("kmask2", 0)
        self.seq.append(("respair", tag, F, km1 != 0 and km2 != 0))
        Cm, Tt = C // F, T * F
        (w1r, b1r), (w2r, b2r) = R.wb(c1), R.wb(c2)
        d = c1.dilation[0]
        si, so = kw.get("in_slope", 0.1), kw.get("out_slope", 0.1)
        pairs = []
        for it, t0, t1 in self.win(Tt, crossing(out, Cm)):
            get = lambda a, c: R.inv_lrelu(_rows_planes(in_planes, Cm, self.prec, it, a, c), si)
            ref = R.resblock1_pair_win(get, w1r, b1r, d, w2r, b2r, t0, t1, Tt, out_slope=so)
            pairs.append((_rows_planes(out, Cm, self.prec, it, t0, t1), ref, t0))
        r_out = 16384 // C - (k2 - 1)          # output rows of one pair-kernel tile
        self._judge(f"{tag} F={F} kmask={km1 != 0} [pair]", "pair",
                    Regions(Tt, R.pair_halo(w1r, d, w2r), "cpu", tile=r_out * F, phase=F, phase_name="f"), pairs)

    def mrf_finish(self, orig, ins, out, *, in_slope=0.1, scale=1.0, out_slope=0.1, prec=N.PREC_F16):
        orig(ins, out, in_slope=in_slope, scale=scale, out_slope=out_slope, prec=prec)
        torch.cuda.synchronize()
        self.seq.append(("mrf", len(ins), round(in_slope, 6), round(scale, 6), round(out_slope, 6)))
        C = out.shape[-1]
        T = out.shape[-2]
        pairs = []
        for it, t0, t1 in self.win(T, crossing(out, C)):
            ref = R.mrf([_rows_planes(a, C, prec, it, t0, t1) for a in ins], in_slope, scale, out_slope)
            pairs.append((_rows_planes(out, C, prec, it, t0, t1), ref, t0))
        self._judge(f"mrf_finish n={len(ins)} out_slope={out_slope}", "mrf", Regions(T, 1, "cpu"), pairs)

    def sinegen(self, orig, *a):
        rc = orig(*a)
        torch.cuda.synchronize()
        B, T, hop = a[7], a[8], a[9]
        self.seq.append(("sinegen",))
        har = _view(a[5], (B, T * hop), torch.float32)
        self.har = har.clone() if self.full else har
        return rc

    def source_conv(self, orig, har, w_t, bias, out, B, S, C, k, s, p, st):
        rc = orig(har, w_t, bias, out, B, S, C, k, s, p, st)
        torch.cuda.synchronize()
        if self.idx is None:
            self._index()
        i = self.idx[("src", int(w_t))]
        self.seq.append(("source", i))
        nc = self.gen.noise_convs[i]
        w, b = R.wb(nc)
        So = (S + 2 * nc.padding[0] - nc.kernel_size[0]) // nc.stride[0] + 1
        hv = _view(har, (B, S), torch.float32)
        ov = _view(out, (B, So, C), torch.float32)
        pairs = []
        for it, t0, t1 in self.win(So, crossing(ov, C)):
            ref = R.source_conv_win(lambda a, c: _rows_f32(hv, 1, it, a, c), w, b, nc.stride[0], nc.padding[0], t0, t1)
            pairs.append((_rows_f32(ov, C, it, t0, t1), ref, t0))
        edge = -(-nc.kernel_size[0] // nc.stride[0])
        self._judge(f"noise_convs[{i}] k={k} s={s}", "source", Regions(So, edge, "cpu"), pairs)
        return rc

    def conv_post(self, orig, in_planes, w, bias, wav, B, S, C, k, prec, st):
        rc = orig(in_planes, w, bias, wav, B, S, C, k, prec, st)
        torch.cuda.synchronize()
        self.seq.append(("post",))
        ip = _view(in_planes, (2, B, S, C), torch.int16)
        wv = _view(wav, (B, S), torch.float32)
        wr, br = R.wb(self.gen.conv_post)
        pairs = []
        for it, t0, t1 in self.win(S, crossing(ip, C)):
            ref = R.conv_post_win(lambda a, c: _rows_planes(ip, C, prec, it, a, c), wr, br, t0, t1)
            pairs.append((_rows_f32(wv, 1, it, t0, t1), ref, t0))
        self._judge("conv_post + tanh", "post", Regions(S, 3, "cpu"), pairs)
        if self.full:
            self.bound["post_in"] = _rows_planes(ip, C, prec, list(range(B)), 0, S)
            self.bound["wav"] = _rows_f32(wv, 1, list(range(B)), 0, S)
        return rc

    # -------------------------------------------------------------------------------- installation
    def install(self, monkeypatch):
        real = N.lib()
        cap = self

        class LibProxy:
            def __getattr__(self, name):
                f = getattr(real, name)
                hook = {"fd_source_conv_fwd": cap.source_conv, "fd_conv_post_fwd": cap.conv_post,
                        "fd_sinegen_fwd": cap.sinegen}.get(name)
                return f if hook is None else (lambda *a: hook(f, *a))

        proxy = LibProxy()
        for name in ("conv_cl", "respair", "mrf_finish", "split_ncw"):
            orig = getattr(N, name)
            monkeypatch.setattr(N, name, (lambda o, h: lambda *a, **k: h(o, *a, **k))(orig, getattr(self, name)))
        monkeypatch.setattr(N, "lib", lambda: proxy)


# ------------------------------------------------------------------------------------------------ the expected path
def _fold(path, C, K, d):
    """time-folding factor of a conv-by-conv ResBlock conv (Generator._fold_factor, tensor cores only)"""
    if path == "simt":
        return 1
    if C == 16:
        return 8
    if C == 32 and d == 1:
        return 4
    if C == 64 and d == 1 and K >= 11:
        return 2
    return 1


def expected_launches(h, path):
    """The launches of Generator.forward, in order, for path "auto" (fused ResBlock pairs where the pair kernel takes
    the stage), "unfused" (FD_VOC_FUSED=0) or "simt".  Tensor cores run every tap-GEMM whose input and output widths are
    multiples of 16 except on "simt"; the pair kernel takes ResBlock1 stages of C = 16 ... 128, time-folded with kmask
    hints at C = 16; the last stage's output LeakyReLU has slope 0.01."""
    be = lambda cin, n: "tc" if path != "simt" and cin % 16 == 0 and n % 16 == 0 else "simt"
    nk = len(h["resblock_kernel_sizes"])
    C = h["upsample_initial_channel"]
    n_up = len(h["upsample_rates"])
    seq = [("sinegen",), ("split",), ("conv", "pre", 1, be(h["num_mels"], C))]
    for i, u in enumerate(h["upsample_rates"]):
        Co = C // 2
        slope = 0.01 if i == n_up - 1 else 0.1
        seq += [("source", i), ("conv", f"ups{i}", 1, be(C, u * Co))]
        fused = path == "auto" and str(h["resblock"]) == "1" and Co in (16, 32, 64, 128)
        for j, (K, dil) in enumerate(zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"])):
            r = i * nk + j
            fin = (round(slope, 6),) if j == nk - 1 else ()
            for m, d in enumerate(dil):
                if fused:
                    seq.append(("respair", f"res{r}.pair{m}", 2 if Co == 16 else 1, Co == 16))
                    continue
                fb = lambda dd: _fold(path, Co, K, dd) if be(Co, Co) == "tc" else 1
                last = m == len(dil) - 1
                if str(h["resblock"]) == "1":
                    seq.append(("conv", f"res{r}.c1.{m}", fb(d), be(Co, Co)))
                    seq.append(("conv", f"res{r}.c2.{m}", fb(1), be(Co, Co)) + (fin if last else ()))
                else:
                    if m == 0 and j > 0:
                        seq.append(("mrf", 1, 1.0, 1.0, 0.1))
                    seq.append(("conv", f"res{r}.c.{m}", fb(d), be(Co, Co)) + (fin if last else ()))
        if fused:
            seq.append(("mrf", nk, 0.1, round(1.0 / nk, 6), slope))
        C = Co
    return seq + [("post",)]


# ------------------------------------------------------------------------------------------------ cases
def _config(name, golden, golden_cfg):
    if name == "small":
        h = golden_cfg["VOC_SMALL"]
        return h, ovoc.make_generator_weights(41, h)
    if name == "resblock2":
        g = golden("r2_voc_resblock2")
        return json.loads(str(g["rb2_cfg"])), {k[len("rb2_sd_"):]: v for k, v in g.items() if k.startswith("rb2_sd_")}
    with open(os.path.join(GOLDEN, "nsf_configs", name + ".json")) as f:
        h = json.load(f)
    return h, ovoc.make_generator_weights(42, h)


def _generator(h, sd, path, precision, monkeypatch):
    monkeypatch.setenv("FD_VOC_FUSED", "0" if path == "unfused" else "1")
    monkeypatch.delenv("FD_BACKEND", raising=False)
    gen = Generator(h, precision=precision, backend="simt" if path == "simt" else "auto")
    gen.remove_weight_norm()
    res = gen.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    return gen.to(dev()).eval()


def _inputs(h, B, T, seed):
    """mel, f0 with voiced / unvoiced transitions (unvoiced first and last frames), rand_ini, sine_noise -- on the device"""
    g = torch.Generator(device=dev()).manual_seed(seed)
    hop = int(np.prod(h["upsample_rates"]))
    mel = (torch.randn(B, h["num_mels"], T, generator=g, device=dev()) - 2.5).clamp(-11.5, 2.0)
    t = torch.arange(T, device=dev(), dtype=torch.float32)
    f0 = (160.0 + 60.0 * torch.sin(t / 7.0))[None].repeat(B, 1) * (1.0 + 0.1 * torch.arange(B, device=dev()))[:, None]
    f0[:, 0] = 0
    f0[:, -1] = 0
    if T > 8:
        f0[:, T // 3:T // 3 + max(1, T // 8)] = 0
    ri = torch.rand(B, 9, generator=g, device=dev())
    nz = torch.randn(B, T * hop, 9, generator=g, device=dev())
    return mel, f0, ri, nz


def _arith(path, precision):
    return "simt" if path == "simt" else {"f16": "x3", "bf16": "bf16", "f16x1": "x1"}[precision]


CASES = ([("config_v1", p, "f16", T) for p in ("auto", "unfused", "simt") for T in (1, 3, 37)]
         + [("config_v1_256", p, "f16", T) for p in ("auto", "unfused", "simt") for T in (1, 5, 128)]
         + [("config_v1_256", "auto", pr, T) for pr in ("bf16", "f16x1") for T in (1, 5, 128)]
         + [("small", p, "f16", T) for p in ("auto", "simt") for T in (1, 24, 77)]
         + [("resblock2", p, "f16", T) for p in ("auto", "simt") for T in (1, 40)])

def _check_path(cap, want):
    print("  path: " + " ".join("/".join(str(x) for x in s) for s in cap.seq))
    if cap.seq != want:
        n = next((i for i, (a, b) in enumerate(zip(cap.seq, want)) if a != b), min(len(cap.seq), len(want)))
        got = cap.seq[n] if n < len(cap.seq) else None
        cap.bad.append(f"path: launch {n} is {got}, expected {want[n] if n < len(want) else None}")


@pytest.mark.parametrize("name,path,precision,T", CASES)
def test_generator_launches_vs_float64(golden, golden_cfg, monkeypatch, name, path, precision, T):
    h, sd = _config(name, golden, golden_cfg)
    gen = _generator(h, sd, path, precision, monkeypatch)
    B = 3
    mel, f0, ri, nz = _inputs(h, B, T, seed=T + 100)
    arith = _arith(path, precision)
    cap = Capture(gen, Windows(B), arith)
    print(f"\n{name} path={path} precision={precision} B={B} T={T}")
    with monkeypatch.context() as mp:
        cap.install(mp)
        wav = gen(mel, f0, rand_ini=ri, sine_noise=nz)
    torch.cuda.synchronize()
    _check_path(cap, expected_launches(h, path))
    if name.startswith("config_v1") and path != "simt":
        assert all(s[3] == "tc" for s in cap.seq if s[0] == "conv"), "a shipped config left the tensor cores"
    # the wiring: each stage boundary against the float64 chain run from the mel (the kernel's own excitation)
    ch = R.generator_chain(gen, mel, cap.har)
    tol = TOL[arith]["chain"]
    bound = [(f"ups[{i}] input", got, ch["ups_in"][i]) for i, got in enumerate(cap.bound["ups_in"])]
    bound += [("conv_post input", cap.bound["post_in"], ch["post_in"]), ("wav", cap.bound["wav"], ch["wav"])]
    for what, got, ref in bound:
        reg = Regions(ref.shape[1], 8, "cpu")
        reg.add(got, ref)
        cap.bad += reg.check(f"chain {what}", tol)
    assert torch.equal(cap.bound["wav"], wav.to(F64).cpu().reshape(B, -1, 1))
    assert not cap.bad, "\n".join(cap.bad)


def test_generator_launches_production_shape_windows(monkeypatch):
    """config_v1 at B = 32 x T = 4000 (2 048 000 samples per item), auto path: every launch judged on windows of items 0,
    15 and 31 (start, middle, end) and around the row where the flat byte offset of its output crosses 2^31 -- in the
    C = 16 planes [2, 32, 2 048 000, 16] that is item 0, row 1 572 864 of the lo plane."""
    with open(os.path.join(GOLDEN, "nsf_configs", "config_v1.json")) as f:
        h = json.load(f)
    gen = _generator(h, ovoc.make_generator_weights(43, h), "auto", "f16", monkeypatch)
    B, T = 32, 4000
    mel, f0, ri, nz = _inputs(h, B, T, seed=7)
    planes16 = torch.empty((2, B, T * 512, 16), dtype=torch.int16, device="meta")
    assert crossing(planes16, 16) == [(0, 1572864)]
    cap = Capture(gen, Windows(B, items=(0, 15, 31), width=1024), "x3")
    with monkeypatch.context() as mp:
        cap.install(mp)
        wav = gen(mel, f0, rand_ini=ri, sine_noise=nz)
    torch.cuda.synchronize()
    del nz
    _check_path(cap, expected_launches(h, "auto"))
    assert wav.shape == (B, 1, T * 512) and bool(torch.isfinite(wav).all())
    assert not cap.bad, "\n".join(cap.bad)
