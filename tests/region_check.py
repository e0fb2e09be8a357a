"""Error reports of the float64 block and stage tests (test_gpu_wavenet_block.py, test_gpu_wavenet_block_bwd.py,
test_gpu_voc_stages.py): plane values in float64, and errors per row region of a [B, T, n] tensor or per named part of
a weight gradient, since an error confined to a few rows or to one tap's columns vanishes in a whole-tensor rel-L2.
"max" is max|err| in units of the whole tensor's RMS."""
import math

import torch

from fish_diffusion_b200 import _native as N

F64 = torch.float64


def pf64(planes, pc, hi_only=False):
    """split planes int16 [2, ...] -> float64 hi + lo (or hi alone), on the planes' device"""
    dt = torch.float16 if pc == N.PREC_F16 else torch.bfloat16
    hi = planes[0].view(dt).to(F64)
    return hi if hi_only else hi + planes[1].view(dt).to(F64)


class Regions:
    """Per-row-region error accumulation over item chunks: rows [0, dil), [T-dil, T), the last tile (128 rows unless
    `tile` says otherwise), the rest; with `phase` = P > 1 also each residue class t mod P (a polyphase phase of an
    upsample, a fold sub-step of a time-folded conv), named f"{phase_name}{r}".  add() takes row windows [t0, t0 + n)
    of the items, so a few windows of a long tensor are judged by the same regions."""

    def __init__(self, T, dil, device, tile=128, phase=1, phase_name="r"):
        self.T, self.dil, self.tile, self.phase, self.phase_name = T, dil, tile, phase, phase_name
        names = ["all", "lo_edge", "hi_edge", "last_tile", "interior"]
        if phase > 1:
            names += [f"{phase_name}{r}" for r in range(phase)]
        self.se = {k: 0.0 for k in names}
        self.sr = {k: 0.0 for k in names}
        self.mx = {k: 0.0 for k in names}
        self.n_all = 0

    def _masks(self, t):
        T, dil = self.T, self.dil
        lo, hi, last = t < dil, t >= T - dil, t >= (T - 1) // self.tile * self.tile
        masks = {"all": torch.ones_like(lo), "lo_edge": lo, "hi_edge": hi, "last_tile": last,
                 "interior": ~(lo | hi | last)}
        if self.phase > 1:
            for r in range(self.phase):
                masks[f"{self.phase_name}{r}"] = t % self.phase == r
        return masks

    def add(self, got, ref, t0=0):
        """got / ref [b, n, c] float64: rows [t0, t0 + n) of b items"""
        e = got - ref
        for k, m in self._masks(torch.arange(t0, t0 + ref.shape[1], device=ref.device)).items():
            if not bool(m.any()):
                continue
            em, rm = e[:, m], ref[:, m]
            self.se[k] += float((em * em).sum())
            self.sr[k] += float((rm * rm).sum())
            self.mx[k] = max(self.mx[k], float(em.abs().max()))
        self.n_all += ref.numel()

    def check(self, what, tol):
        rtol, mtol = tol
        rms = math.sqrt(self.sr["all"] / max(self.n_all, 1))
        msgs, bad = [], []
        for k in self.se:
            if self.sr[k] == 0.0 and self.se[k] == 0.0:
                continue
            rel = math.sqrt(self.se[k] / max(self.sr[k], 1e-300))
            mx = self.mx[k] / max(rms, 1e-300)
            msgs.append(f"{k} {rel:.2e}/{mx:.2e}")
            if not (rel < rtol and mx < mtol):
                bad.append(f"{k}: rel-L2 {rel:.2e} (bar {rtol:.1e}), max {mx:.2e} (bar {mtol:.1e})")
        print(f"  {what}: " + ", ".join(msgs))
        return [f"{what} {x}" for x in bad]


def check_parts(what, got, ref, parts, tol, exact_zero=True):
    """Like Regions.check for a tensor cut into named parts (index expressions into got / ref): rel-L2 of each part and
    its max|err| in units of the whole tensor's RMS.  A part whose reference is exactly zero must be exactly zero, or
    (exact_zero False) is judged by its max alone."""
    rtol, mtol = tol
    rms = max(float(ref.pow(2).mean().sqrt()), 1e-300)
    msgs, bad = [], []
    for k, ix in {"all": (...,), **parts}.items():
        e, r = got[ix] - ref[ix], ref[ix]
        se, sr = float(e.pow(2).sum()), float(r.pow(2).sum())
        if sr == 0.0 and se == 0.0:
            msgs.append(f"{k} exact 0")
            continue
        rel = math.sqrt(se / max(sr, 1e-300))
        mx = float(e.abs().max()) / rms
        if sr == 0.0 and not exact_zero:
            rel = 0.0
            msgs.append(f"{k} (zero reference) max {mx:.2e}")
        else:
            msgs.append(f"{k} {rel:.2e}/{mx:.2e}")
        if not (rel < rtol and mx < mtol):
            bad.append(f"{k}: rel-L2 {rel:.2e} (bar {rtol:.1e}), max {mx:.2e} (bar {mtol:.1e})")
    print(f"  {what}: " + ", ".join(msgs))
    return [f"{what} {x}" for x in bad]
