"""H100-native GaussianDiffusion + noise predictors: drop-in for the reference
``fish_diffusion/archs/diffsinger/diffusions/{diffusion,noise_predictor}.py``.

Same constructor, buffers (state_dict keys), attributes and ``forward`` / ``train_step`` contracts
(diffusion.py:48-118,172-313; SURVEY.md section 8b), registered as ``DIFFUSIONS["GaussianDiffusion"]``.
The sampler state lives channels-last on the device for the whole loop; the conditioner is split once per call (and,
with three GEMM products where it fits, projected for every layer once per call); every update (DDPM posterior step,
PLMS / UniPC linear combinations, norm/denorm) is one fused native kernel.
Scalar coefficient math stays on the host exactly like the reference's float32 buffers.
"""
from __future__ import annotations

import json
from functools import partial

import numpy as np
import torch
from torch import nn

from . import _native as N
from .registry import DENOISERS, DIFFUSIONS
from .uni_pc import NoiseScheduleVP, unipc_sample_native


def get_noise_schedule_list(schedule_mode, timesteps, max_beta=0.01, s=0.008):
    """float64 numpy schedule, same formulas as the reference (diffusion.py:18-31)."""
    if schedule_mode == "linear":
        schedule_list = np.linspace(1e-4, max_beta, timesteps)
    elif schedule_mode == "cosine":
        steps = timesteps + 1
        x = np.linspace(0, steps, steps)
        alphas_cumprod = np.cos(((x / steps) + s) / (1 + s) * np.pi * 0.5) ** 2
        alphas_cumprod = alphas_cumprod / alphas_cumprod[0]
        betas = 1 - (alphas_cumprod[1:] / alphas_cumprod[:-1])
        schedule_list = np.clip(betas, a_min=0, a_max=0.999)
    else:
        raise NotImplementedError
    return schedule_list


to_torch = partial(torch.tensor, dtype=torch.float32)


def hoist_cond_proj(denoiser, B: int, T: int, device) -> bool:
    """Whether a sampler call keeps the conditioner projection of all layers resident and computes it once instead of
    inside every GEMM1 launch.  Only with three tensor-core products: there the projection is a seventh of GEMM1's MMA
    work; single-product GEMM1 gains less than the fp32 projection costs to read (at B=32, T=4000 the f16x1 sampler ran
    3.34 s hoisted against 3.23 s fused, DESIGN.md section 5).  And only when the buffer takes at most a quarter of the
    card's total memory (not of the free memory, which other processes on a shared GPU change from run to run), so a
    given shape takes the same path every time."""
    if N.mma_code(denoiser.precision) & N.PREC_SINGLE:
        return False
    nbytes = 4 * int(np.prod(denoiser.cond_proj_shape(B, T)))
    return nbytes <= torch.cuda.mem_get_info(device)[1] // 4


class NaiveNoisePredictor(nn.Module):
    """Buffers of the reference NaiveNoisePredictor (noise_predictor.py:19-71); the update itself is the fused
    kernel fd_ddpm_step."""

    def __init__(self, betas, clip_min=-1.0, clip_max=1.0):
        super().__init__()
        alphas = 1.0 - betas
        alphas_cumprod = np.cumprod(alphas, axis=0)
        alphas_cumprod_prev = np.append(1.0, alphas_cumprod[:-1])
        self.register_buffer("clip_min", to_torch(clip_min))
        self.register_buffer("clip_max", to_torch(clip_max))
        self.register_buffer("alphas_cumprod_prev", to_torch(alphas_cumprod_prev))
        self.register_buffer("log_one_minus_alphas_cumprod", to_torch(np.log(1.0 - alphas_cumprod)))
        self.register_buffer("sqrt_recip_alphas_cumprod", to_torch(np.sqrt(1.0 / alphas_cumprod)))
        self.register_buffer("sqrt_recipm1_alphas_cumprod", to_torch(np.sqrt(1.0 / alphas_cumprod - 1)))
        posterior_variance = betas * (1.0 - alphas_cumprod_prev) / (1.0 - alphas_cumprod)
        self.register_buffer("posterior_variance", to_torch(posterior_variance))
        self.register_buffer("posterior_log_variance_clipped", to_torch(np.log(np.maximum(posterior_variance, 1e-20))))
        self.register_buffer("posterior_mean_coef1",
                             to_torch(betas * np.sqrt(alphas_cumprod_prev) / (1.0 - alphas_cumprod)))
        self.register_buffer("posterior_mean_coef2",
                             to_torch((1.0 - alphas_cumprod_prev) * np.sqrt(alphas) / (1.0 - alphas_cumprod)))
        self._host = None

    def host_tables(self):
        """float32 host copies (read once; the per-step scalars are kernel arguments, no device sync per step)."""
        if self._host is None:
            self._host = {k: v.detach().cpu().numpy() for k, v in self.state_dict().items()}
        return self._host

    def _load_from_state_dict(self, *a, **k):
        self._host = None
        return super()._load_from_state_dict(*a, **k)

    def step_cl(self, x, t: int, eps, noise=None, x_planes=None, prec=N.PREC_F16, seed=0, offset=0, subseq0=0):
        """x' = NaiveNoisePredictor.forward(x, t, eps) (noise_predictor.py:73-104) on fp32 tensors of any layout
        (elementwise); in place on x.  `noise` None -> in-kernel Philox."""
        h = self.host_tables()
        sigma = float(np.exp(np.float32(0.5) * h["posterior_log_variance_clipped"][t])) if t > 0 else 0.0
        N.check(N.lib().fd_ddpm_step(
            N.ptr(x), N.ptr(eps), N.ptr(noise), N.ptr(x), N.ptr(x_planes), x.numel(),
            float(h["sqrt_recip_alphas_cumprod"][t]), float(h["sqrt_recipm1_alphas_cumprod"][t]),
            float(h["posterior_mean_coef1"][t]), float(h["posterior_mean_coef2"][t]), sigma,
            float(h["clip_min"]), float(h["clip_max"]), seed, offset, subseq0, prec, N.stream_ptr(x.device)),
            "fd_ddpm_step")
        return x


class PLMSNoisePredictor(nn.Module):
    """Buffer of the reference PLMSNoisePredictor (noise_predictor.py:107-116); updates are fd_lincomb calls."""

    def __init__(self, betas):
        super().__init__()
        alphas = 1.0 - betas
        self.register_buffer("alphas_cumprod", to_torch(np.cumprod(alphas, axis=0)))
        self._host = None

    def host_table(self):
        if self._host is None:
            self._host = self.alphas_cumprod.detach().cpu().numpy()
        return self._host

    def _load_from_state_dict(self, *a, **k):
        self._host = None
        return super()._load_from_state_dict(*a, **k)

    def coefs(self, t: int, t_prev: int):
        """(cx, cn) with x_pred = cx * x + cn * noise  -- noise_predictor.py:118-131 in float32 scalars."""
        ac = self.host_table()
        f = np.float32
        a_t, a_prev = f(ac[t]), f(ac[t_prev])
        a_t_sq, a_prev_sq = np.sqrt(a_t), np.sqrt(a_prev)
        d = f(a_prev - a_t)
        cx = f(1) + d * (f(1) / (a_t_sq * (a_t_sq + a_prev_sq)))
        cn = -d * (f(1) / (a_t_sq * (np.sqrt((f(1) - a_prev) * a_t) + np.sqrt((f(1) - a_t) * a_prev))))
        return float(cx), float(cn)


class UNIPCNoisePredictor(nn.Module):
    """Holds the discrete VP schedule like the reference (noise_predictor.py:151-158); no buffers."""

    def __init__(self, betas, condition_key="conditioner"):
        super().__init__()
        self.noise_schedule = NoiseScheduleVP(betas)
        self.condition_key = condition_key


def lincomb(out, terms, planes=None, prec=N.PREC_F16):
    """out = sum coef_i * tensor_i (fd_lincomb); terms = [(coef, tensor), ...], tensors may alias out."""
    import ctypes
    n = len(terms)
    ptrs = (ctypes.c_void_p * n)(*[t.data_ptr() for _, t in terms])
    coefs = (ctypes.c_float * n)(*[float(c) for c, _ in terms])
    ref = terms[0][1]
    N.check(N.lib().fd_lincomb(N.ptr(out), N.ptr(planes), ptrs, coefs, n, ref.numel(), prec,
                               N.stream_ptr(ref.device)), "fd_lincomb")
    return out


@DIFFUSIONS.register_module(name="GaussianDiffusion", force=True)
class GaussianDiffusion(nn.Module):
    def __init__(self, denoiser, mel_channels=128, noise_schedule="linear", timesteps=1000, max_beta=0.01, s=0.008,
                 noise_loss="l1", sampler_interval=10, spec_stats_path="dataset/stats.json", spec_min=None,
                 spec_max=None, noise_predictor=None):
        super().__init__()
        self.denoise_fn = denoiser if isinstance(denoiser, nn.Module) else DENOISERS.build(denoiser)
        self.mel_bins = mel_channels
        betas = get_noise_schedule_list(noise_schedule, timesteps, max_beta, s)
        alphas = 1.0 - betas
        alphas_cumprod = np.cumprod(alphas, axis=0)
        (timesteps,) = betas.shape
        self.num_timesteps = int(timesteps)
        self.noise_loss = noise_loss
        self.register_buffer("betas", to_torch(betas))
        self.register_buffer("alphas_cumprod", to_torch(alphas_cumprod))
        self.register_buffer("sqrt_alphas_cumprod", to_torch(np.sqrt(alphas_cumprod)))
        self.register_buffer("sqrt_one_minus_alphas_cumprod", to_torch(np.sqrt(1.0 - alphas_cumprod)))
        assert (spec_min is None and spec_max is None) or (spec_min is not None and spec_max is not None), \
            "spec_min and spec_max must be both None or both not None"
        if spec_min is None:
            with open(spec_stats_path) as f:
                stats = json.load(f)
            spec_min, spec_max = stats["spec_min"], stats["spec_max"]
        assert len(spec_min) == len(spec_max) == mel_channels or len(spec_min) == len(spec_max) == 1, \
            "spec_min and spec_max must be either of length 1 or mel_channels"
        self.register_buffer("spec_min", torch.FloatTensor(spec_min).view(1, 1, -1))
        self.register_buffer("spec_max", torch.FloatTensor(spec_max).view(1, 1, -1))
        self.sampler_interval = sampler_interval
        self.naive_noise_predictor = NaiveNoisePredictor(betas=betas)
        self.plms_noise_predictor = PLMSNoisePredictor(betas=betas)
        self.unipc_noise_predictor = UNIPCNoisePredictor(betas=betas)
        if noise_predictor is None:
            noise_predictor = "naive" if sampler_interval == 1 else "unipc"
        self.noise_predictor = noise_predictor
        self._philox_calls = 0

    # ------------------------------------------------------------------------------------ helpers
    def _prec(self):
        return N.prec_code(getattr(self.denoise_fn, "precision", "f16"))

    def _affine(self, x_cl, inverse: bool):
        """norm_spec / denorm_spec (diffusion.py:315-319) over channels-last [B,T,M] as y = x*scale + shift."""
        smin = self.spec_min.reshape(-1).to(torch.float32)
        smax = self.spec_max.reshape(-1).to(torch.float32)
        if inverse:   # (x + 1) / 2 * (max - min) + min
            scale = (smax - smin) / 2
            shift = scale + smin
        else:         # (x - min) / (max - min) * 2 - 1
            scale = 2 / (smax - smin)
            shift = -smin * scale - 1
        scale, shift = scale.contiguous(), shift.contiguous()
        y = torch.empty_like(x_cl)
        B, T, M = x_cl.shape
        N.check(N.lib().fd_affine_cl(N.ptr(x_cl.contiguous()), N.ptr(y), N.ptr(scale), N.ptr(shift), scale.numel(),
                                     B * T, M, N.stream_ptr(x_cl.device)), "fd_affine_cl")
        return y

    def norm_spec(self, x):
        return self._affine(x, inverse=False)

    def denorm_spec(self, x):
        return self._affine(x, inverse=True)

    def _rng_seed(self):
        """Philox key of the current call.  An explicit `seed=` wins; otherwise ONE int64 is drawn from torch's default
        (CPU) generator at the start of every sampler / train_step call (`_begin_call`), so `torch.manual_seed(s)`
        followed by the same calls reproduces the same outputs (as it does for the reference's torch.randn draws), two
        consecutive calls differ, and a resumed run continues from the restored generator state.  Ranks that share a
        torch seed draw the same key; their items are told apart by the global element index (first_item)."""
        s = getattr(self, "_seed_override", None)
        if s is None:
            s = getattr(self, "_call_seed", None)
        if s is None:
            s = self._begin_call()
        return int(s) & (2 ** 63 - 1)

    def _begin_call(self):
        self._call_seed = int(torch.randint(0, 2 ** 62, (1,), dtype=torch.int64).item())
        self._philox_calls = 0
        return self._call_seed

    def _sampler_ws(self, dev, B, T, M, E):
        key = (str(dev), B, T, M, E)
        ws = getattr(self, "_sws", None)
        if ws is None or ws["key"] != key:
            ws = {"key": key, "x": torch.empty((B, T, M), dtype=torch.float32, device=dev),
                  "eps": torch.empty((B, T, M), dtype=torch.float32, device=dev),
                  "x_planes": torch.empty((2, B, T, M), dtype=torch.int16, device=dev),
                  "cond_planes": torch.empty((2, B, T, E), dtype=torch.int16, device=dev)}
            self._sws = ws
        return ws

    def _randn(self, shape, device, out=None):
        if out is None:
            out = torch.empty(shape, dtype=torch.float32, device=device)
        self._philox_calls += 1
        N.check(N.lib().fd_randn(N.ptr(out), out.numel(), self._rng_seed(), self._philox_calls << 20,
                                 getattr(self, "_subseq0", 0), N.stream_ptr(device)), "fd_randn")
        return out

    @staticmethod
    def _to_cl(t_bmt):
        """[B,M,T] tensor (the reference's layout for injected noise / x_T) -> contiguous channels-last [B,T,M]."""
        B, M, T = t_bmt.shape
        t_bmt = t_bmt.to(torch.float32).contiguous()
        out = torch.empty((B, T, M), dtype=torch.float32, device=t_bmt.device)
        N.check(N.lib().fd_transpose_ncw_to_nwc(N.ptr(t_bmt), N.ptr(out), B, M, T, N.stream_ptr(t_bmt.device)),
                "fd_transpose_ncw_to_nwc")
        return out

    def q_sample(self, x_start, t, noise=None):
        """diffusion.py:120-127 on any layout with batch leading; t int64 [B] or [1]."""
        if noise is None:
            noise = self._randn(tuple(x_start.shape), x_start.device)
        B = x_start.shape[0]
        t = t.reshape(-1).to(x_start.device)
        if t.numel() == 1:
            t = t.expand(B)
        a = self.sqrt_alphas_cumprod.gather(-1, t).contiguous()
        s = self.sqrt_one_minus_alphas_cumprod.gather(-1, t).contiguous()
        x_start, noise = x_start.contiguous(), noise.contiguous()
        y = torch.empty_like(x_start)
        N.check(N.lib().fd_q_sample(N.ptr(x_start), N.ptr(noise), N.ptr(a), N.ptr(s), N.ptr(y), B,
                                    x_start.numel() // B, N.stream_ptr(x_start.device)), "fd_q_sample")
        return y

    # ------------------------------------------------------------------------------------ training step
    def get_mel_loss(self, loss_fn, noise, epsilon):
        import torch.nn.functional as F
        if isinstance(loss_fn, list):
            return sum(self.get_mel_loss(fn, noise, epsilon) * weight for weight, fn in loss_fn)
        if loss_fn == "l1":
            return F.l1_loss(noise, epsilon)
        if loss_fn == "smoothed-l1":
            return F.smooth_l1_loss(noise, epsilon)
        if loss_fn == "l2":
            return F.mse_loss(noise, epsilon)
        if callable(loss_fn):
            return loss_fn(noise, epsilon)
        raise NotImplementedError()

    def train_step(self, features, mel, x_masks=None, cond_masks=None, t=None, noise=None):
        """Reference train_step / p_losses (diffusion.py:129-190): t ~ U{0..N-1}[B], x_t = q_sample(norm_spec(mel)),
        eps = denoise_fn(x_t, t, cond) (no masks, SURVEY.md D10), masked loss.  `t` / `noise` ([B,M,T]) may be
        injected for parity tests.  With grad enabled the loss carries the autograd graph through the native
        forward/backward kernels (WaveNetTrainFn); under no_grad only the forward runs."""
        B, T, E = features.shape
        dev = features.device
        prec = self._prec()
        self._subseq0 = 0
        self._begin_call()
        if t is None:
            t = torch.randint(0, self.num_timesteps, (B,), device=dev).long()
        with torch.no_grad():
            x = self.norm_spec(mel.to(torch.float32))                   # [B,T,M] channels-last
            noise_cl = self._randn(tuple(x.shape), dev) if noise is None else self._to_cl(noise)
            noised = self.q_sample(x, t, noise_cl)
        if torch.is_grad_enabled():
            eps = self.denoise_fn.forward_train_cl(noised, t.to(torch.float32), features.to(torch.float32))
        else:
            cond_planes = N.split_nwc(features.to(torch.float32), prec)
            eps = self.denoise_fn.forward_cl(N.split_nwc(noised, prec), t.to(torch.float32), cond_planes)
        if x_masks is not None:
            m = x_masks[:, :, None]
            noised = noised.masked_fill(m, 0.0)
            eps = eps.masked_fill(m, 0.0)
        loss = self.get_mel_loss(self.noise_loss, noise_cl, eps)
        return dict(loss=loss, noised_mels=noised, epsilon=eps, t=t)

    # ------------------------------------------------------------------------------------ sampling
    @torch.no_grad()
    def forward(self, features, sampler_interval=None, progress: bool = False, skip_steps: int = 0,
                original_mel: torch.Tensor = None, noise_predictor: str = None, x_masks: torch.Tensor = None,
                cond_masks: torch.Tensor = None, x_T: torch.Tensor = None, step_noises=None, seed: int = None,
                first_item: int = 0, cond_planes: torch.Tensor = None):
        """Reference contract (diffusion.py:196-313): features [B,T,E] -> mel [B,T,M].
        Extra (parity tests): x_T [B,M,T] replaces the initial randn / the q_sample noise of shallow diffusion,
        step_noises[i] [B,M,T] replaces the i-th randn_like of the naive predictor.
        first_item: index of features[0] inside the global batch.  The in-kernel Philox draws are indexed by the
        global element (SURVEY.md section 8e), so with the same `seed` a batch sharded over ranks / split into calls of
        the same T reproduces the unsharded result bit for bit.
        cond_planes: the conditioner already as split planes [2,B,T,E] (DiffSinger.conditioner_planes: the feature
        projections written straight into the sampler's plane buffer by one GEMM); `features` may then be None and
        `cond_masks` must already have been applied."""
        if seed is not None:
            # reproducible call: Philox streams are (seed, draw index within this call) instead of the running counter
            self._seed_override, self._philox_calls = int(seed), 0
            try:
                return self.forward(features, sampler_interval, progress, skip_steps, original_mel, noise_predictor,
                                    x_masks, cond_masks, x_T, step_noises, None, first_item, cond_planes)
            finally:
                self._seed_override = None
        if getattr(self, "_seed_override", None) is None:
            self._begin_call()
        if sampler_interval is None:
            sampler_interval = self.sampler_interval
        if noise_predictor is None:
            noise_predictor = self.noise_predictor
        noise_predictor = noise_predictor.lower()
        if noise_predictor not in ("naive", "unipc", "plms"):
            raise NotImplementedError(f"Unknown noise predictor: {noise_predictor}")
        N.require_cuda(features if cond_planes is None else cond_planes, "features")
        dev = (features if cond_planes is None else cond_planes).device
        den = self.denoise_fn
        prec = self._prec()
        B, T, E = features.shape if cond_planes is None else tuple(cond_planes.shape[1:])
        M = self.mel_bins
        self._subseq0 = int(first_item) * ((T * M + 3) // 4)      # first Philox subsequence (one per 4 elements)
        cmask = None if cond_masks is None else cond_masks.to(torch.uint8).contiguous()
        # per-shape work buffers are kept between calls: stable pointers let the denoiser replay its captured CUDA
        # graph from the first evaluation of every later call (one in-flight sampler call per module instance)
        ws = self._sampler_ws(dev, B, T, M, E)
        if cond_planes is None:
            cond_planes = N.split_nwc(features.to(torch.float32), prec, mask=cmask, out=ws["cond_planes"])   # once per call
        elif cond_planes.data_ptr() != ws["cond_planes"].data_ptr():
            ws["cond_planes"].copy_(cond_planes)
            cond_planes = ws["cond_planes"]
        # every evaluation of this call sees the same conditioner: its projection (all layers) is computed here, once
        # per call and under the current weights, and GEMM1 then sums the conv taps only
        cond_proj = None
        if hoist_cond_proj(den, B, T, dev):
            shape = den.cond_proj_shape(B, T)
            if ws.get("cond_proj") is None or tuple(ws["cond_proj"].shape) != shape:
                ws["cond_proj"] = torch.empty(shape, dtype=torch.float32, device=dev)
            cond_proj = den.cond_projection(cond_planes, ws["cond_proj"])
        else:
            ws["cond_proj"] = None
        if original_mel is None:
            x = self._to_cl(x_T) if x_T is not None else self._randn((B, T, M), dev, out=ws["x"])
        else:
            # the reference passes original_mel as [B,M,T]-normalisable; it is normalised then used as x [B,M,T]
            # the reference's own callers hand original_mel over as [B, M, T] (tools/diffusion/inference.py: the mel is
            # transposed before the call); [B, T, M] is accepted only when the shape is unambiguous
            om = original_mel.to(torch.float32)
            x = self.norm_spec(self._to_cl(om) if om.shape[1] == M and (om.shape[2] == T or M != T) else om)
        if skip_steps:
            t0 = torch.tensor([self.num_timesteps - skip_steps], device=dev, dtype=torch.long)
            qn = self._to_cl(x_T) if (x_T is not None and original_mel is not None) else None
            x = self.q_sample(x_start=x, t=t0, noise=qn)
        x = x.contiguous()
        if x.data_ptr() != ws["x"].data_ptr():
            ws["x"].copy_(x)
            x = ws["x"]
        x_planes = ws["x_planes"]
        N.split_nwc(x, prec, out=x_planes)
        chunks = torch.arange(0, self.num_timesteps - skip_steps, sampler_interval, dtype=torch.long).flip(0).tolist()
        it = chunks
        if progress and noise_predictor in ("naive", "plms"):
            from tqdm import tqdm
            it = tqdm(chunks)
        eps = ws["eps"]
        seed = self._rng_seed()
        # converted once per call: the denoiser replays a captured CUDA graph when it sees the same buffers again
        if x_masks is not None:
            x_masks = x_masks.to(device=dev, dtype=torch.uint8).contiguous()
        step_table = {}      # diffusion step (float) -> 1-element device tensor, uploaded once per sampler call

        def denoise(xp, t_float, masks=True, out=eps):
            steps = step_table.get(t_float)
            if steps is None:
                steps = step_table[t_float] = torch.tensor([t_float], dtype=torch.float32, device=dev)
            return den.forward_cl(xp, steps, cond_planes, x_mask=x_masks if masks else None, out=out,
                                  cond_proj=cond_proj)

        if noise_predictor in ("naive", "plms") and len(chunks) > 1:   # one upload for the whole schedule
            tab = torch.tensor([float(t) for t in chunks], dtype=torch.float32, device=dev)
            for i, t in enumerate(chunks):
                step_table[float(t)] = tab[i:i + 1]

        if noise_predictor == "naive":
            for i, t in enumerate(it):
                denoise(x_planes, float(t))
                nz = None if step_noises is None else self._to_cl(step_noises[i])
                self._philox_calls += 1
                self.naive_noise_predictor.step_cl(x, int(t), eps, noise=nz, x_planes=x_planes, prec=prec, seed=seed,
                                                   offset=self._philox_calls << 20, subseq0=self._subseq0)
            return self.denorm_spec(x)

        if noise_predictor == "unipc":
            x = unipc_sample_native(self.unipc_noise_predictor.noise_schedule, x, x_planes,
                                    lambda xp, t_in, out: denoise(xp, t_in, out=out), sampler_interval, prec,
                                    progress=progress)
            return self.denorm_spec(x)

        # ---- PLMS (diffusion.py:269-311, credit OpenVPI in the reference)
        plms = self.plms_noise_predictor
        stage = 0
        hist = []                                       # previous eps tensors, newest last
        x_pred = torch.empty_like(x)
        xp_planes = torch.empty_like(x_planes)
        prime = torch.empty_like(x)
        for t in it:
            cur = torch.empty_like(x)
            denoise(x_planes, float(t), out=cur)
            t_prev = t - sampler_interval
            t_prev = t_prev * (t_prev > 0)
            cx, cn = plms.coefs(int(t), int(t_prev))
            if stage == 0:
                lincomb(x_pred, [(cx, x), (cn, cur)], planes=xp_planes, prec=prec)
                prev = torch.empty_like(x)
                denoise(xp_planes, float(t_prev), masks=False, out=prev)     # no masks here (diffusion.py:285)
                lincomb(prime, [(0.5, cur), (0.5, prev)])
            elif stage == 1:
                lincomb(prime, [(1.5, cur), (-0.5, hist[-1])])
            elif stage == 2:
                lincomb(prime, [(23 / 12, cur), (-16 / 12, hist[-1]), (5 / 12, hist[-2])])
            else:
                lincomb(prime, [(55 / 24, cur), (-59 / 24, hist[-1]), (37 / 24, hist[-2]), (-9 / 24, hist[-3])])
            if stage < 3:
                hist.append(cur)
                stage += 1
            else:
                hist = hist[-2:] + [cur]
            lincomb(x, [(cx, x), (cn, prime)], planes=x_planes, prec=prec)
        return self.denorm_spec(x)
