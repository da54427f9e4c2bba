"""Drop-in for ``modules.diff.shallow_diffusion_tts.GaussianDiffusion``.

Reference: /root/reference/NeuralSeq/modules/diff/shallow_diffusion_tts.py:71-289
(identical p_sample in modules/diff/diffusion.py:264-271).  Kept: constructor
signature, buffer names (:103-126), ``p_sample`` / ``p_sample_plms`` / ``q_sample`` /
``norm_spec`` / ``denorm_spec`` / ``forward(..., infer=True)`` signatures, the module-level
``noise_like`` hook, the ``denoise_fn(x, t, cond=cond)`` call convention and the
``denoise_fn.*`` / ``fs2.*`` state-dict prefixes.

The epsilon network and every elementwise update run in libagpt_b200.so; the schedule
tables are computed exactly as the reference does (numpy float64, cast to fp32).
Training (``p_losses``) is out of scope.  One documented extension: ``p_sample_plms``
uses clamp_min(0) semantics for ``t - interval`` so that it also works for B > 1 (the
reference's Python ``max`` on a tensor only works for B == 1; SURVEY.md 8a-12).
"""
from __future__ import annotations

import ctypes as C
from collections import deque

import numpy as np
import torch
from torch import nn

from ... import _lib
from ...utils import hparams as _hp


def noise_like(shape, device, repeat=False):
    if repeat:
        n = torch.randn((1, *shape[1:]), device=device)
        return n.repeat(shape[0], *((1,) * (len(shape) - 1)))
    return torch.randn(shape, device=device)


def linear_beta_schedule(timesteps, max_beta=None):
    if max_beta is None:
        max_beta = _hp.resolve().get("max_beta", 0.01)
    return np.linspace(1e-4, max_beta, timesteps)


def cosine_beta_schedule(timesteps, s=0.008):
    steps = timesteps + 1
    x = np.linspace(0, steps, steps)
    ac = np.cos(((x / steps) + s) / (1 + s) * np.pi * 0.5) ** 2
    ac = ac / ac[0]
    return np.clip(1 - (ac[1:] / ac[:-1]), a_min=0, a_max=0.999)


beta_schedule = {"cosine": cosine_beta_schedule, "linear": linear_beta_schedule}


def _fs2_factory(phone_encoder, out_dims, use_midi):
    """The acoustic front-end is outside the accelerated path (SURVEY.md 8f-4); reuse the
    reference's FastSpeech2 when its package is importable, otherwise leave it unset."""
    if phone_encoder is None:
        return None
    try:
        if use_midi:
            from modules.diffsinger_midi.fs2 import FastSpeech2MIDI as F
        else:
            from modules.fastspeech.fs2 import FastSpeech2 as F
    except Exception:
        return None
    return F(phone_encoder, out_dims)


class GaussianDiffusion(nn.Module):
    def __init__(self, phone_encoder, out_dims, denoise_fn, timesteps=1000, K_step=1000,
                 loss_type=None, betas=None, spec_min=None, spec_max=None):
        super().__init__()
        hp = _hp.resolve()
        self.denoise_fn = denoise_fn
        fs2 = _fs2_factory(phone_encoder, out_dims, bool(hp.get("use_midi")))
        if fs2 is not None:
            self.fs2 = fs2
        self.mel_bins = out_dims
        if betas is not None:
            betas = betas.detach().cpu().numpy() if isinstance(betas, torch.Tensor) else np.asarray(betas)
        elif "schedule_type" in hp:
            betas = beta_schedule[hp["schedule_type"]](timesteps)
        else:
            betas = cosine_beta_schedule(timesteps)
        betas = np.asarray(betas, dtype=np.float64)
        alphas = 1.0 - betas
        ac = np.cumprod(alphas, axis=0)
        ac_prev = np.append(1.0, ac[:-1])
        self.num_timesteps = int(betas.shape[0])
        self.K_step = K_step
        self.loss_type = loss_type if loss_type is not None else hp.get("diff_loss_type", "l1")
        self.noise_list = deque(maxlen=4)
        f32 = lambda a: torch.tensor(a, dtype=torch.float32)
        post_var = betas * (1.0 - ac_prev) / (1.0 - ac)
        for name, val in (
                ("betas", betas), ("alphas_cumprod", ac), ("alphas_cumprod_prev", ac_prev),
                ("sqrt_alphas_cumprod", np.sqrt(ac)),
                ("sqrt_one_minus_alphas_cumprod", np.sqrt(1.0 - ac)),
                ("log_one_minus_alphas_cumprod", np.log(1.0 - ac)),
                ("sqrt_recip_alphas_cumprod", np.sqrt(1.0 / ac)),
                ("sqrt_recipm1_alphas_cumprod", np.sqrt(1.0 / ac - 1)),
                ("posterior_variance", post_var),
                ("posterior_log_variance_clipped", np.log(np.maximum(post_var, 1e-20))),
                ("posterior_mean_coef1", betas * np.sqrt(ac_prev) / (1.0 - ac)),
                ("posterior_mean_coef2", (1.0 - ac_prev) * np.sqrt(alphas) / (1.0 - ac))):
            self.register_buffer(name, f32(val))
        keep = hp.get("keep_bins", out_dims)
        self.register_buffer("spec_min", torch.FloatTensor(spec_min)[None, None, :keep])
        self.register_buffer("spec_max", torch.FloatTensor(spec_max)[None, None, :keep])
        self._host = None

    # ------------------------------------------------------------------ host tables
    def _tables(self):
        """fp32 CPU copies of the buffers, for the per-step scalar gathers."""
        if self._host is None:
            g = lambda n: getattr(self, n).detach().float().cpu()
            sigma = (0.5 * g("posterior_log_variance_clipped")).exp()
            self._host = dict(A=g("sqrt_recip_alphas_cumprod"), B=g("sqrt_recipm1_alphas_cumprod"),
                              c1=g("posterior_mean_coef1"), c2=g("posterior_mean_coef2"), sigma=sigma,
                              ac=g("alphas_cumprod"))
        return self._host

    def _apply(self, fn, *a, **k):
        self._host = None
        return super()._apply(fn, *a, **k)

    @staticmethod
    def _t_list(t, b):
        if torch.is_tensor(t):
            t = t.tolist()          # device sync; the fast loop below passes Python ints instead
        elif isinstance(t, int):
            t = [t] * b
        return [int(v) for v in t]

    def _fast(self):
        from .net import DiffNet
        return isinstance(self.denoise_fn, DiffNet)

    # ------------------------------------------------------------------ reference API
    def predict_start_from_noise(self, x_t, t, noise):
        tl = self._t_list(t, x_t.shape[0])
        tb = self._tables()
        shp = (-1,) + (1,) * (x_t.dim() - 1)
        a = tb["A"][tl].to(x_t.device).reshape(shp)
        b = tb["B"][tl].to(x_t.device).reshape(shp)
        return a * x_t - b * noise

    @torch.no_grad()
    def p_sample(self, x, t, cond, clip_denoised=True, repeat_noise=False):
        b = x.shape[0]
        tl = self._t_list(t, b)
        noise = noise_like(x.shape, x.device, repeat_noise)
        return self._p_sample_core(x, tl, cond, noise, clip_denoised)

    def _p_sample_core(self, x, tl, cond, noise, clip_denoised=True):
        if not x.is_cuda:
            raise RuntimeError("audiogpt_b200.GaussianDiffusion runs on CUDA only (no CPU fallback)")
        tb = self._tables()
        b = x.shape[0]
        coef = np.empty((b, 5), dtype=np.float32)
        for i, tv in enumerate(tl):
            coef[i] = (tb["A"][tv], tb["B"][tv], tb["c1"][tv], tb["c2"][tv],
                       float(tb["sigma"][tv]) if tv != 0 else 0.0)
        x = x.contiguous().float()
        out = torch.empty_like(x)
        tt = (C.c_int * b)(*tl)
        n = x[0].numel()
        if self._fast():
            self.denoise_fn.set_cond(cond)
            h, eps = self.denoise_fn._h, None
        else:
            eps = self.denoise_fn(x, torch.tensor(tl, device=x.device, dtype=torch.long), cond=cond)
            h, eps = None, eps.contiguous().float()
        _lib.call("gd_p_sample", x.device, h, _lib.fptr(x), _lib.fptr(eps) if eps is not None else None, tt,
                  coef.ctypes.data_as(C.c_void_p), _lib.fptr(noise) if noise is not None else None,
                  1 if clip_denoised else 0, b, n, _lib.fptr(out))
        return out

    def _eps(self, x, tl, cond):
        if self._fast():
            return self.denoise_fn(x, tl, cond)
        return self.denoise_fn(x, torch.tensor(tl, device=x.device, dtype=torch.long), cond=cond).contiguous().float()

    def _axpby(self, x, es, rows):
        b = x.shape[0]
        coef = np.zeros((b, 5), dtype=np.float32)
        coef[:, :len(rows[0])] = np.asarray(rows, dtype=np.float32)
        ptrs = [_lib.fptr(e) for e in es] + [None] * (4 - len(es))
        out = torch.empty_like(x)
        _lib.call("axpby5", x.device, _lib.fptr(x), *ptrs, coef.ctypes.data_as(C.c_void_p), b, x[0].numel(), _lib.fptr(out))
        return out

    def _plms_scalars(self, tv, interval):
        """(alpha, beta) with x_pred = alpha*x + beta*eps -- get_x_pred (:174-185) in fp32 torch scalars."""
        ac = self._tables()["ac"]
        a_t = ac[tv]
        a_prev = torch.ones_like(a_t) if tv < interval else ac[max(tv - interval, 0)]
        a_t_sq, a_prev_sq = a_t.sqrt(), a_prev.sqrt()
        cx = 1 / (a_t_sq * (a_t_sq + a_prev_sq))
        ce = 1 / (a_t_sq * (((1 - a_prev) * a_t).sqrt() + ((1 - a_t) * a_prev).sqrt()))
        d = a_prev - a_t
        return float(1 + d * cx), float(-(d * ce))

    @torch.no_grad()
    def p_sample_plms(self, x, t, interval, cond, clip_denoised=True, repeat_noise=False):
        b = x.shape[0]
        tl = self._t_list(t, b)
        x = x.contiguous().float()
        ab = [self._plms_scalars(tv, interval) for tv in tl]
        hist = self.noise_list
        eps = self._eps(x, tl, cond)
        if len(hist) == 0:
            x_pred = self._axpby(x, [eps], [(a, bb) for a, bb in ab])
            eps_prev = self._eps(x_pred, [max(tv - interval, 0) for tv in tl], cond)
            out = self._axpby(x, [eps, eps_prev], [(a, bb / 2, bb / 2) for a, bb in ab])
        elif len(hist) == 1:
            out = self._axpby(x, [eps, hist[-1]], [(a, 3 * bb / 2, -bb / 2) for a, bb in ab])
        elif len(hist) == 2:
            out = self._axpby(x, [eps, hist[-1], hist[-2]],
                              [(a, 23 * bb / 12, -16 * bb / 12, 5 * bb / 12) for a, bb in ab])
        else:
            out = self._axpby(x, [eps, hist[-1], hist[-2], hist[-3]],
                              [(a, 55 * bb / 24, -59 * bb / 24, 37 * bb / 24, -9 * bb / 24) for a, bb in ab])
        hist.append(eps)
        return out

    def q_sample(self, x_start, t, noise=None):
        if noise is None:
            noise = torch.randn_like(x_start)
        shp = (-1,) + (1,) * (x_start.dim() - 1)
        a = self.sqrt_alphas_cumprod.gather(-1, t).reshape(shp)
        s = self.sqrt_one_minus_alphas_cumprod.gather(-1, t).reshape(shp)
        return a * x_start + s * noise

    def norm_spec(self, x):
        return (x - self.spec_min) / (self.spec_max - self.spec_min) * 2 - 1

    def denorm_spec(self, x):
        return (x + 1) / 2 * (self.spec_max - self.spec_min) + self.spec_min

    def out2mel(self, x):
        return x

    # ------------------------------------------------------------------ sampling loops
    @torch.no_grad()
    def sample(self, cond, x_start=None, t_start=None, noises=None, pndm_speedup=None):
        """Run the reverse process for ``cond`` [B,H,T] and return the normalised mel
        x_0 [B,1,M,T].  ``x_start`` defaults to N(0,1) ('gaussian_start'); ``noises``
        optionally supplies the per-step noise ([steps,B,1,M,T], indexed by t)."""
        b, _, T = cond.shape
        t0 = self.K_step if t_start is None else t_start
        x = x_start if x_start is not None else torch.randn((b, 1, self.mel_bins, T), device=cond.device)
        if pndm_speedup:
            self.noise_list = deque(maxlen=4)
            for i in reversed(range(0, t0, pndm_speedup)):
                x = self.p_sample_plms(x, [i] * b, pndm_speedup, cond)
        elif self._fast() and x.is_cuda and t0 > 0:
            x = self._sample_loop_device(x, cond, t0, noises)
        else:
            for i in reversed(range(0, t0)):
                noise = noises[i] if noises is not None else noise_like(x.shape, x.device, False)
                x = self._p_sample_core(x, [i] * b, cond, noise)
        return x

    # per-call budget for pre-drawn noise of the on-device loop (bytes); longer chains run in chunks of steps
    NOISE_CHUNK_BYTES = 512 << 20

    def _sample_loop_device(self, x, cond, t0, noises):
        """The ancestral loop inside the library (agpt_gd_sample_loop: one captured step replayed, step tables on
        the device).  Noise is drawn HERE, one ``noise_like`` call per step in the reference's order (t0-1 .. 0),
        so a monkey-patched ``noise_like`` and the torch RNG stream see exactly what the step-wise loop shows them."""
        tb = self._tables()
        b = x.shape[0]
        n = x[0].numel()
        x = x.contiguous().float().clone()
        self.denoise_fn.set_cond(cond)
        per_step = b * n * 4
        chunk = max(1, min(t0, self.NOISE_CHUNK_BYTES // max(per_step, 1)))
        t_hi = t0
        while t_hi > 0:
            t_lo = max(0, t_hi - chunk)
            ns = t_hi - t_lo
            if noises is not None and torch.is_tensor(noises) and noises.is_cuda and noises.is_contiguous() \
                    and noises.dtype == torch.float32:
                bank = noises[t_lo:t_hi]                      # indexed by t
            else:
                bank = torch.empty((ns,) + tuple(x.shape), device=x.device, dtype=torch.float32)
                for i in reversed(range(t_lo, t_hi)):
                    bank[i - t_lo].copy_(noises[i] if noises is not None else noise_like(x.shape, x.device, False))
            coef = np.empty((ns, 5), dtype=np.float32)
            for k in range(ns):
                tv = t_hi - 1 - k
                coef[k] = (tb["A"][tv], tb["B"][tv], tb["c1"][tv], tb["c2"][tv],
                           float(tb["sigma"][tv]) if tv != 0 else 0.0)
            _lib.call("gd_sample_loop", x.device, self.denoise_fn._h, _lib.fptr(x), t_hi, t_lo,
                      coef.ctypes.data_as(C.c_void_p), _lib.fptr(bank), b * n, 1)
            t_hi = t_lo
        return x

    def forward(self, txt_tokens, mel2ph=None, spk_embed=None, ref_mels=None, f0=None, uv=None,
                energy=None, infer=False, **kwargs):
        if not infer:
            raise NotImplementedError("audiogpt_b200 accelerates inference only (p_losses is out of scope)")
        if not hasattr(self, "fs2"):
            raise RuntimeError("GaussianDiffusion was built without the FastSpeech2 front-end "
                               "(reference package not importable); call .sample(cond, ...) directly")
        hp = _hp.resolve()
        ret = self.fs2(txt_tokens, mel2ph, spk_embed, ref_mels, f0, uv, energy,
                       skip_decoder=False, infer=True, **kwargs)
        cond = ret["decoder_inp"].transpose(1, 2)
        ret["fs2_mel"] = ret["mel_out"]
        t = self.K_step
        fs2_mels = self.norm_spec(ret["mel_out"]).transpose(1, 2)[:, None, :, :]
        x = self.q_sample(x_start=fs2_mels, t=torch.tensor([t - 1], device=cond.device).long())
        if hp.get("gaussian_start"):
            x = torch.randn((cond.shape[0], 1, self.mel_bins, cond.shape[2]), device=cond.device)
        x = self.sample(cond, x_start=x, t_start=t, pndm_speedup=hp.get("pndm_speedup"))
        x = x[:, 0].transpose(1, 2)
        mel = self.denorm_spec(x)
        if mel2ph is not None:
            mel = mel * ((mel2ph > 0).float()[:, :, None])
        ret["mel_out"] = mel
        return ret
