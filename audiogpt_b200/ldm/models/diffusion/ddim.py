"""Drop-in for ``ldm.models.diffusion.ddim.DDIMSampler``.

Reference: /root/reference/text_to_audio/Make_An_Audio/ldm/models/diffusion/ddim.py:12-262
with make_ddim_timesteps / make_ddim_sampling_parameters from
ldm/modules/diffusionmodules/util.py:46-74.

Same constructor, ``make_schedule``, ``sample(...) -> (samples, intermediates)``,
``ddim_sampling``, ``p_sample_ddim``, ``stochastic_encode`` and ``decode`` signatures; the
``model`` object only needs what the reference reads from it (num_timesteps, betas,
alphas_cumprod, alphas_cumprod_prev, device, apply_model, q_sample for mask mode).

* The elementwise update (CFG combine, pred_x0, dir_xt, x_prev) is one CUDA kernel
  (agpt_ddim_update) instead of ~12 tiny torch kernels + 4 torch.full per step.
* When the model's denoiser is audiogpt_b200's UNetModel behind a 'crossattn'
  DiffusionWrapper and no per-step Python hook is requested (callbacks, mask,
  score_corrector, quantize, dropout), ``sample`` runs the whole loop inside the library
  (agpt_unet_ddim_sample): K/V of the context are projected once, timesteps never leave
  the host, no device->host sync per step.  The same holds for AttentionUNetModel (the
  inpainting UNet) behind a 'concat' DiffusionWrapper with a tensor conditioning and no
  guidance: the conditioning channels are handed to the engine once per call
  (agpt_unet_set_concat).  Guided or dict conditionings take the step-wise path.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from .... import _lib


def make_ddim_timesteps(ddim_discr_method, num_ddim_timesteps, num_ddpm_timesteps, verbose=True):
    if ddim_discr_method == "uniform":
        c = num_ddpm_timesteps // num_ddim_timesteps
        steps = np.asarray(list(range(0, num_ddpm_timesteps, c)))
    elif ddim_discr_method == "quad":
        steps = ((np.linspace(0, np.sqrt(num_ddpm_timesteps * .8), num_ddim_timesteps)) ** 2).astype(int)
    else:
        raise NotImplementedError(f'There is no ddim discretization method called "{ddim_discr_method}"')
    out = steps + 1   # "+1 to get the final alpha values right" (util.py:57-58)
    if verbose:
        print(f"Selected timesteps for ddim sampler: {out}")
    return out


def make_ddim_sampling_parameters(alphacums, ddim_timesteps, eta, verbose=True):
    """alphacums: fp32 CPU tensor.  Returns fp32 tensors (the reference mixes tensor/numpy
    types here; values are identical: fp32 gathers, sigma algebra in fp32)."""
    alphacums = torch.as_tensor(alphacums, dtype=torch.float32).cpu()
    idx = torch.as_tensor(np.asarray(ddim_timesteps), dtype=torch.long)
    alphas = alphacums[idx]
    alphas_prev = torch.cat([alphacums[:1], alphacums[idx[:-1]]])
    sigmas = eta * torch.sqrt((1 - alphas_prev) / (1 - alphas) * (1 - alphas / alphas_prev))
    if verbose:
        print(f"Selected alphas for ddim sampler: a_t: {alphas}; a_(t-1): {alphas_prev}")
        print(f"For the chosen value of eta, which is {eta}, this results in the following sigma_t schedule "
              f"for ddim sampler {sigmas}")
    return sigmas, alphas, alphas_prev


def noise_like(shape, device, repeat=False):
    if repeat:
        return torch.randn((1, *shape[1:]), device=device).repeat(shape[0], *((1,) * (len(shape) - 1)))
    return torch.randn(shape, device=device)


def _agpt_unet_of(model):
    """Our UNetModel if `model` routes apply_model(x,t,c) -> diffusion_model(x,t,context=c), or our AttentionUNetModel
    if it routes apply_model(x,t,c) -> diffusion_model(cat([x] + c_concat, 1), t) ('concat')."""
    from ...modules.diffusionmodules.openaimodel import AttentionUNetModel, UNetModel
    wrapper = getattr(model, "model", None)
    unet = getattr(wrapper, "diffusion_model", None)
    key = getattr(wrapper, "conditioning_key", "crossattn")
    if isinstance(unet, AttentionUNetModel):
        return unet if key == "concat" and unet.in_channels > unet.out_channels else None
    if isinstance(unet, UNetModel) and key == "crossattn":
        return unet
    return None


def _concat_tensor(cond):
    """The conditioning tensor of a 'concat' call: a tensor, or a one-element list holding one (else None)."""
    if isinstance(cond, list) and len(cond) == 1:
        cond = cond[0]
    return cond if torch.is_tensor(cond) else None


class DDIMSampler(object):
    def __init__(self, model, schedule="linear", **kwargs):
        super().__init__()
        self.model = model
        self.device = torch.device("cuda") if torch.cuda.is_available() else torch.device("cpu")
        self.ddpm_num_timesteps = model.num_timesteps
        self.schedule = schedule

    def register_buffer(self, name, attr):
        if type(attr) == torch.Tensor:
            attr = attr.to(self.device)
        setattr(self, name, attr)

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0., verbose=True):
        self.ddim_timesteps = make_ddim_timesteps(ddim_discretize, ddim_num_steps, self.ddpm_num_timesteps, verbose)
        ac = self.model.alphas_cumprod
        assert ac.shape[0] == self.ddpm_num_timesteps, "alphas have to be defined for each timestep"
        f32 = lambda x: x.clone().detach().to(torch.float32).to(self.model.device)
        acc = ac.detach().float().cpu()
        self.register_buffer("betas", f32(self.model.betas))
        self.register_buffer("alphas_cumprod", f32(ac))
        self.register_buffer("alphas_cumprod_prev", f32(self.model.alphas_cumprod_prev))
        self.register_buffer("sqrt_alphas_cumprod", f32(acc.sqrt()))
        self.register_buffer("sqrt_one_minus_alphas_cumprod", f32((1. - acc).sqrt()))
        self.register_buffer("log_one_minus_alphas_cumprod", f32((1. - acc).log()))
        self.register_buffer("sqrt_recip_alphas_cumprod", f32((1. / acc).sqrt()))
        self.register_buffer("sqrt_recipm1_alphas_cumprod", f32((1. / acc - 1).sqrt()))
        sig, a, ap = make_ddim_sampling_parameters(acc, self.ddim_timesteps, ddim_eta, verbose)
        # private host-side fp32 tables: per-step scalars are read from these (no device sync per step) ...
        self._h_sigmas, self._h_alphas, self._h_alphas_prev = sig, a, ap
        self._h_sqrt_one_minus_alphas = (1. - a).sqrt()
        # ... and the reference's registered attributes, on the sampler's device like ddim.py:46-52 keeps them
        # (external code indexes them with CUDA tensors)
        self.register_buffer("ddim_sigmas", sig.clone())
        self.register_buffer("ddim_alphas", a.clone())
        self.ddim_alphas_prev = ap.double().numpy()        # a float64 numpy array of the fp32 values in the reference too (util.py:66)
        self.register_buffer("ddim_sqrt_one_minus_alphas", self._h_sqrt_one_minus_alphas.clone())
        acp = self.model.alphas_cumprod_prev.detach().float().cpu()
        self._h_sigmas_orig = ddim_eta * torch.sqrt((1 - acp) / (1 - acc) * (1 - acc / acp))
        self.register_buffer("ddim_sigmas_for_original_num_steps", self._h_sigmas_orig.clone())

    # ------------------------------------------------------------------ sampling
    @torch.no_grad()
    def sample(self, S, batch_size, shape, conditioning=None, callback=None, normals_sequence=None,
               img_callback=None, quantize_x0=False, eta=0., mask=None, x0=None, temperature=1.,
               noise_dropout=0., score_corrector=None, corrector_kwargs=None, verbose=True, x_T=None,
               log_every_t=100, unconditional_guidance_scale=1., unconditional_conditioning=None, **kwargs):
        if conditioning is not None:
            c0 = conditioning
            if isinstance(c0, dict):
                c0 = c0[list(c0.keys())[0]]
                while isinstance(c0, list):
                    c0 = c0[0]
            if c0.shape[0] != batch_size:
                print(f"Warning: Got {c0.shape[0]} conditionings but batch-size is {batch_size}")
        self.make_schedule(ddim_num_steps=S, ddim_eta=eta, verbose=verbose)
        Cc, H, W = shape
        size = (batch_size, Cc, H, W)
        return self.ddim_sampling(conditioning, size, callback=callback, img_callback=img_callback,
                                  quantize_denoised=quantize_x0, mask=mask, x0=x0,
                                  ddim_use_original_steps=False, noise_dropout=noise_dropout,
                                  temperature=temperature, score_corrector=score_corrector,
                                  corrector_kwargs=corrector_kwargs, x_T=x_T, log_every_t=log_every_t,
                                  unconditional_guidance_scale=unconditional_guidance_scale,
                                  unconditional_conditioning=unconditional_conditioning)

    def _fused_ok(self, cond, callback, img_callback, quantize_denoised, mask, noise_dropout, score_corrector,
                  timesteps, ddim_use_original_steps, temperature, unconditional_conditioning, scale):
        if any(v is not None for v in (callback, img_callback, mask, score_corrector, timesteps)):
            return None
        if quantize_denoised or noise_dropout > 0. or ddim_use_original_steps:
            return None
        if float(self._h_sigmas.abs().max()) != 0.0:        # eta > 0 draws noise per step in torch
            return None
        unet = _agpt_unet_of(self.model)
        if unet is not None and unet.in_channels > unet.out_channels:
            # concat conditioning: fused without guidance only (guided concat sampling takes the step-wise path)
            c = _concat_tensor(cond)
            guided = unconditional_conditioning is not None and scale != 1.
            return unet if c is not None and c.is_cuda and not guided else None
        if not torch.is_tensor(cond) or not cond.is_cuda:
            return None
        if unconditional_conditioning is not None and not torch.is_tensor(unconditional_conditioning):
            return None
        return unet

    @torch.no_grad()
    def ddim_sampling(self, cond, shape, x_T=None, ddim_use_original_steps=False, callback=None, timesteps=None,
                      quantize_denoised=False, mask=None, x0=None, img_callback=None, log_every_t=100,
                      temperature=1., noise_dropout=0., score_corrector=None, corrector_kwargs=None,
                      unconditional_guidance_scale=1., unconditional_conditioning=None):
        device = self.model.betas.device
        b = shape[0]
        img = torch.randn(shape, device=device) if x_T is None else x_T
        unet = self._fused_ok(cond, callback, img_callback, quantize_denoised, mask, noise_dropout, score_corrector,
                              timesteps, ddim_use_original_steps, temperature, unconditional_conditioning,
                              unconditional_guidance_scale)
        if unet is not None:
            out, p0 = self._fused_loop(unet, img, cond, unconditional_conditioning, unconditional_guidance_scale)
            # The reference appends (x, pred_x0) at index % log_every_t == 0 and at the first step
            # (ddim.py:162-164); with the loop on device only the end points exist: the lists hold the start
            # and the LAST step's (x_prev, pred_x0) -- the entries callers read ([-1]).  Per-step logging
            # (any callback / img_callback) selects the step-wise path below, which logs exactly like the
            # reference.  Note: the on-device loop calls the UNet engine directly, not model.apply_model.
            return out, {"x_inter": [img, out], "pred_x0": [img, p0]}

        if timesteps is None:
            timesteps = self.ddpm_num_timesteps if ddim_use_original_steps else self.ddim_timesteps
        elif not ddim_use_original_steps:
            subset_end = int(min(timesteps / self.ddim_timesteps.shape[0], 1) * self.ddim_timesteps.shape[0]) - 1
            timesteps = self.ddim_timesteps[:subset_end]
        intermediates = {"x_inter": [img], "pred_x0": [img]}
        time_range = reversed(range(0, timesteps)) if ddim_use_original_steps else np.flip(timesteps)
        total_steps = timesteps if ddim_use_original_steps else timesteps.shape[0]
        for i, step in enumerate(time_range):
            index = total_steps - i - 1
            ts = torch.full((b,), int(step), device=device, dtype=torch.long)
            if mask is not None:
                assert x0 is not None
                img_orig = self.model.q_sample(x0, ts)
                img = img_orig * mask + (1. - mask) * img
            img, pred_x0 = self.p_sample_ddim(
                img, cond, ts, index=index, use_original_steps=ddim_use_original_steps,
                quantize_denoised=quantize_denoised, temperature=temperature, noise_dropout=noise_dropout,
                score_corrector=score_corrector, corrector_kwargs=corrector_kwargs,
                unconditional_guidance_scale=unconditional_guidance_scale,
                unconditional_conditioning=unconditional_conditioning)
            if callback: callback(i)
            if img_callback: img_callback(pred_x0, i)
            if index % log_every_t == 0 or index == total_steps - 1:
                intermediates["x_inter"].append(img)
                intermediates["pred_x0"].append(pred_x0)
        return img, intermediates

    def _fused_loop(self, unet, x_T, cond, uncond, scale):
        x = x_T.contiguous().float()
        B, _, H, W = x.shape
        guided = uncond is not None and scale != 1.
        if unet.in_channels > unet.out_channels:
            unet.set_concat(_concat_tensor(cond))
        else:
            unet.set_context(torch.cat([uncond, cond]).contiguous() if guided else cond)
        order = np.flip(self.ddim_timesteps)
        S = len(order)
        idx = [S - i - 1 for i in range(S)]
        ci = (C.c_int * S)(*[int(s) for s in order])
        fa = lambda t: (C.c_float * S)(*[float(t[j]) for j in idx])
        out, p0 = torch.empty_like(x), torch.empty_like(x)
        _lib.call("unet_ddim_sample", x.device, unet._h, _lib.fptr(x), B, H, W, S, ci, fa(self._h_alphas),
                  fa(self._h_alphas_prev), fa(self._h_sigmas), fa(self._h_sqrt_one_minus_alphas),
                  float(scale) if guided else 1.0, _lib.fptr(out), _lib.fptr(p0))
        return out, p0

    @torch.no_grad()
    def p_sample_ddim(self, x, c, t, index, repeat_noise=False, use_original_steps=False, quantize_denoised=False,
                      temperature=1., noise_dropout=0., score_corrector=None, corrector_kwargs=None,
                      unconditional_guidance_scale=1., unconditional_conditioning=None):
        b, device = x.shape[0], x.device
        single = unconditional_conditioning is None or unconditional_guidance_scale == 1.
        if single:
            e2 = self.model.apply_model(x, t, c)
        else:
            x_in, t_in = torch.cat([x] * 2), torch.cat([t] * 2)
            if isinstance(c, dict):
                assert isinstance(unconditional_conditioning, dict)
                c_in = {k: ([torch.cat([unconditional_conditioning[k][i], c[k][i]]) for i in range(len(c[k]))]
                            if isinstance(c[k], list) else torch.cat([unconditional_conditioning[k], c[k]]))
                        for k in c}
            elif isinstance(c, list):
                assert isinstance(unconditional_conditioning, list)
                c_in = [torch.cat([unconditional_conditioning[i], c[i]]) for i in range(len(c))]
            else:
                c_in = torch.cat([unconditional_conditioning, c])
            e2 = self.model.apply_model(x_in, t_in, c_in)
        if score_corrector is not None:
            assert self.model.parameterization == "eps"
            if not single:
                eu, ec = e2.chunk(2)
                e2, single = eu + unconditional_guidance_scale * (ec - eu), True
            e2 = score_corrector.modify_score(self.model, e2, x, t, c, **corrector_kwargs)

        if use_original_steps:
            a_t = float(self.model.alphas_cumprod[index]); a_prev = float(self.model.alphas_cumprod_prev[index])
            sq = float(self.model.sqrt_one_minus_alphas_cumprod[index])
            sg = float(self._h_sigmas_orig[index])
        else:
            a_t, a_prev = float(self._h_alphas[index]), float(self._h_alphas_prev[index])
            sq, sg = float(self._h_sqrt_one_minus_alphas[index]), float(self._h_sigmas[index])
        if not x.is_cuda:
            raise RuntimeError("audiogpt_b200.DDIMSampler runs on CUDA only (no CPU fallback)")
        noise = noise_like(x.shape, device, repeat_noise) if (sg != 0. or noise_dropout > 0.) else None
        if noise is not None and noise_dropout > 0.:
            noise = torch.nn.functional.dropout(noise, p=noise_dropout)
        x = x.contiguous().float(); e2 = e2.contiguous().float()
        x_prev, pred_x0 = torch.empty_like(x), torch.empty_like(x)
        _lib.call("ddim_update", device, _lib.fptr(x), _lib.fptr(e2), 1 if single else 0, float(unconditional_guidance_scale),
                  a_t, a_prev, sg, sq, _lib.fptr(noise) if noise is not None else None, float(temperature), b,
                  x[0].numel(), _lib.fptr(x_prev), _lib.fptr(pred_x0))
        if quantize_denoised:
            raise NotImplementedError("quantize_denoised needs a VQ first stage (not on the AudioGPT path)")
        return x_prev, pred_x0

    @torch.no_grad()
    def stochastic_encode(self, x0, t, use_original_steps=False, noise=None):
        if use_original_steps:
            sa, som = self.sqrt_alphas_cumprod, self.sqrt_one_minus_alphas_cumprod
        else:
            sa, som = torch.sqrt(self._h_alphas).to(x0.device), self._h_sqrt_one_minus_alphas.to(x0.device)
        if noise is None:
            noise = torch.randn_like(x0)
        shp = (-1,) + (1,) * (x0.dim() - 1)
        return sa.to(x0.device)[t].reshape(shp) * x0 + som.to(x0.device)[t].reshape(shp) * noise

    @torch.no_grad()
    def decode(self, x_latent, cond, t_start, unconditional_guidance_scale=1.0, unconditional_conditioning=None,
               use_original_steps=False):
        timesteps = np.arange(self.ddpm_num_timesteps) if use_original_steps else self.ddim_timesteps
        timesteps = timesteps[:t_start]
        x_dec = x_latent
        total = timesteps.shape[0]
        for i, step in enumerate(np.flip(timesteps)):
            index = total - i - 1
            ts = torch.full((x_latent.shape[0],), int(step), device=x_latent.device, dtype=torch.long)
            x_dec, _ = self.p_sample_ddim(x_dec, cond, ts, index=index, use_original_steps=use_original_steps,
                                          unconditional_guidance_scale=unconditional_guidance_scale,
                                          unconditional_conditioning=unconditional_conditioning)
        return x_dec


class LatentDiffusionShim(torch.nn.Module):
    """Minimal stand-in for ``LatentDiffusion_audio`` (ldm/models/diffusion/ddpm_audio.py) exposing exactly
    what DDIMSampler reads (ddim.py:17,30-36,124,175): schedule buffers as ddpm.py:115-167 registers them
    and ``apply_model`` -> ``DiffusionWrapper('crossattn')`` -> UNet (ddpm.py:1400-1409).  Used by the
    benchmark and tests; inside AudioGPT the real LatentDiffusion object plays this role."""

    class _Wrapper(torch.nn.Module):
        """DiffusionWrapper.forward (ddpm.py:1400-1409) for the conditioning keys: 'crossattn' (text-to-audio),
        'hybrid' (channel-concatenated conditioning + cross-attention) and 'concat' (channel-concatenated conditioning
        only: the inpainting UNet)."""

        def __init__(self, unet, conditioning_key="crossattn"):
            super().__init__()
            assert conditioning_key in ("crossattn", "hybrid", "concat")
            self.diffusion_model = unet
            self.conditioning_key = conditioning_key

        def forward(self, x, t, c_concat=None, c_crossattn=None):
            if self.conditioning_key == "concat":
                return self.diffusion_model(torch.cat([x] + c_concat, dim=1), t)
            cc = torch.cat(c_crossattn, 1)
            if self.conditioning_key == "hybrid":
                x = torch.cat([x] + c_concat, dim=1)
            return self.diffusion_model(x, t, context=cc)

    def __init__(self, unet, timesteps=1000, linear_start=0.00085, linear_end=0.012, conditioning_key="crossattn"):
        super().__init__()
        self.model = self._Wrapper(unet, conditioning_key)
        betas = (torch.linspace(linear_start ** 0.5, linear_end ** 0.5, timesteps, dtype=torch.float64) ** 2).numpy()
        ac = np.cumprod(1. - betas, axis=0)
        f32 = lambda a: torch.tensor(a, dtype=torch.float32)
        self.register_buffer("betas", f32(betas))
        self.register_buffer("alphas_cumprod", f32(ac))
        self.register_buffer("alphas_cumprod_prev", f32(np.append(1., ac[:-1])))
        self.num_timesteps = int(timesteps)
        self.parameterization = "eps"

    @property
    def device(self):
        return self.betas.device

    def apply_model(self, x_noisy, t, cond):
        if not isinstance(cond, dict):      # the key choice of ddpm_audio.py:561-570
            key = "c_concat" if self.model.conditioning_key == "concat" else "c_crossattn"
            cond = {key: cond if isinstance(cond, list) else [cond]}
        return self.model(x_noisy, t, **cond)

    def q_sample(self, x_start, t, noise=None):
        noise = torch.randn_like(x_start) if noise is None else noise
        shp = (-1,) + (1,) * (x_start.dim() - 1)
        return (self.alphas_cumprod.sqrt()[t].reshape(shp) * x_start +
                (1. - self.alphas_cumprod).sqrt()[t].reshape(shp) * noise)
