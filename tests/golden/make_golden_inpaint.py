#!/usr/bin/env python
"""Generate the Make-An-Audio Inpaint UNet golden fixtures (ldm_inpaint*.npz) by running the REFERENCE's own UNetModel
(AttentionBlock, resblock_updown) and DDIMSampler on CPU fp32, with the shims and helpers of make_golden.py.

Run in the build container only (needs /root/reference, which does not travel to the GPU box):

    python tests/golden/make_golden_inpaint.py

ldm_inpaint_small: UNET_INPAINT_SMALL forwards at 2x9x6x10 in both attention orders (QKVAttentionLegacy / QKVAttention)
with resblock_updown on and off, and a DDIM-10 end point through the 'concat' shim at B = 2.
ldm_inpaint: the shipped config (configs/inpaint/txt2audio_args.yaml) -- its forward at 1x9x10x106, its state-dict keys and
shapes, the head count of every AttentionBlock, and the DDIM-100 end point and last pred_x0 of the Inpaint tool's
sampling call (x_T = RandomState(55).randn(1, 4, 10, 106), seeded masked-mel latent + mask conditioning).
Weights are not stored: tests rebuild them with specs.synth_unet and the seeds below.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF, LDMShim, import_ldm, save, specs  # noqa: E402

SMALL_SEED, FULL_SEED = 5050, 6060
# the small forwards: (use_new_attention_order, resblock_updown)
VARIANTS = [(False, True), (True, True), (False, False), (True, False)]


def variant_cfg(new_order, updown):
    return dict(specs.UNET_INPAINT_SMALL, use_new_attention_order=new_order, resblock_updown=updown)


def inpaint_cond(B, H, W, seed):
    """[B, 5, H, W]: a masked-mel latent and the Inpaint tool's mask channel (mask * 2 - 1 after nearest interpolation,
    audio-chatgpt.py:438-445,504-506), one masked band of columns per sample"""
    lat = specs.synth_tensor((B, 4, H, W), seed=seed)
    mask = -torch.ones((B, 1, H, W))
    for b in range(B):
        lo = int(W * (0.3 + 0.1 * b)) % W
        mask[b, :, :, lo:lo + max(1, W // 5)] = 1.0
    return torch.cat([lat, mask], dim=1)


class ConcatLDMShim(LDMShim):
    """LatentDiffusion.apply_model's key choice (ddpm_audio.py:561-570) and DiffusionWrapper 'concat'
    (ddpm.py:1404-1406): ddpm.py itself does not import here (it needs pytorch_lightning.utilities)."""

    def apply_model(self, x, t, c):
        if not isinstance(c, dict):
            c = {"c_concat": c if isinstance(c, list) else [c]}
        return self.unet(torch.cat([x] + c["c_concat"], dim=1), timesteps=t)


def golden_inpaint():
    from ldm.modules.diffusionmodules.openaimodel import AttentionBlock, UNetModel
    from ldm.modules.diffusionmodules.util import make_beta_schedule
    from ldm.models.diffusion.ddim import DDIMSampler

    betas = make_beta_schedule("linear", 1000, linear_start=0.0015, linear_end=0.0205)
    ac = np.cumprod(1.0 - betas, axis=0)
    tab = dict(betas=torch.tensor(betas, dtype=torch.float32),
               alphas_cumprod=torch.tensor(ac, dtype=torch.float32),
               alphas_cumprod_prev=torch.tensor(np.append(1.0, ac[:-1]), dtype=torch.float32))

    def build(cfg, seed):
        u = UNetModel(image_size=32, use_checkpoint=True, **cfg)
        u.load_state_dict(specs.synth_unet(cfg, seed), strict=True)
        return u.eval()

    # ---- small: four forwards, DDIM-10 through the concat shim ----
    N, H, W = 2, 6, 10
    x = specs.synth_tensor((N, 9, H, W), seed=71)
    t = torch.tensor([991, 1], dtype=torch.long)
    eps = {}
    for new_order, updown in VARIANTS:
        u = build(variant_cfg(new_order, updown), SMALL_SEED)
        with torch.no_grad():
            e = u(x, timesteps=t)
        eps[f"eps_order{int(new_order)}_updown{int(updown)}"] = e
        print(f"inpaint small order={int(new_order)} updown={int(updown)} eps rms", e.pow(2).mean().sqrt().item())
    u = build(specs.UNET_INPAINT_SMALL, SMALL_SEED)
    smp = DDIMSampler(ConcatLDMShim(u, tab))
    xT = torch.tensor(np.random.RandomState(55).randn(N, 4, H, W), dtype=torch.float32)
    c = inpaint_cond(N, H, W, seed=72)
    out, inter = smp.sample(S=10, batch_size=N, shape=(4, H, W), conditioning=c, verbose=False, eta=0.0, x_T=xT)
    print("inpaint small ddim-10 rms", out.pow(2).mean().sqrt().item())
    save("ldm_inpaint_small", x=x, t=t, x_T=xT, c=c, ddim10=out, pred_x0_last=inter["pred_x0"][-1],
         alphas_cumprod=tab["alphas_cumprod"], **eps)

    # ---- the shipped config ----
    cfg = specs.UNET_INPAINT
    u = build(cfg, FULL_SEED)
    ref_sd = u.state_dict()
    names, heads = [], []
    for name, m in u.named_modules():
        if isinstance(m, AttentionBlock):
            names.append(name)
            heads.append(m.num_heads)
    print(len(names), "AttentionBlocks, heads", heads, "params", sum(p.numel() for p in u.parameters()))
    H, W = 10, 106
    xf = specs.synth_tensor((1, 9, H, W), seed=73)
    with torch.no_grad():
        ef = u(xf, timesteps=torch.tensor([991]))
    print("inpaint full eps rms", ef.pow(2).mean().sqrt().item())
    xT = torch.tensor(np.random.RandomState(55).randn(1, 4, H, W), dtype=torch.float32)
    cf = inpaint_cond(1, H, W, seed=74)
    smp = DDIMSampler(ConcatLDMShim(u, tab))
    out, inter = smp.sample(S=100, batch_size=1, shape=(4, H, W), conditioning=cf, verbose=False, eta=0.0, x_T=xT)
    print("inpaint ddim-100 end point rms", out.pow(2).mean().sqrt().item(), "absmax", out.abs().max().item())
    save("ldm_inpaint", x=xf, eps=ef, x_T=xT, c=cf, ddim100=out, pred_x0_last=inter["pred_x0"][-1],
         ref_keys=np.array(list(ref_sd.keys())),
         ref_shapes=np.array([",".join(str(v) for v in t.shape) for t in ref_sd.values()]),
         attn_names=np.array(names), attn_heads=np.array(heads, dtype=np.int64))


if __name__ == "__main__":
    import_ldm()
    cwd = os.getcwd()
    os.chdir(os.path.join(REF, "text_to_audio", "Make_An_Audio"))
    try:
        golden_inpaint()
    finally:
        os.chdir(cwd)
