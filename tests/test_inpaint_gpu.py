"""Make-An-Audio Inpaint UNet (AttentionBlock, resblock_updown, 'concat' conditioning) and its DDIM loop on the GPU
against golden vectors from the reference's own UNetModel / DDIMSampler (tests/golden/make_golden_inpaint.py) and
against the CPU oracle.  Stated tolerance: relative RMSE <= 1e-4 on a single UNet forward; <= 1e-3 after DDIM-10 and
<= 2e-3 after DDIM-100 (fp32 everywhere; summation order and the d^-1/2 vs d^-1/4 * d^-1/4 score scale differ)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from audiogpt_b200 import _lib, specs
from audiogpt_b200.ldm.models.diffusion.ddim import DDIMSampler, LatentDiffusionShim
from audiogpt_b200.ldm.modules.diffusionmodules.openaimodel import AttentionUNetModel
from conftest import load_golden, rel_rmse

pytestmark = pytest.mark.gpu
T = torch.tensor
SMALL_SEED, FULL_SEED = 5050, 6060
SCHEDULE = dict(linear_start=0.0015, linear_end=0.0205)     # configs/inpaint/txt2audio_args.yaml:5-6


def build(cfg, seed):
    u = AttentionUNetModel(image_size=32, use_checkpoint=True, **cfg)
    u.load_state_dict(specs.synth_unet(cfg, seed), strict=True)
    return u.eval().to("cuda")


def sampler(u):
    return DDIMSampler(LatentDiffusionShim(u, conditioning_key="concat", **SCHEDULE).to("cuda"))


def launches_per_step(u):
    return int(_lib.lib().agpt_unet_launches_per_step(u._h))


@pytest.mark.parametrize("new_order,updown", [(False, True), (True, True), (False, False), (True, False)])
def test_small_forward_vs_reference(new_order, updown):
    g = load_golden("ldm_inpaint_small")
    u = build(dict(specs.UNET_INPAINT_SMALL, use_new_attention_order=new_order, resblock_updown=updown), SMALL_SEED)
    eps = u(T(g["x"]).cuda(), timesteps=T(g["t"]).cuda()).cpu()
    e = rel_rmse(eps, g[f"eps_order{int(new_order)}_updown{int(updown)}"])
    print(f"inpaint small order={int(new_order)} updown={int(updown)} eps rel-RMSE: {e:.3e}")
    assert e < 1e-4


def test_shipped_forward_vs_reference():
    g = load_golden("ldm_inpaint")
    u = build(specs.UNET_INPAINT, FULL_SEED)
    eps = u(T(g["x"]).cuda(), timesteps=[991]).cpu()
    e = rel_rmse(eps, g["eps"])
    print(f"inpaint UNet 1x9x10x106 eps rel-RMSE: {e:.3e}")
    assert e < 1e-4


def _fused_and_stepwise(u, S, c, xT, g, gate):
    smp = sampler(u)
    B, _, H, W = xT.shape
    kw = dict(S=S, batch_size=B, shape=(4, H, W), conditioning=c, verbose=False, eta=0.0, x_T=xT)
    out, inter = smp.sample(**kw)
    # the on-device loop ran: only its two end points are logged, and it counted its launches
    assert len(inter["x_inter"]) == 2 and len(inter["pred_x0"]) == 2 and launches_per_step(u) > 0
    calls = []
    out2, inter2 = smp.sample(callback=calls.append, **kw)                       # step-wise path
    assert calls == list(range(S)) and len(inter2["x_inter"]) >= 2
    e, e0 = rel_rmse(out.cpu(), g["ddim%d" % S]), rel_rmse(inter["pred_x0"][-1].cpu(), g["pred_x0_last"])
    e2, e20 = rel_rmse(out2.cpu(), g["ddim%d" % S]), rel_rmse(inter2["pred_x0"][-1].cpu(), g["pred_x0_last"])
    ea = rel_rmse(out.cpu(), out2.cpu())
    print(f"DDIM-{S} concat: fused {e:.3e} (pred_x0 {e0:.3e})  step-wise {e2:.3e} (pred_x0 {e20:.3e})  fused vs step-wise {ea:.3e}")
    assert e < gate and e0 < gate and e2 < gate and e20 < gate
    assert ea < 1e-3


def test_ddim10_small_fused_and_stepwise():
    g = load_golden("ldm_inpaint_small")
    u = build(specs.UNET_INPAINT_SMALL, SMALL_SEED)
    _fused_and_stepwise(u, 10, T(g["c"]).cuda(), T(g["x_T"]).cuda(), g, 1e-3)
    # ddim_sampling may also get a one-element list (apply_model's c_concat list; sample() itself reads .shape, as the
    # reference's does)
    smp = sampler(u)
    smp.make_schedule(ddim_num_steps=10, ddim_eta=0.0, verbose=False)
    out, inter = smp.ddim_sampling([T(g["c"]).cuda()], (2, 4, 6, 10), x_T=T(g["x_T"]).cuda())
    assert len(inter["x_inter"]) == 2 and rel_rmse(out.cpu(), g["ddim10"]) < 1e-3


def test_ddim100_shipped_fused_and_stepwise():
    """The Inpaint tool's DDIMSampler.sample(S=100) on the shipped 107 M-parameter UNet (1x4x10x106 latent)."""
    g = load_golden("ldm_inpaint")
    u = build(specs.UNET_INPAINT, FULL_SEED)
    _fused_and_stepwise(u, 100, T(g["c"]).cuda(), T(g["x_T"]).cuda(), g, 2e-3)


def test_guided_concat_takes_stepwise_path_vs_oracle():
    """classifier-free guidance with concat conditioning is not fused: the step-wise path, against the oracle"""
    from oracle import inpaint_ref as ir, ldm_ref as lr
    cfg = specs.UNET_INPAINT_SMALL
    u = build(cfg, SMALL_SEED)
    sd = specs.synth_unet(cfg, SMALL_SEED)
    xT, c, uc = (specs.synth_tensor(s, seed=k) for k, s in ((1, (2, 4, 6, 10)), (2, (2, 5, 6, 10)), (3, (2, 5, 6, 10))))
    out, inter = sampler(u).sample(S=5, batch_size=2, shape=(4, 6, 10), conditioning=c.cuda(), verbose=False, eta=0.0,
                                   x_T=xT.cuda(), unconditional_guidance_scale=1.5, unconditional_conditioning=uc.cuda())
    assert len(inter["x_inter"]) > 2
    eps_fn = lambda x, t, cc: ir.unet_forward(sd, cfg, torch.cat([x, cc], 1), t)
    ref = lr.ddim_sample(eps_fn, lr.ldm_schedule(**SCHEDULE)["alphas_cumprod"], 5, xT, c, uc, 1.5)
    e = rel_rmse(out.cpu(), ref)
    print(f"guided concat DDIM-5 rel-RMSE vs oracle: {e:.3e}")
    assert e < 1e-3


def test_batch_independence():
    u = build(specs.UNET_INPAINT_SMALL, SMALL_SEED)
    x = specs.synth_tensor((3, 9, 10, 106), seed=9).cuda()
    e = u(x, timesteps=[501, 17, 900])
    for i, t in enumerate((501, 17, 900)):
        e1 = u(x[i:i + 1].contiguous(), timesteps=[t])
        assert torch.allclose(e1[0], e[i], atol=2e-5, rtol=1e-4), i


@pytest.mark.parametrize("N,H,W,updown", [(1, 2, 4, True), (3, 4, 14, True), (2, 10, 106, False), (1, 6, 18, False)])
def test_ragged_shapes_vs_oracle(N, H, W, updown):
    from oracle import inpaint_ref as ir
    cfg = dict(specs.UNET_INPAINT_SMALL, resblock_updown=updown)
    u = build(cfg, SMALL_SEED)
    sd = specs.synth_unet(cfg, SMALL_SEED)
    x = specs.synth_tensor((N, 9, H, W), seed=200 + H + W)
    t = [(37 * i + 11) % 1000 for i in range(N)]
    e = rel_rmse(u(x.cuda(), timesteps=t).cpu(), ir.unet_forward(sd, cfg, x, torch.tensor(t)))
    print(f"inpaint small {N}x9x{H}x{W} updown={updown}: rel-RMSE vs oracle {e:.3e}")
    assert e < 1e-4


def test_concat_loop_rejects_missing_or_mismatched_conditioning():
    u = build(specs.UNET_INPAINT_SMALL, SMALL_SEED)
    with pytest.raises(AssertionError):
        u.set_concat(torch.zeros(1, 4, 6, 10, device="cuda"))             # 4 channels, the model concatenates 5
    u.set_concat(torch.zeros(1, 5, 6, 10, device="cuda"))
    x = torch.zeros(2, 4, 6, 10, device="cuda")
    import ctypes as C
    ci, f1 = (C.c_int * 1)(1), (C.c_float * 1)(0.5)
    z = (C.c_float * 1)(0.0)
    with pytest.raises(RuntimeError, match="agpt_unet_set_concat"):          # conditioning of another batch size
        _lib.call("unet_ddim_sample", x.device, u._h, _lib.fptr(x), 2, 6, 10, 1, ci, f1, f1, z, f1, 1.0,
                  _lib.fptr(torch.empty_like(x)), None)


def test_inpaint_chain_vs_oracle():
    """Wired like Inpaint.inpaint (audio-chatgpt.py:498-516) on the small configs: engine encode of the masked mel,
    posterior mode, the mask nearest-interpolated to the latent and concatenated, the concat DDIM loop, engine decode;
    against the same chain on the CPU oracles."""
    from oracle import inpaint_ref as ir, ldm_ref as lr, vae_enc_ref, vae_ref
    from audiogpt_b200.ldm.models.autoencoder import AutoencoderKLWithEncoder
    vcfg, ucfg = specs.VAE_SMALL, specs.UNET_INPAINT_SMALL
    vae = AutoencoderKLWithEncoder(ddconfig={k: v for k, v in vcfg.items() if k != "embed_dim"},
                                   lossconfig={"target": "torch.nn.Identity"}, embed_dim=vcfg["embed_dim"])
    vsd = dict(specs.synth_vae_encoder(vcfg), **specs.synth_vae_decoder(vcfg))
    vae.load_state_dict(vsd, strict=True)
    vae = vae.eval().to("cuda")
    u = build(ucfg, SMALL_SEED)
    usd = specs.synth_unet(ucfg, SMALL_SEED)
    B, S = 2, 8
    masked_mel = specs.synth_masked_mel(B, 80, 848, 848)
    mask = -torch.ones(B, 1, 80, 848)
    mask[0, :, :, 300:420] = 1.0
    mask[1, :, :, 600:700] = 1.0
    xT = torch.tensor(np.random.RandomState(55).randn(B, 4, 10, 106), dtype=torch.float32)

    c = vae.encode(masked_mel.cuda()).mode()
    c = torch.cat((c, F.interpolate(mask.cuda(), size=c.shape[-2:])), dim=1)
    lat, _ = sampler(u).sample(S=S, batch_size=B, shape=(c.shape[1] - 1,) + tuple(c.shape[2:]), conditioning=c,
                               verbose=False, x_T=xT.cuda())
    mel = vae.decode(lat).cpu()

    rc = vae_enc_ref.vae_encode(vsd, vcfg, masked_mel)[:, :vcfg["embed_dim"]]
    rc = torch.cat((rc, F.interpolate(mask, size=rc.shape[-2:])), dim=1)
    eps_fn = lambda x, t, cc: ir.unet_forward(usd, ucfg, torch.cat([x, cc], 1), t)
    rlat = lr.ddim_sample(eps_fn, lr.ldm_schedule(**SCHEDULE)["alphas_cumprod"], S, xT, rc)
    rmel = vae_ref.vae_decode(vsd, vcfg, rlat)
    el, em = rel_rmse(lat.cpu(), rlat), rel_rmse(mel, rmel)
    print(f"inpaint chain: latent rel-RMSE {el:.3e}, decoded mel rel-RMSE {em:.3e}")
    assert el < 1e-3 and em < 1e-3
