"""Make-An-Audio UNet + DDIM parity on the GPU (through the C ABI) vs golden vectors from the
reference classes and vs the CPU oracle.  Stated tolerance: relative RMSE <= 1e-4 on a single
UNet forward; <= 1e-3 after recursive DDIM steps (fp32 everywhere; summation order differs)."""
import numpy as np
import pytest
import torch

from audiogpt_b200 import specs
from audiogpt_b200.ldm.models.diffusion.ddim import DDIMSampler, LatentDiffusionShim
from audiogpt_b200.ldm.modules.diffusionmodules.openaimodel import UNetModel
from conftest import load_golden, rel_rmse

pytestmark = pytest.mark.gpu
T = torch.tensor


def build(cfg, seed):
    u = UNetModel(image_size=32, use_checkpoint=True, **cfg)
    u.load_state_dict(specs.synth_unet(cfg, seed), strict=True)
    return u.eval().to("cuda")


def test_state_dict_keys_match_reference_layout():
    cfg = specs.UNET_TXT2AUDIO
    u = UNetModel(image_size=32, **cfg)
    keys = list(u.state_dict().keys())
    assert keys == list(specs.unet_param_shapes(cfg).keys())
    assert "input_blocks.1.1.transformer_blocks.0.attn2.to_k.weight" in keys
    assert "output_blocks.2.2.conv.weight" in keys and "input_blocks.3.0.op.weight" in keys
    assert sum(p.numel() for p in u.parameters()) == 160_223_684


def test_unet_small_forward():
    g = load_golden("ldm_small")
    u = build(specs.UNET_SMALL, 3030)
    eps = u(T(g["x"]).cuda(), timesteps=T(g["t"]).cuda(), context=T(g["ctx"]).cuda()).cpu()
    e = rel_rmse(eps, g["eps"])
    print("unet small eps rel-RMSE:", e)
    assert e < 1e-4


def test_ddim_small_cfg_fused_and_stepwise():
    g = load_golden("ldm_small")
    u = build(specs.UNET_SMALL, 3030)
    ldm = LatentDiffusionShim(u).to("cuda")
    assert torch.equal(ldm.alphas_cumprod.cpu(), T(g["alphas_cumprod"]))
    smp = DDIMSampler(ldm)
    N, H, W = 2, 6, 10
    ctx, uc, xT = T(g["ctx"]).cuda(), T(g["uc"]).cuda(), T(g["x_T"]).cuda()
    out, inter = smp.sample(S=10, batch_size=N, shape=(4, H, W), conditioning=ctx, verbose=False,
                            unconditional_guidance_scale=1.5, unconditional_conditioning=uc, eta=0.0, x_T=xT)
    assert np.array_equal(smp.ddim_timesteps, g["ddim_timesteps"])
    assert torch.equal(smp.ddim_alphas.cpu(), T(g["ddim_alphas"]))
    assert np.array_equal(np.asarray(smp.ddim_alphas_prev, dtype=np.float64), g["ddim_alphas_prev"])
    assert torch.equal(smp.ddim_sqrt_one_minus_alphas.cpu(), T(g["ddim_sqrt_one_minus_alphas"]))
    e = rel_rmse(out.cpu(), g["ddim10"])
    print("ddim-10 CFG (fused loop) rel-RMSE:", e)
    assert e < 1e-3
    # step-wise path (a callback forces the Python loop + agpt_ddim_update)
    calls = []
    out2, inter2 = smp.sample(S=10, batch_size=N, shape=(4, H, W), conditioning=ctx, verbose=False,
                              unconditional_guidance_scale=1.5, unconditional_conditioning=uc, eta=0.0, x_T=xT,
                              callback=lambda i: calls.append(i))
    assert calls == list(range(10))
    assert rel_rmse(out2.cpu(), g["ddim10"]) < 1e-3
    assert len(inter2["x_inter"]) >= 2
    out5, _ = smp.sample(S=5, batch_size=N, shape=(4, H, W), conditioning=ctx, verbose=False, eta=0.0, x_T=xT)
    assert rel_rmse(out5.cpu(), g["ddim5_nocfg"]) < 1e-3


def test_unet_txt2audio_cfg_pair_and_first_steps():
    """BASELINE configs[3] network (160 M params) on the 4x10x78 latent."""
    g = load_golden("ldm_txt2audio")
    u = build(specs.UNET_TXT2AUDIO, 4040)
    xf = torch.tensor(np.random.RandomState(55).randn(1, 4, 10, 78), dtype=torch.float32).cuda()
    cf = specs.synth_tensor((1, 77, 1024), seed=5).cuda()
    ucf = specs.synth_tensor((1, 77, 1024), seed=6).cuda()
    ef = u(torch.cat([xf, xf]), timesteps=[991, 991], context=torch.cat([ucf, cf])).cpu()
    e = rel_rmse(ef, g["eps_pair"])
    print("unet txt2audio eps rel-RMSE:", e)
    assert e < 1e-4
    ldm = LatentDiffusionShim(u).to("cuda")
    smp = DDIMSampler(ldm)
    smp.make_schedule(ddim_num_steps=100, ddim_eta=0.0, verbose=False)
    img = xf
    for i, step in enumerate(np.flip(smp.ddim_timesteps)[:4]):
        ts = torch.full((1,), int(step), device="cuda", dtype=torch.long)
        img, _ = smp.p_sample_ddim(img, cf, ts, index=100 - i - 1, unconditional_guidance_scale=1.5,
                                   unconditional_conditioning=ucf)
    e4 = rel_rmse(img.cpu(), g["ddim100_first4"])
    print("ddim-100 first 4 steps rel-RMSE:", e4)
    assert e4 < 1e-3


def test_ddim100_full_chain_vs_reference():
    """The WHOLE DDIM-100 + CFG 1.5 chain of BASELINE configs[3] (B = 1 clip, 200 UNet forwards of the 160 M-param
    network) against the end point the reference's own DDIMSampler + UNetModel produced on CPU
    (tests/golden/ldm_txt2audio_ddim100.npz).  Stated tolerance: rel-RMSE <= 2e-3 after 100 recursive steps
    (single forward: <= 1e-4); on-device graph loop and the step-wise Python loop must both hold it."""
    g = load_golden("ldm_txt2audio_ddim100")
    u = build(specs.UNET_TXT2AUDIO, 4040)
    ldm = LatentDiffusionShim(u).to("cuda")
    smp = DDIMSampler(ldm)
    xf = T(g["x_T"]).cuda()
    cf = specs.synth_tensor((1, 77, 1024), seed=5).cuda()
    ucf = specs.synth_tensor((1, 77, 1024), seed=6).cuda()
    kw = dict(S=100, batch_size=1, shape=(4, 10, 78), conditioning=cf, verbose=False, x_T=xf, eta=0.0,
              unconditional_guidance_scale=1.5, unconditional_conditioning=ucf)
    out, inter = smp.sample(**kw)
    e = rel_rmse(out.cpu(), g["ddim100"])
    e0 = rel_rmse(inter["pred_x0"][-1].cpu(), g["pred_x0_last"])
    print("ddim-100 end point rel-RMSE (graph loop):", e, " last pred_x0:", e0)
    assert e < 2e-3 and e0 < 2e-3
    out2, inter2 = smp.sample(callback=lambda i: None, **kw)        # step-wise path
    e2 = rel_rmse(out2.cpu(), g["ddim100"])
    print("ddim-100 end point rel-RMSE (step-wise):", e2, " graph vs step-wise:", rel_rmse(out.cpu(), out2.cpu()))
    assert e2 < 2e-3
    # (the loop's fused out-conv + guidance + update kernel accumulates the 4-channel conv in plain fp32 FMA order, the
    # step-wise path through the tap-GEMM: ~1e-6 per step, amplified like any perturbation by this chain)
    assert rel_rmse(out.cpu(), out2.cpu()) < 1e-3
    assert rel_rmse(inter2["pred_x0"][-1].cpu(), g["pred_x0_last"]) < 2e-3


def test_hybrid_conditioning_stepwise_path_vs_oracle():
    """DiffusionWrapper 'hybrid' mode (ddpm.py:1404-1408: channel-concatenated conditioning + cross-attention) with
    dict conditionings through DDIMSampler: not the fused crossattn case, so the sampler takes the step-wise path
    (apply_model -> UNet forward -> agpt_ddim_update per step), with classifier-free guidance on dict conditionings
    (ddim.py:183-195).  Compared with the oracle sampler driving the oracle UNet the same way."""
    from oracle import ldm_ref as lr
    cfg = dict(specs.UNET_SMALL, in_channels=8)            # 4 latent + 4 concatenated conditioning channels
    u = build(cfg, 3131)
    sd = specs.synth_unet(cfg, 3131)
    ldm = LatentDiffusionShim(u, conditioning_key="hybrid").to("cuda")
    smp = DDIMSampler(ldm)
    N, H, W, S = 2, 6, 10, 7
    xT = specs.synth_tensor((N, 4, H, W), seed=1)
    cc = specs.synth_tensor((N, 4, H, W), seed=2)          # e.g. a masked-mel latent
    ctx = specs.synth_tensor((N, S, cfg["context_dim"]), seed=3)
    uctx = specs.synth_tensor((1, S, cfg["context_dim"]), seed=4).expand(N, -1, -1).contiguous()
    cond = {"c_concat": [cc.cuda()], "c_crossattn": [ctx.cuda()]}
    ucond = {"c_concat": [cc.cuda()], "c_crossattn": [uctx.cuda()]}
    out, inter = smp.sample(S=10, batch_size=N, shape=(4, H, W), conditioning=cond, verbose=False, x_T=xT.cuda(), eta=0.0,
                            unconditional_guidance_scale=1.5, unconditional_conditioning=ucond)
    assert len(inter["x_inter"]) >= 2                       # the step-wise path logs like the reference
    eps_fn = lambda x, t, c: lr.unet_forward(sd, cfg, torch.cat([x, torch.cat([cc] * (x.shape[0] // N))], 1), t, c)
    ref = lr.ddim_sample(eps_fn, lr.ldm_schedule()["alphas_cumprod"], 10, xT, ctx, uctx, 1.5)
    e = rel_rmse(out.cpu(), ref)
    print("hybrid conditioning DDIM-10 + CFG rel-RMSE vs oracle:", e)
    assert e < 1e-3


def test_context_cache_survives_freed_source():
    """ADVICE r1: the hoisted K/V cache is keyed on the caller's tensor; a half-precision context is converted,
    so the source could be freed and its address reused by another prompt of the same shape."""
    cfg = specs.UNET_SMALL
    u = build(cfg, 3030)
    x = specs.synth_tensor((1, 4, 6, 10), seed=41).cuda()
    outs = []
    for seed in (1, 2, 3):
        ctx16 = specs.synth_tensor((1, 7, cfg["context_dim"]), seed=seed).cuda().half()
        ref_ctx = ctx16.float()
        e = u(x, timesteps=[10], context=ctx16)
        del ctx16                                    # the next iteration's tensor may land on the same address
        e_ref = u(x, timesteps=[10], context=ref_ctx.clone())
        assert torch.equal(e, e_ref)
        outs.append(e)
    assert not torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("N,H,W,S", [(1, 2, 4, 1), (3, 4, 6, 5), (2, 10, 78, 77)])
def test_shapes_vs_oracle(N, H, W, S):
    from oracle import ldm_ref as lr
    cfg = specs.UNET_SMALL
    u = build(cfg, 3030)
    sd = specs.synth_unet(cfg, 3030)
    x = specs.synth_tensor((N, 4, H, W), seed=200 + H)
    ctx = specs.synth_tensor((N, S, cfg["context_dim"]), seed=300 + S)
    t = [(37 * i + 11) % 1000 for i in range(N)]
    ref = lr.unet_forward(sd, cfg, x, torch.tensor(t), ctx)
    got = u(x.cuda(), timesteps=t, context=ctx.cuda()).cpu()
    assert rel_rmse(got, ref) < 1e-4


def test_eta_noise_path_vs_oracle():
    """eta > 0: sigma_t * noise term (ddim.py:221-224) with injected noise."""
    from oracle import ldm_ref as lr
    x = specs.synth_tensor((2, 4, 6, 10), seed=1)
    e2 = specs.synth_tensor((4, 4, 6, 10), seed=2)
    nz = specs.synth_tensor((2, 4, 6, 10), seed=3)
    from audiogpt_b200 import _lib
    a_t, a_prev, sg = 0.37, 0.52, 0.11
    sq = float(np.sqrt(np.float32(1 - np.float32(a_t))))
    eu, ec = e2.chunk(2)
    ref, ref0 = lr.ddim_step(x, eu + 1.5 * (ec - eu), a_t, a_prev, sg, sq, nz, 0.9)
    xc, ec2, nc = x.cuda(), e2.cuda(), nz.cuda()
    xp, p0 = torch.empty_like(xc), torch.empty_like(xc)
    _lib.check(_lib.lib().agpt_ddim_update(_lib.fptr(xc), _lib.fptr(ec2), 0, 1.5, a_t, a_prev, sg, sq, _lib.fptr(nc),
                                            0.9, 2, x[0].numel(), _lib.fptr(xp), _lib.fptr(p0),
                                            _lib.cur_stream()))
    assert rel_rmse(xp.cpu(), ref) < 1e-6 and rel_rmse(p0.cpu(), ref0) < 1e-6


def test_c4_full_size_properties():
    """C4 per-GPU shape: B=4 clips -> CFG batch 8 on 4x10x78; batch independence."""
    u = build(specs.UNET_TXT2AUDIO, 4040)
    x = specs.synth_tensor((8, 4, 10, 78), seed=9).cuda()
    ctx = specs.synth_tensor((8, 77, 1024), seed=10).cuda()
    e = u(x, timesteps=[501] * 8, context=ctx)
    assert e.shape == (8, 4, 10, 78) and torch.isfinite(e).all()
    e1 = u(x[2:3].contiguous(), timesteps=[501], context=ctx[2:3].contiguous())
    assert torch.allclose(e1[0], e[2], atol=2e-5, rtol=1e-4)


def attention_operands(N, heads, d, Lq, Lk, layout, seed):
    """device (q, q_pitch, k, v, kv_pitch) pointers and their fp64 CPU heads [N][h][L][d].  layout "kv": q [N][Lq][C]
    and K | V interleaved rows [N][Lk][2C] (the hoisted context projection); "packed": q | k | v rows [N][L][3C] (the
    UNet self-attention, FS2, CLAP, GenerSpeech); "peaky": "kv" with q scaled so that the scores have sigma ~ 8 (the
    running max jumps between key blocks and most p underflow)."""
    import ctypes as C
    C_ = heads * d
    heads_of = lambda t, L: t.double().cpu().reshape(N, L, heads, d).permute(0, 2, 1, 3)
    if layout == "packed":
        assert Lq == Lk
        qkv = specs.synth_tensor((N, Lq, 3 * C_), seed=seed).cuda()
        base = qkv.data_ptr()
        ptrs = (C.c_void_p(base), 3 * C_, C.c_void_p(base + 4 * C_), C.c_void_p(base + 8 * C_), 3 * C_)
        return ptrs, (heads_of(qkv[..., :C_], Lq), heads_of(qkv[..., C_:2 * C_], Lk), heads_of(qkv[..., 2 * C_:], Lk)), qkv
    q = specs.synth_tensor((N, Lq, C_), seed=seed, scale=8.0 if layout == "peaky" else 1.0).cuda()
    kv = specs.synth_tensor((N, Lk, 2 * C_), seed=seed + 1).cuda()
    ptrs = (C.c_void_p(q.data_ptr()), C_, C.c_void_p(kv.data_ptr()), C.c_void_p(kv.data_ptr() + 4 * C_), 2 * C_)
    return ptrs, (heads_of(q, Lq), heads_of(kv[..., :C_], Lk), heads_of(kv[..., C_:], Lk)), (q, kv)


ATTN_KV = [(2, 8, 40, 780, 780), (2, 8, 40, 780, 77), (2, 8, 80, 195, 195), (1, 8, 80, 195, 77), (1, 2, 8, 5, 3),
           (2, 3, 16, 130, 70), (1, 4, 32, 64, 129), (1, 2, 64, 200, 64)]
ATTN_MORE = [(2, 8, 40, 780, 780, "packed"), (2, 12, 64, 77, 77, "packed"), (3, 2, 128, 150, 150, "packed"),
             (2, 8, 40, 780, 780, "peaky"), (1, 2, 64, 200, 300, "peaky"), (2, 2, 128, 150, 150, "kv"),
             (1, 2, 128, 65, 200, "peaky"), (2, 8, 40, 1, 77, "kv"), (2, 4, 80, 70, 1, "kv"), (1, 8, 40, 1, 1, "packed"),
             (2, 4, 64, 100, 65, "kv"), (1, 2, 40, 65, 65, "peaky")]


@pytest.mark.parametrize("N,heads,d,Lq,Lk,layout", [c + ("kv",) for c in ATTN_KV] + ATTN_MORE,
                         ids=["-".join(map(str, c)) for c in ATTN_KV + ATTN_MORE])
def test_tensor_core_attention_vs_fp64(N, heads, d, Lq, Lk, layout):
    """agpt_attention (QK^T and PV on wgmma, online softmax) against softmax(q k^T d^-0.5) v evaluated in fp64, for the
    UNet's shapes (8 heads of 40 / 80 channels; 780 / 195 queries; 780 / 195 / 77 keys), ragged small ones, packed
    q | k | v rows, peaky scores, d = 128, and Lq = 1, Lk = 1, Lk = 65; the fp32-FMA kernel is held to the same gate.
    Stated tolerance: rel-RMSE <= 1e-5 (3 x fp16-part products, 2^-22)."""
    from audiogpt_b200 import _lib
    L = _lib.lib()
    C_ = heads * d
    (qp, q_pitch, kp, vp, kv_pitch), (qh, kh, vh), _keep = attention_operands(N, heads, d, Lq, Lk, layout, 1)
    ref = (torch.softmax(qh @ kh.transpose(-1, -2) * d ** -0.5, dim=-1) @ vh).permute(0, 2, 1, 3).reshape(N, Lq, C_)
    errs = []
    for tc in (1, 0):     # 1: wgmma kernel, 0: fp32-FMA kernel
        _lib.check(L.agpt_set_attention_tc(tc))
        try:
            o = torch.full((N, Lq, C_), float("nan"), device="cuda")
            _lib.check(L.agpt_attention(qp, q_pitch, kp, kv_pitch, vp, kv_pitch, _lib.fptr(o), C_, N, heads, d, Lq, Lk,
                                        _lib.cur_stream()))
            torch.cuda.synchronize()
        finally:
            _lib.check(L.agpt_set_attention_tc(-1))
        errs.append(rel_rmse(o.cpu(), ref))
    print(f"attention N={N} h={heads} d={d} {Lq}x{Lk} {layout}: rel-RMSE wgmma {errs[0]:.2e}  fp32 kernel {errs[1]:.2e}")
    assert errs[0] < 1e-5 and errs[1] < 1e-5
