"""State-dict layouts of the hot-path networks + seeded synthetic weights.

Host-side logic only (no arithmetic of the path lives here).  The layouts are
the ones the reference's checkpoints carry, so that the drop-in classes accept
them unchanged:

* HiFi-GAN generator   NeuralSeq/modules/hifigan/hifigan.py:104-142 (ctor)
* DiffNet              NeuralSeq/modules/diff/net.py:58-105
* UNetModel            text_to_audio/Make_An_Audio/ldm/modules/diffusionmodules/openaimodel.py:443-693
  (+ SpatialTransformer ldm/modules/attention.py:152-248)

There is no network in the build/bench environment and the reference ships no
weights (download.sh), so parity tests and the benchmark use *seeded random*
state dicts produced by :func:`synth_state_dict`; zero-initialised layers of
the reference are re-randomised so that parity is not vacuous (SURVEY.md 8c).
"""
from __future__ import annotations

import math
from collections import OrderedDict
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

# --------------------------------------------------------------------------
# configs named by BASELINE.json / SURVEY.md section 8
# --------------------------------------------------------------------------

HIFIGAN_V1 = dict(  # NeuralSeq/egs/egs_bases/tts/vocoder/hifigan.yaml:3-12
    resblock="1",
    upsample_rates=[8, 8, 2, 2],
    upsample_kernel_sizes=[16, 16, 4, 4],
    upsample_initial_channel=512,
    resblock_kernel_sizes=[3, 7, 11],
    resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]],
    use_pitch_embed=False,
    audio_sample_rate=22050,
)

HIFIGAN_SMALL = dict(  # same topology, 8x narrower: CPU-second parity fixture
    resblock="1",
    upsample_rates=[8, 8, 2, 2],
    upsample_kernel_sizes=[16, 16, 4, 4],
    upsample_initial_channel=64,
    resblock_kernel_sizes=[3, 7, 11],
    resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]],
    use_pitch_embed=False,
    audio_sample_rate=22050,
)

BIGVGAN_BASE = dict(  # BigVGAN-base 22 kHz / 80 band (the args.yml that ships with the Make-An-Audio vocoder
    # checkpoint is download-only; topology of text_to_audio/Make_An_Audio/vocoder/bigvgan/models.py:133-203)
    resblock="1", num_mels=80,
    upsample_rates=[8, 8, 2, 2],
    upsample_kernel_sizes=[16, 16, 4, 4],
    upsample_initial_channel=512,
    resblock_kernel_sizes=[3, 7, 11],
    resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]],
    activation="snakebeta", snake_logscale=True,
)

BIGVGAN_SMALL = dict(BIGVGAN_BASE, upsample_initial_channel=64)   # CPU-second parity fixture

VAE_TXT2AUDIO = dict(  # first_stage_config.ddconfig, configs/text_to_audio/txt2audio_args.yaml:52-68
    embed_dim=4, z_channels=4, resolution=848, in_channels=1, out_ch=1, ch=128, ch_mult=[1, 2, 2, 4],
    num_res_blocks=2, attn_resolutions=[106, 212], dropout=0.0, double_z=True,
)

VAE_SMALL = dict(VAE_TXT2AUDIO, ch=32)   # same topology (attention at the same levels), 4x narrower

DIFFNET_BASE = dict(  # egs/egs_bases/svs/base.yaml:3-9, configs/tts/fs2.yaml:5
    in_dims=80, hidden_size=256, residual_layers=20, residual_channels=256,
    dilation_cycle_length=1,
)
DIFFNET_SMALL = dict(in_dims=80, hidden_size=32, residual_layers=4,
                     residual_channels=32, dilation_cycle_length=2)

UNET_TXT2AUDIO = dict(  # configs/text_to_audio/txt2audio_args.yaml:31-50
    in_channels=4, out_channels=4, model_channels=320,
    attention_resolutions=[1, 2], num_res_blocks=2, channel_mult=[1, 2],
    num_heads=8, num_head_channels=-1, use_spatial_transformer=True,
    transformer_depth=1, context_dim=1024, legacy=False,
)
UNET_SMALL = dict(
    in_channels=4, out_channels=4, model_channels=32,
    attention_resolutions=[1, 2], num_res_blocks=2, channel_mult=[1, 2],
    num_heads=4, num_head_channels=-1, use_spatial_transformer=True,
    transformer_depth=1, context_dim=48, legacy=False,
)
# Make-An-Audio Inpaint (configs/inpaint/txt2audio_args.yaml:30-45): AttentionBlock UNet, resblock_updown, legacy
# per-head qkv order, 'concat' conditioning of 5 channels (masked-mel latent + mask) onto the 4-channel latent
UNET_INPAINT = dict(
    in_channels=9, out_channels=4, model_channels=320,
    attention_resolutions=[1, 2], num_res_blocks=2, channel_mult=[1, 2],
    num_heads=8, resblock_updown=True,
)
# same structure, 5x narrower (head dims 16 / 32)
UNET_INPAINT_SMALL = dict(UNET_INPAINT, model_channels=64, num_heads=4)

# lj_ds_beta6.yaml:5-24 (DiffSpeech mel normalisation range)
SPEC_MIN = [-4.7574, -4.6783, -4.6431, -4.5832, -4.5390, -4.6771, -4.8089, -4.7672,
            -4.5784, -4.7755, -4.7150, -4.8919, -4.8271, -4.7389, -4.6047, -4.7759,
            -4.6799, -4.8201, -4.7823, -4.8262, -4.7857, -4.7545, -4.9358, -4.9733,
            -5.1134, -5.1395, -4.9016, -4.8434, -5.0189, -4.8460, -5.0529, -4.9510,
            -5.0217, -5.0049, -5.1831, -5.1445, -5.1015, -5.0281, -4.9887, -4.9916,
            -4.9785, -4.9071, -4.9488, -5.0342, -4.9332, -5.0650, -4.8924, -5.0875,
            -5.0483, -5.0848, -5.1809, -5.0677, -5.0015, -5.0792, -5.0636, -5.2413,
            -5.1421, -5.1710, -5.3256, -5.0511, -5.1186, -5.0057, -5.0446, -5.1173,
            -5.0325, -5.1085, -5.0053, -5.0755, -5.1176, -5.1004, -5.2153, -5.2757,
            -5.3025, -5.2867, -5.2918, -5.3328, -5.2731, -5.2985, -5.2400, -5.2211]
SPEC_MAX = [-0.5982, -0.0778, 0.1205, 0.2747, 0.4657, 0.5123, 0.5684, 0.7093,
            0.6461, 0.6420, 0.7316, 0.7715, 0.7681, 0.8349, 0.7815, 0.7591,
            0.7910, 0.7433, 0.7352, 0.6869, 0.6854, 0.6623, 0.5353, 0.6492,
            0.6909, 0.6106, 0.5761, 0.5936, 0.5638, 0.4054, 0.4545, 0.3589,
            0.3037, 0.3380, 0.1599, 0.2433, 0.2741, 0.2130, 0.1569, 0.1911,
            0.2324, 0.1586, 0.1221, 0.0341, -0.0558, 0.0553, -0.1153, -0.0933,
            -0.1171, -0.0050, -0.1519, -0.1629, -0.0522, -0.0739, -0.2069, -0.2405,
            -0.1244, -0.2116, -0.1361, -0.1575, -0.1442, 0.0513, -0.1567, -0.2000,
            0.0086, -0.0698, 0.1385, 0.0941, 0.1864, 0.1225, 0.2176, 0.2566,
            0.1670, 0.1007, 0.1444, 0.0888, 0.1998, 0.2414, 0.2932, 0.3047]


# --------------------------------------------------------------------------
# HiFi-GAN
# --------------------------------------------------------------------------

def hifigan_stage_channels(h) -> List[int]:
    c0 = int(h["upsample_initial_channel"])
    return [c0 // (2 ** (i + 1)) for i in range(len(h["upsample_rates"]))]


def hifigan_param_shapes(h, c_out: int = 1, n_mels: int = 80) -> "OrderedDict[str, Tuple[int, ...]]":
    """Keys/shapes after remove_weight_norm() (hifigan.py:171-178)."""
    s: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    c0 = int(h["upsample_initial_channel"])
    rates = list(h["upsample_rates"])
    s["conv_pre.weight"] = (c0, n_mels, 7)
    s["conv_pre.bias"] = (c0,)
    chans = hifigan_stage_channels(h)
    for i, (u, k) in enumerate(zip(rates, h["upsample_kernel_sizes"])):
        s[f"ups.{i}.weight"] = (chans[i] * 2, chans[i], int(k))
        s[f"ups.{i}.bias"] = (chans[i],)
    nk = len(h["resblock_kernel_sizes"])
    for i, ch in enumerate(chans):
        for j, (ks, dil) in enumerate(zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"])):
            p = f"resblocks.{i * nk + j}"
            if str(h["resblock"]) == "1":
                for n in range(len(dil)):
                    s[f"{p}.convs1.{n}.weight"] = (ch, ch, int(ks))
                    s[f"{p}.convs1.{n}.bias"] = (ch,)
                for n in range(len(dil)):
                    s[f"{p}.convs2.{n}.weight"] = (ch, ch, int(ks))
                    s[f"{p}.convs2.{n}.bias"] = (ch,)
            else:
                for n in range(len(dil)):
                    s[f"{p}.convs.{n}.weight"] = (ch, ch, int(ks))
                    s[f"{p}.convs.{n}.bias"] = (ch,)
    s["conv_post.weight"] = (c_out, chans[-1], 7)
    s["conv_post.bias"] = (c_out,)
    if h.get("use_pitch_embed"):
        s["m_source.l_linear.weight"] = (1, 9)
        s["m_source.l_linear.bias"] = (1,)
        for i in range(len(rates)):
            if i + 1 < len(rates):
                st = int(math.prod(rates[i + 1:]))
                s[f"noise_convs.{i}.weight"] = (chans[i], 1, 2 * st)
            else:
                s[f"noise_convs.{i}.weight"] = (chans[i], 1, 1)
            s[f"noise_convs.{i}.bias"] = (chans[i],)
    return s


def kaiser_sinc_filter12() -> torch.Tensor:
    """The 12-tap Kaiser-windowed sinc low-pass (cutoff 0.25, half-width 0.3) that both halves of
    Activation1d register as a buffer (vocoder/bigvgan/alias_free_torch/filter.py:19-47, resample.py:17-19,
    38-41): shape [1, 1, 12]."""
    ks, cutoff, half_width = 12, 0.25, 0.3
    half = ks // 2
    A = 2.285 * (half - 1) * math.pi * (4 * half_width) + 7.95
    beta = 0.1102 * (A - 8.7) if A > 50.0 else (0.5842 * (A - 21) ** 0.4 + 0.07886 * (A - 21.0) if A >= 21.0 else 0.0)
    window = torch.kaiser_window(ks, beta=beta, periodic=False)
    time = torch.arange(-half, half) + 0.5
    f = 2 * cutoff * window * torch.sinc(2 * cutoff * time)
    f = f / f.sum()
    return f.view(1, 1, ks)


def bigvgan_param_shapes(h) -> "OrderedDict[str, Tuple[int, ...]]":
    """Keys/shapes of BigVGAN.state_dict() after remove_weight_norm() (vocoder/bigvgan/models.py:133-175;
    AMPBlock1 :29-83, AMPBlock2 :86-130; Activation1d buffers alias_free_torch/resample.py:19,41)."""
    s: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    c0 = int(h["upsample_initial_channel"])
    n_mels = int(h.get("num_mels", 80))
    beta = str(h["activation"]) == "snakebeta"
    s["conv_pre.weight"] = (c0, n_mels, 7)
    s["conv_pre.bias"] = (c0,)
    chans = hifigan_stage_channels(h)
    for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"])):
        s[f"ups.{i}.0.weight"] = (chans[i] * 2, chans[i], int(k))
        s[f"ups.{i}.0.bias"] = (chans[i],)

    def act(prefix, ch):
        s[f"{prefix}.act.alpha"] = (ch,)
        if beta:
            s[f"{prefix}.act.beta"] = (ch,)
        s[f"{prefix}.upsample.filter"] = (1, 1, 12)
        s[f"{prefix}.downsample.lowpass.filter"] = (1, 1, 12)

    nk = len(h["resblock_kernel_sizes"])
    for i, ch in enumerate(chans):
        for j, (ks, dil) in enumerate(zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"])):
            p = f"resblocks.{i * nk + j}"
            if str(h["resblock"]) == "1":
                for n in range(len(dil)):
                    s[f"{p}.convs1.{n}.weight"] = (ch, ch, int(ks))
                    s[f"{p}.convs1.{n}.bias"] = (ch,)
                for n in range(len(dil)):
                    s[f"{p}.convs2.{n}.weight"] = (ch, ch, int(ks))
                    s[f"{p}.convs2.{n}.bias"] = (ch,)
                for m in range(2 * len(dil)):
                    act(f"{p}.activations.{m}", ch)
            else:
                for n in range(len(dil)):
                    s[f"{p}.convs.{n}.weight"] = (ch, ch, int(ks))
                    s[f"{p}.convs.{n}.bias"] = (ch,)
                for m in range(len(dil)):
                    act(f"{p}.activations.{m}", ch)
    act("activation_post", chans[-1])
    s["conv_post.weight"] = (1, chans[-1], 7)
    s["conv_post.bias"] = (1,)
    return s


def synth_bigvgan(h, seed: int = 4321):
    """Seeded BigVGAN weights: convs as synth_hifigan; snake alpha/beta ~ N(0, 0.3^2) (log scale) or
    1 + 0.3 N (linear scale); the filter buffers hold the Kaiser-sinc taps."""
    shapes = bigvgan_param_shapes(h)
    # gain 0.7: the snake activations do not attenuate like leaky-relu; keeps tanh unsaturated (rms ~0.1)
    sd = synth_state_dict(shapes, seed, gain=0.7, gains={"conv_post.weight": 0.143})
    logscale = bool(h.get("snake_logscale", False))
    filt = kaiser_sinc_filter12()
    for idx, key in enumerate(shapes):
        if key.endswith(".filter"):
            sd[key] = filt.clone()
        elif key.endswith(".act.alpha") or key.endswith(".act.beta"):
            g = torch.Generator(device="cpu")
            g.manual_seed(int(seed) * 7919 + idx)
            t = 0.3 * torch.randn(shapes[key], generator=g, dtype=torch.float32)
            sd[key] = t if logscale else (1.0 + t).abs() + 0.1
    return sd


# --------------------------------------------------------------------------
# DiffNet
# --------------------------------------------------------------------------

def diffnet_param_shapes(cfg) -> "OrderedDict[str, Tuple[int, ...]]":
    C, H, M = cfg["residual_channels"], cfg["hidden_size"], cfg["in_dims"]
    s: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    s["input_projection.weight"] = (C, M, 1)
    s["input_projection.bias"] = (C,)
    s["mlp.0.weight"] = (4 * C, C)
    s["mlp.0.bias"] = (4 * C,)
    s["mlp.2.weight"] = (C, 4 * C)
    s["mlp.2.bias"] = (C,)
    for i in range(cfg["residual_layers"]):
        p = f"residual_layers.{i}"
        s[f"{p}.dilated_conv.weight"] = (2 * C, C, 3)
        s[f"{p}.dilated_conv.bias"] = (2 * C,)
        s[f"{p}.diffusion_projection.weight"] = (C, C)
        s[f"{p}.diffusion_projection.bias"] = (C,)
        s[f"{p}.conditioner_projection.weight"] = (2 * C, H, 1)
        s[f"{p}.conditioner_projection.bias"] = (2 * C,)
        s[f"{p}.output_projection.weight"] = (2 * C, C, 1)
        s[f"{p}.output_projection.bias"] = (2 * C,)
    s["skip_projection.weight"] = (C, C, 1)
    s["skip_projection.bias"] = (C,)
    s["output_projection.weight"] = (M, C, 1)
    s["output_projection.bias"] = (M,)
    return s


# --------------------------------------------------------------------------
# UNet (openaimodel.UNetModel with SpatialTransformer blocks)
# --------------------------------------------------------------------------

def unet_plan(cfg) -> dict:
    """Walk the constructor logic of openaimodel.py:516-693 and return the block
    list as plain data: each block is a list of layers
    ('conv_in', cin, cout) | ('res', cin, cout) | ('st', ch, heads, dhead, depth) |
    ('attn', ch, heads, dhead) | ('down', ch) | ('up', ch) | ('resdown', ch) | ('resup', ch).
    Only the options the shipped configs use are supported (dims=2, conv_resample, no class labels,
    use_scale_shift_norm=False)."""
    mc = cfg["model_channels"]
    mult = list(cfg["channel_mult"])
    nres = cfg["num_res_blocks"]
    attn_res = set(cfg["attention_resolutions"])
    num_heads = cfg.get("num_heads", -1)
    nhc = cfg.get("num_head_channels", -1)
    nh_up = cfg.get("num_heads_upsample", -1)
    nh_up = num_heads if nh_up == -1 else nh_up
    legacy = cfg.get("legacy", True)
    st = cfg.get("use_spatial_transformer", False)
    updown = cfg.get("resblock_updown", False)
    depth = cfg.get("transformer_depth", 1)

    def heads_for(ch):
        if nhc == -1:
            return num_heads, ch // num_heads
        return ch // nhc, nhc

    def attn(ch, upsample):
        if st:
            nh, dh = heads_for(ch)
            return ("st", ch, nh, dh, depth)
        # AttentionBlock(num_heads=..., num_head_channels=dim_head) as the constructor builds it (openaimodel.py:543-561,
        # 590-597, 643-662): with legacy and num_head_channels == -1 it receives -1 and uses num_heads (num_heads_upsample
        # in the output blocks); otherwise dim_head is a channel count and the head count is ch // dim_head
        if nhc == -1 and legacy:
            nh = nh_up if upsample else num_heads
        else:
            nh = ch // heads_for(ch)[1]
        return ("attn", ch, nh, ch // nh)

    inp: List[list] = [[("conv_in", cfg["in_channels"], mc)]]
    chans = [mc]
    ch, ds = mc, 1
    for level, m in enumerate(mult):
        for _ in range(nres):
            layers = [("res", ch, m * mc)]
            ch = m * mc
            if ds in attn_res:
                layers.append(attn(ch, False))
            inp.append(layers)
            chans.append(ch)
        if level != len(mult) - 1:
            inp.append([("resdown" if updown else "down", ch)])
            chans.append(ch)
            ds *= 2
    mid = [("res", ch, ch), attn(ch, False), ("res", ch, ch)]
    out: List[list] = []
    for level, m in list(enumerate(mult))[::-1]:
        for i in range(nres + 1):
            ich = chans.pop()
            layers = [("res", ch + ich, mc * m)]
            ch = mc * m
            if ds in attn_res:
                layers.append(attn(ch, True))
            if level and i == nres:
                layers.append(("resup" if updown else "up", ch))
                ds //= 2
            out.append(layers)
    return dict(input_blocks=inp, middle_block=mid, output_blocks=out,
                model_channels=mc, time_embed_dim=4 * mc, final_ch=ch,
                context_dim=cfg.get("context_dim"), out_channels=cfg["out_channels"],
                in_channels=cfg["in_channels"])


def _res_shapes(s, p, cin, cout, temb):
    s[f"{p}.in_layers.0.weight"] = (cin,)
    s[f"{p}.in_layers.0.bias"] = (cin,)
    s[f"{p}.in_layers.2.weight"] = (cout, cin, 3, 3)
    s[f"{p}.in_layers.2.bias"] = (cout,)
    s[f"{p}.emb_layers.1.weight"] = (cout, temb)
    s[f"{p}.emb_layers.1.bias"] = (cout,)
    s[f"{p}.out_layers.0.weight"] = (cout,)
    s[f"{p}.out_layers.0.bias"] = (cout,)
    s[f"{p}.out_layers.3.weight"] = (cout, cout, 3, 3)
    s[f"{p}.out_layers.3.bias"] = (cout,)
    if cin != cout:
        s[f"{p}.skip_connection.weight"] = (cout, cin, 1, 1)
        s[f"{p}.skip_connection.bias"] = (cout,)


def _st_shapes(s, p, ch, nh, dh, depth, ctx):
    inner = nh * dh
    s[f"{p}.norm.weight"] = (ch,)
    s[f"{p}.norm.bias"] = (ch,)
    s[f"{p}.proj_in.weight"] = (inner, ch, 1, 1)
    s[f"{p}.proj_in.bias"] = (inner,)
    for d in range(depth):
        q = f"{p}.transformer_blocks.{d}"
        for name, cdim in (("attn1", inner), ("attn2", ctx)):
            s[f"{q}.{name}.to_q.weight"] = (inner, inner)
            s[f"{q}.{name}.to_k.weight"] = (inner, cdim)
            s[f"{q}.{name}.to_v.weight"] = (inner, cdim)
            s[f"{q}.{name}.to_out.0.weight"] = (inner, inner)
            s[f"{q}.{name}.to_out.0.bias"] = (inner,)
        s[f"{q}.ff.net.0.proj.weight"] = (8 * inner, inner)
        s[f"{q}.ff.net.0.proj.bias"] = (8 * inner,)
        s[f"{q}.ff.net.2.weight"] = (inner, 4 * inner)
        s[f"{q}.ff.net.2.bias"] = (inner,)
        for n in ("norm1", "norm2", "norm3"):
            s[f"{q}.{n}.weight"] = (inner,)
            s[f"{q}.{n}.bias"] = (inner,)
    s[f"{p}.proj_out.weight"] = (ch, inner, 1, 1)
    s[f"{p}.proj_out.bias"] = (ch,)


def unet_param_shapes(cfg) -> "OrderedDict[str, Tuple[int, ...]]":
    plan = unet_plan(cfg)
    mc, temb, ctx = plan["model_channels"], plan["time_embed_dim"], plan["context_dim"]
    s: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    s["time_embed.0.weight"] = (temb, mc)
    s["time_embed.0.bias"] = (temb,)
    s["time_embed.2.weight"] = (temb, temb)
    s["time_embed.2.bias"] = (temb,)

    def block(prefix, layers):
        for j, l in enumerate(layers):
            p = f"{prefix}.{j}"
            if l[0] == "conv_in":
                s[f"{p}.weight"] = (l[2], l[1], 3, 3)
                s[f"{p}.bias"] = (l[2],)
            elif l[0] == "res":
                _res_shapes(s, p, l[1], l[2], temb)
            elif l[0] in ("resdown", "resup"):
                _res_shapes(s, p, l[1], l[1], temb)
            elif l[0] == "st":
                _st_shapes(s, p, l[1], l[2], l[3], l[4], ctx)
            elif l[0] == "attn":       # AttentionBlock (openaimodel.py:303-312): Conv1d 1x1 qkv / proj_out
                s[f"{p}.norm.weight"] = (l[1],)
                s[f"{p}.norm.bias"] = (l[1],)
                s[f"{p}.qkv.weight"] = (3 * l[1], l[1], 1)
                s[f"{p}.qkv.bias"] = (3 * l[1],)
                s[f"{p}.proj_out.weight"] = (l[1], l[1], 1)
                s[f"{p}.proj_out.bias"] = (l[1],)
            elif l[0] == "down":
                s[f"{p}.op.weight"] = (l[1], l[1], 3, 3)
                s[f"{p}.op.bias"] = (l[1],)
            elif l[0] == "up":
                s[f"{p}.conv.weight"] = (l[1], l[1], 3, 3)
                s[f"{p}.conv.bias"] = (l[1],)

    for i, layers in enumerate(plan["input_blocks"]):
        block(f"input_blocks.{i}", layers)
    block("middle_block", plan["middle_block"])
    for i, layers in enumerate(plan["output_blocks"]):
        block(f"output_blocks.{i}", layers)
    s["out.0.weight"] = (plan["final_ch"],)
    s["out.0.bias"] = (plan["final_ch"],)
    s["out.2.weight"] = (plan["out_channels"], mc, 3, 3)
    s["out.2.bias"] = (plan["out_channels"],)
    return s


# --------------------------------------------------------------------------
# seeded synthetic weights
# --------------------------------------------------------------------------

def synth_state_dict(shapes: Dict[str, Sequence[int]], seed: int, gain: float = 1.0,
                     convtranspose_prefixes: Sequence[str] = ("ups.",),
                     gains: Dict[str, float] = None) -> "OrderedDict[str, torch.Tensor]":
    """Deterministic fp32 weights (CPU torch.Generator => identical on every box).

    weights ~ N(0, gain^2 / fan_in); biases ~ N(0, 0.05^2); normalisation
    scales ~ 1 + 0.1 N(0,1).  Every tensor is drawn from its own generator
    seeded by (seed, index) so that adding keys does not reshuffle the rest."""
    out: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    for idx, (key, shape) in enumerate(shapes.items()):
        g = torch.Generator(device="cpu")
        g.manual_seed(int(seed) * 100003 + idx)
        shape = tuple(int(v) for v in shape)
        if len(shape) == 1:
            t = torch.randn(shape, generator=g, dtype=torch.float32)
            if key.endswith(".weight"):      # GroupNorm / LayerNorm scale
                t = 1.0 + 0.1 * t
            else:
                t = 0.05 * t
        else:
            if any(key.startswith(p) for p in convtranspose_prefixes):
                # ConvTranspose1d weight [C_in, C_out, k], stride u=k/2: two taps per output
                fan_in = shape[0] * 2
            else:
                fan_in = 1
                for v in shape[1:]:
                    fan_in *= v
            gk = gain
            for pref, mul in (gains or {}).items():
                if key.startswith(pref):
                    gk = gain * mul
            t = torch.randn(shape, generator=g, dtype=torch.float32) * (gk / math.sqrt(fan_in))
        out[key] = t
    return out


def synth_tensor(shape: Sequence[int], seed: int, scale: float = 1.0, shift: float = 0.0) -> torch.Tensor:
    g = torch.Generator(device="cpu")
    g.manual_seed(int(seed))
    return torch.randn(tuple(shape), generator=g, dtype=torch.float32) * scale + shift


def synth_hifigan(h, seed: int = 1234, c_out: int = 1):
    """Seeded generator weights; conv_post is scaled down so that tanh is not
    saturated (pre-tanh rms ~0.35) and waveform RMSE is a meaningful metric."""
    return synth_state_dict(hifigan_param_shapes(h, c_out), seed, gains={"conv_post.weight": 0.35})


def vae_decoder_plan(cfg):
    """Block list of ldm Decoder.__init__ (ldm/modules/diffusionmodules/model.py:462-536): returns
    (block_in at the bottom, [(level, [(cin, cout, has_attn), ...], has_upsample), ...] in execution order)."""
    ch, mult = int(cfg["ch"]), list(cfg["ch_mult"])
    nres = len(mult)
    block_in = ch * mult[-1]
    curr_res = int(cfg["resolution"]) // 2 ** (nres - 1)
    levels = []
    bi = block_in
    for i_level in reversed(range(nres)):
        bo = ch * mult[i_level]
        blocks = []
        for _ in range(int(cfg["num_res_blocks"]) + 1):
            blocks.append((bi, bo, curr_res in cfg["attn_resolutions"]))
            bi = bo
        up = i_level != 0
        levels.append((i_level, blocks, up))
        if up:
            curr_res *= 2
    return block_in, levels


def _vae_res_shapes(s, p, cin, cout):
    """ResnetBlock without time embedding (model.py:82-119)"""
    s[f"{p}.norm1.weight"] = (cin,); s[f"{p}.norm1.bias"] = (cin,)
    s[f"{p}.conv1.weight"] = (cout, cin, 3, 3); s[f"{p}.conv1.bias"] = (cout,)
    s[f"{p}.norm2.weight"] = (cout,); s[f"{p}.norm2.bias"] = (cout,)
    s[f"{p}.conv2.weight"] = (cout, cout, 3, 3); s[f"{p}.conv2.bias"] = (cout,)
    if cin != cout:
        s[f"{p}.nin_shortcut.weight"] = (cout, cin, 1, 1); s[f"{p}.nin_shortcut.bias"] = (cout,)


def _vae_attn_shapes(s, p, c):
    """AttnBlock (model.py:150-175)"""
    s[f"{p}.norm.weight"] = (c,); s[f"{p}.norm.bias"] = (c,)
    for n in ("q", "k", "v", "proj_out"):
        s[f"{p}.{n}.weight"] = (c, c, 1, 1); s[f"{p}.{n}.bias"] = (c,)


def vae_decoder_param_shapes(cfg) -> "OrderedDict[str, Tuple[int, ...]]":
    """post_quant_conv (ldm/models/autoencoder.py:307) + decoder.* (model.py:462-536) of AutoencoderKL."""
    s: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    zc, ed = int(cfg["z_channels"]), int(cfg["embed_dim"])
    s["post_quant_conv.weight"] = (zc, ed, 1, 1)
    s["post_quant_conv.bias"] = (zc,)
    block_in, levels = vae_decoder_plan(cfg)

    s["decoder.conv_in.weight"] = (block_in, zc, 3, 3)
    s["decoder.conv_in.bias"] = (block_in,)
    _vae_res_shapes(s, "decoder.mid.block_1", block_in, block_in)
    _vae_attn_shapes(s, "decoder.mid.attn_1", block_in)
    _vae_res_shapes(s, "decoder.mid.block_2", block_in, block_in)
    last = block_in
    for i_level, blocks, up in levels:
        for j, (cin, cout, has_attn) in enumerate(blocks):
            _vae_res_shapes(s, f"decoder.up.{i_level}.block.{j}", cin, cout)
            if has_attn:
                _vae_attn_shapes(s, f"decoder.up.{i_level}.attn.{j}", cout)
            last = cout
        if up:
            s[f"decoder.up.{i_level}.upsample.conv.weight"] = (last, last, 3, 3)
            s[f"decoder.up.{i_level}.upsample.conv.bias"] = (last,)
    s["decoder.norm_out.weight"] = (last,); s["decoder.norm_out.bias"] = (last,)
    s["decoder.conv_out.weight"] = (int(cfg["out_ch"]), last, 3, 3)
    s["decoder.conv_out.bias"] = (int(cfg["out_ch"]),)
    return s


def synth_vae_decoder(cfg, seed: int = 5150):
    return synth_state_dict(vae_decoder_param_shapes(cfg), seed, convtranspose_prefixes=())


def vae_encoder_plan(cfg):
    """Block list of ldm Encoder.__init__ (model.py:368-437): returns
    (block_in at the bottom, [(level, [(cin, cout, has_attn), ...], has_downsample), ...] in execution order).
    Every level has num_res_blocks blocks (in_ch_mult = (1,) + ch_mult); all but the last end in a Downsample."""
    ch, mult = int(cfg["ch"]), list(cfg["ch_mult"])
    curr_res = int(cfg["resolution"])
    levels = []
    bi = ch
    for i_level in range(len(mult)):
        bo = ch * mult[i_level]
        blocks = []
        for _ in range(int(cfg["num_res_blocks"])):
            blocks.append((bi, bo, curr_res in cfg["attn_resolutions"]))
            bi = bo
        down = i_level != len(mult) - 1
        levels.append((i_level, blocks, down))
        if down:
            curr_res //= 2
    return bi, levels


def vae_encoder_param_shapes(cfg) -> "OrderedDict[str, Tuple[int, ...]]":
    """encoder.* (model.py:368-437) + quant_conv (ldm/models/autoencoder.py:322) of AutoencoderKL, in the order the
    engine consumes them (each level's blocks interleaved with their attention blocks)."""
    s: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    ch, zc, ed = int(cfg["ch"]), int(cfg["z_channels"]), int(cfg["embed_dim"])
    s["encoder.conv_in.weight"] = (ch, int(cfg.get("in_channels", 1)), 3, 3)
    s["encoder.conv_in.bias"] = (ch,)
    block_in, levels = vae_encoder_plan(cfg)
    for i_level, blocks, down in levels:
        for j, (cin, cout, has_attn) in enumerate(blocks):
            _vae_res_shapes(s, f"encoder.down.{i_level}.block.{j}", cin, cout)
            if has_attn:
                _vae_attn_shapes(s, f"encoder.down.{i_level}.attn.{j}", cout)
        if down:
            c = blocks[-1][1]
            s[f"encoder.down.{i_level}.downsample.conv.weight"] = (c, c, 3, 3)
            s[f"encoder.down.{i_level}.downsample.conv.bias"] = (c,)
    _vae_res_shapes(s, "encoder.mid.block_1", block_in, block_in)
    _vae_attn_shapes(s, "encoder.mid.attn_1", block_in)
    _vae_res_shapes(s, "encoder.mid.block_2", block_in, block_in)
    s["encoder.norm_out.weight"] = (block_in,); s["encoder.norm_out.bias"] = (block_in,)
    s["encoder.conv_out.weight"] = (2 * zc, block_in, 3, 3)
    s["encoder.conv_out.bias"] = (2 * zc,)
    s["quant_conv.weight"] = (2 * ed, 2 * zc, 1, 1)
    s["quant_conv.bias"] = (2 * ed,)
    return s


def synth_vae_encoder(cfg, seed: int = 5151):
    return synth_state_dict(vae_encoder_param_shapes(cfg), seed, convtranspose_prefixes=())


def synth_masked_mel(B: int, H: int, W: int, seed: int) -> torch.Tensor:
    """Seeded mel-like image [B, 1, H, W] in [-1, 1] with a band of frames masked to -1, prepared the way the Inpaint
    tool prepares its encoder input (audio-chatgpt.py:437-444: masked_mel = (1 - mask) * mel in [0, 1], then * 2 - 1).
    Row b masks frames [W * (0.3 + 0.1 b), + W / 6) (modulo W)."""
    g = torch.Generator(device="cpu")
    g.manual_seed(int(seed))
    mel = torch.sigmoid(1.5 * torch.randn((B, 1, H, W), generator=g, dtype=torch.float32))
    mask = torch.zeros((B, 1, H, W), dtype=torch.float32)
    for b in range(B):
        lo = int(W * (0.3 + 0.1 * b)) % W
        mask[b, :, :, lo:lo + max(1, W // 6)] = 1.0
    return ((1.0 - mask) * mel) * 2.0 - 1.0


# ---------------------------------------------------------------------------------------------- PitchExtractor
PE_BASE = dict(n_mel_bins=80, hidden_size=256, conv_layers=2, predictor_hidden=256, predictor_layers=5, predictor_kernel=5)
PE_SMALL = dict(n_mel_bins=80, hidden_size=32, conv_layers=2, predictor_hidden=32, predictor_layers=5, predictor_kernel=5)


def pe_param_shapes(cfg) -> "OrderedDict[str, Tuple[int, ...]]":
    """State-dict layout (incl. the BatchNorm buffers) of NeuralSeq/modules/fastspeech/pe.py:119-134 PitchExtractor:
    mel_prenet (Prenet :7-42), mel_encoder (ConvStacks :82-116) and pitch_predictor (tts_modules.py:217-245)."""
    s: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    H, M, P = int(cfg["hidden_size"]), int(cfg["n_mel_bins"]), int(cfg["predictor_hidden"])
    k = int(cfg["predictor_kernel"])
    cin = M
    for l in range(3):
        s[f"mel_prenet.layers.{l}.0.weight"] = (H, cin, 5); s[f"mel_prenet.layers.{l}.0.bias"] = (H,)
        s[f"mel_prenet.layers.{l}.2.weight"] = (H,); s[f"mel_prenet.layers.{l}.2.bias"] = (H,)
        s[f"mel_prenet.layers.{l}.2.running_mean"] = (H,); s[f"mel_prenet.layers.{l}.2.running_var"] = (H,)
        s[f"mel_prenet.layers.{l}.2.num_batches_tracked"] = ()
        cin = H
    s["mel_prenet.out_proj.weight"] = (H, H); s["mel_prenet.out_proj.bias"] = (H,)
    for l in range(int(cfg["conv_layers"])):
        s[f"mel_encoder.conv.{l}.conv.conv.weight"] = (H, H, 5); s[f"mel_encoder.conv.{l}.conv.conv.bias"] = (H,)
        s[f"mel_encoder.conv.{l}.norm.weight"] = (H,); s[f"mel_encoder.conv.{l}.norm.bias"] = (H,)
    if int(cfg["conv_layers"]) > 0:
        s["mel_encoder.in_proj.weight"] = (H, H); s["mel_encoder.in_proj.bias"] = (H,)
        s["mel_encoder.out_proj.weight"] = (H, H); s["mel_encoder.out_proj.bias"] = (H,)
    s["pitch_predictor.pos_embed_alpha"] = (1,)
    cin = H
    for l in range(int(cfg["predictor_layers"])):
        s[f"pitch_predictor.conv.{l}.1.weight"] = (P, cin, k); s[f"pitch_predictor.conv.{l}.1.bias"] = (P,)
        s[f"pitch_predictor.conv.{l}.3.weight"] = (P,); s[f"pitch_predictor.conv.{l}.3.bias"] = (P,)
        cin = P
    s["pitch_predictor.linear.weight"] = (2, P); s["pitch_predictor.linear.bias"] = (2,)
    s["pitch_predictor.embed_positions._float_tensor"] = (1,)
    return s


def synth_pe(cfg, seed: int = 606):
    """Seeded PitchExtractor weights; BatchNorm running statistics are made valid (var > 0)."""
    shapes = pe_param_shapes(cfg)
    sd = synth_state_dict({k: v for k, v in shapes.items() if len(v) > 0}, seed)
    out: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    for i, (k, shp) in enumerate(shapes.items()):
        if k.endswith("num_batches_tracked"):
            out[k] = torch.tensor(0, dtype=torch.long)
        elif k.endswith("running_var"):
            g = torch.Generator().manual_seed(seed * 7919 + i)
            out[k] = 0.5 + torch.rand(shp, generator=g)
        elif k.endswith("running_mean"):
            out[k] = sd[k] * 4.0                  # N(0, 0.2^2)
        elif k.endswith("pos_embed_alpha"):
            out[k] = torch.tensor([0.7])
        elif k.endswith("_float_tensor"):
            out[k] = torch.zeros(1)
        else:
            out[k] = sd[k]
    return out


def synth_diffnet(cfg, seed: int = 2024):
    return synth_state_dict(diffnet_param_shapes(cfg), seed)


def synth_unet(cfg, seed: int = 4040):
    return synth_state_dict(unet_param_shapes(cfg), seed)


# ---------------------------------------------------------------------------------------------- FastSpeech2 / FastSpeech2MIDI
# hidden 64, 2 heads (head dim 32), every optional branch of the frame path on: pitch 'frame' + energy
FS2_SMALL = dict(hidden_size=64, num_heads=2, enc_layers=2, dec_layers=2, enc_ffn_kernel=9, dec_ffn_kernel=9, n_tokens=40,
                 out_dims=80, predictor_hidden=64, dur_predictor_layers=2, dur_predictor_kernel=3, predictor_layers=2,
                 predictor_kernel=5, use_pos_embed=1, rel_pos=0, pitch_type="frame", use_energy_embed=1, use_midi=0)
# egs/egs_bases/tts/fs2.yaml (BASELINE config C2): hidden 256, 2 heads, 4 + 4 FFT layers, pitch 'frame' (standard norm, uv)
FS2_C2 = dict(FS2_SMALL, hidden_size=256, enc_layers=4, dec_layers=4, n_tokens=80, predictor_hidden=256, use_energy_embed=0)
# configs/tts/fs2.yaml: pitch 'ph' with log norm
FS2_PH = dict(FS2_C2, pitch_type="ph")
# egs/egs_bases/svs/midi/e2e/opencpop/ds1000.yaml (AudioGPT's text-to-singing tool): MIDI encoder, rel_pos, no pitch embedding,
# 5-layer duration / pitch predictors
FS2_DS1000 = dict(FS2_C2, rel_pos=1, pitch_type=None, dur_predictor_layers=5, predictor_layers=5, use_midi=1)


def _fft_shapes(s, p, H, L, k):
    for i in range(L):
        q = f"{p}.layers.{i}.op"
        s[f"{q}.layer_norm1.weight"] = (H,); s[f"{q}.layer_norm1.bias"] = (H,)
        s[f"{q}.self_attn.in_proj_weight"] = (3 * H, H)
        s[f"{q}.self_attn.out_proj.weight"] = (H, H)
        s[f"{q}.layer_norm2.weight"] = (H,); s[f"{q}.layer_norm2.bias"] = (H,)
        s[f"{q}.ffn.ffn_1.weight"] = (4 * H, H, k); s[f"{q}.ffn.ffn_1.bias"] = (4 * H,)
        s[f"{q}.ffn.ffn_2.weight"] = (H, 4 * H); s[f"{q}.ffn.ffn_2.bias"] = (H,)
    s[f"{p}.layer_norm.weight"] = (H,); s[f"{p}.layer_norm.bias"] = (H,)


def _predictor_shapes(s, p, H, P, k, layers, odim):
    s[f"{p}.pos_embed_alpha"] = (1,)
    cin = H
    for l in range(layers):
        s[f"{p}.conv.{l}.1.weight"] = (P, cin, k); s[f"{p}.conv.{l}.1.bias"] = (P,)
        s[f"{p}.conv.{l}.3.weight"] = (P,); s[f"{p}.conv.{l}.3.bias"] = (P,)
        cin = P
    s[f"{p}.linear.weight"] = (odim, P); s[f"{p}.linear.bias"] = (odim,)
    s[f"{p}.embed_positions._float_tensor"] = (1,)


def fs2_param_shapes(cfg) -> "OrderedDict[str, Tuple[int, ...]]":
    """State-dict keys and shapes of NeuralSeq/modules/fastspeech/fs2.py:22-72 FastSpeech2 (FastspeechEncoder /
    FastspeechDecoder of EncSALayers, DurationPredictor, Pitch / EnergyPredictor) and, with use_midi, of
    modules/diffsinger_midi/fs2.py:46-53 FastSpeech2MIDI.  The shared token embedding appears under both of its names.
    The order is the one agpt_fs2_create consumes (strict load_state_dict does not depend on it)."""
    s: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    H, P = int(cfg["hidden_size"]), int(cfg["predictor_hidden"])
    s["encoder_embed_tokens.weight"] = (int(cfg["n_tokens"]), H)
    s["encoder.embed_tokens.weight"] = (int(cfg["n_tokens"]), H)
    if not cfg["rel_pos"]:
        s["encoder.embed_positions._float_tensor"] = (1,)
    _fft_shapes(s, "encoder", H, int(cfg["enc_layers"]), int(cfg["enc_ffn_kernel"]))
    s["decoder.pos_embed_alpha"] = (1,)
    s["decoder.embed_positions._float_tensor"] = (1,)
    _fft_shapes(s, "decoder", H, int(cfg["dec_layers"]), int(cfg["dec_ffn_kernel"]))
    s["mel_out.weight"] = (int(cfg["out_dims"]), H); s["mel_out.bias"] = (int(cfg["out_dims"]),)
    cin = H
    for l in range(int(cfg["dur_predictor_layers"])):
        s[f"dur_predictor.conv.{l}.1.weight"] = (P, cin, int(cfg["dur_predictor_kernel"]))
        s[f"dur_predictor.conv.{l}.1.bias"] = (P,)
        s[f"dur_predictor.conv.{l}.3.weight"] = (P,); s[f"dur_predictor.conv.{l}.3.bias"] = (P,)
        cin = P
    s["dur_predictor.linear.weight"] = (1, P); s["dur_predictor.linear.bias"] = (1,)
    k, nl = int(cfg["predictor_kernel"]), int(cfg["predictor_layers"])
    if cfg["pitch_type"]:
        s["pitch_embed.weight"] = (300, H)
        _predictor_shapes(s, "pitch_predictor", H, P, k, nl, 2 if cfg["pitch_type"] == "frame" else 1)
    if cfg["use_energy_embed"]:
        s["energy_embed.weight"] = (256, H)
        _predictor_shapes(s, "energy_predictor", H, P, k, nl, 1)
    if cfg["use_midi"]:
        s["midi_embed.weight"] = (300, H)
        s["midi_dur_layer.weight"] = (H, 1); s["midi_dur_layer.bias"] = (H,)
        s["is_slur_embed.weight"] = (2, H)
    return s


def synth_fs2(cfg, seed: int = 808):
    """Seeded FastSpeech2 weights with realistic operating points: the duration Linear gives exp(xs) - 1 of about 4-8
    frames per token (else mel2ph is empty), the energy Linear a positive energy (the reference indexes its embedding
    with it), the 'ph' pitch Linear log2 F0 around 7.5 (about 180 Hz).  Padding rows of the token embedding are zero, as
    Embedding(padding_idx=0) initialises them, and both names of the shared embedding hold the same tensor."""
    shapes = fs2_param_shapes(cfg)
    sd = synth_state_dict(shapes, seed, convtranspose_prefixes=())
    emb = sd["encoder_embed_tokens.weight"].clone()
    emb[0] = 0
    sd["encoder_embed_tokens.weight"] = emb
    sd["encoder.embed_tokens.weight"] = emb
    for k in sd:
        if k.endswith("pos_embed_alpha"):
            sd[k] = torch.tensor([0.7])
        elif k.endswith("_float_tensor"):
            sd[k] = torch.zeros(1)
    sd["dur_predictor.linear.weight"] = sd["dur_predictor.linear.weight"] * 0.3
    sd["dur_predictor.linear.bias"] = torch.tensor([1.9])
    if cfg["use_energy_embed"]:
        sd["energy_predictor.linear.weight"] = sd["energy_predictor.linear.weight"] * 0.3
        sd["energy_predictor.linear.bias"] = torch.tensor([2.0])
    if cfg["pitch_type"] == "ph":
        sd["pitch_predictor.linear.weight"] = sd["pitch_predictor.linear.weight"] * 0.3
        sd["pitch_predictor.linear.bias"] = torch.tensor([7.5])
    return sd


def fs2_hparams(cfg):
    """The hparams a reference FastSpeech2 / FastSpeech2MIDI of this engine config is built from (the shipped configs'
    values for everything the config does not vary)."""
    return dict(hidden_size=cfg["hidden_size"], num_heads=cfg["num_heads"], enc_layers=cfg["enc_layers"],
                dec_layers=cfg["dec_layers"], enc_ffn_kernel_size=cfg["enc_ffn_kernel"], dec_ffn_kernel_size=cfg["dec_ffn_kernel"],
                audio_num_mel_bins=cfg["out_dims"], predictor_hidden=cfg["predictor_hidden"],
                dur_predictor_layers=cfg["dur_predictor_layers"], dur_predictor_kernel=cfg["dur_predictor_kernel"],
                predictor_layers=cfg["predictor_layers"], predictor_kernel=cfg["predictor_kernel"],
                use_pos_embed=bool(cfg["use_pos_embed"]), rel_pos=bool(cfg["rel_pos"]), encoder_type="fft", decoder_type="fft",
                ffn_act="gelu", ffn_padding="SAME", dur_loss="mse", use_spk_id=False, use_spk_embed=False, use_split_spk_id=False,
                num_spk=1, dropout=0.1, predictor_dropout=0.5, predictor_grad=0.1, use_pitch_embed=cfg["pitch_type"] is not None,
                pitch_type=cfg["pitch_type"] or "frame", use_uv=True, pitch_norm="log" if cfg["pitch_type"] == "ph" else "standard",
                f0_mean=220.0, f0_std=60.0, use_energy_embed=bool(cfg["use_energy_embed"]), pitch_ar=False,
                use_midi=bool(cfg["use_midi"]))


class TokenDictionary:
    """The two methods FastSpeech2.__init__ reads from its phone encoder: len() and pad() (= 0)."""

    def __init__(self, n):
        self.n = int(n)

    def __len__(self):
        return self.n

    def pad(self):
        return 0


def synth_fs2_inputs(cfg, B, T, seed):
    """Ragged token batch with a padded tail: lengths T, T - 3, T // 2 (cycled), ids in [1, n_tokens); MIDI inputs
    (pitch_midi 40..79, midi_dur 0.1..1.0 s, is_slur) zero on padding.  CPU tensors."""
    g = torch.Generator().manual_seed(int(seed))
    lens = [(T, T - 3, T // 2)[i % 3] for i in range(B)]
    valid = torch.arange(T)[None, :] < torch.tensor(lens)[:, None]
    tok = torch.randint(1, int(cfg["n_tokens"]), (B, T), generator=g) * valid
    out = dict(txt_tokens=tok)
    if cfg["use_midi"]:
        out["pitch_midi"] = torch.randint(40, 80, (B, T), generator=g) * valid
        out["midi_dur"] = (0.1 + 0.9 * torch.rand((B, T), generator=g)) * valid
        out["is_slur"] = torch.randint(0, 2, (B, T), generator=g) * valid
    return out


# ---------------------------------------------------------------------------------------------- GenerSpeech
# NeuralSeq/modules/GenerSpeech/config/generspeech.yaml over egs/egs_bases/tts/fs2.yaml: the FS2_C2 front-end plus three
# LocalStyleAdaptors (128 VQ codes), three ProsodyAligners and an 8-block Glow post-flow (hidden 128, k 3, 3 layers,
# in_layers / res_skip_layers shared by blocks 0-3 and 4-7)
GS_C2 = dict(FS2_C2, n_vq=128, glow_hidden=128, glow_kernel=3, glow_blocks=8, glow_layers=3, share_wn_layers=4)
# same topology, narrower: hidden 64 (aligner head dim 32), 16 codes, a 4-block post-flow of hidden 32
GS_SMALL = dict(FS2_SMALL, use_energy_embed=0, n_vq=16, glow_hidden=32, glow_kernel=3, glow_blocks=4, glow_layers=2,
                share_wn_layers=2)
GS_LEVELS = ("utter", "ph", "word")
GS_STYLE_C = 80          # LocalStyleAdaptor: WN / ConvBlocks width (prosody_util.py:175-178)
GS_ALIGN_FFN = 2048      # CrossAttenLayer dim_feedforward


def _wn_shapes(s, p, hid, k, layers, gin):
    """modules/GenerSpeech/model/wavenet.py WN with weight norm (bias, weight_g, weight_v per conv)"""
    for i in range(layers):
        s[f"{p}.in_layers.{i}.bias"] = (2 * hid,)
        s[f"{p}.in_layers.{i}.weight_g"] = (2 * hid, 1, 1)
        s[f"{p}.in_layers.{i}.weight_v"] = (2 * hid, hid, k)
    for i in range(layers):
        rc = 2 * hid if i < layers - 1 else hid
        s[f"{p}.res_skip_layers.{i}.bias"] = (rc,)
        s[f"{p}.res_skip_layers.{i}.weight_g"] = (rc, 1, 1)
        s[f"{p}.res_skip_layers.{i}.weight_v"] = (rc, hid, 1)
    if gin:
        s[f"{p}.cond_layer.bias"] = (2 * hid * layers,)
        s[f"{p}.cond_layer.weight_g"] = (2 * hid * layers, 1, 1)
        s[f"{p}.cond_layer.weight_v"] = (2 * hid * layers, gin, 1)


def gs_glow_cond_channels(cfg):
    """channels of the post-flow conditioning g = cat[mel_out, decoder_inp, spk, emo, ref_prosody] (generspeech.py:58-62)"""
    return int(cfg["out_dims"]) + 4 * int(cfg["hidden_size"])


def generspeech_param_shapes(cfg) -> "OrderedDict[str, Tuple[int, ...]]":
    """State-dict keys and shapes of NeuralSeq/modules/GenerSpeech/model/generspeech.py GenerSpeech: the FastSpeech2 keys
    (fs2_param_shapes, with spk_embed_proj), MixStyle's affine layer (unused at inference), the three LocalStyleAdaptors
    (ConvBlocks, VQEmbeddingEMA buffers, a weight-normed WN whose cond_layer is unused), l1_* and ProsodyAligners, the
    pitch inpainter, and the Glow post-flow.  Tensors a coupling block shares with the block that owns them (its WN
    in_layers / res_skip_layers) appear under every name, as in the reference's state dict."""
    s = fs2_param_shapes(cfg)
    H, C, k = int(cfg["hidden_size"]), GS_STYLE_C, int(cfg["predictor_kernel"])
    s["spk_embed_proj.weight"] = (H, 256); s["spk_embed_proj.bias"] = (H,)
    s["norm.affine_layer.linear_layer.weight"] = (2 * H, H); s["norm.affine_layer.linear_layer.bias"] = (2 * H,)
    s["emo_embed_proj.weight"] = (H, 256); s["emo_embed_proj.bias"] = (H,)
    for lvl in GS_LEVELS:
        p = f"prosody_extractor_{lvl}"
        for r in range(5):
            for j in range(2):
                q = f"{p}.encoder.res_blocks.{r}.blocks.{j}"
                s[f"{q}.0.weight"] = (C,); s[f"{q}.0.bias"] = (C,)
                s[f"{q}.1.weight"] = (2 * C, C, 5); s[f"{q}.1.bias"] = (2 * C,)
                s[f"{q}.4.weight"] = (C, 2 * C, 1); s[f"{q}.4.bias"] = (C,)
        s[f"{p}.encoder.last_norm.weight"] = (C,); s[f"{p}.encoder.last_norm.bias"] = (C,)
        s[f"{p}.encoder.post_net1.weight"] = (H, C, 3); s[f"{p}.encoder.post_net1.bias"] = (H,)
        n = int(cfg["n_vq"])
        s[f"{p}.vqvae.data_initialized"] = (1,)
        s[f"{p}.vqvae.embedding"] = (n, H); s[f"{p}.vqvae.ema_count"] = (n,); s[f"{p}.vqvae.ema_weight"] = (n, H)
        _wn_shapes(s, f"{p}.wavenet", C, 3, 4, C)
        s[f"l1_{lvl}.weight"] = (H, 2 * H); s[f"l1_{lvl}.bias"] = (H,)
        for i in range(2):
            q = f"align_{lvl}.layers.{i}"
            s[f"{q}.multihead_attn.in_proj_weight"] = (3 * H, H); s[f"{q}.multihead_attn.in_proj_bias"] = (3 * H,)
            s[f"{q}.multihead_attn.out_proj.weight"] = (H, H); s[f"{q}.multihead_attn.out_proj.bias"] = (H,)
            s[f"{q}.linear1.weight"] = (GS_ALIGN_FFN, H); s[f"{q}.linear1.bias"] = (GS_ALIGN_FFN,)
            s[f"{q}.norm1.weight"] = (H,); s[f"{q}.norm1.bias"] = (H,)
            s[f"{q}.linear2.weight"] = (H, GS_ALIGN_FFN); s[f"{q}.linear2.bias"] = (H,)
            s[f"{q}.norm2.weight"] = (H,); s[f"{q}.norm2.bias"] = (H,)
    _predictor_shapes(s, "pitch_inpainter_predictor", H, H, k, 3, 2)
    s["embed_positions._float_tensor"] = (1,)
    c2, hid, L = 2 * int(cfg["out_dims"]), int(cfg["glow_hidden"]), int(cfg["glow_layers"])
    for b in range(int(cfg["glow_blocks"])):
        p = f"post_flow.flows.{3 * b}"
        s[f"{p}.logs"] = (1, c2, 1); s[f"{p}.bias"] = (1, c2, 1)
        p = f"post_flow.flows.{3 * b + 1}"
        for n_ in ("l", "log_s", "u", "p", "sign_s", "l_mask", "eye"):
            s[f"{p}.{n_}"] = (4,) if n_ in ("log_s", "sign_s") else (4, 4)
        p = f"post_flow.flows.{3 * b + 2}"
        s[f"{p}.start.bias"] = (hid,); s[f"{p}.start.weight_g"] = (hid, 1, 1); s[f"{p}.start.weight_v"] = (hid, c2 // 2, 1)
        s[f"{p}.end.weight"] = (c2, hid, 1); s[f"{p}.end.bias"] = (c2,)
        _wn_shapes(s, f"{p}.wn", hid, int(cfg["glow_kernel"]), L, 2 * gs_glow_cond_channels(cfg))
    return s


def gs_wn_owner(cfg, b):
    """the coupling block whose WN in_layers / res_skip_layers block b uses (glow_modules.py:538-553)"""
    share = int(cfg["share_wn_layers"])
    return b - b % share if share > 0 else b


def synth_generspeech(cfg, seed: int = 909):
    """Seeded GenerSpeech weights.  The FastSpeech2 part as synth_fs2 (durations of a few frames per token); weight-norm
    gains near the direction's norm; VQ codebooks on the scale of the style encoder's output (about 1), with the
    VQEmbeddingEMA buffers consistent (initialised, ema_weight = embedding); InvConvNear factors of a well-conditioned
    4x4 (a permutation, unit lower / upper triangles, log-scales about 0); ActNorm and the coupling end layers small
    so that the reverse flow stays O(1) over every block.  Shared WN tensors hold the same tensor under every name."""
    shapes = generspeech_param_shapes(cfg)
    sd = synth_state_dict(shapes, seed, convtranspose_prefixes=())
    sd.update(synth_fs2(cfg, seed))
    g = torch.Generator().manual_seed(int(seed) + 17)
    for key, shape in shapes.items():
        if key.endswith(".weight_g"):
            v = sd[key[:-1] + "v"]
            n = v.reshape(v.shape[0], -1).norm(dim=1).reshape(shape)
            sd[key] = n * (0.6 + 0.8 * torch.rand(shape, generator=g))
        elif key.endswith("vqvae.embedding"):   # codes of norm sqrt(H) x 0.5..3: distances far apart between codes
            sd[key] = torch.randn(shape, generator=g) * (0.5 + 2.5 * torch.rand((shape[0], 1), generator=g))
        elif key.endswith("vqvae.data_initialized") or key.endswith("vqvae.ema_count"):
            sd[key] = torch.ones(shape)
        elif key.endswith("_float_tensor"):
            sd[key] = torch.zeros(shape)
        elif key.endswith(("pos_embed_alpha",)):
            sd[key] = torch.tensor([0.7])
    for key in shapes:
        if key.endswith("vqvae.ema_weight"):
            sd[key] = sd[key[:-len("ema_weight")] + "embedding"].clone()
    for b in range(int(cfg["glow_blocks"])):
        p = f"post_flow.flows.{3 * b}"
        sd[p + ".logs"] = 0.1 * torch.randn(sd[p + ".logs"].shape, generator=g)
        sd[p + ".bias"] = 0.1 * torch.randn(sd[p + ".bias"].shape, generator=g)
        p = f"post_flow.flows.{3 * b + 1}"
        sd[p + ".p"] = torch.eye(4)[torch.randperm(4, generator=g)]
        sd[p + ".sign_s"] = torch.where(torch.rand(4, generator=g) > 0.5, 1.0, -1.0)
        sd[p + ".log_s"] = 0.2 * torch.randn(4, generator=g)
        sd[p + ".l"] = 0.3 * torch.randn(4, 4, generator=g)
        sd[p + ".u"] = 0.3 * torch.randn(4, 4, generator=g)
        sd[p + ".l_mask"] = torch.tril(torch.ones(4, 4), -1)
        sd[p + ".eye"] = torch.eye(4)
        p = f"post_flow.flows.{3 * b + 2}"
        sd[p + ".end.weight"] = 0.3 * sd[p + ".end.weight"]
        own = f"post_flow.flows.{3 * gs_wn_owner(cfg, b) + 2}.wn."
        for key in shapes:
            if key.startswith(p + ".wn.") and not key.startswith(p + ".wn.cond_layer"):
                sd[key] = sd[own + key[len(p + ".wn."):]]
    return sd


def generspeech_hparams(cfg):
    """The hparams a reference GenerSpeech of this engine config is built from: fs2_hparams plus the generspeech.yaml keys
    (speaker embedding on, predictor_grad 1)."""
    hp = fs2_hparams(cfg)
    hp.update(use_spk_embed=True, predictor_grad=1.0, ffn_padding="SAME", nVQ=int(cfg["n_vq"]), vae_dropout=0.0,
              lambda_commit=0.25, post_glow_hidden=int(cfg["glow_hidden"]), post_glow_kernel_size=int(cfg["glow_kernel"]),
              post_glow_n_blocks=int(cfg["glow_blocks"]), post_glow_n_block_layers=int(cfg["glow_layers"]),
              share_wn_layers=int(cfg["share_wn_layers"]), sigmoid_scale=False, post_share_cond_layers=False,
              use_txt_cond=True, vq_start=20500, forcing=20000, noise_scale=0.8)
    return hp


def _segments(n_frames, n_segs, g, empty=None):
    """segment ids 1..n_segs over n_frames frames in order (each at least one frame; `empty` is skipped), 0 after"""
    ids = [i for i in range(1, n_segs + 1) if i != empty]
    cuts = torch.sort(torch.randperm(n_frames - 1, generator=g)[:len(ids) - 1] + 1).values.tolist()
    seg = torch.zeros(n_frames, dtype=torch.long)
    for i, (a, b) in enumerate(zip([0] + cuts, cuts + [n_frames])):
        seg[a:b] = ids[i]
    return seg


def synth_generspeech_inputs(cfg, B, T, T_ref, seed):
    """A ragged TTS_OOD batch (GenerSpeechInfer.input_to_batch's tensors): txt_tokens as synth_fs2_inputs; ref_mels
    [B, T_ref, 80] of log-mel scale with zero frames past each row's length (T_ref, T_ref - 5, 2 T_ref / 3, cycled);
    ref_mel2ph with T_ref // 4 segments per row (row 1 skips one id: an empty phoneme segment) and ref_mel2word with
    T_ref // 10, both 0 on the padding frames; spk_embed / emo_embed [B, 256].  Every row reaches the same largest
    segment id, so each row's B = 1 run sees the batch's segment count.  CPU tensors."""
    out = synth_fs2_inputs(cfg, B, T, seed)
    g = torch.Generator().manual_seed(int(seed) + 1)
    lens = [(T_ref, T_ref - 5, (2 * T_ref) // 3)[i % 3] for i in range(B)]
    mels = torch.zeros(B, T_ref, 80)
    m2p = torch.zeros(B, T_ref, dtype=torch.long)
    m2w = torch.zeros(B, T_ref, dtype=torch.long)
    for i, n in enumerate(lens):
        mels[i, :n] = -4.0 + 1.5 * torch.randn(n, 80, generator=g)
        m2p[i, :n] = _segments(n, T_ref // 4, g, empty=3 if i == 1 else None)
        m2w[i, :n] = _segments(n, T_ref // 10, g)
    out.update(ref_mels=mels, ref_mel2ph=m2p, ref_mel2word=m2w, spk_embed=torch.randn(B, 256, generator=g),
               emo_embed=torch.randn(B, 256, generator=g))
    return out


# ---------------------------------------------------------------------------------------------- CLAP text encoder
# FrozenCLAPEmbedder (text_to_audio/Make_An_Audio/ldm/modules/encoders/modules.py:173-212): bert-base-uncased (the
# BertConfig() defaults) and CLAP's Projection 768 -> 1024 (CLAP/config.yml d_proj), tokens padded to max_length 77
CLAP_BASE = dict(vocab_size=30522, max_position_embeddings=512, type_vocab_size=2, hidden_size=768, num_layers=12,
                 num_heads=12, intermediate_size=3072, d_proj=1024, layer_norm_eps=1e-12, proj_layer_norm_eps=1e-5,
                 max_length=77)
# same structure, head dim 16; d_proj 48 is UNET_SMALL's context_dim, so it conditions the small UNet
CLAP_SMALL = dict(CLAP_BASE, vocab_size=1000, max_position_embeddings=80, hidden_size=64, num_layers=2, num_heads=4,
                  intermediate_size=256, d_proj=48)
# the fields of agpt_clap_cfg (max_length belongs to the tokenizer)
CLAP_ENGINE_KEYS = ("vocab_size", "max_position_embeddings", "type_vocab_size", "hidden_size", "num_layers", "num_heads",
                    "intermediate_size", "d_proj", "layer_norm_eps", "proj_layer_norm_eps")


def clap_param_shapes(cfg) -> "OrderedDict[str, Tuple[int, ...]]":
    """State-dict keys and shapes of FrozenCLAPEmbedder: caption_encoder.base (HF BertModel: embeddings, encoder
    layers, pooler) and caption_encoder.projection (CLAP/clap.py:8-14 Projection), in state-dict order, which is the
    order agpt_clap_create consumes."""
    s: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    H, I, D = int(cfg["hidden_size"]), int(cfg["intermediate_size"]), int(cfg["d_proj"])
    b = "caption_encoder.base."
    s[b + "embeddings.word_embeddings.weight"] = (int(cfg["vocab_size"]), H)
    s[b + "embeddings.position_embeddings.weight"] = (int(cfg["max_position_embeddings"]), H)
    s[b + "embeddings.token_type_embeddings.weight"] = (int(cfg["type_vocab_size"]), H)
    s[b + "embeddings.LayerNorm.weight"] = (H,); s[b + "embeddings.LayerNorm.bias"] = (H,)
    for i in range(int(cfg["num_layers"])):
        p = f"{b}encoder.layer.{i}."
        for n in ("query", "key", "value"):
            s[f"{p}attention.self.{n}.weight"] = (H, H); s[f"{p}attention.self.{n}.bias"] = (H,)
        s[p + "attention.output.dense.weight"] = (H, H); s[p + "attention.output.dense.bias"] = (H,)
        s[p + "attention.output.LayerNorm.weight"] = (H,); s[p + "attention.output.LayerNorm.bias"] = (H,)
        s[p + "intermediate.dense.weight"] = (I, H); s[p + "intermediate.dense.bias"] = (I,)
        s[p + "output.dense.weight"] = (H, I); s[p + "output.dense.bias"] = (H,)
        s[p + "output.LayerNorm.weight"] = (H,); s[p + "output.LayerNorm.bias"] = (H,)
    s[b + "pooler.dense.weight"] = (H, H); s[b + "pooler.dense.bias"] = (H,)
    q = "caption_encoder.projection."
    s[q + "linear1.weight"] = (D, H)
    s[q + "linear2.weight"] = (D, D)
    s[q + "layer_norm.weight"] = (D,); s[q + "layer_norm.bias"] = (D,)
    return s


def synth_clap(cfg, seed: int = 7070):
    """Seeded FrozenCLAPEmbedder weights (synth_state_dict: embedding rows and Linears N(0, 1 / fan_in), LayerNorm
    scales 1 + 0.1 N, biases 0.05 N)."""
    return synth_state_dict(clap_param_shapes(cfg), seed, convtranspose_prefixes=())


# ---------------------------------------------------------------------------------------------- CLAP candidate scorer
# wav_evaluation/models/CLAPWrapper.py: the CLAP model T2A.select_best_audio scores its candidates with
# (useful_ckpts/CLAP/config.yml).  bert = the text tower's BertConfig (bert-base-uncased: BertConfig() defaults);
# Projection LayerNorms use nn.LayerNorm's default eps.
CLAP_SCORER = dict(text_model="bert-base-uncased", text_len=100, transformer_embed_dim=768,
                   freeze_text_encoder_weights=True, audioenc_name="Cnn14", out_emb=2048, sampling_rate=44100,
                   duration=9, fmin=50, fmax=14000, n_fft=1028, hop_size=320, mel_bins=64, window_size=1024,
                   d_proj=1024, temperature=0.003, num_classes=527, batch_size=1024, demo=False,
                   bert=dict(CLAP_BASE, proj_layer_norm_eps=1e-5))
# the same audio tower with a CLAP_SMALL-sized BERT (positions for text_len 100 and one longer prompt)
CLAP_SCORER_SMALL = dict(CLAP_SCORER, transformer_embed_dim=64,
                         bert=dict(CLAP_SMALL, max_position_embeddings=128, d_proj=1024))
CNN14_CHANNELS = (64, 128, 256, 512, 1024, 2048)   # conv_block1..6 (audio.py:132-137)
BN_EPS = 1e-5                                       # nn.BatchNorm2d default


def clap_scorer_bert_cfg(cfg):
    """The agpt_clap_cfg of the scorer's text tower (its Projection is transformer_embed_dim -> d_proj)."""
    b = dict(cfg["bert"], d_proj=int(cfg["d_proj"]))
    assert b["hidden_size"] == cfg["transformer_embed_dim"], "transformer_embed_dim must equal the BERT width"
    return {k: b[k] for k in CLAP_ENGINE_KEYS}


def _projection_shapes(s, p, d_in, d_out):
    s[p + "linear1.weight"] = (d_out, d_in)
    s[p + "linear2.weight"] = (d_out, d_out)
    s[p + "layer_norm.weight"] = (d_out,); s[p + "layer_norm.bias"] = (d_out,)


def _bn_shapes(s, p, c):
    for n in ("weight", "bias", "running_mean", "running_var"):
        s[f"{p}.{n}"] = (c,)
    s[p + ".num_batches_tracked"] = ()


def clap_scorer_param_shapes(cfg) -> "OrderedDict[str, Tuple[int, ...]]":
    """State-dict keys and shapes of wav_evaluation.models.clap.CLAP (the checkpoint's "model" dict) in state-dict
    order: logit_scale, audio_encoder (Cnn14 with torchlibrosa's Spectrogram / LogmelFilterBank, then Projection),
    caption_encoder (HF BertModel without the position_ids buffer, then Projection).  A 2022 checkpoint also holds
    caption_encoder.base.embeddings.position_ids, which current transformers no longer registers."""
    s: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    s["logit_scale"] = ()
    a = "audio_encoder.base."
    nb = int(cfg["window_size"]) // 2 + 1
    s[a + "spectrogram_extractor.stft.conv_real.weight"] = (nb, 1, int(cfg["window_size"]))
    s[a + "spectrogram_extractor.stft.conv_imag.weight"] = (nb, 1, int(cfg["window_size"]))
    s[a + "logmel_extractor.melW"] = (nb, int(cfg["mel_bins"]))
    _bn_shapes(s, a + "bn0", int(cfg["mel_bins"]))
    cin = 1
    for i, c in enumerate(CNN14_CHANNELS):
        p = f"{a}conv_block{i + 1}."
        s[p + "conv1.weight"] = (c, cin, 3, 3)
        s[p + "conv2.weight"] = (c, c, 3, 3)
        _bn_shapes(s, p + "bn1", c)
        _bn_shapes(s, p + "bn2", c)
        cin = c
    E = int(cfg["out_emb"])
    s[a + "fc1.weight"] = (E, cin); s[a + "fc1.bias"] = (E,)
    s[a + "fc_audioset.weight"] = (int(cfg["num_classes"]), E); s[a + "fc_audioset.bias"] = (int(cfg["num_classes"]),)
    _projection_shapes(s, "audio_encoder.projection.", E, int(cfg["d_proj"]))
    for k, v in clap_param_shapes(clap_scorer_bert_cfg(cfg)).items():
        s[k] = v
    return s


def cnn14_engine_keys(cfg):
    """The audio-tower keys agpt_cnn14_create consumes, in its order: the clap_scorer_param_shapes order without
    fc_audioset (the scorer never uses clipwise_output) and num_batches_tracked."""
    return [k for k in clap_scorer_param_shapes(cfg) if k.startswith("audio_encoder.")
            and ".fc_audioset." not in k and not k.endswith("num_batches_tracked")]


def sinc_resample_kernel(orig_freq: int, new_freq: int, lowpass_filter_width: int = 6, rolloff: float = 0.99):
    """torchaudio.transforms.Resample(orig_freq, new_freq)'s polyphase filter at its defaults (sinc_interp_hann),
    restated from torchaudio.functional.functional._get_sinc_resample_kernel: returns (kernel [new][2 width + orig]
    fp32, width, orig, new), the rates reduced by their gcd.  Output sample k * new + p is
    sum_j kernel[p][j] * x[k * orig + j - width] (zero outside the clip); there are ceil(new * L / orig) of them."""
    g = math.gcd(int(orig_freq), int(new_freq))
    orig, new = int(orig_freq) // g, int(new_freq) // g
    base = min(orig, new) * rolloff
    width = math.ceil(lowpass_filter_width * orig / base)
    idx = torch.arange(-width, width + orig, dtype=torch.float64)[None, None] / orig
    t = torch.arange(0, -new, -1)[:, None, None] / new + idx
    t *= base
    t = t.clamp_(-lowpass_filter_width, lowpass_filter_width)
    window = torch.cos(t * math.pi / lowpass_filter_width / 2) ** 2
    t *= math.pi
    kernels = torch.where(t == 0, torch.tensor(1.0).to(t), t.sin() / t)
    kernels *= window * (base / orig)
    return kernels.to(torch.float32)[:, 0], width, orig, new


def stft_dft_weights(n_fft: int):
    """torchlibrosa STFT's conv_real / conv_imag weights [n_fft/2 + 1][1][n_fft]: the DFT rows exp(-2 pi i k n / N)
    times the periodic Hann window (librosa get_window('hann', fftbins=True))."""
    n = np.arange(n_fft)
    win = 0.5 - 0.5 * np.cos(2 * np.pi * n / n_fft)
    k = np.arange(n_fft // 2 + 1)
    ph = 2 * np.pi * ((k[:, None] * n[None, :]) % n_fft) / n_fft
    real = np.cos(ph) * win[None, :]
    imag = -np.sin(ph) * win[None, :]
    return (torch.from_numpy(real.astype(np.float32))[:, None, :], torch.from_numpy(imag.astype(np.float32))[:, None, :])


def slaney_mel(sr: float, n_fft: int, n_mels: int, fmin: float, fmax: float) -> np.ndarray:
    """librosa.filters.mel(sr=sr, n_fft=n_fft, n_mels=n_mels, fmin=fmin, fmax=fmax) (Slaney scale and area
    normalisation, its defaults) restated in numpy: [n_mels][n_fft/2 + 1] fp32."""
    f_sp, min_log_hz, min_log_mel, logstep = 200.0 / 3, 1000.0, 15.0, math.log(6.4) / 27.0

    def hz_to_mel(f):
        f = np.asanyarray(f, dtype=np.float64)
        return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-10) / min_log_hz) / logstep, f / f_sp)

    def mel_to_hz(m):
        return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)

    fftfreqs = np.fft.rfftfreq(n=n_fft, d=1.0 / sr)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(fmin), hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    w = np.zeros((n_mels, len(fftfreqs)))
    for i in range(n_mels):
        w[i] = np.maximum(0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    w *= (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]
    return w.astype(np.float32)


def synth_clap_scorer(cfg, seed: int = 9090):
    """Seeded CLAP scorer weights in the checkpoint's layout (synth_state_dict draws, then): the real periodic-Hann DFT
    rows and Slaney mel matrix of the config; convs and fc1 at He gain; BatchNorm running statistics with positive
    variance (bn0's centred on the log-mel range of a speech-level clip), so log-mels and activations keep O(1)
    magnitudes through the 12 convs; logit_scale = log(1 / 0.07) as CLAP initialises it."""
    shapes = clap_scorer_param_shapes(cfg)
    sd = synth_state_dict(shapes, seed, convtranspose_prefixes=(),
                          gains={"audio_encoder.base.conv_block": math.sqrt(2.0), "audio_encoder.base.fc1": math.sqrt(2.0)})
    a = "audio_encoder.base."
    sd[a + "spectrogram_extractor.stft.conv_real.weight"], sd[a + "spectrogram_extractor.stft.conv_imag.weight"] = \
        stft_dft_weights(int(cfg["window_size"]))
    sd[a + "logmel_extractor.melW"] = torch.from_numpy(np.ascontiguousarray(slaney_mel(
        cfg["sampling_rate"], cfg["window_size"], cfg["mel_bins"], cfg["fmin"], cfg["fmax"]).T))
    g = torch.Generator().manual_seed(int(seed) + 1)
    for k, shape in shapes.items():
        if k.endswith("num_batches_tracked"):
            sd[k] = torch.tensor(0, dtype=torch.long)
        elif k.endswith("running_mean"):
            sd[k] = (-5.0 + 3.0 * torch.randn(shape, generator=g)) if k.startswith(a + "bn0") else 0.1 * torch.randn(shape, generator=g)
        elif k.endswith("running_var"):
            sd[k] = (100.0 if k.startswith(a + "bn0") else 1.0) * (0.5 + torch.rand(shape, generator=g))
    sd["logit_scale"] = torch.tensor(math.log(1 / 0.07), dtype=torch.float32)
    return sd


def synth_scorer_clips(lens=(159744, 40000, 159744), sr: int = 16000, seed: int = 31):
    """Seeded mono test clips for the scorer (float32 numpy, one per length): a few sines with a slow amplitude
    envelope plus noise, different in every clip.  The default lengths are T2A's candidates (80 x 624 mel frames at
    hop 256: cropped) and a short clip (tiled)."""
    rs = np.random.RandomState(int(seed))
    clips = []
    for i, n in enumerate(lens):
        t = np.arange(int(n)) / sr
        x = sum(0.2 / (j + 1) * np.sin(2 * np.pi * rs.uniform(80, 4000) * t + rs.uniform(0, 6)) for j in range(4 + 2 * i))
        x = x * (0.6 + 0.4 * np.sin(2 * np.pi * rs.uniform(0.5, 3) * t)) + 0.02 * (i + 1) * rs.randn(int(n))
        clips.append(x.astype(np.float32))
    return clips


# ---------------------------------------------------------------------------------------------- sound extraction
# LASSNet of the SoundExtraction tool (sound_extraction/model/LASSNet.py, text_encoder.py, resunet_film.py,
# modules.py:169-379, film.py): bert-mini (prajjwal1/bert-mini: 4 layers, hidden 256, 4 heads, FFN 1024, no pooler),
# Linear(256, 256) + ReLU, and UNetRes_FiLM(channels=1, cond_embedding_dim=256).  The STFT is filter_length 1024, hop
# 512, periodic Hann (sound_extraction/utils/stft.py).
LASS = dict(vocab_size=30522, max_position_embeddings=512, type_vocab_size=2, hidden_size=256, num_layers=4, num_heads=4,
            intermediate_size=1024, layer_norm_eps=1e-12)
# the same network with a 1000-token vocabulary (the UNet's widths are fixed by the reference class)
LASS_SMALL = dict(LASS, vocab_size=1000, max_position_embeddings=64)
LASS_COND = 256
LASS_ENC = ((1, 32), (32, 64), (64, 128), (128, 256), (256, 384), (384, 384))   # encoder_block1..6 (in, out)
LASS_DEC = ((384, 384), (384, 384), (384, 256), (256, 128), (128, 64), (64, 32))  # decoder_block1..6 (in, out)
LASS_FFT, LASS_HOP = 1024, 512


def lass_blocks():
    """The 26 ConvBlockResCond of UNetRes_FiLM in forward order: (state-dict prefix, C_in, C_out)."""
    out = []
    for i, (ci, co) in enumerate(LASS_ENC):
        out += [(f"UNet.encoder_block{i + 1}.conv_block1", ci, co), (f"UNet.encoder_block{i + 1}.conv_block2", co, co)]
    out.append(("UNet.conv_block7", 384, 384))
    for j, (ci, co) in enumerate(LASS_DEC):
        out += [(f"UNet.decoder_block{j + 1}.conv_block2", 2 * co, co), (f"UNet.decoder_block{j + 1}.conv_block3", co, co)]
    out.append(("UNet.after_conv_block1", 32, 32))
    return out


def _film_shapes(s, p, c, d=LASS_COND):
    s[p + ".linear.0.weight"] = (2 * c, d); s[p + ".linear.0.bias"] = (2 * c,)
    s[p + ".linear.2.weight"] = (c, 2 * c); s[p + ".linear.2.bias"] = (c,)


def _resblock_cond_shapes(s, p, ci, co):
    _bn_shapes(s, p + ".bn1", ci)
    _bn_shapes(s, p + ".bn2", co)
    s[p + ".conv1.weight"] = (co, ci, 3, 3)
    _film_shapes(s, p + ".film1", co)
    s[p + ".conv2.weight"] = (co, co, 3, 3)
    _film_shapes(s, p + ".film2", co)
    if ci != co:
        s[p + ".shortcut.weight"] = (co, ci, 1, 1); s[p + ".shortcut.bias"] = (co,)
        _film_shapes(s, p + ".film_res", co)


def lass_param_shapes(cfg) -> "OrderedDict[str, Tuple[int, ...]]":
    """State-dict keys and shapes of LASSNet in state-dict order, which is the order agpt_lass_create consumes (without
    the num_batches_tracked counters): text_embedder.bert_layer (HF BertModel without pooler and without the
    position_ids buffer current transformers no longer saves), text_embedder.linear_layer, then UNet."""
    s: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    H, I = int(cfg["hidden_size"]), int(cfg["intermediate_size"])
    b = "text_embedder.bert_layer."
    s[b + "embeddings.word_embeddings.weight"] = (int(cfg["vocab_size"]), H)
    s[b + "embeddings.position_embeddings.weight"] = (int(cfg["max_position_embeddings"]), H)
    s[b + "embeddings.token_type_embeddings.weight"] = (int(cfg["type_vocab_size"]), H)
    s[b + "embeddings.LayerNorm.weight"] = (H,); s[b + "embeddings.LayerNorm.bias"] = (H,)
    for i in range(int(cfg["num_layers"])):
        p = f"{b}encoder.layer.{i}."
        for n in ("query", "key", "value"):
            s[f"{p}attention.self.{n}.weight"] = (H, H); s[f"{p}attention.self.{n}.bias"] = (H,)
        s[p + "attention.output.dense.weight"] = (H, H); s[p + "attention.output.dense.bias"] = (H,)
        s[p + "attention.output.LayerNorm.weight"] = (H,); s[p + "attention.output.LayerNorm.bias"] = (H,)
        s[p + "intermediate.dense.weight"] = (I, H); s[p + "intermediate.dense.bias"] = (I,)
        s[p + "output.dense.weight"] = (H, I); s[p + "output.dense.bias"] = (H,)
        s[p + "output.LayerNorm.weight"] = (H,); s[p + "output.LayerNorm.bias"] = (H,)
    s["text_embedder.linear_layer.0.weight"] = (LASS_COND, H); s["text_embedder.linear_layer.0.bias"] = (LASS_COND,)
    blocks = {p: (ci, co) for p, ci, co in lass_blocks()}
    for i in range(len(LASS_ENC)):
        for k in (1, 2):
            p = f"UNet.encoder_block{i + 1}.conv_block{k}"
            _resblock_cond_shapes(s, p, *blocks[p])
    _resblock_cond_shapes(s, "UNet.conv_block7", 384, 384)
    for j, (ci, co) in enumerate(LASS_DEC):
        p = f"UNet.decoder_block{j + 1}"
        s[p + ".conv1.weight"] = (ci, co, 3, 3)
        _bn_shapes(s, p + ".bn1", ci)
        _resblock_cond_shapes(s, p + ".conv_block2", 2 * co, co)
        _resblock_cond_shapes(s, p + ".conv_block3", co, co)
    _resblock_cond_shapes(s, "UNet.after_conv_block1", 32, 32)
    s["UNet.after_conv2.weight"] = (1, 32, 1, 1); s["UNet.after_conv2.bias"] = (1,)
    return s


def lass_engine_keys(cfg):
    """The keys agpt_lass_create consumes, in its order: lass_param_shapes without num_batches_tracked."""
    return [k for k in lass_param_shapes(cfg) if not k.endswith("num_batches_tracked")]


def synth_lass(cfg, seed: int = 6060):
    """Seeded LASSNet weights: synth_state_dict draws (convs and Linears N(0, 1 / fan_in)), then every BatchNorm gets
    gamma 1 + 0.2 N, beta 0.1 N, running mean 0.2 N and running variance in [0.5, 1.5) (the first block's bn1, which
    sees raw magnitudes, mean 1 and variance in [4, 6)), and the FiLM layers' second Linear is scaled by 0.5 so the
    62 additive vectors stay O(0.1), and after_conv2 by 0.25, so the mask logits stay O(1) and the sigmoid does not
    saturate."""
    shapes = lass_param_shapes(cfg)
    sd = synth_state_dict(shapes, seed, convtranspose_prefixes=())
    g = torch.Generator().manual_seed(int(seed) + 1)
    first = "UNet.encoder_block1.conv_block1.bn1."
    for k, shape in shapes.items():
        if ".bn" not in k:
            continue
        if k.endswith("num_batches_tracked"):
            sd[k] = torch.tensor(0, dtype=torch.long)
        elif k.endswith(".weight"):
            sd[k] = 1.0 + 0.2 * torch.randn(shape, generator=g)
        elif k.endswith(".bias"):
            sd[k] = 0.1 * torch.randn(shape, generator=g)
        elif k.endswith("running_mean"):
            sd[k] = torch.ones(shape) if k.startswith(first) else 0.2 * torch.randn(shape, generator=g)
        elif k.endswith("running_var"):
            sd[k] = (4.0 if k.startswith(first) else 0.5) + (2.0 if k.startswith(first) else 1.0) * torch.rand(shape, generator=g)
    for k in shapes:
        if ".film" in k and ".linear.2." in k:
            sd[k] = sd[k] * 0.5
    sd["UNet.after_conv2.weight"] = sd["UNet.after_conv2.weight"] * 0.25
    return sd


def stft_bases(filter_length: int = LASS_FFT, hop_length: int = LASS_HOP):
    """sound_extraction/utils/stft.py STFT's forward_basis / inverse_basis buffers [filter_length + 2][1][filter_length]
    (win_length = filter_length, window 'hann'): built in numpy float64 the reference's way, cast to fp32, windowed
    with the fp32 periodic Hann window."""
    scale = filter_length / hop_length
    fb = np.fft.fft(np.eye(filter_length))
    cutoff = filter_length // 2 + 1
    fb = np.vstack([np.real(fb[:cutoff, :]), np.imag(fb[:cutoff, :])])
    fwd = torch.FloatTensor(fb[:, None, :])
    inv = torch.FloatTensor(np.linalg.pinv(scale * fb).T[:, None, :])
    from scipy.signal import get_window
    win = torch.from_numpy(get_window("hann", filter_length, fftbins=True)).float()
    return (fwd * win).float(), (inv * win).float()


def stft_window_sum(n_frames: int, filter_length: int = LASS_FFT, hop_length: int = LASS_HOP) -> np.ndarray:
    """stft.py window_sumsquare('hann', n_frames, ...) with norm None: the fp32 envelope, each frame's float64 squared
    window added in float64 and stored back to fp32, as numpy's in-place add does."""
    n = filter_length + hop_length * (n_frames - 1)
    x = np.zeros(n, dtype=np.float32)
    from scipy.signal import get_window
    win_sq = get_window("hann", filter_length, fftbins=True) ** 2
    for i in range(n_frames):
        s = i * hop_length
        x[s:min(n, s + filter_length)] += win_sq[:max(0, min(filter_length, n - s))]
    return x


def synth_lass_ids(cfg, lens, seed: int = 61):
    """Seeded query rows as the tool tokenizes them (add_special_tokens=False, padding=True): [N, max(lens)] ids with
    [CLS] (101, or 1 for a vocabulary without it) first, and the attention mask."""
    rs = np.random.RandomState(int(seed))
    V = int(cfg["vocab_size"])
    cls = 101 if V > 101 else 1
    L = max(lens)
    ids = np.zeros((len(lens), L), np.int64)
    mask = np.zeros((len(lens), L), np.int64)
    for i, n in enumerate(lens):
        ids[i, 0] = cls
        ids[i, 1:n] = rs.randint(1000 if V > 2000 else 2, V, size=n - 1)
        mask[i, :n] = 1
    return torch.from_numpy(ids), torch.from_numpy(mask)


def synth_lass_wav(n_samples: int, seed: int = 62) -> torch.Tensor:
    """A seeded mono clip at 32 kHz: a few sines under a slow envelope plus noise, [n_samples] fp32."""
    rs = np.random.RandomState(int(seed))
    t = np.arange(int(n_samples)) / 32000.0
    x = sum(0.15 / (j + 1) * np.sin(2 * np.pi * rs.uniform(60, 6000) * t + rs.uniform(0, 6)) for j in range(6))
    x = x * (0.6 + 0.4 * np.sin(2 * np.pi * rs.uniform(0.3, 2) * t)) + 0.02 * rs.randn(int(n_samples))
    return torch.from_numpy(x.astype(np.float32))


# ---------------------------------------------------------------------------------------------- sound event detection
# PVT of the SoundDetection tool (audio_detection/audio_infer/pytorch/models.py:141-237; audio-chatgpt.py:612-673 builds
# PVT(sample_rate=32000, window_size=1024, hop_size=320, mel_bins=64, fmin=50, fmax=14000, classes_num=527)).  The
# transformer sizes are fixed inside the reference class (PyramidVisionTransformerV2(...) at :170-188); bn0 is
# BatchNorm2d(64), so mel_bins is 64.  Block norms and stage norms use eps 1e-6 (the norm_layer partial), the
# patch-embedding norm and Attention.norm are plain nn.LayerNorm (1e-5).
PVT_SHIPPED = dict(sample_rate=32000, window_size=1024, hop_size=320, mel_bins=64, fmin=50, fmax=14000, classes_num=527,
                   embed_dims=(64, 128, 320, 512), depths=(3, 4, 6, 3), num_heads=(1, 2, 5, 8), mlp_ratios=(8, 8, 4, 4),
                   sr_ratios=(8, 4, 2, 1), interpolate_ratio=32, layer_norm_eps=1e-6, embed_norm_eps=1e-5)
# the same four-stage structure (sr 8 / 4 / 2 / 1, head dim 64), narrower and one block per stage, with a short window
PVT_SMALL = dict(PVT_SHIPPED, window_size=256, hop_size=80, classes_num=23, embed_dims=(64, 64, 128, 128),
                 depths=(1, 1, 1, 1), num_heads=(1, 1, 2, 2), mlp_ratios=(4, 4, 2, 2))
PVT_STAGES = 4


def pvt_grids(cfg, n_samples: int):
    """The token grid (H = time, W = mel) of every stage for a clip of n_samples: the Python twin of agpt_pvt_frames.
    T = n // hop + 1 frames; stage 1 is Conv2d(k 7, stride 4, padding 2), stages 2-4 Conv2d(k 3, stride 2, padding 1).
    Raises ValueError for a clip the network cannot take: no more than window_size // 2 samples (reflect padding), or a
    stage whose grid is smaller than its sr_ratio (Attention.sr would leave no key)."""
    n = int(n_samples)
    if n <= int(cfg["window_size"]) // 2:
        raise ValueError(f"clip of {n} samples: reflect padding needs more than {int(cfg['window_size']) // 2}")
    H, W = n // int(cfg["hop_size"]) + 1, int(cfg["mel_bins"])
    grids = []
    for i in range(PVT_STAGES):
        if min(H, W) < (3 if i == 0 else 1):
            raise ValueError(f"clip of {n} samples is too short: stage {i + 1} has no tokens")
        H, W = ((H - 3) // 4 + 1, (W - 3) // 4 + 1) if i == 0 else ((H - 1) // 2 + 1, (W - 1) // 2 + 1)
        sr = int(cfg["sr_ratios"][i])
        if H < sr or W < sr:
            raise ValueError(f"clip of {n} samples is too short: stage {i + 1}'s {H} x {W} grid is smaller than its sr_ratio {sr}")
        grids.append((H, W))
    return grids


def pvt_min_samples(cfg) -> int:
    """The shortest clip pvt_grids accepts (9600 samples, 0.3 s, for PVT_SHIPPED: stage 1 needs 8 rows, so 31 frames)."""
    need = 1
    for i in reversed(range(PVT_STAGES)):
        need = max(need, int(cfg["sr_ratios"][i]))
        need = 4 * (need - 1) + 3 if i == 0 else 2 * (need - 1) + 1      # the fewest input rows that give `need` rows
    return max((need - 1) * int(cfg["hop_size"]), int(cfg["window_size"]) // 2 + 1)


def pvt_param_shapes(cfg) -> "OrderedDict[str, Tuple[int, ...]]":
    """State-dict keys and shapes of the reference PVT in state-dict order: the frozen front-end buffers the checkpoint
    carries, bn0, pvt_transformer.patch_embed{i} / block{i}.{j} / norm{i}, fc_audioset."""
    s: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    n = int(cfg["window_size"])
    nb = n // 2 + 1
    s["spectrogram_extractor.stft.conv_real.weight"] = (nb, 1, n)
    s["spectrogram_extractor.stft.conv_imag.weight"] = (nb, 1, n)
    s["logmel_extractor.melW"] = (nb, int(cfg["mel_bins"]))
    _bn_shapes(s, "bn0", int(cfg["mel_bins"]))
    cin = 1
    for i in range(PVT_STAGES):
        C, sr, hid = int(cfg["embed_dims"][i]), int(cfg["sr_ratios"][i]), int(cfg["embed_dims"][i]) * int(cfg["mlp_ratios"][i])
        k = 7 if i == 0 else 3
        p = f"pvt_transformer.patch_embed{i + 1}."
        s[p + "proj.weight"] = (C, cin, k, k); s[p + "proj.bias"] = (C,)
        s[p + "norm.weight"] = (C,); s[p + "norm.bias"] = (C,)
        for j in range(int(cfg["depths"][i])):
            p = f"pvt_transformer.block{i + 1}.{j}."
            s[p + "norm1.weight"] = (C,); s[p + "norm1.bias"] = (C,)
            s[p + "attn.q.weight"] = (C, C); s[p + "attn.q.bias"] = (C,)
            s[p + "attn.kv.weight"] = (2 * C, C); s[p + "attn.kv.bias"] = (2 * C,)
            s[p + "attn.proj.weight"] = (C, C); s[p + "attn.proj.bias"] = (C,)
            if sr > 1:
                s[p + "attn.sr.weight"] = (C, C, sr, sr); s[p + "attn.sr.bias"] = (C,)
                s[p + "attn.norm.weight"] = (C,); s[p + "attn.norm.bias"] = (C,)
            s[p + "norm2.weight"] = (C,); s[p + "norm2.bias"] = (C,)
            s[p + "mlp.fc1.weight"] = (hid, C); s[p + "mlp.fc1.bias"] = (hid,)
            s[p + "mlp.dwconv.dwconv.weight"] = (hid, 1, 3, 3); s[p + "mlp.dwconv.dwconv.bias"] = (hid,)
            s[p + "mlp.fc2.weight"] = (C, hid); s[p + "mlp.fc2.bias"] = (C,)
        s[f"pvt_transformer.norm{i + 1}.weight"] = (C,); s[f"pvt_transformer.norm{i + 1}.bias"] = (C,)
        cin = C
    s["fc_audioset.weight"] = (int(cfg["classes_num"]), cin); s["fc_audioset.bias"] = (int(cfg["classes_num"]),)
    return s


def pvt_engine_keys(cfg):
    """The keys agpt_pvt_create consumes, in its order: the state dict without bn0.num_batches_tracked."""
    return [k for k in pvt_param_shapes(cfg) if not k.endswith("num_batches_tracked")]


def synth_pvt(cfg, seed: int = 3030):
    """Seeded PVT weights in the checkpoint's layout: the config's periodic-Hann DFT rows and Slaney mel matrix, and
    random values for everything the reference initialises to a constant (LayerNorm and bn0 affine, bn0's running
    statistics -- centred on the log-mel range of a speech-level clip --, every bias), so no term is absent."""
    shapes = pvt_param_shapes(cfg)
    sd = synth_state_dict(shapes, seed, convtranspose_prefixes=(), gains={"fc_audioset.weight": 3.0})
    sd["spectrogram_extractor.stft.conv_real.weight"], sd["spectrogram_extractor.stft.conv_imag.weight"] = \
        stft_dft_weights(int(cfg["window_size"]))
    sd["logmel_extractor.melW"] = torch.from_numpy(np.ascontiguousarray(slaney_mel(
        cfg["sample_rate"], cfg["window_size"], cfg["mel_bins"], cfg["fmin"], cfg["fmax"]).T))
    g = torch.Generator().manual_seed(int(seed) + 1)
    sd["bn0.running_mean"] = -30.0 + 5.0 * torch.randn(shapes["bn0.running_mean"], generator=g)
    sd["bn0.running_var"] = 200.0 * (0.5 + torch.rand(shapes["bn0.running_var"], generator=g))
    sd["bn0.num_batches_tracked"] = torch.tensor(0, dtype=torch.long)
    return sd


def synth_pvt_wav(n_samples: int, seed: int = 33, sr: int = 32000) -> torch.Tensor:
    """A seeded mono test clip [n_samples] fp32: a few sines under a slow envelope plus noise."""
    rs = np.random.RandomState(int(seed))
    t = np.arange(int(n_samples)) / sr
    x = sum(0.2 / (j + 1) * np.sin(2 * np.pi * rs.uniform(80, 6000) * t + rs.uniform(0, 6)) for j in range(5))
    x = x * (0.6 + 0.4 * np.sin(2 * np.pi * rs.uniform(0.5, 3) * t)) + 0.03 * rs.randn(int(n_samples))
    return torch.from_numpy(x.astype(np.float32))


# ---------------------------------------------------------------------------------------------- target sound detection
# RaDur_fusion of the TargetSoundDetection tool (audio_detection/target_sound_detection/src/models.py:1109-1291;
# audio-chatgpt.py:775-806 builds it with inputdim=64, outputdim=2 and tao = 0.6).  The checkpoint's run_config.pth,
# which holds att_pool, enhancement, top and time_resolution, is not in the reference tree: TSD_DEFAULT takes the
# heaviest path (attention pooling and the enhancement pass) with the tool's default time_resolution and tao, and top
# is a stand-in.  The network sizes are fixed inside the reference classes.
TSD_DEFAULT = dict(time_resolution=125, att_pool=True, enhancement=True, top=10, tao=0.6, mel_bins=64, outputdim=2)
TSD_DET_CHANNELS = (128, 256, 512)       # Cnn10_mul_scale.conv_block2..4
TSD_EMB = 128                            # Cnn14.fc1 width
TSD_GRU = 512
# Cnn10_mul_scale's pool sizes by scale (models.py:436-455); CDur_CNN_mul_scale_fusion maps time_resolution 125 / 250 /
# 500 / anything else to scale 8 / 4 / 2 / 0
TSD_POOLS = {8: ((2, 2), (2, 2), (2, 4), (1, 4)), 4: ((2, 2), (2, 2), (1, 4), (1, 4)),
             2: ((2, 2), (1, 2), (1, 4), (1, 4)), 0: ((1, 2), (1, 2), (1, 4), (1, 4))}
TSD_ENC_POOLS = ((2, 2),) * 3 + ((1, 2),) * 3


def tsd_scale(time_resolution) -> int:
    return {125: 8, 250: 4, 500: 2}.get(int(time_resolution), 0)


def tsd_stem_rows(T: int, ph: int):
    """The stem's pooled row counts (H1, H2, H3, m) for a T-frame mel: the 1 x 1 / 3 x 3 / 5 x 5 GLU branches (all with
    padding 1) pooled by ph rows, and m = min(min(H1, 500), H2, H3 + 1), the rows the concat keeps."""
    if T < 3 or T - 2 < ph:
        raise ValueError(f"clip of {T} frames is too short: the 5 x 5 stem branch has no pooled row")
    H1, H2, H3 = (T + 2) // ph, T // ph, (T - 2) // ph
    return H1, H2, H3, min(min(H1, 500), H2, H3 + 1)


def tsd_frames(cfg, T: int, Tr: int):
    """(T', Tr', Te): the detection frames of a T-frame clip, the reference encoder's frames of a Tr-frame reference and
    the mixture encoder's frames (0 without enhancement) -- the Python twin of agpt_tsd_frames.  Raises ValueError when
    any of them would be 0."""
    T, Tr = int(T), int(Tr)
    pools = TSD_POOLS[tsd_scale(cfg["time_resolution"])]
    H = tsd_stem_rows(T, pools[0][0])[3]
    for ph, _ in pools[1:]:
        if H < ph:
            raise ValueError(f"clip of {T} frames is too short: a detection pool has no output row")
        H //= ph
    if Tr < 8:
        raise ValueError(f"reference of {Tr} frames is too short: Cnn14 needs 8 frames for one output frame")
    Te = 0
    if cfg["enhancement"]:
        if T < 8:
            raise ValueError(f"clip of {T} frames is too short: the enhancement's Cnn14 needs 8 frames")
        Te = T // 8
    return H, Tr // 8, Te


def tsd_param_shapes(cfg) -> "OrderedDict[str, Tuple[int, ...]]":
    """State-dict keys and shapes of the reference RaDur_fusion in state-dict order: encoder (Cnn14 with the
    torchlibrosa front end and fc_audioset it never runs), detection (Cnn10_mul_scale, GRU, fc, fusion, outputlayer),
    q, k, q_ee, k_ee, bn, EE_fusion."""
    s: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    e = "encoder."
    s[e + "spectrogram_extractor.stft.conv_real.weight"] = (513, 1, 1024)     # Cnn14() defaults: window 1024, 32 kHz
    s[e + "spectrogram_extractor.stft.conv_imag.weight"] = (513, 1, 1024)
    s[e + "logmel_extractor.melW"] = (513, 64)
    _bn_shapes(s, e + "bn0", 64)
    cin = 1
    for i, c in enumerate(CNN14_CHANNELS):
        p = f"{e}conv_block{i + 1}."
        s[p + "conv1.weight"] = (c, cin, 3, 3)
        s[p + "conv2.weight"] = (c, c, 3, 3)
        _bn_shapes(s, p + "bn1", c)
        _bn_shapes(s, p + "bn2", c)
        cin = c
    s[e + "fc1.weight"] = (TSD_EMB, cin); s[e + "fc1.bias"] = (TSD_EMB,)
    s[e + "fc_audioset.weight"] = (527, TSD_EMB); s[e + "fc_audioset.bias"] = (527,)
    f = "detection.features."
    for j, k in enumerate((1, 3, 5)):
        s[f"{f}conv_block1_{j + 1}.conv1.weight"] = (64, 1, k, k)
        _bn_shapes(s, f"{f}conv_block1_{j + 1}.bn1", 64)
    cin = 96
    for i, c in enumerate(TSD_DET_CHANNELS):
        p = f"{f}conv_block{i + 2}."
        s[p + "conv1.weight"] = (c, cin, 3, 3)
        s[p + "conv2.weight"] = (c, c, 3, 3)
        _bn_shapes(s, p + "bn1", c)
        _bn_shapes(s, p + "bn2", c)
        cin = c
    for sfx in ("", "_reverse"):
        s[f"detection.gru.weight_ih_l0{sfx}"] = (3 * TSD_GRU, TSD_GRU)
        s[f"detection.gru.weight_hh_l0{sfx}"] = (3 * TSD_GRU, TSD_GRU)
        s[f"detection.gru.bias_ih_l0{sfx}"] = (3 * TSD_GRU,)
        s[f"detection.gru.bias_hh_l0{sfx}"] = (3 * TSD_GRU,)
    s["detection.fc.weight"] = (256, 2 * TSD_GRU); s["detection.fc.bias"] = (256,)
    s["detection.fusion.fuse_layer1.conv.weight"] = (1024, TSD_EMB, 1); s["detection.fusion.fuse_layer1.conv.bias"] = (1024,)
    s["detection.fusion.fuse_layer2.conv.weight"] = (1024, 512, 1); s["detection.fusion.fuse_layer2.conv.bias"] = (1024,)
    O = int(cfg["outputdim"])
    s["detection.outputlayer.weight"] = (O, 256); s["detection.outputlayer.bias"] = (O,)
    for n in ("q", "k", "q_ee", "k_ee"):
        s[n + ".weight"] = (TSD_EMB, TSD_EMB); s[n + ".bias"] = (TSD_EMB,)
    _bn_shapes(s, "bn", TSD_EMB)
    for n in ("fuse_layer1", "fuse_layer2"):
        s[f"EE_fusion.{n}.conv.weight"] = (4 * TSD_EMB, TSD_EMB, 1); s[f"EE_fusion.{n}.conv.bias"] = (4 * TSD_EMB,)
    return s


def tsd_engine_keys(cfg):
    """The keys agpt_tsd_create consumes, in its order: the state dict without the encoder's front end (its forward takes
    a mel), encoder.fc_audioset and every num_batches_tracked."""
    skip = ("encoder.spectrogram_extractor.", "encoder.logmel_extractor.", "encoder.bn0.", "encoder.fc_audioset.")
    return [k for k in tsd_param_shapes(cfg) if not k.startswith(skip) and not k.endswith("num_batches_tracked")]


def synth_tsd(cfg, seed: int = 7171, out_shift: float = 0.0):
    """Seeded RaDur_fusion weights in the checkpoint's layout: convs at He gain, BatchNorm running statistics with
    positive variance, the encoder's front end as torchlibrosa builds it for Cnn14()'s defaults, and an outputlayer at 4x
    gain whose class-0 bias is moved by out_shift (the fixtures use it to put the gate tao inside the top-k scores)."""
    shapes = tsd_param_shapes(cfg)
    sd = synth_state_dict(shapes, seed, convtranspose_prefixes=(),
                          gains={"encoder.conv_block": math.sqrt(2.0), "detection.features.conv_block": math.sqrt(2.0),
                                 "detection.outputlayer.weight": 4.0})
    sd["encoder.spectrogram_extractor.stft.conv_real.weight"], sd["encoder.spectrogram_extractor.stft.conv_imag.weight"] = \
        stft_dft_weights(1024)
    sd["encoder.logmel_extractor.melW"] = torch.from_numpy(np.ascontiguousarray(slaney_mel(32000, 1024, 64, 50, 14000).T))
    g = torch.Generator().manual_seed(int(seed) + 1)
    for k, shape in shapes.items():
        if k.endswith("num_batches_tracked"):
            sd[k] = torch.tensor(0, dtype=torch.long)
        elif k.endswith("running_mean"):
            sd[k] = 0.1 * torch.randn(shape, generator=g)
        elif k.endswith("running_var"):
            sd[k] = 0.5 + torch.rand(shape, generator=g)
    sd["detection.outputlayer.bias"] = sd["detection.outputlayer.bias"].clone()
    sd["detection.outputlayer.bias"][0] += float(out_shift)
    return sd


def synth_tsd_mel(T: int, seed: int, B: int = 1) -> torch.Tensor:
    """Seeded log-mel clips [B][T][64] fp32 on the scale of the tool's log(mel + eps) features: a per-band floor, a few
    sustained events with their own spectral shape, and noise."""
    rs = np.random.RandomState(int(seed))
    T = int(T)
    t = np.arange(T)[:, None]
    x = np.empty((B, T, 64))
    for b in range(B):
        v = -7.0 + 1.5 * np.cos(np.arange(64) / 64 * np.pi)[None, :] + 0.8 * rs.randn(T, 64)
        for _ in range(3):
            on = rs.randint(0, max(T - 4, 1))
            dur = rs.randint(4, max(T // 3, 5))
            env = ((t >= on) & (t < on + dur)).astype(np.float64)
            v = v + env * (3.0 + 2.0 * rs.rand(1, 64) + 0.5 * np.sin(t / rs.uniform(2, 10)))
        x[b] = v
    return torch.from_numpy(x.astype(np.float32))


# ---------------------------------------------------------------------------------------------------------- Binaural
# mono2binaural/src/models.py BinauralNetwork(view_dim=7, warpnet_layers=4, warpnet_channels=64): the Binaural tool's
# network (audio-chatgpt.py:713-773).  The view is 7 x K: a position (metres) and a scalar-last quaternion per frame,
# one frame per 400 samples at 48 kHz.
BINAURAL = dict(layers=4, channels=64)
BINAURAL_SMALL = dict(layers=2, channels=16)
BINAURAL_VIEW_DIM = 7
BINAURAL_HOP = 400


def binaural_param_shapes(cfg) -> "OrderedDict[str, Tuple[int, ...]]":
    """The state-dict keys and shapes of BinauralNetwork (Warpnet's convs; its warpers hold no parameters), in the order
    agpt_binaural_create consumes them."""
    C = int(cfg["channels"])
    out: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    for l in range(int(cfg["layers"])):
        out[f"warper.layers.{l}.weight"] = (C, BINAURAL_VIEW_DIM if l == 0 else C, 2)
        out[f"warper.layers.{l}.bias"] = (C,)
    out["warper.linear.weight"] = (2, C, 1)
    out["warper.linear.bias"] = (2,)
    return out


def synth_binaural(cfg, seed: int = 4242, warp_gain: float = 250.0):
    """Seeded BinauralNetwork weights: He-gain convs and a linear head at warp_gain, so the neural warp spans about a
    few hundred samples either side of zero -- enough to push some frames' total warp above 0, where the reference clips
    it."""
    return synth_state_dict(binaural_param_shapes(cfg), seed, convtranspose_prefixes=(),
                            gains={"warper.layers.": math.sqrt(2.0), "warper.linear.": warp_gain})


def synth_binaural_view(K: int, seed: int, B: int = 1) -> torch.Tensor:
    """A seeded trajectory [B][7][K] fp32: the transmitter wanders 0.5-3 m from the listener (a smooth random walk in
    direction and distance) and turns through random unit quaternions (x, y, z, w), a new one every few frames."""
    rs = np.random.RandomState(int(seed))
    out = np.empty((B, BINAURAL_VIEW_DIM, int(K)), dtype=np.float64)
    for b in range(B):
        d = np.cumsum(rs.randn(int(K), 3) * 0.05, axis=0) + rs.randn(3)
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        r = 1.75 + 1.25 * np.sin(np.cumsum(rs.uniform(0.0, 0.2, int(K))) + rs.uniform(0, 2 * np.pi))
        out[b, 0:3] = (d * r[:, None]).T
        q = rs.randn(int(K), 4)
        hold = rs.randint(1, 6)
        q = np.repeat(q[::hold], hold, axis=0)[: int(K)]
        out[b, 3:7] = (q / np.linalg.norm(q, axis=1, keepdims=True)).T
    return torch.from_numpy(out.astype(np.float32))


def synth_binaural_mono(L: int, seed: int, B: int = 1) -> torch.Tensor:
    """Seeded mono clips [B][L] as a loaded 16-bit wav is: int16 PCM / 32768.  A few sines up to 2 kHz under a slow
    envelope, plus a little noise."""
    rs = np.random.RandomState(int(seed))
    t = np.arange(int(L)) / 48000.0
    out = np.empty((B, int(L)))
    for b in range(B):
        x = sum(rs.uniform(0.05, 0.25) * np.sin(2 * np.pi * rs.uniform(50, 2000) * t + rs.uniform(0, 2 * np.pi)) for _ in range(4))
        x = x * (0.6 + 0.4 * np.sin(2 * np.pi * rs.uniform(0.2, 2.0) * t)) + 0.01 * rs.randn(int(L))
        out[b] = x
    pcm = np.clip(np.round(out * 32768.0), -32768, 32767).astype(np.int16)
    return torch.from_numpy(pcm.astype(np.float32) / 32768.0)


def binaural_nearest(T: int, K: int) -> np.ndarray:
    """F.interpolate(mode='nearest', size=T) source frame of each of T samples from K frames (UpSample.h nearest_idx:
    the identity when K == T, i >> 1 when T == 2K, else min(floor(float(i) * (float(K) / float(T))), K - 1) in fp32)."""
    i = np.arange(int(T), dtype=np.int64)
    if K == T:
        return i
    if T == 2 * K:
        return i >> 1
    scale = np.float32(K) / np.float32(T)
    return np.minimum(np.floor(i.astype(np.float32) * scale).astype(np.int64), int(K) - 1)


def binaural_chunks(L: int, Kv: int, chunk_size: int = 48000, rec_field: int = 800):
    """The Binaural tool's chunk plan (audio-chatgpt.py:729-766) for a mono clip of L samples and a view of Kv frames.

    When Kv * 400 != L the clip is trimmed to a multiple of 400 and a longer view keeps its last L' / 400 frames (the
    tool slices from m_a; its random start is never used); a shorter view is left as it is.  Chunk i (a multiple of
    chunk_size) reads mono[max(0, i - rec_field) : i + chunk_size] and view[max(0, i - rec_field) // 400 : (i +
    chunk_size) // 400]; every chunk after the first keeps binaural[:, -(T - rec_field):].

    Returns (L_out, rows): rows are dicts of mono_off, T, view_off (a frame of the untrimmed view), K, keep (the first
    kept sample) and out_off, in the output's order.  A chunk whose view slice is empty has K = 0: the reference's
    F.interpolate raises there."""
    L, Kv, cs, rf = int(L), int(Kv), int(chunk_size), int(rec_field)
    vs, kv = 0, Kv
    if Kv * BINAURAL_HOP != L:
        L = (L // BINAURAL_HOP) * BINAURAL_HOP
        if Kv * BINAURAL_HOP > L:
            vs = Kv - L // BINAURAL_HOP
            kv = L // BINAURAL_HOP
    rows, out = [], 0
    for n, i in enumerate(range(0, L, cs)):
        m0, m1 = max(0, i - rf), min(L, i + cs)
        v0, v1 = max(0, i - rf) // BINAURAL_HOP, min(kv, (i + cs) // BINAURAL_HOP)
        T = m1 - m0
        keep = 0 if n == 0 else slice(-(T - rf), None).indices(T)[0]
        rows.append(dict(mono_off=m0, T=T, view_off=vs + min(v0, kv), K=max(0, v1 - v0), keep=keep, out_off=out))
        out += T - keep
    return out, rows


# --------------------------------------------------------------------------------------------------- wav2vec2 ASR
# transformers' Wav2Vec2ForCTC with facebook/wav2vec2-base-960h's config (the Wav2Vec2Config() defaults): the model
# GenerSpeechInfer.preprocess_input transcribes the reference clip with (NeuralSeq/inference/tts/base_tts_infer.py:38-42,
# 83-101).  Keys are Wav2Vec2Config's attribute names.
W2V_BASE = dict(conv_dim=(512,) * 7, conv_kernel=(10, 3, 3, 3, 3, 2, 2), conv_stride=(5, 2, 2, 2, 2, 2, 2),
                hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
                num_conv_pos_embeddings=128, num_conv_pos_embedding_groups=16, vocab_size=32, layer_norm_eps=1e-5,
                feat_extract_norm="group", do_stable_layer_norm=False, hidden_act="gelu", feat_extract_activation="gelu",
                conv_bias=False)
W2V_SMALL = dict(W2V_BASE, num_hidden_layers=2)     # base widths (the positional conv's 48-channel groups), 2 layers
W2V_SR = 16000                                      # the processor's (and GenerSpeech's) sampling rate
W2V_POS_GROUP = 48                                  # channels per positional-conv group the engine runs
W2V_HEAD_DIMS = (8, 16, 32, 40, 64, 80, 128)        # head dims of the attention kernel


def _w2v(cfg, key):
    return cfg[key] if isinstance(cfg, dict) else getattr(cfg, key)


def w2v_check(cfg):
    """Raise ValueError unless the engine covers cfg (a W2V_* dict or a Wav2Vec2Config): the "group" feature-extractor
    norm, post-LN layers, GELU everywhere, bias-free convs of one width, 48-channel positional-conv groups and a head dim
    the attention kernel takes.  wav2vec2-large-960h-lv60-self (stable layer norm, LayerNorm conv encoder) is refused."""
    def need(ok, what):
        if not ok:
            raise ValueError(f"audiogpt_b200.Wav2Vec2ForCTC does not cover this config: {what}")
    need(_w2v(cfg, "feat_extract_norm") == "group", f"feat_extract_norm={_w2v(cfg, 'feat_extract_norm')!r} (needs 'group')")
    need(not _w2v(cfg, "do_stable_layer_norm"), "do_stable_layer_norm=True (the large / lv60 layout)")
    need(_w2v(cfg, "hidden_act") == "gelu" and _w2v(cfg, "feat_extract_activation") == "gelu", "activations other than gelu")
    need(not _w2v(cfg, "conv_bias"), "conv_bias=True")
    dims, ks, ss = list(_w2v(cfg, "conv_dim")), list(_w2v(cfg, "conv_kernel")), list(_w2v(cfg, "conv_stride"))
    need(len(dims) == len(ks) == len(ss) and 1 <= len(dims) <= 8, "1..8 conv layers of matching conv_dim / kernel / stride")
    need(len(set(dims)) == 1 and dims[0] % 32 == 0 and 32 <= dims[0] <= 1024, "conv widths must be equal (a multiple of 32, <= 1024)")
    need(1 <= ks[0] <= 16 and 1 <= ss[0] <= 64, "conv_kernel[0] must be <= 16")
    need(all(1 <= s <= 8 and -(-k // s) <= 12 for k, s in zip(ks[1:], ss[1:])), "conv_kernel / conv_stride past layer 0 "
         "must give at most 12 super-row taps")
    H, nh = int(_w2v(cfg, "hidden_size")), int(_w2v(cfg, "num_attention_heads"))
    need(H % nh == 0 and H // nh in W2V_HEAD_DIMS, f"head dim {H / nh:g} (needs one of {W2V_HEAD_DIMS})")
    need(H == W2V_POS_GROUP * int(_w2v(cfg, "num_conv_pos_embedding_groups")),
         "hidden_size must be 48 * num_conv_pos_embedding_groups")
    need(1 <= int(_w2v(cfg, "num_conv_pos_embeddings")) <= 128, "num_conv_pos_embeddings must be <= 128")
    if not isinstance(cfg, dict):
        need(not getattr(cfg, "add_adapter", False), "add_adapter=True")


def w2v_param_shapes(cfg) -> "OrderedDict[str, Tuple[int, ...]]":
    """State-dict keys and shapes of Wav2Vec2ForCTC (group-norm, post-LN layout) in state-dict order."""
    s: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    dims, ks = [int(v) for v in _w2v(cfg, "conv_dim")], [int(v) for v in _w2v(cfg, "conv_kernel")]
    H, I, K = int(_w2v(cfg, "hidden_size")), int(_w2v(cfg, "intermediate_size")), int(_w2v(cfg, "num_conv_pos_embeddings"))
    G = int(_w2v(cfg, "num_conv_pos_embedding_groups"))
    w = "wav2vec2."
    s[w + "masked_spec_embed"] = (H,)
    for i, (c, k) in enumerate(zip(dims, ks)):
        p = f"{w}feature_extractor.conv_layers.{i}."
        s[p + "conv.weight"] = (c, 1 if i == 0 else dims[i - 1], k)
        if i == 0:
            s[p + "layer_norm.weight"] = (c,); s[p + "layer_norm.bias"] = (c,)
    C = dims[-1]
    s[w + "feature_projection.layer_norm.weight"] = (C,); s[w + "feature_projection.layer_norm.bias"] = (C,)
    s[w + "feature_projection.projection.weight"] = (H, C); s[w + "feature_projection.projection.bias"] = (H,)
    p = w + "encoder.pos_conv_embed.conv."
    s[p + "bias"] = (H,)
    s[p + "parametrizations.weight.original0"] = (1, 1, K)
    s[p + "parametrizations.weight.original1"] = (H, H // G, K)
    s[w + "encoder.layer_norm.weight"] = (H,); s[w + "encoder.layer_norm.bias"] = (H,)
    for i in range(int(_w2v(cfg, "num_hidden_layers"))):
        p = f"{w}encoder.layers.{i}."
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            s[f"{p}attention.{n}.weight"] = (H, H); s[f"{p}attention.{n}.bias"] = (H,)
        s[p + "layer_norm.weight"] = (H,); s[p + "layer_norm.bias"] = (H,)
        s[p + "feed_forward.intermediate_dense.weight"] = (I, H); s[p + "feed_forward.intermediate_dense.bias"] = (I,)
        s[p + "feed_forward.output_dense.weight"] = (H, I); s[p + "feed_forward.output_dense.bias"] = (H,)
        s[p + "final_layer_norm.weight"] = (H,); s[p + "final_layer_norm.bias"] = (H,)
    s["lm_head.weight"] = (int(_w2v(cfg, "vocab_size")), H); s["lm_head.bias"] = (int(_w2v(cfg, "vocab_size")),)
    return s


def w2v_lengths(cfg, n_samples: int) -> List[int]:
    """Output length of each conv of the feature encoder for n_samples of input ((T - k) // s + 1 in turn; 0 from the
    first layer without a frame on) -- the twin of agpt_w2v_frames, whose answer is the last entry."""
    out, t = [], int(n_samples)
    for k, s in zip(_w2v(cfg, "conv_kernel"), _w2v(cfg, "conv_stride")):
        t = (t - int(k)) // int(s) + 1 if t >= int(k) else 0
        out.append(t)
    return out


def w2v_superrow_weight(w: torch.Tensor, stride: int) -> torch.Tensor:
    """A stride-s Conv1d weight [Co][Ci][k] as the stride-1 conv over super-rows (s consecutive rows of [T][Ci] read as
    one row of s Ci channels): [Co][s Ci][ceil(k / s)], tap t's channel block j holding w[:, :, t s + j] (zero past k).
    Output row p then reads super-rows p .. p + ceil(k / s) - 1.  The engine's only copy of this packing."""
    Co, Ci, k = w.shape
    s = int(stride)
    nt = -(-k // s)
    out = w.new_zeros((Co, s, Ci, nt))
    for t in range(nt):
        for j in range(s):
            if t * s + j < k:
                out[:, j, :, t] = w[:, :, t * s + j]
    return out.reshape(Co, s * Ci, nt)


def w2v_fold_pos_weight(g: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """The positional conv's weight_norm(dim=2) folded: g v / |v|, the norm over dims (0, 1) per tap (what the module's
    parametrization computes)."""
    return torch._weight_norm(v, g, 2)


def w2v_engine_cfg(cfg) -> dict:
    """The fields of agpt_w2v_cfg for cfg (after w2v_check)."""
    w2v_check(cfg)
    return dict(conv_layers=len(_w2v(cfg, "conv_dim")), conv_dim=int(_w2v(cfg, "conv_dim")[0]),
                conv_kernel=[int(v) for v in _w2v(cfg, "conv_kernel")], conv_stride=[int(v) for v in _w2v(cfg, "conv_stride")],
                hidden_size=int(_w2v(cfg, "hidden_size")), num_layers=int(_w2v(cfg, "num_hidden_layers")),
                num_heads=int(_w2v(cfg, "num_attention_heads")), intermediate_size=int(_w2v(cfg, "intermediate_size")),
                num_conv_pos_embeddings=int(_w2v(cfg, "num_conv_pos_embeddings")),
                num_conv_pos_embedding_groups=int(_w2v(cfg, "num_conv_pos_embedding_groups")),
                vocab_size=int(_w2v(cfg, "vocab_size")), layer_norm_eps=float(_w2v(cfg, "layer_norm_eps")))


def w2v_engine_weights(cfg, sd) -> List[torch.Tensor]:
    """The arrays agpt_w2v_create consumes, in its order, from a Wav2Vec2ForCTC state dict: conv0 and its GroupNorm;
    conv 1.. packed by w2v_superrow_weight; the feature projection; the positional conv's folded weight, then its bias;
    encoder.layer_norm; per layer q, k, v (reordered from the state dict's k, v, q into the [Q | K | V] GEMM), out_proj,
    layer_norm, intermediate_dense, output_dense, final_layer_norm; lm_head.  masked_spec_embed (training only) is
    left out."""
    w = "wav2vec2."
    out = []
    fe = w + "feature_extractor.conv_layers."
    out += [sd[fe + "0.conv.weight"], sd[fe + "0.layer_norm.weight"], sd[fe + "0.layer_norm.bias"]]
    for i, s in enumerate(_w2v(cfg, "conv_stride")):
        if i:
            out.append(w2v_superrow_weight(sd[f"{fe}{i}.conv.weight"], int(s)))
    fp = w + "feature_projection."
    out += [sd[fp + "layer_norm.weight"], sd[fp + "layer_norm.bias"], sd[fp + "projection.weight"], sd[fp + "projection.bias"]]
    pc = w + "encoder.pos_conv_embed.conv."
    out += [w2v_fold_pos_weight(sd[pc + "parametrizations.weight.original0"], sd[pc + "parametrizations.weight.original1"]),
            sd[pc + "bias"]]
    out += [sd[w + "encoder.layer_norm.weight"], sd[w + "encoder.layer_norm.bias"]]
    for i in range(int(_w2v(cfg, "num_hidden_layers"))):
        p = f"{w}encoder.layers.{i}."
        for n in ("attention.q_proj", "attention.k_proj", "attention.v_proj", "attention.out_proj", "layer_norm",
                  "feed_forward.intermediate_dense", "feed_forward.output_dense", "final_layer_norm"):
            out += [sd[f"{p}{n}.weight"], sd[f"{p}{n}.bias"]]
    out += [sd["lm_head.weight"], sd["lm_head.bias"]]
    return out


def synth_w2v(cfg, seed: int = 2626):
    """Seeded Wav2Vec2ForCTC weights (synth_state_dict) with He-gain feature-encoder convs, so the GELU stack keeps its
    scale, and positional weight-norm gains g in [1.5, 2.5], so that conv is O(1) next to the projection it is added to."""
    sd = synth_state_dict(w2v_param_shapes(cfg), seed, convtranspose_prefixes=(),
                          gains={"wav2vec2.feature_extractor.conv_layers.": math.sqrt(2.0)})
    k = "wav2vec2.encoder.pos_conv_embed.conv.parametrizations.weight.original0"
    sd[k] = 1.5 + torch.rand(sd[k].shape, generator=torch.Generator().manual_seed(int(seed) + 1))
    return sd


def synth_w2v_wav(n_samples: int, seed: int, B: int = 1, offset: float = 0.0) -> torch.Tensor:
    """Seeded input_values [B][n_samples] as the base-960h processor returns them (zero mean, unit variance per clip): a
    few sines under a slow envelope plus noise, then offset added (a DC offset the GroupNorm statistics must survive)."""
    rs = np.random.RandomState(int(seed))
    t = np.arange(int(n_samples)) / float(W2V_SR)
    out = np.empty((B, int(n_samples)))
    for b in range(B):
        x = sum(rs.uniform(0.2, 1.0) * np.sin(2 * np.pi * rs.uniform(80, 3000) * t + rs.uniform(0, 2 * np.pi)) for _ in range(5))
        x = x * (0.6 + 0.4 * np.sin(2 * np.pi * rs.uniform(0.5, 4.0) * t)) + 0.1 * rs.randn(int(n_samples))
        out[b] = (x - x.mean()) / np.sqrt(x.var() + 1e-7)
    return torch.from_numpy((out + offset).astype(np.float32))


# ------------------------------------------------------------------------------------------------ emotion encoder
# The TTS_OOD tool's emotion encoder (NeuralSeq/data_gen/tts/emotion/: params_data.py, params_model.py, model.py,
# inference.py, audio.py): embed_utterance's partial slices, librosa's power mel and EmotionEncoder's nn.LSTM(40, 256, 3).
# Keys are the engine config's (agpt_emo_cfg).
EMO = dict(input_size=40, hidden_size=256, num_layers=3, embedding_size=256)
EMO_SR = 16000                # sampling_rate
EMO_N_FFT = 400               # mel_window_length 25 ms (win_length = n_fft)
EMO_HOP = 160                 # mel_window_step 10 ms
EMO_MELS = 40                 # mel_n_channels
EMO_PARTIAL_FRAMES = 160      # partials_n_frames
EMO_DBFS = -30                # audio_norm_target_dBFS: the level preprocess_wav normalises to
# librosa.feature.melspectrogram's stft padding.  audio.py passes wav and sr positionally, which only runs on librosa
# < 0.10 (numpy is pinned to 1.23.1), and those versions pad 'reflect' (0.10 changed the default to 'constant').
EMO_PAD_MODE = "reflect"


def emo_check(cfg):
    """Raise ValueError unless the engine covers cfg (an EMO-style dict): 40 mel inputs, hidden size 256, at least one
    layer, and a linear width in [1, 4096]."""
    if int(cfg["input_size"]) != EMO_MELS:
        raise ValueError(f"EmotionEncoder: input_size must be {EMO_MELS} (mel_n_channels), got {cfg['input_size']}")
    if int(cfg["hidden_size"]) != 256:
        raise ValueError(f"EmotionEncoder: the engine's LSTM has hidden_size 256, got {cfg['hidden_size']}")
    if not 1 <= int(cfg["num_layers"]) <= 16:
        raise ValueError(f"EmotionEncoder: num_layers must be in [1, 16], got {cfg['num_layers']}")
    if not 1 <= int(cfg["embedding_size"]) <= 4096:
        raise ValueError(f"EmotionEncoder: embedding_size must be in [1, 4096], got {cfg['embedding_size']}")


def emo_param_shapes(cfg) -> "OrderedDict[str, Tuple[int, ...]]":
    """EmotionEncoder's state-dict keys and shapes in state-dict order: its own parameters (the similarity scaling)
    first, then lstm (gate order i, f, g, o in every [1024] axis) and linear."""
    s: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    s["similarity_weight"] = (1,)
    s["similarity_bias"] = (1,)
    H, G = int(cfg["hidden_size"]), 4 * int(cfg["hidden_size"])
    for k in range(int(cfg["num_layers"])):
        s[f"lstm.weight_ih_l{k}"] = (G, int(cfg["input_size"]) if k == 0 else H)
        s[f"lstm.weight_hh_l{k}"] = (G, H)
        s[f"lstm.bias_ih_l{k}"] = (G,)
        s[f"lstm.bias_hh_l{k}"] = (G,)
    s["linear.weight"] = (int(cfg["embedding_size"]), H)
    s["linear.bias"] = (int(cfg["embedding_size"]),)
    return s


def emo_partials(n_samples: int, partial_utterance_n_frames: int = EMO_PARTIAL_FRAMES, min_pad_coverage: float = 0.75,
                 overlap: float = 0.5):
    """compute_partial_slices (inference.py:59-108): (wav_slices, mel_slices), lists of slices in samples and in mel
    frames of 160 samples -- the twin of agpt_emo_partials."""
    assert 0 <= overlap < 1
    assert 0 < min_pad_coverage <= 1
    n_frames = int(np.ceil((n_samples + 1) / EMO_HOP))
    frame_step = max(int(np.round(partial_utterance_n_frames * (1 - overlap))), 1)
    wav_slices, mel_slices = [], []
    steps = max(1, n_frames - partial_utterance_n_frames + frame_step + 1)
    for i in range(0, steps, frame_step):
        mel_slices.append(slice(i, i + partial_utterance_n_frames))
        wav_slices.append(slice(i * EMO_HOP, (i + partial_utterance_n_frames) * EMO_HOP))
    last = wav_slices[-1]
    coverage = (n_samples - last.start) / (last.stop - last.start)
    if coverage < min_pad_coverage and len(mel_slices) > 1:
        mel_slices, wav_slices = mel_slices[:-1], wav_slices[:-1]
    return wav_slices, mel_slices


def emo_padded_length(n_samples: int, wav_slices) -> int:
    """The length embed_utterance zero-pads the wav to: wav_slices[-1].stop when that is at least n_samples."""
    return max(int(n_samples), int(wav_slices[-1].stop))


def emo_fold_bias(b_ih: torch.Tensor, b_hh: torch.Tensor) -> torch.Tensor:
    """The one bias of a layer's input projection: b_ih + b_hh (both are added to every gate pre-activation)."""
    return b_ih + b_hh


def emo_front_weights():
    """The front end's constant arrays: the periodic-Hann DFT rows for n_fft 400, real and imaginary [201][400], and
    librosa's Slaney mel matrix (0 .. 8 kHz, area-normalised) transposed, [201][40]."""
    re, im = stft_dft_weights(EMO_N_FFT)
    mel = torch.from_numpy(np.ascontiguousarray(slaney_mel(EMO_SR, EMO_N_FFT, EMO_MELS, 0.0, EMO_SR / 2.0).T))
    return re[:, 0], im[:, 0], mel


def emo_engine_weights(cfg, sd) -> List[torch.Tensor]:
    """The arrays agpt_emo_create consumes, in its order: per layer weight_ih, weight_hh and the folded bias; linear's
    weight and bias; then emo_front_weights().  The similarity scaling (training only) is left out."""
    out = []
    for k in range(int(cfg["num_layers"])):
        p = "lstm."
        out += [sd[f"{p}weight_ih_l{k}"], sd[f"{p}weight_hh_l{k}"], emo_fold_bias(sd[f"{p}bias_ih_l{k}"], sd[f"{p}bias_hh_l{k}"])]
    out += [sd["linear.weight"], sd["linear.bias"]]
    out += list(emo_front_weights())
    return out


# weight_ih_l0's gain over N(0, 1 / 40): a -30 dBFS power mel is O(1e-2), where PyTorch's own U(-1/16, 1/16) init
# leaves every gate almost linear; this puts a real fraction of the pre-activations past |z| > 1 for synth_emotion_wav
EMO_INPUT_GAIN = 60.0


def synth_emotion(cfg=EMO, seed: int = 5353):
    """Seeded EmotionEncoder weights (synth_state_dict): weight_ih_l0 at EMO_INPUT_GAIN, the deeper layers' weight_ih
    and every weight_hh at gain 2 (so layers 1.. see O(1) pre-activations from |h| < 1), and the similarity scaling at
    its initial values (10, -5)."""
    # synth_state_dict applies the last matching prefix: weight_ih_l0 takes EMO_INPUT_GAIN
    sd = synth_state_dict(emo_param_shapes(cfg), seed, convtranspose_prefixes=(),
                          gains={"lstm.weight_ih_l": 2.0, "lstm.weight_hh_l": 2.0, "lstm.weight_ih_l0": EMO_INPUT_GAIN})
    sd["similarity_weight"] = torch.tensor([10.0])
    sd["similarity_bias"] = torch.tensor([-5.0])
    return sd


def synth_emotion_wav(n_samples: int, seed: int) -> np.ndarray:
    """A seeded speech-like clip, float32 numpy at 16 kHz, as preprocess_wav returns one: voiced harmonics of a gliding
    f0 (80-250 Hz) with a 1/k spectral tilt, a little noise, and a syllable-rate (3-6 Hz) envelope with short pauses,
    normalised to -30 dBFS."""
    rs = np.random.RandomState(int(seed))
    n = int(n_samples)
    t = np.arange(n) / float(EMO_SR)
    f0 = rs.uniform(90, 200) * (1.0 + 0.15 * np.sin(2 * np.pi * rs.uniform(0.2, 0.8) * t + rs.uniform(0, 6)))
    ph = 2 * np.pi * np.cumsum(f0) / EMO_SR
    x = sum(np.sin(k * ph + rs.uniform(0, 6)) / k for k in range(1, 30) if k * f0.max() < 0.45 * EMO_SR)
    env = np.maximum(0.0, np.sin(2 * np.pi * rs.uniform(3, 6) * t + rs.uniform(0, 6))) ** 0.7
    x = x * (0.1 + env) + 0.05 * rs.randn(n)
    x = x * 10 ** ((EMO_DBFS - 10 * np.log10(np.mean(x ** 2) + 1e-20)) / 20)
    return x.astype(np.float32)
