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
