"""CPU fp32 oracle for the Make-An-Audio Inpaint UNet (TEST INFRASTRUCTURE ONLY): the UNetModel built with
AttentionBlocks (use_spatial_transformer=False, no context) and, optionally, resblock_updown.

Restates, over a plain state dict (all paths under text_to_audio/Make_An_Audio/ of the reference):
  UNetModel.forward                       ldm/modules/diffusionmodules/openaimodel.py:711-744
  ResBlock._forward with up / down        openaimodel.py:207-216, 255-275 (AvgPool2d(2, 2) / nearest x2)
  AttentionBlock._forward                 openaimodel.py:278-324
  QKVAttentionLegacy / QKVAttention       openaimodel.py:347-372 / 379-406
The plain ResBlock, Downsample / Upsample, time embedding and GroupNorm come from oracle/ldm_ref.py, and so does the
DDIM sampler (ldm_schedule / ddim_sample) that drives this UNet.  The block list is re-derived from the config by
walking the constructor's rules (openaimodel.py:516-693), independent of audiogpt_b200.specs.unet_plan.  Pinned by
tests/test_inpaint_cpu.py against tests/golden/ldm_inpaint*.npz produced by the reference classes.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle.ldm_ref import _gn, resblock, timestep_embedding


def resblock_updown(sd, p, x, emb, updown):
    """ResBlock(up=True / down=True): h_upd after GN + SiLU, x_upd on the input, then in_layers.2 at the new
    resolution; the skip is the identity (the channel count does not change)."""
    h = F.silu(_gn(sd, p + ".in_layers.0", x, 1e-5))
    if updown == "down":
        h, x = F.avg_pool2d(h, 2, 2), F.avg_pool2d(x, 2, 2)
    else:
        h, x = F.interpolate(h, scale_factor=2, mode="nearest"), F.interpolate(x, scale_factor=2, mode="nearest")
    h = F.conv2d(h, sd[p + ".in_layers.2.weight"], sd[p + ".in_layers.2.bias"], padding=1)
    e = F.linear(F.silu(emb), sd[p + ".emb_layers.1.weight"], sd[p + ".emb_layers.1.bias"])
    h = h + e[:, :, None, None]
    h = F.conv2d(F.silu(_gn(sd, p + ".out_layers.0", h, 1e-5)),
                 sd[p + ".out_layers.3.weight"], sd[p + ".out_layers.3.bias"], padding=1)
    return x + h


def attention_block(sd, p, x, heads, new_order=False):
    """AttentionBlock with QKVAttentionLegacy (qkv channels [q_h; k_h; v_h] per head) or QKVAttention ([Q | K | V]);
    q and k each scaled by d^-1/4."""
    B, C, H, W = x.shape
    xf = x.reshape(B, C, H * W)
    qkv = F.conv1d(_gn(sd, p + ".norm", xf, 1e-5), sd[p + ".qkv.weight"], sd[p + ".qkv.bias"])
    d = C // heads
    if new_order:
        q, k, v = (t.reshape(B * heads, d, H * W) for t in qkv.chunk(3, dim=1))
    else:
        q, k, v = qkv.reshape(B * heads, 3 * d, H * W).split(d, dim=1)
    s = 1.0 / math.sqrt(math.sqrt(d))
    w = torch.softmax(torch.einsum("bct,bcs->bts", q * s, k * s), dim=-1)
    a = torch.einsum("bts,bcs->bct", w, v).reshape(B, C, H * W)
    h = F.conv1d(a, sd[p + ".proj_out.weight"], sd[p + ".proj_out.bias"])
    return (xf + h).reshape(B, C, H, W)


def _layout(cfg):
    """Block lists of the constructor's walk.  ('attn', heads): with legacy and num_head_channels == -1 the
    AttentionBlock receives num_head_channels=-1 and uses num_heads (num_heads_upsample in the output blocks);
    otherwise dim_head is a channel count and the head count is ch // dim_head."""
    mc, mult, nres = cfg["model_channels"], list(cfg["channel_mult"]), cfg["num_res_blocks"]
    ares = set(cfg["attention_resolutions"])
    nhc = cfg.get("num_head_channels", -1)
    updown = cfg.get("resblock_updown", False)

    def nheads(ch, upsample=False):
        if nhc != -1:
            return ch // nhc
        if cfg.get("legacy", True):
            if upsample and cfg.get("num_heads_upsample", -1) != -1:
                return cfg["num_heads_upsample"]
            return cfg["num_heads"]
        return ch // (ch // cfg["num_heads"])

    ins, ch, ds = [["conv"]], mc, 1
    for lvl, m in enumerate(mult):
        for _ in range(nres):
            ch = m * mc
            ins.append(["res"] + ([("attn", nheads(ch))] if ds in ares else []))
        if lvl != len(mult) - 1:
            ins.append(["resdown" if updown else "down"])
            ds *= 2
    mid = ["res", ("attn", nheads(ch)), "res"]
    outs = []
    for lvl, m in list(enumerate(mult))[::-1]:
        for i in range(nres + 1):
            ch = mc * m
            blk = ["res"] + ([("attn", nheads(ch, True))] if ds in ares else [])
            if lvl and i == nres:
                blk.append("resup" if updown else "up")
                ds //= 2
            outs.append(blk)
    return ins, mid, outs


def unet_forward(sd, cfg, x, t):
    """x [N, in_channels, H, W] (the latent with its concat conditioning), t [N] -> eps [N, out_channels, H, W]."""
    new_order = cfg.get("use_new_attention_order", False)
    ins, mid, outs = _layout(cfg)
    with torch.no_grad():
        emb = timestep_embedding(t, cfg["model_channels"])
        emb = F.linear(F.silu(F.linear(emb, sd["time_embed.0.weight"], sd["time_embed.0.bias"])),
                       sd["time_embed.2.weight"], sd["time_embed.2.bias"])

        def run(prefix, blk, h):
            for j, l in enumerate(blk):
                p = f"{prefix}.{j}"
                if l == "conv":
                    h = F.conv2d(h, sd[p + ".weight"], sd[p + ".bias"], padding=1)
                elif l == "res":
                    h = resblock(sd, p, h, emb)
                elif l in ("resdown", "resup"):
                    h = resblock_updown(sd, p, h, emb, l[3:])
                elif l == "down":
                    h = F.conv2d(h, sd[p + ".op.weight"], sd[p + ".op.bias"], stride=2, padding=1)
                elif l == "up":
                    h = F.interpolate(h, scale_factor=2, mode="nearest")
                    h = F.conv2d(h, sd[p + ".conv.weight"], sd[p + ".conv.bias"], padding=1)
                else:
                    h = attention_block(sd, p, h, l[1], new_order)
            return h

        hs, h = [], x
        for i, blk in enumerate(ins):
            h = run(f"input_blocks.{i}", blk, h)
            hs.append(h)
        h = run("middle_block", mid, h)
        for i, blk in enumerate(outs):
            h = torch.cat([h, hs.pop()], dim=1)
            h = run(f"output_blocks.{i}", blk, h)
        h = F.silu(_gn(sd, "out.0", h, 1e-5))
        return F.conv2d(h, sd["out.2.weight"], sd["out.2.bias"], padding=1)
