"""CPU restatement of AutoencoderKL.encode (TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py).

The encoder half of the first stage: the Inpaint tool encodes its masked mel with it (audio-chatgpt.py:507) and
AutoencoderKL.forward runs it before decoding.  Follows text_to_audio/Make_An_Audio/ldm/models/autoencoder.py:345-349
(encode = quant_conv(encoder(x)), the posterior is built from the moments), ldm/modules/diffusionmodules/model.py:
438-459 (Encoder.forward) and :60-79 (Downsample: F.pad (0,1,0,1) then a 3x3 stride-2 conv without padding); the
ResnetBlock / AttnBlock / GroupNorm helpers are the decoder oracle's (oracle/vae_ref.py).  Functional: state dict in,
moments [B, 2*embed_dim, h, w] out.  Pinned against the reference's own Encoder + quant_conv in
tests/golden/vae_enc_small.npz / vae_enc_txt2audio.npz.
"""
import torch.nn.functional as F

from audiogpt_b200.specs import vae_encoder_plan
from oracle.vae_ref import _attn, _gn, _res, _swish


def vae_encode(sd, cfg, x):
    """x [B, in_channels, H, W] -> moments [B, 2*embed_dim, H // 8, W // 8] (for ch_mult of length 4)."""
    block_in, levels = vae_encoder_plan(cfg)
    h = F.conv2d(x, sd["encoder.conv_in.weight"], sd["encoder.conv_in.bias"], padding=1)
    for i_level, blocks, down in levels:
        for j, (cin, cout, has_attn) in enumerate(blocks):
            h = _res(h, sd, f"encoder.down.{i_level}.block.{j}", cin, cout)
            if has_attn:
                h = _attn(h, sd, f"encoder.down.{i_level}.attn.{j}")
        if down:
            h = F.conv2d(F.pad(h, (0, 1, 0, 1)), sd[f"encoder.down.{i_level}.downsample.conv.weight"],
                         sd[f"encoder.down.{i_level}.downsample.conv.bias"], stride=2)
    h = _res(h, sd, "encoder.mid.block_1", block_in, block_in)
    h = _attn(h, sd, "encoder.mid.attn_1")
    h = _res(h, sd, "encoder.mid.block_2", block_in, block_in)
    h = _swish(_gn(h, sd, "encoder.norm_out"))
    h = F.conv2d(h, sd["encoder.conv_out.weight"], sd["encoder.conv_out.bias"], padding=1)
    return F.conv2d(h, sd["quant_conv.weight"], sd["quant_conv.bias"])


def vae_encode_flops(cfg, H, W):
    """2 x MAC count of one encode (convs + attention GEMMs, quant_conv unfolded) for the measurement row."""
    block_in, levels = vae_encoder_plan(cfg)
    ch, zc, ed = cfg["ch"], cfg["z_channels"], cfg["embed_dim"]

    def res(cin, cout, n):
        return 2 * n * (9 * cin * cout + 9 * cout * cout + (cin * cout if cin != cout else 0))

    def attn(c, n):
        return 2 * n * (4 * c * c) + 2 * 2 * n * n * c

    h, w = H, W
    fl = 2 * h * w * 9 * cfg.get("in_channels", 1) * ch
    for _, blocks, down in levels:
        for cin, cout, has_attn in blocks:
            fl += res(cin, cout, h * w) + (attn(cout, h * w) if has_attn else 0)
        if down:
            c = blocks[-1][1]
            h, w = h // 2, w // 2
            fl += 2 * h * w * 9 * c * c
    hw = h * w
    fl += 2 * res(block_in, block_in, hw) + attn(block_in, hw)
    fl += 2 * hw * 9 * block_in * 2 * zc + 2 * hw * 2 * zc * 2 * ed
    return fl
