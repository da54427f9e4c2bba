"""CPU restatement of GenerSpeech's inference forward (TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py).

Follows NeuralSeq/modules/GenerSpeech/model/generspeech.py:75-260 with infer=True and global_steps past `forcing` (the
path GenerSpeechInfer.forward_model takes): the FastSpeech2 encoder and duration predictor on (enc + spk + emo), the
three LocalStyleAdaptors (prosody_util.py:172-199: WN, group_hidden_by_segs, ConvBlocks, VQEmbeddingEMA.encode), the
fairseq positions + l1_* + ProsodyAligner (nn.MultiheadAttention branch), the two pitch predictors, the FFT decoder, and
the Glow post-flow run in reverse (glow_modules.py:68-192, 282-335, 496-592, 742-767).  MixStyle is the identity in
eval.  Functional: state dict in, dict out.  Pinned against the reference module in tests/golden/generspeech_*.npz.
"""
import math

import torch
import torch.nn.functional as F

from oracle.fs2_ref import _conv_stack, _denorm, _fft, _predictor, coarse_margin, f0_to_coarse, make_positions, sinusoidal


def fold_wn(sd, p):
    """torch.nn.utils.weight_norm (dim 0): w = g * v / ||v||"""
    v, g = sd[p + ".weight_v"], sd[p + ".weight_g"]
    return g * v / v.reshape(v.shape[0], -1).norm(dim=1).reshape(-1, *([1] * (v.dim() - 1)))


def wn(sd, p, x, mask, cond, hid, layers, k):
    """WN (wavenet.py:54-78): x [B, hid, T], mask [B, 1, T] or None (= ones), cond [B, 2 hid layers, T] or None"""
    out = torch.zeros_like(x)
    for i in range(layers):
        a = F.conv1d(x, fold_wn(sd, f"{p}.in_layers.{i}"), sd[f"{p}.in_layers.{i}.bias"], padding=(k - 1) // 2)
        if cond is not None:
            a = a + cond[:, i * 2 * hid:(i + 1) * 2 * hid]
        acts = torch.tanh(a[:, :hid]) * torch.sigmoid(a[:, hid:])
        rs = F.conv1d(acts, fold_wn(sd, f"{p}.res_skip_layers.{i}"), sd[f"{p}.res_skip_layers.{i}.bias"])
        if i < layers - 1:
            x = x + rs[:, :hid]
            if mask is not None:
                x = x * mask
            out = out + rs[:, hid:]
        else:
            out = out + rs
    return out if mask is None else out * mask


def conv_blocks(sd, p, x):
    """ConvBlocks(80 -> H), 5 ResidualBlocks of 2 LN -> conv k5 -> x 5^-0.5 -> GELU -> 1x1 layers (prosody_util.py:231-335).
    x [B, T, 80] -> [B, T, H]"""
    x = x.transpose(1, 2)
    nonpad = (x.abs().sum(1) > 0).float()[:, None, :]

    def ln(y, q):
        return F.layer_norm(y.transpose(1, 2), (y.shape[1],), sd[q + ".weight"], sd[q + ".bias"], eps=1e-5).transpose(1, 2)
    for r in range(5):
        rp = (x.abs().sum(1) > 0).float()[:, None, :]
        for j in range(2):
            q = f"{p}.res_blocks.{r}.blocks.{j}"
            h = F.conv1d(ln(x, q + ".0"), sd[q + ".1.weight"], sd[q + ".1.bias"], padding=2) * 5 ** -0.5
            h = F.conv1d(F.gelu(h), sd[q + ".4.weight"], sd[q + ".4.bias"])
            x = (x + h) * rp
    x = x * nonpad
    x = ln(x, p + ".last_norm") * nonpad
    x = F.conv1d(x, sd[p + ".post_net1.weight"], sd[p + ".post_net1.bias"], padding=1) * nonpad
    return x.transpose(1, 2)


def vq_encode(emb, x):
    """VQEmbeddingEMA.encode + the straight-through output: -> (x + (q - x), indices [B, T], relative margin of the
    best distance against the second best)"""
    B, T, D = x.shape
    xf = x.reshape(-1, D)
    d = torch.addmm(torch.sum(emb ** 2, dim=1) + torch.sum(xf ** 2, dim=1, keepdim=True), xf, emb.t(), alpha=-2.0, beta=1.0)
    idx = torch.argmin(d, dim=-1)
    two = torch.topk(d.double(), 2, dim=-1, largest=False).values
    margin = float(((two[:, 1] - two[:, 0]) / two[:, 1].abs().clamp_min(1e-30)).min())
    q = F.embedding(idx, emb).view_as(x)
    return x + (q - x), idx.reshape(B, T), margin


def local_style(sd, p, ref_mels, seg):
    """LocalStyleAdaptor.forward(ref_mels, seg, no_vq=False) -> (pre-VQ prosody, quantised, indices, margin)"""
    mask = (~ref_mels[:, :, 0].eq(0)).float()[:, None, :]
    h = wn(sd, p + ".wavenet", ref_mels.transpose(1, 2), mask, None, 80, 4, 3).transpose(1, 2)
    if seg is not None:
        n = int(seg.max())
        B, T, C = h.shape
        s = h.new_zeros(B, n + 1, C).scatter_add_(1, seg[:, :, None].repeat(1, 1, C), h)
        c = h.new_zeros(B, n + 1).scatter_add_(1, seg, h.new_ones(B, T))
        h = s[:, 1:] / torch.clamp(c[:, 1:, None], min=1)
    pros = conv_blocks(sd, p + ".encoder", h)
    z, idx, margin = vq_encode(sd[p + ".vqvae.embedding"], pros)
    return pros, z, idx, margin


def aligner(sd, p, src, kv, kpm, H, nh=2):
    """ProsodyAligner (2 post-norm CrossAttenLayers, nn.MultiheadAttention with key padding): src [B, Tq, H], kv [B, Tk, H]"""
    B, Tq, _ = src.shape
    d = H // nh
    for i in range(2):
        q = f"{p}.layers.{i}"
        w, b = sd[q + ".multihead_attn.in_proj_weight"], sd[q + ".multihead_attn.in_proj_bias"]
        qq = F.linear(src, w[:H], b[:H]).reshape(B, Tq, nh, d).transpose(1, 2)
        kk = F.linear(kv, w[H:2 * H], b[H:2 * H]).reshape(B, -1, nh, d).transpose(1, 2)
        vv = F.linear(kv, w[2 * H:], b[2 * H:]).reshape(B, -1, nh, d).transpose(1, 2)
        a = (qq * d ** -0.5) @ kk.transpose(-1, -2)
        a = a.masked_fill(kpm[:, None, None, :], float("-inf")).softmax(-1)
        o = F.linear((a @ vv).transpose(1, 2).reshape(B, Tq, H), sd[q + ".multihead_attn.out_proj.weight"],
                     sd[q + ".multihead_attn.out_proj.bias"])
        src = F.layer_norm(src + o, (H,), sd[q + ".norm1.weight"], sd[q + ".norm1.bias"])
        f = F.linear(F.relu(F.linear(src, sd[q + ".linear1.weight"], sd[q + ".linear1.bias"])), sd[q + ".linear2.weight"],
                     sd[q + ".linear2.bias"])
        src = F.layer_norm(src + f, (H,), sd[q + ".norm2.weight"], sd[q + ".norm2.bias"])
    return src


def invconv_inverse(sd, p):
    """InvConvNear._get_weight() in fp32, then torch.inverse (glow_modules.py:184-193)"""
    l = sd[p + ".l"] * sd[p + ".l_mask"] + sd[p + ".eye"]
    u = sd[p + ".u"] * sd[p + ".l_mask"].transpose(0, 1).contiguous() + torch.diag(sd[p + ".sign_s"] * torch.exp(sd[p + ".log_s"]))
    return torch.inverse(torch.matmul(sd[p + ".p"], torch.matmul(l, u)).float())


def glow_reverse(sd, cfg, z, g):
    """Glow(...).forward(z, ones, g, reverse=True) with n_sqz 2, n_split 4: z [B, 80, T], g [B, G, T] -> [B, 80, 2 (T // 2)]"""
    def squeeze(x):
        b, c, t = x.shape
        t = (t // 2) * 2
        return x[:, :, :t].reshape(b, c, t // 2, 2).permute(0, 3, 1, 2).reshape(b, c * 2, t // 2)
    x, g = squeeze(z), squeeze(g)
    b_, c, t = x.shape
    hid, L, k = int(cfg["glow_hidden"]), int(cfg["glow_layers"]), int(cfg["glow_kernel"])
    for blk in reversed(range(int(cfg["glow_blocks"]))):
        p = f"post_flow.flows.{3 * blk + 2}"
        x0, x1 = x[:, :c // 2], x[:, c // 2:]
        h = F.conv1d(x0, fold_wn(sd, p + ".start"), sd[p + ".start.bias"])
        cond = F.conv1d(g, fold_wn(sd, p + ".wn.cond_layer"), sd[p + ".wn.cond_layer.bias"])
        h = wn(sd, p + ".wn", h, None, cond, hid, L, k)
        out = F.conv1d(h, sd[p + ".end.weight"], sd[p + ".end.bias"])
        m, logs = out[:, :c // 2], out[:, c // 2:]
        x = torch.cat([x0, (x1 - m) * torch.exp(-logs)], 1)
        w = invconv_inverse(sd, f"post_flow.flows.{3 * blk + 1}")
        y = x.view(b_, 2, c // 4, 2, t).permute(0, 1, 3, 2, 4).contiguous().view(b_, 4, c // 4, t)
        y = F.conv2d(y, w.view(4, 4, 1, 1))
        x = y.view(b_, 2, 2, c // 4, t).permute(0, 1, 3, 2, 4).contiguous().view(b_, c, t)
        p = f"post_flow.flows.{3 * blk}"
        x = (x - sd[p + ".bias"]) * torch.exp(-sd[p + ".logs"])
    return x.view(b_, 2, c // 2, t).permute(0, 2, 3, 1).contiguous().view(b_, c // 2, t * 2)


def generspeech_forward(sd, cfg, txt_tokens, ref_mels, ref_mel2ph, ref_mel2word, spk_embed, emo_embed, z_post, mel2ph=None,
                        f0_mean=220.0, f0_std=60.0):
    """-> (dict with GenerSpeech's inference keys, intermediates, margins).  z_post: the post-flow's input noise
    [B, 80, T_mel], already scaled by noise_scale (None: stop before the post-flow; mel_out is then the decoder's)."""
    H, nh = int(cfg["hidden_size"]), int(cfg["num_heads"])
    ret, mid, margins = {}, {}, {}
    pad = txt_tokens == 0
    src_nonpad = (~pad).float()[:, :, None]
    x = math.sqrt(H) * sd["encoder_embed_tokens.weight"][txt_tokens] + sinusoidal(make_positions(txt_tokens), H)
    enc = _fft(sd, "encoder", x, pad, nh, int(cfg["enc_ffn_kernel"]))
    spk = F.linear(spk_embed, sd["spk_embed_proj.weight"], sd["spk_embed_proj.bias"])[:, None, :]
    emo = F.linear(emo_embed, sd["emo_embed_proj.weight"], sd["emo_embed_proj.bias"])[:, None, :]
    xs = _conv_stack(sd, "dur_predictor", (enc + spk + emo) * src_nonpad, int(cfg["dur_predictor_kernel"]), (~pad).float())
    xs = xs * src_nonpad
    if mel2ph is None:
        e = xs[..., 0].exp() - 1
        margins["dur_margin"] = float((e.double() - e.double().floor() - 0.5).abs()[~pad].min())
        dur = torch.clamp(torch.round(e), min=0).long() * (~pad).long()
        ret["dur"], ret["dur_choice"] = xs, dur
        cum = torch.cumsum(dur, 1)
        prev = F.pad(cum, [1, -1])
        pos_idx = torch.arange(int(dur.sum(-1).max()))[None, None]
        mask = (pos_idx >= prev[:, :, None]) & (pos_idx < cum[:, :, None])
        mel2ph = (torch.arange(1, dur.shape[1] + 1)[None, :, None] * mask.long()).sum(1)
    else:
        ret["dur"] = xs[..., 0]
    ret["mel2ph"] = mel2ph
    dec = torch.gather(F.pad(enc, [0, 0, 1, 0]), 1, mel2ph[..., None].repeat(1, 1, H))
    tgt = (mel2ph > 0).float()[:, :, None]
    pros_sum = 0
    vq_margin = 1.0
    for lvl, seg in (("utter", None), ("ph", ref_mel2ph), ("word", ref_mel2word)):
        pre, zq, idx, m = local_style(sd, f"prosody_extractor_{lvl}", ref_mels, seg)
        vq_margin = min(vq_margin, m)
        mid[f"prosody_{lvl}"], mid[f"vq_idx_{lvl}"] = zq, idx
        pos = sinusoidal(make_positions(zq[:, :, 0]), H)
        pe = F.linear(torch.cat([zq, pos], -1), sd[f"l1_{lvl}.weight"], sd[f"l1_{lvl}.bias"])
        out = aligner(sd, f"align_{lvl}", dec, pe, pe[:, :, 0].eq(0), H)
        mid[f"aligned_{lvl}"] = out
        pros_sum = pros_sum + out
    margins["vq_margin"] = vq_margin
    k = int(cfg["predictor_kernel"])
    pp = _predictor(sd, "pitch_predictor", dec * tgt, k) + \
        _predictor(sd, "pitch_inpainter_predictor", (dec + spk + emo + pros_sum) * tgt, k)
    ret["pitch_pred"] = pp
    ppad = mel2ph == 0
    fd = _denorm(pp[:, :, 0], "standard", f0_mean, f0_std)
    fd[pp[:, :, 1] > 0] = 0
    fd[ppad] = 0
    ret["f0_denorm"] = fd
    ret["f0_denorm_pred"] = fd.clone()
    coarse = f0_to_coarse(fd.clone())
    margins["f0_margin"] = coarse_margin(fd)
    dec = (dec + spk + emo + sd["pitch_embed.weight"][coarse] + pros_sum) * tgt
    ret["decoder_inp"] = dec
    dpad = dec.abs().sum(-1).eq(0)
    x = dec + sd["decoder.pos_embed_alpha"] * sinusoidal(make_positions(dec[..., 0]), H)
    x = _fft(sd, "decoder", x, dpad, nh, int(cfg["dec_ffn_kernel"]))
    mel = F.linear(x, sd["mel_out.weight"], sd["mel_out.bias"]) * tgt
    mid["mel_pre_flow"] = mel
    ret["mel_out"] = mel
    if z_post is None:
        return ret, coarse, mid, margins
    T = mel.shape[1]
    g = torch.cat([mel, dec, spk.expand(-1, T, -1), emo.expand(-1, T, -1), pros_sum], -1).transpose(1, 2)
    ret["mel_out"] = glow_reverse(sd, cfg, z_post, g).transpose(1, 2)
    ret["x_mask"], ret["spk_embed"], ret["emo_embed"], ret["ref_prosody"] = tgt, spk, emo, pros_sum
    return ret, coarse, mid, margins
