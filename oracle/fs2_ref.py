"""CPU restatement of FastSpeech2.forward / FastSpeech2MIDI.forward (TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py).

Follows NeuralSeq/modules/fastspeech/fs2.py:79-226 (FastSpeech2.forward, add_dur, add_pitch, add_energy, run_decoder),
modules/diffsinger_midi/fs2.py:11-118 (MIDI encoder input), modules/fastspeech/tts_modules.py:59-143 (DurationPredictor),
:179-214 (LengthRegulator), :217-264 (Pitch / EnergyPredictor), :276-384 (FFTBlocks, FastspeechEncoder / Decoder),
modules/commons/common_layers.py:541-587 (EncSALayer), :485-521 (TransformerFFNLayer), :87-142 + utils/__init__.py:145-157
(fairseq sinusoidal positions), modules/commons/espnet_positional_embedding.py:89-113 (RelPositionalEncoding: positions
run backwards from max_len - 1), utils/pitch_utils.py:22-76 (f0_to_coarse, denorm_f0).  Functional: state dict in,
dict out.  Pinned against the reference module in tests/golden/fs2_*.npz.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

F0_MEL_MIN = 1127 * np.log(1 + 50.0 / 700)
F0_MEL_MAX = 1127 * np.log(1 + 1100.0 / 700)


def sinusoidal(pos, dim):
    """fairseq table rows for integer positions pos (0 = padding row of zeros)"""
    half = dim // 2
    f = torch.exp(torch.arange(half, dtype=torch.float) * -(math.log(10000) / (half - 1)))
    n = int(pos.max().item()) + 1
    emb = torch.arange(n, dtype=torch.float).unsqueeze(1) * f.unsqueeze(0)
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=1)
    if dim % 2 == 1:
        emb = torch.cat([emb, torch.zeros(n, 1)], dim=1)
    emb[0, :] = 0
    return emb[pos]


def make_positions(x):
    mask = x.ne(0).int()
    return (torch.cumsum(mask, dim=1).type_as(mask) * mask).long()


def rel_pe(T, d, max_len=5000):
    n = max(max_len, T)
    position = torch.arange(n - 1, -1, -1.0, dtype=torch.float32).unsqueeze(1)
    div = torch.exp(torch.arange(0, d, 2, dtype=torch.float32) * -(math.log(10000.0) / d))
    pe = torch.zeros(n, d)
    pe[:, 0::2] = torch.sin(position * div)
    pe[:, 1::2] = torch.cos(position * div)
    return pe[:T]


def f0_to_coarse(f0):
    f0_mel = 1127 * (1 + f0 / 700).log()
    f0_mel[f0_mel > 0] = (f0_mel[f0_mel > 0] - F0_MEL_MIN) * 254 / (F0_MEL_MAX - F0_MEL_MIN) + 1
    f0_mel[f0_mel <= 1] = 1
    f0_mel[f0_mel > 255] = 255
    return (f0_mel + 0.5).long()


def coarse_margin(f0):
    """distance of the scaled f0_mel from the .5 rounding boundary, over the bins that are not clamped"""
    f0_mel = 1127 * (1 + f0.double() / 700).log()
    m = (f0_mel - F0_MEL_MIN) * 254 / (F0_MEL_MAX - F0_MEL_MIN) + 1
    m = m[(f0_mel > 0) & (m > 1) & (m < 255)]
    return float((m - m.floor() - 0.5).abs().min()) if m.numel() else 1.0


def _ln(x, sd, p):
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".weight"], sd[p + ".bias"], eps=1e-5)


def _fft(sd, p, x, pad, nh, k):
    """FFTBlocks body: x [B, T, H] (positions already added), pad [B, T] bool"""
    nonpad = (~pad).float()[:, :, None]
    B, T, H = x.shape
    d = H // nh
    x = x * nonpad
    i = 0
    while f"{p}.layers.{i}.op.layer_norm1.weight" in sd:
        q = f"{p}.layers.{i}.op"
        h = _ln(x, sd, q + ".layer_norm1")
        qkv = h @ sd[q + ".self_attn.in_proj_weight"].t()
        qq, kk, vv = (t.reshape(B, T, nh, d).transpose(1, 2) for t in qkv.split(H, dim=-1))
        a = (qq * d ** -0.5) @ kk.transpose(-1, -2)
        a = a.masked_fill(pad[:, None, None, :], float("-inf")).softmax(-1)
        o = (a @ vv).transpose(1, 2).reshape(B, T, H) @ sd[q + ".self_attn.out_proj.weight"].t()
        x = (x + o) * nonpad
        h = _ln(x, sd, q + ".layer_norm2").transpose(1, 2)
        h = F.conv1d(h, sd[q + ".ffn.ffn_1.weight"], sd[q + ".ffn.ffn_1.bias"], padding=k // 2).transpose(1, 2)
        h = F.gelu(h * k ** -0.5)
        h = F.linear(h, sd[q + ".ffn.ffn_2.weight"], sd[q + ".ffn.ffn_2.bias"])
        x = (x + h) * nonpad
        i += 1
    return _ln(x, sd, p + ".layer_norm") * nonpad


def _conv_stack(sd, p, xs, k, mask=None):
    """[conv SAME -> ReLU -> LayerNorm over channels (-> x nonpad)] x n, then the Linear.  xs [B, T, C]"""
    xs = xs.transpose(1, 2)
    i = 0
    while f"{p}.conv.{i}.1.weight" in sd:
        xs = F.conv1d(F.pad(xs, ((k - 1) // 2, (k - 1) // 2)), sd[f"{p}.conv.{i}.1.weight"], sd[f"{p}.conv.{i}.1.bias"])
        xs = F.relu(xs)
        xs = F.layer_norm(xs.transpose(1, 2), (xs.shape[1],), sd[f"{p}.conv.{i}.3.weight"], sd[f"{p}.conv.{i}.3.bias"],
                          eps=1e-5).transpose(1, 2)
        if mask is not None:
            xs = xs * mask[:, None, :]
        i += 1
    return F.linear(xs.transpose(1, 2), sd[p + ".linear.weight"], sd[p + ".linear.bias"])


def _predictor(sd, p, xs, k):
    xs = xs + sd[p + ".pos_embed_alpha"] * sinusoidal(make_positions(xs[..., 0]), xs.shape[-1])
    return _conv_stack(sd, p, xs, k)


def _denorm(f0, norm, f0_mean, f0_std):
    if norm == "standard":
        return f0 * f0_std + f0_mean
    if norm == "log":
        return 2 ** f0
    return f0.clone()


def fs2_forward(sd, cfg, txt_tokens, mel2ph=None, f0=None, uv=None, energy=None, skip_decoder=False, pitch_midi=None,
                midi_dur=None, is_slur=None, use_uv=True, pitch_norm="standard", f0_mean=0.0, f0_std=1.0):
    """-> (dict with the reference's keys, coarse pitch bins, {'dur_margin', 'f0_margin', 'energy_margin'})"""
    H, nh = int(cfg["hidden_size"]), int(cfg["num_heads"])
    ret, margins = {}, {}
    pad = txt_tokens == 0
    src_nonpad = (~pad).float()[:, :, None]
    # ---- encoder (FastspeechEncoder.forward_embedding + FFTBlocks without positions)
    x = math.sqrt(H) * sd["encoder_embed_tokens.weight"][txt_tokens]
    if cfg["use_midi"]:
        x = x + sd["midi_embed.weight"][pitch_midi]
        if midi_dur is not None:
            x = x + F.linear(midi_dur[:, :, None], sd["midi_dur_layer.weight"], sd["midi_dur_layer.bias"])
        if is_slur is not None:
            x = x + sd["is_slur_embed.weight"][is_slur]
    if cfg["use_pos_embed"]:
        if cfg["rel_pos"]:
            x = x * math.sqrt(H) + rel_pe(x.shape[1], H)[None]
        else:
            x = x + sinusoidal(make_positions(txt_tokens), H)
    enc = _fft(sd, "encoder", x, pad, nh, int(cfg["enc_ffn_kernel"]))
    # ---- durations, length regulator
    xs = _conv_stack(sd, "dur_predictor", enc * src_nonpad, int(cfg["dur_predictor_kernel"]), (~pad).float())
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
    pitch_inp = dec * tgt
    coarse = None
    k = int(cfg["predictor_kernel"])
    if cfg["pitch_type"] == "ph":
        pp = _predictor(sd, "pitch_predictor", enc * src_nonpad, k)
        ret["pitch_pred"] = pp
        ff = pp[:, :, 0] if f0 is None else f0
        ret["f0_denorm"] = fd = _denorm(ff, pitch_norm, f0_mean, f0_std)
        coarse = f0_to_coarse(fd.clone())
        margins["f0_margin"] = coarse_margin(fd)
        dec = dec + sd["pitch_embed.weight"][torch.gather(F.pad(coarse, [1, 0]), 1, mel2ph)]
    elif cfg["pitch_type"] == "frame":
        pp = _predictor(sd, "pitch_predictor", pitch_inp, k)
        ppad = mel2ph == 0
        ff = pp[:, :, 0] if f0 is None else f0.clone()
        if use_uv and uv is None:
            uv = pp[:, :, 1] > 0
        fd = _denorm(ff, pitch_norm, f0_mean, f0_std)
        if uv is not None and use_uv:
            fd[uv > 0] = 0
        fd[ppad] = 0
        ff[ppad] = 0            # the reference's in-place write: zeroes pitch_pred[..., 0] when it is the f0 used
        ret["pitch_pred"], ret["f0_denorm"] = pp, fd
        coarse = f0_to_coarse(fd.clone())
        margins["f0_margin"] = coarse_margin(fd)
        dec = dec + sd["pitch_embed.weight"][coarse]
    if cfg["use_energy_embed"]:
        ep = _predictor(sd, "energy_predictor", pitch_inp, k)[:, :, 0]
        ret["energy_pred"] = ep
        ee = ep if energy is None else energy
        s = ee.double() * 64
        margins["energy_margin"] = float((s - s.round()).abs().min())
        dec = dec + sd["energy_embed.weight"][torch.clamp(ee * 256 // 4, max=255).long()]
    ret["decoder_inp"] = dec = dec * tgt
    if skip_decoder:
        return ret, coarse, margins
    dpad = dec.abs().sum(-1).eq(0)
    x = dec + sd["decoder.pos_embed_alpha"] * sinusoidal(make_positions(dec[..., 0]), H)
    x = _fft(sd, "decoder", x, dpad, nh, int(cfg["dec_ffn_kernel"]))
    ret["mel_out"] = F.linear(x, sd["mel_out.weight"], sd["mel_out.bias"]) * tgt
    return ret, coarse, margins
