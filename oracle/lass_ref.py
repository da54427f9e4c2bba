"""Oracle of the SoundExtraction tool (audio-chatgpt.py:675-710): sound_extraction/utils/stft.py STFT.transform /
inverse and sound_extraction/model/LASSNet.py (bert-mini text encoder, UNetRes_FiLM with eval BatchNorm), restated
with torch fp32 ops from a state dict in the layout of audiogpt_b200.specs.lass_param_shapes.  It does not use
transformers or librosa.  Device-agnostic: the tensors decide where it runs (scripts/lass_time.py runs it on the GPU
as the eager arm)."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from audiogpt_b200 import specs


def stft_transform(wav, fwd_basis, hop):
    """STFT.transform: wav [B, N] -> (magnitude, phase) [B, n_fft/2 + 1, N // hop + 1]."""
    B, N = wav.shape
    n = fwd_basis.shape[-1]
    x = F.pad(wav.reshape(B, 1, 1, N), (n // 2, n // 2, 0, 0), mode="reflect").squeeze(1)
    y = F.conv1d(x, fwd_basis, stride=hop)
    c = n // 2 + 1
    re, im = y[:, :c], y[:, c:]
    return torch.sqrt(re ** 2 + im ** 2), torch.atan2(im, re)


def stft_inverse(mag, phase, inv_basis, hop):
    """STFT.inverse: (magnitude, phase) [B, n_fft/2 + 1, T] -> [B, 1, (T - 1) * hop]."""
    n = inv_basis.shape[-1]
    x = torch.cat([mag * torch.cos(phase), mag * torch.sin(phase)], dim=1)
    y = F.conv_transpose1d(x, inv_basis, stride=hop)
    ws = specs.stft_window_sum(mag.shape[-1], n, hop)
    idx = torch.from_numpy(np.where(ws > np.finfo(np.float32).tiny)[0]).to(y.device)
    ws = torch.from_numpy(ws).to(y.device)
    y[:, :, idx] /= ws[idx]
    y *= float(n) / hop
    return y[:, :, n // 2:][:, :, :-(n // 2)]


def text_cond(sd, cfg, input_ids, attention_mask):
    """Text_Encoder.forward(...)[0]: relu(Linear(BertModel(input_ids, attention_mask)[0][:, 0])) -> [N, 256]."""
    ids = input_ids.long()
    N, L = ids.shape
    H, nh = int(cfg["hidden_size"]), int(cfg["num_heads"])
    dh = H // nh
    eps = float(cfg["layer_norm_eps"])
    w = lambda k: sd["text_embedder.bert_layer." + k]   # noqa: E731

    def ln(x, p):
        return F.layer_norm(x, (H,), w(p + ".weight"), w(p + ".bias"), eps)

    x = w("embeddings.word_embeddings.weight")[ids] + w("embeddings.token_type_embeddings.weight")[0]
    x = ln(x + w("embeddings.position_embeddings.weight")[:L], "embeddings.LayerNorm")
    bias = torch.zeros(N, 1, 1, L, dtype=x.dtype, device=x.device).masked_fill(
        attention_mask.reshape(N, 1, 1, L).to(x.device) == 0, float("-inf"))
    for i in range(int(cfg["num_layers"])):
        p = f"encoder.layer.{i}."
        q, k, v = (F.linear(x, w(p + f"attention.self.{n}.weight"), w(p + f"attention.self.{n}.bias"))
                   .view(N, L, nh, dh).transpose(1, 2) for n in ("query", "key", "value"))
        a = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(dh) + bias, dim=-1) @ v
        a = a.transpose(1, 2).reshape(N, L, H)
        x = ln(F.linear(a, w(p + "attention.output.dense.weight"), w(p + "attention.output.dense.bias")) + x,
               p + "attention.output.LayerNorm")
        h = F.gelu(F.linear(x, w(p + "intermediate.dense.weight"), w(p + "intermediate.dense.bias")))
        x = ln(F.linear(h, w(p + "output.dense.weight"), w(p + "output.dense.bias")) + x, p + "output.LayerNorm")
    return F.relu(F.linear(x[:, 0], sd["text_embedder.linear_layer.0.weight"], sd["text_embedder.linear_layer.0.bias"]))


def _bn(sd, p, x):
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"], False, 0.0, 1e-5)


def _film(sd, p, c):
    h = F.relu(F.linear(c, sd[p + ".linear.0.weight"], sd[p + ".linear.0.bias"]))
    return F.relu(F.linear(h, sd[p + ".linear.2.weight"], sd[p + ".linear.2.bias"]))[:, :, None, None]


def _block(sd, p, x, c):
    """ConvBlockResCond.forward (modules.py:368-379)."""
    h = F.conv2d(F.leaky_relu(_bn(sd, p + ".bn1", x), 0.01), sd[p + ".conv1.weight"], padding=1) + _film(sd, p + ".film1", c)
    y = F.conv2d(F.leaky_relu(_bn(sd, p + ".bn2", h), 0.01), sd[p + ".conv2.weight"], padding=1) + _film(sd, p + ".film2", c)
    if p + ".shortcut.weight" in sd:
        r = F.conv2d(x, sd[p + ".shortcut.weight"], sd[p + ".shortcut.bias"]) + _film(sd, p + ".film_res", c)
        return r + y
    return x + y


def unet_logits(sd, sp, cond):
    """UNetRes_FiLM.forward(sp, cond, cond): sp [B, 1, T, F] -> the pre-sigmoid mask [B, 1, T, F]."""
    x = sp
    T = x.shape[2]
    x = F.pad(x, (0, 0, 0, int(np.ceil(T / 64)) * 64 - T))
    x = x[..., :x.shape[-1] - 2]
    skips = []
    for i in range(len(specs.LASS_ENC)):
        p = f"UNet.encoder_block{i + 1}"
        x = _block(sd, p + ".conv_block2", _block(sd, p + ".conv_block1", x, cond), cond)
        skips.append(x)
        x = F.avg_pool2d(x, 2)
    x = _block(sd, "UNet.conv_block7", x, cond)
    for j in range(len(specs.LASS_DEC)):
        p = f"UNet.decoder_block{j + 1}"
        x = F.conv_transpose2d(F.relu(_bn(sd, p + ".bn1", x)), sd[p + ".conv1.weight"], stride=2)[:, :, :-1, :]
        x = torch.cat([x, skips[-1 - j]], dim=1)
        x = _block(sd, p + ".conv_block3", _block(sd, p + ".conv_block2", x, cond), cond)
    x = _block(sd, "UNet.after_conv_block1", x, cond)
    x = F.conv2d(x, sd["UNet.after_conv2.weight"], sd["UNet.after_conv2.bias"])
    return F.pad(x, (0, 2))[:, :, :T, :]


def lass_forward(sd, cfg, sp, input_ids, attention_mask):
    """LASSNet.forward after tokenization: (mask, logits, cond)."""
    cond = text_cond(sd, cfg, input_ids, attention_mask)
    logits = unet_logits(sd, sp, cond)
    return torch.sigmoid(logits), logits, cond


def extract(sd, cfg, wav, input_ids, attention_mask, fwd_basis, inv_basis, hop):
    """SoundExtraction.inference after loading and tokenization: wav [1, N] -> the separated waveform [(T - 1) * hop]."""
    mag, phase = stft_transform(wav, fwd_basis, hop)
    mixed = mag.transpose(2, 1).unsqueeze(0)
    mask, _, _ = lass_forward(sd, cfg, mixed, input_ids, attention_mask)
    est = (mask * mixed).squeeze(1).permute(0, 2, 1)
    return stft_inverse(est, phase, inv_basis, hop).reshape(-1)
