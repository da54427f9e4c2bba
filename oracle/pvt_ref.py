"""Plain-torch restatement of the SoundDetection tool's PVT in eval mode (audio_detection/audio_infer/pytorch/models.py:
PVT.forward, PyramidVisionTransformerV2, Block, Attention, Mlp, DWConv, OverlapPatchEmbed): log-mel front end, four
pyramid stages, framewise head.  Works on a {key: tensor} state dict in the reference's layout, in the dtype of the
weights (fp32, or fp64 for tolerance setting: ``to_double``).  Written from the network's description, independent of
the engine."""
import torch
import torch.nn.functional as F

from audiogpt_b200 import specs


def to_double(sd):
    return {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}


def logmel(sd, cfg, x):
    """x [B, n] -> bn0(log-mel) [B, 1, T, mel_bins], T = n // hop + 1."""
    n = int(cfg["window_size"])
    xp = F.pad(x[:, None, :], (n // 2, n // 2), mode="reflect")
    re = F.conv1d(xp, sd["spectrogram_extractor.stft.conv_real.weight"], stride=int(cfg["hop_size"]))
    im = F.conv1d(xp, sd["spectrogram_extractor.stft.conv_imag.weight"], stride=int(cfg["hop_size"]))
    power = (re ** 2 + im ** 2).transpose(1, 2)[:, None]                      # [B, 1, T, n/2 + 1]
    lm = 10.0 * torch.log10(torch.clamp(torch.matmul(power, sd["logmel_extractor.melW"]), min=1e-10))
    bn = F.batch_norm(lm.transpose(1, 3), sd["bn0.running_mean"], sd["bn0.running_var"], sd["bn0.weight"], sd["bn0.bias"],
                      False, 0.0, specs.BN_EPS)
    return bn.transpose(1, 3)


def _ln(sd, p, x, eps):
    return F.layer_norm(x, x.shape[-1:], sd[p + ".weight"], sd[p + ".bias"], eps)


def _lin(sd, p, x):
    return F.linear(x, sd[p + ".weight"], sd[p + ".bias"])


def _image(x, H, W):
    B, _, C = x.shape
    return x.transpose(1, 2).reshape(B, C, H, W)


def _tokens(img):
    return img.flatten(2).transpose(1, 2)


def attention(sd, p, x, H, W, heads, sr, eps_sr):
    B, N, C = x.shape
    d = C // heads
    q = _lin(sd, p + "q", x).reshape(B, N, heads, d).transpose(1, 2)
    if sr > 1:
        x = _tokens(F.conv2d(_image(x, H, W), sd[p + "sr.weight"], sd[p + "sr.bias"], stride=sr))
        x = _ln(sd, p + "norm", x, eps_sr)
    kv = _lin(sd, p + "kv", x).reshape(B, -1, 2, heads, d).permute(2, 0, 3, 1, 4)
    a = torch.softmax(q @ kv[0].transpose(-2, -1) * d ** -0.5, dim=-1)
    return _lin(sd, p + "proj", (a @ kv[1]).transpose(1, 2).reshape(B, N, C))


def mlp(sd, p, x, H, W):
    h = _lin(sd, p + "fc1", x)
    h = _tokens(F.conv2d(_image(h, H, W), sd[p + "dwconv.dwconv.weight"], sd[p + "dwconv.dwconv.bias"], padding=1,
                         groups=h.shape[-1]))
    return _lin(sd, p + "fc2", F.gelu(h))


def features(sd, cfg, img):
    """forward_features: img [B, 1, T, mel] -> the list of the four stage outputs [B, C_i, H_i, W_i]."""
    outs = []
    x = img
    for i in range(specs.PVT_STAGES):
        pe = f"pvt_transformer.patch_embed{i + 1}."
        x = F.conv2d(x, sd[pe + "proj.weight"], sd[pe + "proj.bias"], stride=4 if i == 0 else 2, padding=2 if i == 0 else 1)
        B, _, H, W = x.shape
        x = _ln(sd, pe + "norm", _tokens(x), cfg["embed_norm_eps"])
        for j in range(int(cfg["depths"][i])):
            p = f"pvt_transformer.block{i + 1}.{j}."
            x = x + attention(sd, p + "attn.", _ln(sd, p + "norm1", x, cfg["layer_norm_eps"]), H, W, int(cfg["num_heads"][i]),
                              int(cfg["sr_ratios"][i]), cfg["embed_norm_eps"])
            x = x + mlp(sd, p + "mlp.", _ln(sd, p + "norm2", x, cfg["layer_norm_eps"]), H, W)
        x = _ln(sd, f"pvt_transformer.norm{i + 1}", x, cfg["layer_norm_eps"])
        x = x.reshape(B, H, W, -1).permute(0, 3, 1, 2)
        outs.append(x)
    return outs


def forward(sd, cfg, wav):
    """wav [B, n] -> dict(framewise_output [B, ratio * H4, classes], clipwise_output [B, classes], logits
    [B, H4, classes], stages: the four stage outputs)."""
    stages = features(sd, cfg, logmel(sd, cfg, wav.to(sd["fc_audioset.weight"].dtype)))
    x = stages[-1].mean(dim=3).transpose(1, 2)                                 # [B, H4, C]
    logits = _lin(sd, "fc_audioset", x)
    frame = torch.sigmoid(logits)
    return dict(framewise_output=frame.repeat_interleave(int(cfg["interpolate_ratio"]), dim=1), clipwise_output=frame.mean(dim=1),
                logits=logits, stages=stages)
