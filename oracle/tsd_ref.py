"""CPU restatement of the target-sound-detection RaDur_fusion in eval mode, in functional torch (fp32 or fp64).

Reference: audio_detection/target_sound_detection/src/models.py:175-218 (ConvBlock), :220-256 (ConvBlock_GLU), :304-377
(Cnn14.forward: the mel goes straight into conv_block1), :422-479 (Cnn10_mul_scale), :698-718 (conv1d), :770-788
(Fusion), :1058-1106 (CDur_CNN_mul_scale_fusion), :1109-1291 (RaDur_fusion: get_w / get_w_ee, attention_pooling,
select_topk_embeddings, sum_with_attention, orcal_EE, forward).  Every time_resolution branch and both flags.
``forward`` also returns the intermediates the tests localise errors with."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from audiogpt_b200 import specs

TEMPERATURE = 11.3     # RaDur_fusion.temperature, as written (not sqrt(128))
BN_EPS = 1e-5


def _bn(sd, p, x, dim=1):
    shape = [1] * x.dim()
    shape[dim] = -1
    g, b = sd[p + ".weight"].view(shape), sd[p + ".bias"].view(shape)
    m, v = sd[p + ".running_mean"].view(shape), sd[p + ".running_var"].view(shape)
    return (x - m) / torch.sqrt(v + BN_EPS) * g + b


def conv_block(sd, p, x, pool):
    x = F.relu(_bn(sd, p + "bn1", F.conv2d(x, sd[p + "conv1.weight"], padding=1)))
    x = F.relu(_bn(sd, p + "bn2", F.conv2d(x, sd[p + "conv2.weight"], padding=1)))
    return F.avg_pool2d(x, kernel_size=pool)


def glu_block(sd, p, x, pool):
    """ConvBlock_GLU: padding (1, 1) whatever the kernel size."""
    x = _bn(sd, p + "bn1", F.conv2d(x, sd[p + "conv1.weight"], padding=1))
    c = x.shape[1] // 2
    return F.avg_pool2d(torch.sigmoid(x[:, :c]) * x[:, c:], kernel_size=pool)


def cnn14(sd, x):
    """Cnn14.forward on a mel [B, T, 64] -> per-frame embeddings [B, T // 8, 128] (fc1, no ReLU)."""
    h = x.unsqueeze(1)
    for i, pool in enumerate(specs.TSD_ENC_POOLS):
        h = conv_block(sd, f"encoder.conv_block{i + 1}.", h, pool)
    return F.linear(h.transpose(1, 2).flatten(-2), sd["encoder.fc1.weight"], sd["encoder.fc1.bias"])


def stem(sd, x, ph):
    """Cnn10_mul_scale's three GLU branches, crop / pad and concat on x [B, 1, T, 64] -> [B, 96, m, 32]."""
    f = "detection.features."
    x1 = glu_block(sd, f + "conv_block1_1.", x, (ph, 2))[:, :, :500, :32]
    x2 = glu_block(sd, f + "conv_block1_2.", x, (ph, 2))
    x3 = F.pad(glu_block(sd, f + "conv_block1_3.", x, (ph, 2)), (0, 1, 0, 1), mode="replicate")
    m = min(x3.shape[2], min(x1.shape[2], x2.shape[2]))
    return torch.cat([x1[:, :, :m], x2[:, :, :m], x3[:, :, :m]], dim=1)


def features(sd, cfg, x):
    """detection.features on a mel [B, T, 64], flattened as the reference does -> [B, T', 512]."""
    pools = specs.TSD_POOLS[specs.tsd_scale(cfg["time_resolution"])]
    h = stem(sd, x.unsqueeze(1), pools[0][0])
    for i, pool in enumerate(pools[1:]):
        h = conv_block(sd, f"detection.features.conv_block{i + 2}.", h, pool)
    return h.transpose(1, 2).contiguous().flatten(-2)


def fusion(sd, p, n_fac, embedding, mix_embed):
    """Fusion.forward(embedding, mix_embed) on [B, T, *] rows: relu(1-wide conv) of each, product, AvgPool1d(n_fac)."""
    f1 = F.relu(F.conv1d(embedding.permute(0, 2, 1), sd[p + "fuse_layer1.conv.weight"], sd[p + "fuse_layer1.conv.bias"]))
    f2 = F.relu(F.conv1d(mix_embed.permute(0, 2, 1), sd[p + "fuse_layer2.conv.weight"], sd[p + "fuse_layer2.conv.bias"]))
    return F.avg_pool1d((f1 * f2).permute(0, 2, 1), n_fac, stride=n_fac)


def gru(sd, x):
    """nn.GRU(512, 512, bidirectional=True, batch_first=True) with the state dict's weights, on x's device and dtype."""
    with torch.device("meta"):     # no initialisation: the parameters are the state dict's own tensors
        m = torch.nn.GRU(512, 512, bidirectional=True, batch_first=True)
    m.load_state_dict({k[len("detection.gru."):]: v.to(x.device, x.dtype) for k, v in sd.items() if k.startswith("detection.gru.")},
                      assign=True)
    m.flatten_parameters()
    return m(x)[0]


def detect(sd, feat, emb):
    """One detection pass from the (per-sample constant) embedding: fusion, GRU, fc, outputlayer, softmax -> [B, T', O]."""
    x = fusion(sd, "detection.fusion.", 2, emb.unsqueeze(1).repeat(1, feat.shape[1], 1), feat)
    x = F.linear(gru(sd, x), sd["detection.fc.weight"], sd["detection.fc.bias"])
    return torch.softmax(F.linear(x, sd["detection.outputlayer.weight"], sd["detection.outputlayer.bias"]), dim=2)


def get_w(sd, qn, kn, q, k):
    """get_w / get_w_ee: softmax over the rows of k of (qn(q) . kn(k)) / 11.3 -> [B, 1, rows]."""
    q = F.linear(q, sd[qn + ".weight"], sd[qn + ".bias"])
    k = F.linear(k, sd[kn + ".weight"], sd[kn + ".bias"])
    return torch.softmax(torch.bmm(q.unsqueeze(1), k.transpose(1, 2)) / TEMPERATURE, dim=2)


def topk(scores, k):
    """Descending top-k with ties to the lower index: (values, indices) [B, min(k, T')]."""
    v, i = scores.sort(descending=True, dim=1, stable=True)
    return v[:, :k], i[:, :k]


def reference_embedding(sd, cfg, ref):
    emb = cnn14(sd, ref)
    mean = emb.mean(1)
    if not cfg["att_pool"]:
        return mean
    mean = _bn(sd, "bn", mean)
    emb = _bn(sd, "bn", emb, dim=2)
    return torch.bmm(get_w(sd, "q", "k", mean, emb), emb).squeeze(1)


def interpolate(d, T):
    return F.interpolate(d.transpose(1, 2), T, mode="linear", align_corners=False).transpose(1, 2)


def forward(sd, cfg, x, ref, dtype=torch.float32):
    """RaDur_fusion(cfg).eval()(x, ref) with state dict sd: x [B, T, 64], ref [B, Tr, 64].  Returns a dict with decision
    [B, T'], decision_up [B, T, O], embedding [B, 128] and decision1 (the first pass) [B, T', O]; with enhancement also
    topk_idx / topk_val [B, k], wmix [B] (the second pass's weight) and decision2 [B, T', O]."""
    sd = {k: v.to(dtype) if v.is_floating_point() else v for k, v in sd.items()}
    x, ref = x.to(dtype), ref.to(dtype)
    T = x.shape[1]
    emb = reference_embedding(sd, cfg, ref)
    feat = features(sd, cfg, x)
    d1 = detect(sd, feat, emb)
    out = dict(embedding=emb, decision1=d1)
    d = d1
    if cfg["enhancement"]:
        mixture = _bn(sd, "bn", cnn14(sd, x), dim=2)
        val, idx = topk(d1[:, :, 0], int(cfg["top"]))
        sel = torch.gather(mixture, 1, idx.unsqueeze(2).expand(-1, -1, mixture.shape[2]))
        att = get_w(sd, "q_ee", "k_ee", emb, sel).squeeze(1) * (val * (val > cfg["tao"]))
        mix = (sel * att.unsqueeze(2)).mean(1)
        me = fusion(sd, "EE_fusion.", 4, mix.unsqueeze(1), emb.unsqueeze(1))[:, 0]
        d2 = detect(sd, feat, me)
        m = val.mean(1)
        w = (m * (m > cfg["tao"]) / 2.0)[:, None, None]
        d = d1 * (1 - w) + w * d2
        out.update(topk_idx=idx, topk_val=val, wmix=w[:, 0, 0], decision2=d2)
    out.update(decision=d[:, :, 0], decision_up=interpolate(d, T))
    return out
