"""Oracle of the CLAP candidate scorer of the text-to-audio tool (T2A.select_best_audio, audio-chatgpt.py:185-199):
wav_evaluation/models/CLAPWrapper.py get_audio_embeddings / get_text_embeddings / compute_similarity, restated with
torch ops from a state dict in the layout of audiogpt_b200.specs.clap_scorer_param_shapes.  It does not use
torchaudio, torchlibrosa or transformers: the resampler's filter is specs.sinc_resample_kernel (torchaudio's,
restated), the spectrogram is the checkpoint's conv-STFT, BERT is restated with its attention mask and token types.
Device-agnostic: the tensors decide where it runs (scripts/clap_score_time.py runs it on the GPU as the eager arm)."""
import math

import torch
import torch.nn.functional as F

from audiogpt_b200 import specs


def resample(wav, orig_freq, new_freq):
    """torchaudio.transforms.Resample(orig_freq, new_freq)(wav) for a 1-D clip."""
    if orig_freq == new_freq:
        return wav
    k, width, o, n = specs.sinc_resample_kernel(orig_freq, new_freq)
    L = wav.shape[-1]
    x = F.pad(wav.reshape(1, 1, L), (width, width + o))
    y = F.conv1d(x, k.to(wav)[:, None, :], stride=o).transpose(1, 2).reshape(-1)
    return y[:math.ceil(n * L / o)]


def fit_duration(wav, clip, start):
    """CLAPWrapper.resample_and_duration's second half: start is None -> tile to clip samples, else the crop start."""
    if start is None:
        return wav.repeat(math.ceil(clip / wav.shape[0]))[:clip]
    return wav[start:start + clip]


def crop_start(resampled_len, clip, rng):
    """The reference's draw: random.randrange(len - clip) when the resampled clip is longer than clip, else None."""
    return None if clip >= resampled_len else rng.randrange(resampled_len - clip)


def _l2(x):
    return x / torch.norm(x, dim=-1, keepdim=True)


def _projection(sd, p, x):
    e1 = F.linear(x, sd[p + "linear1.weight"])
    e2 = F.linear(F.gelu(e1), sd[p + "linear2.weight"])
    return F.layer_norm(e1 + e2, (e1.shape[-1],), sd[p + "layer_norm.weight"], sd[p + "layer_norm.bias"], 1e-5)


def _bn(sd, p, x):
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                        False, 0.0, specs.BN_EPS)


def cnn14_logmel(sd, cfg, x):
    """x [B, clip] -> bn0(log-mel) [B, 1, T, mel_bins]: torchlibrosa Spectrogram (center, reflect, power 2) as conv1d
    with the checkpoint's DFT rows, LogmelFilterBank (ref 1, amin 1e-10, no top_db), bn0."""
    a = "audio_encoder.base."
    n = int(cfg["window_size"])
    xp = F.pad(x[:, None, :], (n // 2, n // 2), mode="reflect")
    re = F.conv1d(xp, sd[a + "spectrogram_extractor.stft.conv_real.weight"], stride=int(cfg["hop_size"]))
    im = F.conv1d(xp, sd[a + "spectrogram_extractor.stft.conv_imag.weight"], stride=int(cfg["hop_size"]))
    power = (re ** 2 + im ** 2).transpose(1, 2)[:, None]                      # [B, 1, T, n/2 + 1]
    mel = torch.matmul(power, sd[a + "logmel_extractor.melW"])
    lm = 10.0 * torch.log10(torch.clamp(mel, min=1e-10))
    return _bn(sd, a + "bn0", lm.transpose(1, 3)).transpose(1, 3)


def cnn14_embedding(sd, cfg, x):
    """Cnn14.forward(x)['embedding'] in eval mode: [B, clip] -> [B, out_emb]."""
    a = "audio_encoder.base."
    h = cnn14_logmel(sd, cfg, x)
    for i in range(len(specs.CNN14_CHANNELS)):
        p = f"{a}conv_block{i + 1}."
        h = F.relu(_bn(sd, p + "bn1", F.conv2d(h, sd[p + "conv1.weight"], padding=1)))
        h = F.relu(_bn(sd, p + "bn2", F.conv2d(h, sd[p + "conv2.weight"], padding=1)))
        if i < len(specs.CNN14_CHANNELS) - 1:
            h = F.avg_pool2d(h, 2)
    h = h.mean(dim=3)
    h = h.max(dim=2)[0] + h.mean(dim=2)
    return F.relu(F.linear(h, sd[a + "fc1.weight"], sd[a + "fc1.bias"]))


def audio_embeddings(sd, cfg, clips):
    """clips: [B, clip] already resampled and fitted -> the normalised audio embeddings [B, d_proj]
    (_get_audio_embeddings and get_audio_embeddings each divide by the norm)."""
    e = _projection(sd, "audio_encoder.projection.", cnn14_embedding(sd, cfg, clips))
    return _l2(_l2(e))


def bert_cls(sd, bcfg, input_ids, token_type_ids, attention_mask):
    """HF BertModel(input_ids, token_type_ids, attention_mask)[0][:, 0]: padding keys (mask 0) are masked out."""
    ids = input_ids.long()
    N, L = ids.shape
    H, nh = int(bcfg["hidden_size"]), int(bcfg["num_heads"])
    dh = H // nh
    eps = float(bcfg["layer_norm_eps"])
    b = "caption_encoder.base."
    w = lambda k: sd[b + k]   # noqa: E731

    def ln(x, p):
        return F.layer_norm(x, (x.shape[-1],), w(p + ".weight"), w(p + ".bias"), eps)

    x = w("embeddings.word_embeddings.weight")[ids] + w("embeddings.token_type_embeddings.weight")[token_type_ids.long()]
    x = ln(x + w("embeddings.position_embeddings.weight")[:L], "embeddings.LayerNorm")
    bias = torch.zeros(N, 1, 1, L, dtype=x.dtype, device=x.device).masked_fill(
        attention_mask.reshape(N, 1, 1, L) == 0, float("-inf"))
    for i in range(int(bcfg["num_layers"])):
        p = f"encoder.layer.{i}."
        q, k, v = (F.linear(x, w(p + f"attention.self.{n}.weight"), w(p + f"attention.self.{n}.bias"))
                   .view(N, L, nh, dh).transpose(1, 2) for n in ("query", "key", "value"))
        a = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(dh) + bias, dim=-1) @ v
        a = a.transpose(1, 2).reshape(N, L, H)
        x = ln(F.linear(a, w(p + "attention.output.dense.weight"), w(p + "attention.output.dense.bias")) + x,
               p + "attention.output.LayerNorm")
        h = F.gelu(F.linear(x, w(p + "intermediate.dense.weight"), w(p + "intermediate.dense.bias")))
        x = ln(F.linear(h, w(p + "output.dense.weight"), w(p + "output.dense.bias")) + x, p + "output.LayerNorm")
    return x[:, 0]


def text_embeddings(sd, cfg, input_ids, token_type_ids, attention_mask):
    """get_text_embeddings after tokenization: [N, L] rows -> normalised [N, d_proj]."""
    bcfg = specs.clap_scorer_bert_cfg(cfg)
    e = _projection(sd, "caption_encoder.projection.", bert_cls(sd, bcfg, input_ids, token_type_ids, attention_mask))
    return _l2(_l2(e))


def similarity(audio_emb, text_emb):
    """compute_similarity(a, t, use_logit_scale=False) = (t @ a.T).T, [N_audio, N_text]."""
    return (text_emb @ audio_emb.T).T


def prepare_clip(wav, sr, cfg, rng, resample_on=True):
    """One (wav, sr) entry of get_audio_embeddings(..., resample): the fitted clip and the crop start drawn (or None)."""
    y = resample(wav.reshape(-1).float(), int(sr), int(cfg["sampling_rate"])) if resample_on else wav.reshape(-1).float()
    clip = int(cfg["duration"]) * int(sr)
    start = crop_start(y.shape[0], clip, rng)
    return fit_duration(y, clip, start), start
