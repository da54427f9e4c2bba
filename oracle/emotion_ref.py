"""CPU restatement of the TTS_OOD tool's emotion encoder, fp32 or fp64.

Reference: NeuralSeq/data_gen/tts/emotion/audio.py:43-55 (wav_to_mel_spectrogram: librosa.feature.melspectrogram with
n_fft 400, hop 160, 40 mels -- periodic Hann, center with specs.EMO_PAD_MODE padding, power 2, Slaney mel, no log),
model.py:41-77 (EmotionEncoder.forward / inference) and inference.py:59-164 (compute_partial_slices, embed_utterance).
The mel follows librosa: the DFT of each windowed frame, its squared magnitude and the mel matrix product.  The LSTM is
torch.nn.LSTM loaded with the state dict.  ``embed_utterance`` also returns the intermediates the tests localise
errors with."""
from __future__ import annotations

import numpy as np
import torch

from audiogpt_b200 import specs


def mel(wav: np.ndarray, dtype=torch.float64) -> torch.Tensor:
    """wav [n] -> the power mel [1 + n // 160][40]."""
    fp64 = dtype == torch.float64
    x = np.asarray(wav, dtype=np.float64 if fp64 else np.float32)
    n_fft, hop = specs.EMO_N_FFT, specs.EMO_HOP
    xp = np.pad(x, n_fft // 2, mode=specs.EMO_PAD_MODE)
    F = 1 + (len(xp) - n_fft) // hop
    idx = np.arange(F)[:, None] * hop + np.arange(n_fft)[None, :]
    win = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(n_fft) / n_fft)
    spec = np.fft.rfft(xp[idx] * win, axis=1)
    if not fp64:
        spec = spec.astype(np.complex64)
    power = np.abs(spec) ** 2
    melW = specs.slaney_mel(specs.EMO_SR, n_fft, specs.EMO_MELS, 0.0, specs.EMO_SR / 2.0).astype(power.dtype)
    return torch.from_numpy(np.ascontiguousarray((melW @ power.T).T)).to(dtype)


def lstm_module(sd, cfg=specs.EMO, dtype=torch.float64) -> torch.nn.LSTM:
    m = torch.nn.LSTM(int(cfg["input_size"]), int(cfg["hidden_size"]), int(cfg["num_layers"]), batch_first=True)
    m.load_state_dict({k[len("lstm."):]: v for k, v in sd.items() if k.startswith("lstm.")}, strict=True)
    return m.to(dtype).eval()


def hidden(sd, frames: torch.Tensor, cfg=specs.EMO, dtype=torch.float64) -> torch.Tensor:
    """EmotionEncoder.inference: frames [N][T][40] -> the last layer's final h [N][256]."""
    with torch.no_grad():
        _, (h, _) = lstm_module(sd, cfg, dtype)(frames.to(dtype))
    return h[-1]


def forward(sd, frames: torch.Tensor, cfg=specs.EMO, dtype=torch.float64) -> torch.Tensor:
    """EmotionEncoder.forward: relu(linear(hidden[-1])), L2-normalised per row."""
    h = hidden(sd, frames, cfg, dtype)
    e = torch.relu(h @ sd["linear.weight"].to(dtype).T + sd["linear.bias"].to(dtype))
    return e / torch.norm(e, dim=1, keepdim=True)


def embed_utterance(sd, wav: np.ndarray, using_partials: bool = True, cfg=specs.EMO, dtype=torch.float64, **kwargs) -> dict:
    """embed_utterance(wav, using_partials, return_partials=True, **kwargs): {"embed", "partials" (None without
    partials), "wav_slices", "mel"}."""
    if not using_partials:
        m = mel(wav, dtype)
        return {"embed": hidden(sd, m[None], cfg, dtype)[0], "partials": None, "wav_slices": None, "mel": m}
    wav_slices, mel_slices = specs.emo_partials(len(wav), **kwargs)
    n = specs.emo_padded_length(len(wav), wav_slices)
    x = np.pad(np.asarray(wav), (0, n - len(wav)), "constant")
    m = mel(x, dtype)
    frames = torch.stack([m[s] for s in mel_slices])
    partials = hidden(sd, frames, cfg, dtype)
    raw = partials.mean(0)
    return {"embed": raw / torch.linalg.vector_norm(raw), "partials": partials, "wav_slices": wav_slices, "mel": m}
