"""Drop-in for ``data_gen.tts.emotion.inference``: the TTS_OOD tool's emo_embed on the engine.

Reference: NeuralSeq/data_gen/tts/emotion/inference.py -- load_model, embed_frames_batch, compute_partial_slices and
embed_utterance, with the same signatures and return types.  embed_utterance uploads the wav once and runs the slicing
pad, the mel, the LSTM over every partial, the mean and the norm in one engine call (EmotionEncoder.engine_embed).  A
float64 wav is cast to float32 first (the reference's librosa computes its mel in float64 and casts the result).
preprocess_wav (volume normalisation and webrtcvad trimming) is host work and stays the reference's.

``install(emotion=True)`` sets EmotionEncoder, embed_frames_batch and embed_utterance on the reference module in place
and keeps the loaded model there: the reference's own load_model, which resolves EmotionEncoder through its module's
globals, then builds the drop-in, and these functions read the model it stored."""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import torch

from .... import specs
from .model import EmotionEncoder

__all__ = ["EmotionEncoder", "load_model", "is_loaded", "embed_frames_batch", "compute_partial_slices", "embed_utterance"]

partials_n_frames = specs.EMO_PARTIAL_FRAMES

_model = None    # type: EmotionEncoder
_device = None   # type: torch.device
# the module load_model stores _model / _device in (install(emotion=True) points it at the reference module)
_state = sys.modules[__name__]


def load_model(weights_fpath: Path, device=None):
    """Build EmotionEncoder on ``device`` (default: CUDA when available) from ``torch.load(weights_fpath)["model_state"]``,
    in eval mode."""
    if device is None:
        dev = torch.device("cuda" if torch.cuda.is_available() else "cpu")
    else:
        dev = torch.device(device)
    model = EmotionEncoder(dev, torch.device("cpu"))
    checkpoint = torch.load(weights_fpath)
    model.load_state_dict(checkpoint["model_state"])
    model.eval()
    _state._model, _state._device = model, dev
    print("Loaded encoder trained to step %d" % (checkpoint["step"]))


def is_loaded():
    return _state._model is not None


def _loaded() -> EmotionEncoder:
    model = _state._model
    if model is None:
        raise Exception("Model was not loaded. Call load_model() before inference.")
    if not isinstance(model, EmotionEncoder):
        raise TypeError(f"the loaded model is {type(model).__name__}, not audiogpt_b200's EmotionEncoder: call "
                        "audiogpt_b200.install(emotion=True) before load_model")
    return model


def embed_frames_batch(frames_batch):
    """frames_batch float32 numpy [N][T][40] -> hidden[-1] as float32 numpy [N][256]."""
    model = _loaded()
    frames = torch.from_numpy(frames_batch).to(_state._device)
    return model.inference(frames).detach().cpu().numpy()


def compute_partial_slices(n_samples, partial_utterance_n_frames=partials_n_frames, min_pad_coverage=0.75, overlap=0.5):
    """(wav_slices, mel_slices) of the partial utterances, as the reference computes them (specs.emo_partials)."""
    return specs.emo_partials(n_samples, partial_utterance_n_frames, min_pad_coverage, overlap)


def embed_utterance(wav, using_partials=True, return_partials=False, **kwargs):
    """wav: a preprocessed 16 kHz waveform (numpy) -> the embedding, float32 numpy (256,); with return_partials also
    the partial embeddings [N][256] and the wav slices (both None without partials)."""
    model = _loaded()
    w = np.asarray(wav)
    if w.ndim != 1:
        raise ValueError(f"wav must be 1-D, got shape {w.shape}")
    x = torch.from_numpy(np.ascontiguousarray(w, dtype=np.float32)).to(_state._device)
    if not using_partials:
        embed, _ = model.engine_embed(x, 0)
        embed = embed.cpu().numpy()
        return (embed, None, None) if return_partials else embed
    wave_slices, _ = compute_partial_slices(len(w), **kwargs)
    args = dict(dict(partial_utterance_n_frames=partials_n_frames, min_pad_coverage=0.75, overlap=0.5), **kwargs)
    embed, partials = model.engine_embed(x, args["partial_utterance_n_frames"], args["min_pad_coverage"], args["overlap"])
    if partials.shape[0] != len(wave_slices):
        raise RuntimeError(f"the engine cut {partials.shape[0]} partials where compute_partial_slices cuts {len(wave_slices)}")
    embed = embed.cpu().numpy()
    if return_partials:
        return embed, partials.cpu().numpy(), wave_slices
    return embed
