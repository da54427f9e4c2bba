#!/usr/bin/env python
"""Generate the emotion-encoder fixture (emotion.npz) by running the REFERENCE's own data_gen.tts.emotion.inference
(compute_partial_slices, embed_utterance) and EmotionEncoder (model.py) on CPU fp32, as GenerSpeechInfer calls them
(inference/tts/GenerSpeech.py:37,58).

Run in the build container only (needs the reference tree, which does not travel to the GPU box):

    python tests/golden/make_golden_emotion.py

Stubs: webrtcvad and matplotlib (only preprocess_wav's VAD and the plotting helpers use them) are empty modules, and
librosa.feature.melspectrogram, which is not installed here, is a shim restating librosa 0.9's melspectrogram at the
reference's arguments: stft with win_length = n_fft, a periodic Hann window, center=True and 'reflect' padding (the
pre-0.10 default), |.|^2, then librosa.filters.mel (Slaney, area-normalised, fmin 0, fmax sr / 2) in float32.
inference._model is set directly to a reference EmotionEncoder on the CPU loaded with specs.synth_emotion weights, and
_device to the CPU.  Neither the weights nor the clips are stored: the tests regenerate both from their seeds (the
fixture keeps per-clip sums to confirm the clips come out the same).  Stored per case: the length, the clip seed, the
wav slices, hidden[-1] per partial, the embedding and forward's output on the partials' frames; plus the reference's
state_dict() keys and shapes.
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF, save, specs  # noqa: E402

SEED = 5353                 # weights
# one padded partial; exactly one partial's 25 600 samples; either side of the 0.75-coverage cut of the second
# partial (it starts at 12 800 and covers 25 600: the cut is at 32 000); the unpadded case; 10 s; 17.7 s
LENGTHS = (16000, 25600, 31999, 32000, 40000, 160000, 283200)
WHOLE = 48000               # using_partials=False


def librosa_shim():
    lib = types.ModuleType("librosa")
    feat = types.ModuleType("librosa.feature")

    def melspectrogram(y, sr=22050, n_fft=2048, hop_length=512, n_mels=128):
        y = np.asarray(y)
        x = np.pad(y, n_fft // 2, mode="reflect")
        n = 1 + (len(x) - n_fft) // hop_length
        win = (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(n_fft) / n_fft)).astype(np.float32)
        frames = np.stack([x[i * hop_length:i * hop_length + n_fft] for i in range(n)], axis=1)
        stft = np.fft.rfft(win[:, None] * frames, axis=0).astype(np.complex64 if y.dtype == np.float32 else np.complex128)
        S = np.abs(stft) ** 2
        mel = specs.slaney_mel(sr, n_fft, n_mels, 0.0, sr / 2.0)
        return np.dot(mel, S)
    feat.melspectrogram = melspectrogram
    lib.feature = feat
    return {"librosa": lib, "librosa.feature": feat}


def main():
    sys.path.insert(0, os.path.join(REF, "NeuralSeq"))
    mods = librosa_shim()
    for n in ("webrtcvad", "matplotlib", "matplotlib.pyplot"):
        mods[n] = types.ModuleType(n)
    mods["matplotlib"].cm = types.ModuleType("matplotlib.cm")
    mods["matplotlib"].pyplot = mods["matplotlib.pyplot"]
    mods["matplotlib.cm"] = mods["matplotlib"].cm
    sys.modules.update(mods)
    from data_gen.tts.emotion import inference
    from data_gen.tts.emotion.model import EmotionEncoder

    torch.manual_seed(0)
    model = EmotionEncoder(torch.device("cpu"), torch.device("cpu"))
    sd = model.state_dict()
    model.load_state_dict(specs.synth_emotion(specs.EMO, SEED), strict=True)
    model.eval()
    inference._model, inference._device = model, torch.device("cpu")

    out = {"weight_seed": SEED, "keys": np.array(list(sd)), "shapes": np.array([",".join(map(str, v.shape)) for v in sd.values()]),
           "lengths": np.array(LENGTHS), "whole_length": WHOLE}
    for i, n in enumerate(LENGTHS):
        wav = specs.synth_emotion_wav(n, seed=100 + i)
        embed, partials, wav_slices = inference.embed_utterance(wav, return_partials=True)
        _, mel_slices = inference.compute_partial_slices(n)
        x = wav
        if wav_slices[-1].stop >= n:
            x = np.pad(wav, (0, wav_slices[-1].stop - n), "constant")
        from data_gen.tts.emotion import audio
        frames = audio.wav_to_mel_spectrogram(x)
        with torch.no_grad():
            fwd = model(torch.from_numpy(np.array([frames[s] for s in mel_slices]))).numpy()
        out[f"c{i}_seed"] = 100 + i
        out[f"c{i}_wav_sum"] = float(np.sum(wav, dtype=np.float64))
        out[f"c{i}_slices"] = np.array([[s.start, s.stop] for s in wav_slices])
        out[f"c{i}_partials"] = partials
        out[f"c{i}_embed"] = embed
        out[f"c{i}_forward"] = fwd
        print(f"{n:7d} samples: {len(wav_slices)} partials, padded to {max(n, wav_slices[-1].stop)}")
    wav = specs.synth_emotion_wav(WHOLE, seed=99)
    out["whole_seed"] = 99
    out["whole_embed"] = inference.embed_utterance(wav, using_partials=False)
    save("emotion", **out)


if __name__ == "__main__":
    main()
