"""Drop-in for ``data_gen.tts.emotion.model.EmotionEncoder``: the emotion encoder of the TTS_OOD tool.

Reference: NeuralSeq/data_gen/tts/emotion/model.py -- nn.LSTM(40, 256, 3, batch_first), Linear(256, 256) and ReLU, plus
the similarity scaling and loss of its training.  The constructor, the state-dict keys and the module tree are the
reference's; ``inference`` (the last layer's final h, what embed_utterance uses) and ``forward`` (relu(linear(.)),
L2-normalised) run on libagpt_b200.so (csrc/emotion.cu).  CUDA only, eval only, float32 [N][T][40] input, no
``hidden_init``.  The engine is packed on first use and again after any weight change."""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from .... import _lib, specs

__all__ = ["EmotionEncoder"]

# params_data.py / params_model.py
mel_n_channels = specs.EMO_MELS
model_hidden_size = 256
model_embedding_size = 256
model_num_layers = 3


class EmotionEncoder(nn.Module):
    _h = _lib.engine_handle

    def __init__(self, device, loss_device):
        super().__init__()
        self.loss_device = loss_device
        self.lstm = nn.LSTM(input_size=mel_n_channels, hidden_size=model_hidden_size, num_layers=model_num_layers,
                            batch_first=True).to(device)
        self.linear = nn.Linear(in_features=model_hidden_size, out_features=model_embedding_size).to(device)
        self.relu = torch.nn.ReLU().to(device)
        # as the reference writes it: a Parameter only while loss_device is the CPU
        self.similarity_weight = nn.Parameter(torch.tensor([10.])).to(loss_device)
        self.similarity_bias = nn.Parameter(torch.tensor([-5.])).to(loss_device)
        self.loss_fn = nn.CrossEntropyLoss().to(loss_device)
        self._engine = _lib.Engine("agpt_emo_create")

    def engine_cfg(self) -> dict:
        """The agpt_emo_cfg fields of this module (after specs.emo_check and the layout checks of the LSTM)."""
        m = self.lstm
        if not m.batch_first or m.bidirectional or m.proj_size or not m.bias:
            raise ValueError("audiogpt_b200.EmotionEncoder covers a batch_first, unidirectional LSTM with biases and no projection")
        cfg = dict(input_size=m.input_size, hidden_size=m.hidden_size, num_layers=m.num_layers,
                   embedding_size=self.linear.out_features)
        specs.emo_check(cfg)
        return cfg

    def _ensure(self, dev):
        cfg = self.engine_cfg()
        srcs = list(self.lstm.parameters()) + list(self.linear.parameters())

        def build():
            sd = {k: v.detach() for k, v in self.state_dict(keep_vars=True).items()}
            with torch.no_grad():
                ws = specs.emo_engine_weights(cfg, sd)
            return (C.byref(_lib.EmoConfig(**cfg)),), ws
        self._engine.ensure(dev, srcs, build)

    def _check(self, x, hidden_init=None):
        if self.training:
            raise RuntimeError("audiogpt_b200.EmotionEncoder is inference only: call .eval() first (load_model does)")
        if hidden_init is not None:
            raise NotImplementedError("audiogpt_b200.EmotionEncoder starts from h0 = c0 = 0: hidden_init is not supported")
        if not torch.is_tensor(x):
            raise TypeError("utterances must be a tensor")
        if x.dtype != torch.float32:
            raise TypeError(f"utterances must be float32 (a mel spectrogram), got {x.dtype}")
        if x.dim() != 3 or x.shape[2] != mel_n_channels:
            raise ValueError(f"utterances must be (batch, frames, {mel_n_channels}), got {tuple(x.shape)}")
        if x.shape[0] < 1 or x.shape[1] < 1:
            raise ValueError(f"utterances must hold at least one frame, got {tuple(x.shape)}")
        if not x.is_cuda:
            raise RuntimeError("audiogpt_b200.EmotionEncoder runs on CUDA only (no CPU fallback): pass a CUDA tensor")

    @torch.no_grad()
    def forward(self, utterances, hidden_init=None):
        """utterances [N][T][40] float32 (CUDA) -> relu(linear(hidden[-1])) L2-normalised per row, [N][256]."""
        self._check(utterances, hidden_init)
        dev = utterances.device
        self._ensure(dev)
        x = utterances.contiguous()
        out = torch.empty((x.shape[0], self.linear.out_features), device=dev, dtype=torch.float32)
        self._engine.call("emo_forward", dev, _lib.fptr(x), x.shape[0], x.shape[1], _lib.fptr(out))
        return out

    @torch.no_grad()
    def inference(self, utterances, hidden_init=None):
        """utterances [N][T][40] float32 (CUDA) -> hidden[-1], the last LSTM layer's final h [N][256]."""
        self._check(utterances, hidden_init)
        dev = utterances.device
        self._ensure(dev)
        x = utterances.contiguous()
        out = torch.empty((x.shape[0], self.lstm.hidden_size), device=dev, dtype=torch.float32)
        self._engine.call("emo_hidden", dev, _lib.fptr(x), x.shape[0], x.shape[1], _lib.fptr(out))
        return out

    # ---- the whole utterance and the front end (inference.embed_utterance, tests and scripts/emotion_time.py)
    def _check_wav(self, wav):
        if self.training:
            raise RuntimeError("audiogpt_b200.EmotionEncoder is inference only: call .eval() first (load_model does)")
        if not torch.is_tensor(wav) or wav.dtype != torch.float32 or wav.dim() != 1 or not wav.is_cuda:
            raise ValueError("wav must be a 1-D float32 CUDA tensor")
        if wav.shape[0] < 1:
            raise ValueError("wav is empty")

    @torch.no_grad()
    def engine_embed(self, wav, partial_frames: int = specs.EMO_PARTIAL_FRAMES, min_pad_coverage: float = 0.75,
                     overlap: float = 0.5):
        """wav [n] float32 (CUDA) -> (embed [256], partials [N][256]): embed_utterance in one engine call.
        partial_frames = 0 runs the whole mel as one sequence (using_partials=False; partials is then None)."""
        self._check_wav(wav)
        dev = wav.device
        self._ensure(dev)
        x = wav.contiguous()
        embed = torch.empty(self.lstm.hidden_size, device=dev, dtype=torch.float32)
        partials = None
        if partial_frames:
            n = C.c_int()
            step, padded = C.c_int(), C.c_long()
            _lib.check(_lib.lib().agpt_emo_partials(x.shape[0], int(partial_frames), float(min_pad_coverage), float(overlap),
                                                    C.byref(n), C.byref(step), C.byref(padded)))
            partials = torch.empty((n.value, self.lstm.hidden_size), device=dev, dtype=torch.float32)
        self._engine.call("emo_embed", dev, _lib.fptr(x), x.shape[0], int(partial_frames), float(min_pad_coverage),
                          float(overlap), _lib.fptr(embed), _lib.fptr(partials) if partials is not None else None)
        return embed, partials

    @torch.no_grad()
    def engine_mel(self, wav):
        """wav [n] float32 (CUDA, n >= 201) -> wav_to_mel_spectrogram(wav), [n // 160 + 1][40]."""
        self._check_wav(wav)
        dev = wav.device
        self._ensure(dev)
        x = wav.contiguous()
        out = torch.empty((x.shape[0] // specs.EMO_HOP + 1, mel_n_channels), device=dev, dtype=torch.float32)
        self._engine.call("emo_mel", dev, _lib.fptr(x), x.shape[0], _lib.fptr(out))
        return out
