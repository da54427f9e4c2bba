"""Drop-in for ``inference.tts.base_tts_infer.Wav2Vec2ForCTC``: the reference-audio ASR of the TTS_OOD tool.

Reference: NeuralSeq/inference/tts/base_tts_infer.py -- build_asr (:38-42) loads ``facebook/wav2vec2-base-960h`` with
``Wav2Vec2ForCTC.from_pretrained(...).to(device)``, and asr (:83-101) calls ``self.asr_model(input_values.cuda()).logits``
and takes the argmax.  This class is transformers' Wav2Vec2ForCTC (so ``from_pretrained``, ``.to``, the state dict and
the config are transformers' own) whose ``forward`` runs on libagpt_b200.so (csrc/w2v.cu).  CUDA only, eval only,
float32 input without an attention mask (the base-960h processor returns none); the argmax and decode stay with the
caller, as there.

``install(asr=True)`` sets this class on the reference module in place: that module also holds BaseTTSInfer, which the
TTS inferers import, so it is never replaced by an alias."""
from __future__ import annotations

import ctypes as C

import torch
from transformers import Wav2Vec2ForCTC as _Wav2Vec2ForCTC
from transformers.modeling_outputs import CausalLMOutput

from ... import _lib, specs

__all__ = ["Wav2Vec2ForCTC"]


class Wav2Vec2ForCTC(_Wav2Vec2ForCTC):
    _h = _lib.engine_handle

    def __init__(self, config, *args, **kwargs):
        super().__init__(config, *args, **kwargs)
        self._engine = _lib.Engine("agpt_w2v_create")

    def _engine_cfg(self):
        ec = specs.w2v_engine_cfg(self.config)
        cc = _lib.W2vConfig()
        for k, v in ec.items():
            if k in ("conv_kernel", "conv_stride"):
                getattr(cc, k)[:len(v)] = v
            else:
                setattr(cc, k, v)
        return cc

    def _ensure(self, dev):
        sd = self.state_dict(keep_vars=True)
        srcs = [sd[k] for k in specs.w2v_param_shapes(self.config) if k != "wav2vec2.masked_spec_embed"]

        def build():
            with torch.no_grad():
                ws = specs.w2v_engine_weights(self.config, {k: t.detach() for k, t in sd.items()})
            return (C.byref(self._engine_cfg()),), ws
        self._engine.ensure(dev, srcs, build)

    def _frames(self, n_samples: int) -> int:
        return specs.w2v_lengths(self.config, n_samples)[-1]

    def _check_input(self, x):
        if self.training:
            raise RuntimeError("audiogpt_b200.Wav2Vec2ForCTC is inference only: call .eval() first (from_pretrained does)")
        if not torch.is_tensor(x):
            raise TypeError("input_values must be a tensor")
        if x.dtype != torch.float32:
            raise TypeError(f"input_values must be float32 (the processor's), got {x.dtype}")
        if x.dim() != 2 or x.shape[0] < 1:
            raise ValueError(f"input_values must be (batch, samples), got {tuple(x.shape)}")
        if self._frames(x.shape[1]) < 1:
            raise ValueError(f"{x.shape[1]} samples yield no frame: the conv feature encoder needs at least 400")
        if not x.is_cuda:
            raise RuntimeError("audiogpt_b200.Wav2Vec2ForCTC runs on CUDA only (no CPU fallback): pass input_values.cuda()")

    @torch.no_grad()
    def forward(self, input_values, attention_mask=None, output_attentions=None, output_hidden_states=None, return_dict=None,
                labels=None, **kwargs):
        """input_values [B, S] float32 (CUDA) -> CausalLMOutput(logits [B, frames, vocab_size]) from the engine."""
        if attention_mask is not None:
            raise NotImplementedError("audiogpt_b200.Wav2Vec2ForCTC takes no attention_mask (base-960h's processor returns none)")
        if labels is not None:
            raise NotImplementedError("audiogpt_b200.Wav2Vec2ForCTC is inference only: labels (the CTC loss) are not supported")
        if output_attentions or output_hidden_states:
            raise NotImplementedError("audiogpt_b200.Wav2Vec2ForCTC returns logits only (no attentions / hidden states)")
        if kwargs:
            raise TypeError(f"unsupported arguments: {sorted(kwargs)}")
        self._check_input(input_values)
        dev = input_values.device
        self._ensure(dev)
        x = input_values.contiguous()
        B, S = x.shape
        logits = torch.empty((B, self._frames(S), self.config.vocab_size), device=dev, dtype=torch.float32)
        self._engine.call("w2v_logits", dev, _lib.fptr(x), B, S, _lib.fptr(logits))
        if return_dict is False:
            return (logits,)
        return CausalLMOutput(loss=None, logits=logits)

    # ---- the stages apart (tests and scripts/asr_time.py)
    @torch.no_grad()
    def engine_features(self, input_values):
        """The conv feature encoder's output [B, conv_dim, frames] (feature_extractor's layout) from the engine."""
        self._check_input(input_values)
        dev = input_values.device
        self._ensure(dev)
        x = input_values.contiguous()
        B, S = x.shape
        out = torch.empty((B, self._frames(S), self.config.conv_dim[-1]), device=dev, dtype=torch.float32)
        self._engine.call("w2v_features", dev, _lib.fptr(x), B, S, _lib.fptr(out))
        return out.transpose(1, 2)

    @torch.no_grad()
    def engine_pos_conv(self, hidden):
        """hidden [B, T, hidden_size] (CUDA, float32) -> hidden + pos_conv_embed(hidden) from the engine."""
        if not torch.is_tensor(hidden) or not hidden.is_cuda or hidden.dtype != torch.float32 or hidden.dim() != 3:
            raise ValueError("hidden must be a float32 CUDA tensor (batch, frames, hidden_size)")
        dev = hidden.device
        self._ensure(dev)
        h = hidden.contiguous()
        out = torch.empty_like(h)
        self._engine.call("w2v_pos_conv", dev, _lib.fptr(h), h.shape[0], h.shape[1], _lib.fptr(out))
        return out
