"""Drop-in for ``modules.fastspeech.pe.PitchExtractor`` (SURVEY.md 8f row 3).

Reference: /root/reference/NeuralSeq/modules/fastspeech/pe.py:119-148 (with Prenet :7-42, ConvStacks :82-116 and
PitchPredictor modules/fastspeech/tts_modules.py:217-260).  Same constructor (``n_mel_bins``, ``conv_layers``; reads
``hidden_size``, ``predictor_hidden``, ``predictor_kernel``, ``ffn_padding``, ``pitch_type``, ``use_uv``, ``pitch_norm``,
``f0_mean`` / ``f0_std`` from the global hparams), same ``forward(mel_input) -> {'pitch_pred', 'f0_denorm_pred'}``, same
state-dict keys including the BatchNorm buffers, so ``load_ckpt(pe, hparams['pe_ckpt'], 'model')`` works unchanged
(inference/svs/base_svs_infer.py:62-70).  Arithmetic: libagpt_b200.so (csrc/pe.cu).  CUDA only, inference only.
"""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from ... import _lib, paramtree, specs
from ...utils import hparams as _hp

_BUFFER_SUFFIXES = ("running_mean", "running_var", "num_batches_tracked", "_float_tensor")


class PitchExtractor(nn.Module):
    _h = _lib.engine_handle

    def __init__(self, n_mel_bins=80, conv_layers=2):
        super().__init__()
        hp = _hp.resolve()
        self.hidden_size = int(hp["hidden_size"])
        ph = int(hp.get("predictor_hidden", -1))
        self.predictor_hidden = ph if ph > 0 else self.hidden_size
        self.conv_layers = int(conv_layers)
        if hp.get("ffn_padding", "SAME") != "SAME":
            raise NotImplementedError("audiogpt_b200.PitchExtractor supports ffn_padding='SAME' (the shipped configs)")
        self.cfg = dict(n_mel_bins=int(n_mel_bins), hidden_size=self.hidden_size, conv_layers=self.conv_layers,
                        predictor_hidden=self.predictor_hidden, predictor_layers=5,
                        predictor_kernel=int(hp.get("predictor_kernel", 5)))
        self._shapes = specs.pe_param_shapes(self.cfg)
        for key, shape in self._shapes.items():
            if key.endswith(_BUFFER_SUFFIXES):      # registered as buffers, like the reference's BatchNorm1d / positional table
                val = torch.zeros(shape, dtype=torch.long if key.endswith("num_batches_tracked") else torch.float32)
                if key.endswith("running_var"):
                    val = torch.ones(shape)
                paramtree.add_buffer(self, key, val)
            else:
                paramtree.add_param(self, key, torch.zeros(shape))
        self._engine = _lib.Engine("agpt_pe_create")

    @torch.no_grad()
    def forward(self, mel_input=None):
        """mel_input [B, T, n_mel_bins] -> {'pitch_pred': [B, T, 2], 'f0_denorm_pred': [B, T]}   (pe.py:136-148)"""
        if not mel_input.is_cuda:
            raise RuntimeError("audiogpt_b200.PitchExtractor runs on CUDA only (no CPU fallback)")
        hp = _hp.resolve()
        ws = [paramtree.get_tensor(self, k) for k in self._shapes]
        self._engine.ensure(mel_input.device, ws, lambda: ((C.byref(_lib.PeCfg(**self.cfg)),), ws))
        mel = mel_input.contiguous().float()
        B, T, _ = mel.shape
        pred = torch.empty((B, T, 2), device=mel.device, dtype=torch.float32)
        f0 = torch.empty((B, T), device=mel.device, dtype=torch.float32)
        use_uv = 1 if (hp.get("pitch_type") == "frame" and hp.get("use_uv")) else 0
        norm = {"standard": 1, "log": 2}.get(hp.get("pitch_norm"), 0)
        self._engine.call("pe_forward", mel.device, _lib.fptr(mel), B, T, _lib.fptr(pred), _lib.fptr(f0), use_uv, norm,
                          float(hp.get("f0_mean", 0.0)), float(hp.get("f0_std", 1.0)))
        return {"pitch_pred": pred, "f0_denorm_pred": f0}
