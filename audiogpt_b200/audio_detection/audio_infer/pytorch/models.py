"""Drop-in for ``audio_infer.pytorch.models.PVT``: the pyramid vision transformer of the SoundDetection tool
(audio-chatgpt.py:612-673), which turns a 32 kHz clip into framewise and clipwise probabilities of the 527 AudioSet
classes.

Reference: audio_detection/audio_infer/pytorch/models.py:141-237 (PVT), :619-940 (PyramidVisionTransformerV2 and its
parts).  Same constructor, same ``forward(input, mixup_lambda=None)`` returning ``{'framewise_output',
'clipwise_output'}``, same state-dict keys -- the frozen front-end tensors the checkpoint carries
(``spectrogram_extractor.stft.conv_real / conv_imag.weight``, ``logmel_extractor.melW``), ``bn0``'s running statistics
and ``num_batches_tracked`` included -- so ``model.load_state_dict(checkpoint['model'])`` loads strictly.  It needs none
of torchlibrosa, timm, mmcv and mmdet, which the reference module imports.  Arithmetic: libagpt_b200.so (csrc/pvt.cu).
CUDA only, eval mode only (no time shift, SpecAugment, mixup, Dropout or DropPath).

Only ``PVT`` is provided; the reference file's other variants (PVT2, PVT_2layer, PVT_lr, PVT_nopretrain) and Cnn
detectors are used by no tool.  ``PVT.from_config(cfg)`` builds other sizes (specs.PVT_SMALL)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch
from torch import nn

from .... import _lib, paramtree, specs

__all__ = ["PVT"]


class PVT(nn.Module):
    _h = _lib.engine_handle

    def __init__(self, sample_rate, window_size, hop_size, mel_bins, fmin, fmax, classes_num):
        super().__init__()
        self._setup(dict(specs.PVT_SHIPPED, sample_rate=sample_rate, window_size=window_size, hop_size=hop_size,
                         mel_bins=mel_bins, fmin=fmin, fmax=fmax, classes_num=classes_num))

    @classmethod
    def from_config(cls, cfg):
        """Built from a specs.PVT_SHIPPED-style config (any stage widths the engine accepts)."""
        self = cls.__new__(cls)
        nn.Module.__init__(self)
        self._setup(cfg)
        return self

    def _setup(self, cfg):
        self.cfg = cfg = dict(cfg)
        if int(cfg["mel_bins"]) != 64:
            raise ValueError("PVT: mel_bins must be 64 (bn0 is BatchNorm2d(64))")
        if any(int(d) != 64 * int(h) for d, h in zip(cfg["embed_dims"], cfg["num_heads"])):
            raise ValueError("PVT: the engine runs 64-wide attention heads (embed_dims[i] == 64 * num_heads[i])")
        self._keys = specs.pvt_engine_keys(cfg)
        g = torch.Generator().manual_seed(0)
        for key, shape in specs.pvt_param_shapes(cfg).items():
            if key.endswith("num_batches_tracked"):
                paramtree.add_buffer(self, key, torch.zeros((), dtype=torch.long))
            elif key.endswith("running_mean"):
                paramtree.add_buffer(self, key, torch.zeros(shape))
            elif key.endswith("running_var"):
                paramtree.add_buffer(self, key, torch.ones(shape))
            elif len(shape) == 1:     # LayerNorm / bn0 scales are 1, every bias 0, as the reference initialises them
                paramtree.add_param(self, key, torch.ones(shape) if key.endswith(".weight") else torch.zeros(shape))
            else:
                paramtree.add_param(self, key, 0.02 * torch.randn(shape, generator=g))
        with torch.no_grad():     # the frozen front end is a function of the config, as in torchlibrosa
            re, im = specs.stft_dft_weights(int(cfg["window_size"]))
            self.spectrogram_extractor.stft.conv_real.weight.copy_(re)
            self.spectrogram_extractor.stft.conv_imag.weight.copy_(im)
            self.logmel_extractor.melW.copy_(torch.from_numpy(np.ascontiguousarray(specs.slaney_mel(
                cfg["sample_rate"], cfg["window_size"], cfg["mel_bins"], cfg["fmin"], cfg["fmax"]).T)))
        self._engine = _lib.Engine("agpt_pvt_create")

    def _config(self):
        c = self.cfg
        cc = _lib.PvtConfig(window_size=c["window_size"], hop_size=c["hop_size"], mel_bins=c["mel_bins"],
                            classes_num=c["classes_num"], interpolate_ratio=c["interpolate_ratio"],
                            layer_norm_eps=c["layer_norm_eps"], embed_norm_eps=c["embed_norm_eps"])
        for name in ("embed_dims", "depths", "num_heads", "mlp_ratios", "sr_ratios"):
            getattr(cc, name)[:] = [int(v) for v in c[name]]
        return cc

    @torch.no_grad()
    def forward(self, input, mixup_lambda=None, return_logits=False):
        """input: (batch_size, n_samples) CUDA waveform.  Returns ``{'framewise_output': [B, 32 * H4, classes],
        'clipwise_output': [B, classes]}`` (and ``'logits'`` [B, H4, classes] with return_logits)."""
        if self.training:
            raise RuntimeError("audiogpt_b200.PVT is inference only: call .eval() first (the tool does)")
        if not torch.is_tensor(input) or not input.is_cuda:
            raise RuntimeError("audiogpt_b200.PVT runs on CUDA only (no CPU fallback)")
        if input.dim() != 2 or input.shape[0] < 1:
            raise ValueError(f"input must be (batch_size, n_samples), got {tuple(input.shape)}")
        B, n = input.shape
        H4 = specs.pvt_grids(self.cfg, n)[-1][0]      # raises ValueError for a clip that is too short
        dev = input.device
        srcs = [paramtree.get_tensor(self, k) for k in self._keys]
        cc = self._config()
        self._engine.ensure(dev, srcs, lambda: ((C.byref(cc),), srcs))
        wav = input.to(torch.float32).contiguous()
        K = int(self.cfg["classes_num"])
        frame = torch.empty((B, int(self.cfg["interpolate_ratio"]) * H4, K), device=dev, dtype=torch.float32)
        clip = torch.empty((B, K), device=dev, dtype=torch.float32)
        logits = torch.empty((B, H4, K), device=dev, dtype=torch.float32) if return_logits else None
        self._engine.call("pvt_forward", dev, _lib.fptr(wav), B, n, _lib.fptr(frame), _lib.fptr(clip),
                          _lib.fptr(logits) if return_logits else None)
        out = {"framewise_output": frame, "clipwise_output": clip}
        if return_logits:
            out["logits"] = logits
        return out
