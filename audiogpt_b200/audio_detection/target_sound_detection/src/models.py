"""Drop-in for ``target_sound_detection.src.models.RaDur_fusion``: the target-sound-detection network of the
TargetSoundDetection tool (audio-chatgpt.py:775-875), which finds where an event, given by a reference clip of it, occurs
in a clip.

Reference: audio_detection/target_sound_detection/src/models.py:1109-1291 (RaDur_fusion) and the parts it builds (Cnn14,
CDur_CNN_mul_scale_fusion, Cnn10_mul_scale, Fusion).  Same constructor ``(model_config, inputdim, outputdim,
time_resolution, **kwargs)`` reading ``att_pool``, ``enhancement``, ``tao`` and ``top`` from model_config, same
``forward(x, ref, label=None)`` returning ``(decision, decision_up, logit)``, same state-dict keys -- the encoder's
torchlibrosa front end, bn0 and fc_audioset, which its forward never runs, and every ``num_batches_tracked`` included --
so the checkpoint loads strictly.  Arithmetic: libagpt_b200.so (csrc/tsd.cu).  CUDA only, eval mode only.

Only ``RaDur_fusion`` is provided: the tool also imports ``event_labels`` from the reference module, so
``install(target_detection=True)`` patches that module in place and never stands in for it."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch
from torch import nn

from .... import _lib, paramtree, specs

__all__ = ["RaDur_fusion"]


class RaDur_fusion(nn.Module):
    _h = _lib.engine_handle

    def __init__(self, model_config, inputdim, outputdim, time_resolution, **kwargs):
        super().__init__()
        if int(inputdim) != 64:
            raise ValueError("RaDur_fusion: inputdim must be 64 (both CNNs pool the mel axis down to one column)")
        self.att_pool = model_config["att_pool"]
        self.enhancement = model_config["enhancement"]
        self.tao = model_config["tao"]
        self.top = model_config["top"]
        self.temperature = 11.3
        self.cfg = dict(time_resolution=int(time_resolution), att_pool=bool(self.att_pool), enhancement=bool(self.enhancement),
                        top=int(self.top), tao=float(self.tao), mel_bins=64, outputdim=int(outputdim))
        if self.cfg["top"] < 1 or not 1 <= self.cfg["outputdim"] <= 16:
            raise ValueError("RaDur_fusion: top must be >= 1 and outputdim in [1, 16]")
        self._keys = specs.tsd_engine_keys(self.cfg)
        g = torch.Generator().manual_seed(0)
        for key, shape in specs.tsd_param_shapes(self.cfg).items():
            if key.endswith("num_batches_tracked"):
                paramtree.add_buffer(self, key, torch.zeros((), dtype=torch.long))
            elif key.endswith("running_mean"):
                paramtree.add_buffer(self, key, torch.zeros(shape))
            elif key.endswith("running_var"):
                paramtree.add_buffer(self, key, torch.ones(shape))
            elif len(shape) == 1:     # BatchNorm scales are 1, every bias 0
                is_bn = any(p.startswith("bn") for p in key.split(".")[:-1])
                paramtree.add_param(self, key, torch.ones(shape) if is_bn and key.endswith(".weight") else torch.zeros(shape))
            else:
                paramtree.add_param(self, key, 0.02 * torch.randn(shape, generator=g))
        with torch.no_grad():     # the encoder's frozen front end is a function of Cnn14()'s defaults, as in torchlibrosa
            re, im = specs.stft_dft_weights(1024)
            self.encoder.spectrogram_extractor.stft.conv_real.weight.copy_(re)
            self.encoder.spectrogram_extractor.stft.conv_imag.weight.copy_(im)
            self.encoder.logmel_extractor.melW.copy_(torch.from_numpy(np.ascontiguousarray(specs.slaney_mel(32000, 1024, 64, 50, 14000).T)))
        self._engine = _lib.Engine("agpt_tsd_create")

    def _config(self):
        c = self.cfg
        return _lib.TsdConfig(time_resolution=c["time_resolution"], att_pool=int(c["att_pool"]), enhancement=int(c["enhancement"]),
                              top=c["top"], tao=c["tao"], mel_bins=64, outputdim=c["outputdim"])

    def frames(self, T, Tr):
        """(T', Tr', Te) for a T-frame clip and a Tr-frame reference (specs.tsd_frames)."""
        return specs.tsd_frames(self.cfg, T, Tr)

    @torch.no_grad()
    def forward(self, x, ref, label=None):
        """x [B, T, 64] log-mel of the clip, ref [B, Tr, 64] log-mel of the reference (CUDA) -> (decision [B, T'],
        decision_up [B, T, outputdim], logit = zeros(1)), as the reference returns them."""
        if self.training:
            raise RuntimeError("audiogpt_b200.RaDur_fusion is inference only: call .eval() first (the tool does)")
        for name, t in (("x", x), ("ref", ref)):
            if not torch.is_tensor(t) or not t.is_cuda:
                raise RuntimeError("audiogpt_b200.RaDur_fusion runs on CUDA only (no CPU fallback)")
            if t.dim() != 3 or t.shape[2] != 64 or t.shape[0] < 1:
                raise ValueError(f"{name} must be (batch, frames, 64), got {tuple(t.shape)}")
        if x.shape[0] != ref.shape[0]:
            raise ValueError(f"x and ref must have the same batch size, got {x.shape[0]} and {ref.shape[0]}")
        if x.device != ref.device:
            raise ValueError("x and ref must be on the same device")
        B, T, _ = x.shape
        Tr = ref.shape[1]
        Td = specs.tsd_frames(self.cfg, T, Tr)[0]      # raises ValueError for a clip or reference that is too short
        dev = x.device
        srcs = [paramtree.get_tensor(self, k) for k in self._keys]
        cc = self._config()
        self._engine.ensure(dev, srcs, lambda: ((C.byref(cc),), srcs))
        xx = x.to(torch.float32).contiguous()
        rr = ref.to(torch.float32).contiguous()
        decision = torch.empty((B, Td), device=dev, dtype=torch.float32)
        up = torch.empty((B, T, self.cfg["outputdim"]), device=dev, dtype=torch.float32)
        self._engine.call("tsd_forward", dev, _lib.fptr(xx), _lib.fptr(rr), B, T, Tr, _lib.fptr(decision), _lib.fptr(up))
        return decision, up, torch.zeros(1, device=dev)
