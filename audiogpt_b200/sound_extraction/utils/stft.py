"""Drop-in for ``sound_extraction.utils.stft.STFT``: the conv-STFT and inverse STFT of the SoundExtraction tool
(audio-chatgpt.py:675-710).

Reference: sound_extraction/utils/stft.py:53-147.  Same constructor ``(filter_length=1024, hop_length=512,
win_length=1024, window='hann')``, same ``forward_basis`` / ``inverse_basis`` buffers, same ``transform``, ``inverse``
and ``forward``.  Arithmetic: libagpt_b200.so (csrc/lass.cu; both directions are 2-tap GEMMs over hop-sample rows).

CUDA tensors stay on their device.  The tool calls it with CPU tensors: those run on the current CUDA device and come
back as CPU tensors (the host-buffer contract HifiGAN.spec2wav has); without a CUDA device it raises.  Only the
tool's geometry is covered: window 'hann', win_length = filter_length = 2 hop_length.
"""
from __future__ import annotations

import torch
from torch import nn

from ... import _lib, specs


class STFT(nn.Module):
    """adapted from Prem Seetharaman's https://github.com/pseeth/pytorch-stft (on the engine)"""

    def __init__(self, filter_length=1024, hop_length=512, win_length=1024, window="hann"):
        super().__init__()
        if window != "hann" or win_length != filter_length or filter_length != 2 * hop_length or hop_length % 8:
            raise NotImplementedError("audiogpt_b200.STFT runs window='hann' with win_length = filter_length = 2 hop_length "
                                      f"(hop a multiple of 8), got {filter_length}, {hop_length}, {win_length}, {window!r}")
        self.filter_length = filter_length
        self.hop_length = hop_length
        self.win_length = win_length
        self.window = window
        self.forward_transform = None
        fwd, inv = specs.stft_bases(filter_length, hop_length)
        self.register_buffer("forward_basis", fwd)
        self.register_buffer("inverse_basis", inv)
        self._engine = _lib.Engine("agpt_stft_create")

    def _device(self, t):
        _lib.require_cuda()
        dev = t.device if t.is_cuda else torch.device("cuda", torch.cuda.current_device())
        bufs = [self.forward_basis, self.inverse_basis]
        self._engine.ensure(dev, bufs, lambda: ((self.filter_length, self.hop_length), bufs))
        return dev

    @torch.no_grad()
    def transform(self, input_data):
        """[B, N] -> (magnitude, phase) [B, filter_length / 2 + 1, N // hop + 1] (on input_data's device)."""
        num_batches = input_data.size(0)
        num_samples = input_data.size(1)
        self.num_samples = num_samples
        if input_data.dim() != 2:
            raise ValueError(f"STFT.transform takes [B, N] samples, got {tuple(input_data.shape)}")
        dev = self._device(input_data)
        x = input_data.to(dev, torch.float32).contiguous()
        nb, T = self.filter_length // 2 + 1, num_samples // self.hop_length + 1
        mag = torch.empty((num_batches, nb, T), device=dev, dtype=torch.float32)
        phase = torch.empty_like(mag)
        self._engine.call("stft_transform", dev, _lib.fptr(x), num_batches, num_samples, _lib.fptr(mag), _lib.fptr(phase))
        if not input_data.is_cuda:
            return mag.cpu(), phase.cpu()
        return mag, phase

    @torch.no_grad()
    def inverse(self, magnitude, phase):
        """(magnitude, phase) [B, filter_length / 2 + 1, T] -> [B, 1, (T - 1) hop] (on magnitude's device)."""
        if magnitude.dim() != 3 or phase.shape != magnitude.shape or magnitude.shape[1] != self.filter_length // 2 + 1:
            raise ValueError(f"STFT.inverse takes magnitude and phase [B, {self.filter_length // 2 + 1}, T], got "
                             f"{tuple(magnitude.shape)} and {tuple(phase.shape)}")
        dev = self._device(magnitude)
        B, _, T = magnitude.shape
        m = magnitude.to(dev, torch.float32).contiguous()
        p = phase.to(dev, torch.float32).contiguous()
        out = torch.empty((B, 1, (T - 1) * self.hop_length), device=dev, dtype=torch.float32)
        self._engine.call("stft_inverse", dev, _lib.fptr(m), _lib.fptr(p), B, T, _lib.fptr(out))
        return out if magnitude.is_cuda else out.cpu()

    def forward(self, input_data):
        self.magnitude, self.phase = self.transform(input_data)
        reconstruction = self.inverse(self.magnitude, self.phase)
        return reconstruction
