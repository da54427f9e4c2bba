"""Drop-in for ``vocoder.bigvgan.models`` of Make-An-Audio (SURVEY.md 8f, "next" row 2).

Reference: /root/reference/text_to_audio/Make_An_Audio/vocoder/bigvgan/models.py:133-203 (``BigVGAN``),
:29-130 (``AMPBlock1`` / ``AMPBlock2``), :393-414 (``VocoderBigVGAN``); activations.py:46-57,104-117;
alias_free_torch/{act,resample,filter}.py.  This is the vocoder ``audio-chatgpt.py:145,180`` dispatches for
text-to-audio.

Same constructor (``h`` with attribute or item access), same ``forward(x)`` (``[B, num_mels, T]`` ->
``[B, 1, T * prod(upsample_rates)]``), same ``remove_weight_norm()``, same ``state_dict`` keys before and
after weight-norm removal (including the ``*.filter`` buffers of every ``Activation1d``), so
``generator.load_state_dict(vocoder_sd['generator'])`` works unchanged.

BigVGAN is the HiFi-GAN generator with every leaky-relu replaced by an anti-aliased periodic
activation; the engine is the same C-ABI object (``agpt_hifigan_*`` with ``cfg.activation != 0``): the
convolutions run on the wgmma tap-GEMM kernel, the activations in ``aa_snake_kernel``
(csrc/hifigan.cu).  CUDA only -- no CPU path.
"""
from __future__ import annotations

import os

import numpy as np
import torch
from torch import nn

from ... import specs
from ...modules.hifigan.hifigan import HifiGanGenerator

LRELU_SLOPE = 0.1


def _as_dict(h):
    if isinstance(h, dict):
        return dict(h)
    keys = ("resblock", "num_mels", "upsample_rates", "upsample_kernel_sizes", "upsample_initial_channel",
            "resblock_kernel_sizes", "resblock_dilation_sizes", "activation", "snake_logscale")
    out = {}
    for k in keys:
        try:
            out[k] = h[k] if hasattr(h, "__getitem__") else getattr(h, k)
        except Exception:
            if hasattr(h, k):
                out[k] = getattr(h, k)
    return out


class BigVGAN(HifiGanGenerator):
    def __init__(self, h):
        nn.Module.__init__(self)
        self.h = h
        hd = _as_dict(h)
        hd.setdefault("num_mels", 80)
        hd.setdefault("snake_logscale", False)
        hd["upsample_rates"] = [int(v) for v in hd["upsample_rates"]]
        hd["upsample_kernel_sizes"] = [int(v) for v in hd["upsample_kernel_sizes"]]
        hd["resblock_kernel_sizes"] = [int(v) for v in hd["resblock_kernel_sizes"]]
        hd["resblock_dilation_sizes"] = [[int(d) for d in dl] for dl in hd["resblock_dilation_sizes"]]
        if str(hd["activation"]) not in ("snake", "snakebeta"):
            raise NotImplementedError("activation incorrectly specified. check the config file and look for 'activation'.")
        shapes = specs.bigvgan_param_shapes(hd)
        hd.update(activation=2 if str(hd["activation"]) == "snakebeta" else 1, snake_logscale=int(bool(hd["snake_logscale"])))
        self._init_generator(hd, 1, shapes, False)

    def _initial_value(self, key, shape):
        if key.endswith(".filter"):
            return specs.kaiser_sinc_filter12()
        if key.endswith((".act.alpha", ".act.beta")):
            return torch.zeros(shape) if self._hd["snake_logscale"] else torch.ones(shape)
        return torch.zeros(shape)

    def folded_weights(self):
        """C-ABI order (include/agpt_b200.h, agpt_hifigan_cfg): state-dict order without the filter buffers,
        then the 12 filter taps once."""
        ws = dict(zip(self._shapes, super().folded_weights()))
        filt = [ws.pop(k) for k in list(ws) if k.endswith(".filter")][-1]
        return list(ws.values()) + [filt.reshape(-1)]

    @torch.no_grad()
    def forward(self, x):
        """x: [B, num_mels, T] fp32 CUDA -> [B, 1, T*hop]   (models.py:177-203)"""
        return HifiGanGenerator.forward(self, x, None)


class VocoderBigVGAN(object):
    """models.py:393-414.  ``ckpt_vocoder``: directory with ``best_netG.pt`` and ``args.yml`` (as in the
    reference) -- or pass a ready ``generator``."""

    def __init__(self, ckpt_vocoder=None, device="cuda", generator=None):
        if generator is None:
            import yaml
            vocoder_sd = torch.load(os.path.join(ckpt_vocoder, "best_netG.pt"), map_location="cpu")
            with open(os.path.join(ckpt_vocoder, "args.yml")) as f:
                vocoder_args = yaml.safe_load(f)
            generator = BigVGAN(vocoder_args)
            generator.load_state_dict(vocoder_sd["generator"])
        self.generator = generator.eval()
        self.device = device
        self.generator.to(self.device)

    def vocode(self, spec):
        with torch.no_grad():
            if isinstance(spec, np.ndarray):
                spec = torch.from_numpy(spec).unsqueeze(0)
            spec = spec.to(dtype=torch.float32, device=self.device)
            return self.generator(spec).squeeze().cpu().numpy()

    def __call__(self, wav):
        return self.vocode(wav)
