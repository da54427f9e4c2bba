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

from ... import _lib, paramtree, specs
from ...modules.hifigan.hifigan import HifiGanGenerator, fold_weight_norm, _wn_key

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
        _lib.HandleOwner.__init__(self)
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
        self._hd = hd
        self.c_out = 1
        self.num_kernels = len(hd["resblock_kernel_sizes"])
        self.num_upsamples = len(hd["upsample_rates"])
        self.hop = int(np.prod(hd["upsample_rates"]))
        self._use_nsf = False
        self._shapes = specs.bigvgan_param_shapes(hd)
        self._weight_norm = True
        g = torch.Generator().manual_seed(0)
        filt = specs.kaiser_sinc_filter12()
        for key, shape in self._shapes.items():
            if key.endswith(".filter"):
                paramtree.add_param(self, key, filt.clone())
            elif _wn_key(key):
                v = torch.randn(shape, generator=g) * 0.01
                n = v.reshape(shape[0], -1).norm(dim=1).reshape(-1, *([1] * (len(shape) - 1)))
                paramtree.add_param(self, key + "_g", n.clone())
                paramtree.add_param(self, key + "_v", v)
            elif key.endswith((".act.alpha", ".act.beta")):
                init = torch.zeros(shape) if hd["snake_logscale"] else torch.ones(shape)
                paramtree.add_param(self, key, init)
            else:
                paramtree.add_param(self, key, torch.zeros(shape))
        self._engine_sig = None

    def folded_weights(self):
        """C-ABI order (include/agpt_b200.h, agpt_hifigan_cfg): state-dict order without the filter buffers,
        then the 12 filter taps once."""
        out, filt = [], None
        for key in self._shapes:
            if key.endswith(".filter"):
                filt = paramtree.get_param(self, key).data.reshape(-1)
                continue
            if self._weight_norm and _wn_key(key):
                out.append(fold_weight_norm(paramtree.get_param(self, key + "_g").data,
                                            paramtree.get_param(self, key + "_v").data))
            else:
                out.append(paramtree.get_param(self, key).data)
        out.append(filt)
        return out

    def _cfg(self):
        hd = self._hd
        c = _lib.HifiganCfg()
        c.n_mels, c.c_out = int(hd["num_mels"]), 1
        c.upsample_initial_channel = int(hd["upsample_initial_channel"])
        c.num_upsamples = self.num_upsamples
        for i, (u, k) in enumerate(zip(hd["upsample_rates"], hd["upsample_kernel_sizes"])):
            c.upsample_rates[i], c.upsample_kernel_sizes[i] = int(u), int(k)
        c.resblock_type = 1 if str(hd["resblock"]) == "1" else 2
        c.num_kernels = self.num_kernels
        for j, (ks, dil) in enumerate(zip(hd["resblock_kernel_sizes"], hd["resblock_dilation_sizes"])):
            c.resblock_kernel_sizes[j] = int(ks)
            c.resblock_num_dilations[j] = len(dil)
            for n, d in enumerate(dil):
                c.resblock_dilations[j][n] = int(d)
        c.use_nsf = 0
        c.activation = 2 if str(hd["activation"]) == "snakebeta" else 1
        c.snake_logscale = 1 if hd["snake_logscale"] else 0
        return c

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
