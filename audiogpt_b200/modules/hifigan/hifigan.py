"""Drop-in for ``modules.hifigan.hifigan.HifiGanGenerator``.

Reference: /root/reference/NeuralSeq/modules/hifigan/hifigan.py:104-178 (and the
architecture-identical twin text_to_audio/Make_An_Audio/vocoder/hifigan/modules.py:86-136).

Same constructor (``h`` dict, ``c_out``), same ``forward(x, f0=None)``, same
``remove_weight_norm()``, same ``state_dict`` key layout before *and* after
weight-norm removal (``*.weight_g`` / ``*.weight_v``  vs  ``*.weight``), so
``load_model`` (NeuralSeq/vocoders/hifigan.py:17-33) works unchanged:

    model = HifiGanGenerator(config); model.load_state_dict(state, strict=True)
    model.remove_weight_norm(); model = model.eval().to(device)

The arithmetic runs in libagpt_b200.so (hand-written sm_90a kernels); the
module only stores parameters.  There is no CPU path: ``forward`` on a CPU
tensor raises.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch
from torch import nn

from ... import _lib, paramtree, specs

LRELU_SLOPE = 0.1


def get_padding(kernel_size, dilation=1):
    return (kernel_size * dilation - dilation) // 2


def _wn_key(key: str) -> bool:
    """Which parameters carry weight-norm in the reference: every conv of the generator
    except the NSF noise_convs / m_source (hifigan.py:33-48,118,124,140)."""
    return key.endswith(".weight") and not key.startswith(("noise_convs.", "m_source."))


def fold_weight_norm(g: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """torch.nn.utils.weight_norm(dim=0): w = g * v / ||v||, norm over all dims but 0
    (for ConvTranspose1d weights [C_in, C_out, k] that is per *input* channel)."""
    n = v.reshape(v.shape[0], -1).norm(dim=1).reshape(-1, *([1] * (v.dim() - 1)))
    return g * v / n


class SourceModuleHnNSF(nn.Module):
    """Harmonic-plus-noise excitation, drop-in for ``SourceModuleHnNSF`` + ``SineGen``
    (NeuralSeq/modules/parallel_wavegan/models/source.py:311-441,484-532): same constructor, same
    ``forward(f0 [B, L, 1]) -> (sine_merge [B, L, 1], noise [B, L, 1], uv [B, L, 1])``, same ``l_linear.*`` keys.

    The arithmetic (phase prefix sum, 9 harmonic sines, uv gating, noise mix, Linear(9 -> 1) + tanh) is ONE fused
    pass in libagpt_b200.so (agpt_nsf_source: a three-level fp64 scan over the ~10^5 samples of an utterance); the
    random draws stay in torch, in the reference's call order and shapes -- ``torch.rand(B, dim)`` (initial
    phases), ``torch.randn_like(sines)``, ``torch.randn_like(uv)`` -- so a seeded run consumes the generator exactly
    like the reference does.  CUDA only."""

    def __init__(self, sampling_rate, harmonic_num=0, sine_amp=0.1, add_noise_std=0.003, voiced_threshod=0,
                 voiced_threshold=None):
        super().__init__()
        self.sampling_rate, self.harmonic_num = sampling_rate, harmonic_num
        self.sine_amp, self.noise_std = sine_amp, add_noise_std
        self.voiced_threshold = voiced_threshod if voiced_threshold is None else voiced_threshold
        self.l_linear = nn.Linear(harmonic_num + 1, 1)

    def draw(self, f0):
        """The three RNG draws of the reference, in its order: (rand_ini [B, dim], noise [B, L, dim], noise_src)."""
        B, L, _ = f0.shape
        dim = self.harmonic_num + 1
        rand_ini = torch.rand(B, dim, device=f0.device)
        noise = torch.randn(B, L, dim, device=f0.device, dtype=f0.dtype)
        noise_src = torch.randn(B, L, 1, device=f0.device, dtype=f0.dtype) * self.sine_amp / 3
        return rand_ini, noise, noise_src

    @torch.no_grad()
    def forward(self, f0, rand_ini=None, noise=None):  # f0 [B, L, 1]
        if not f0.is_cuda:
            raise RuntimeError("audiogpt_b200.SourceModuleHnNSF runs on CUDA only (no CPU fallback)")
        B, L, _ = f0.shape
        dim = self.harmonic_num + 1
        noise_src = None
        if rand_ini is None or noise is None:
            rand_ini, noise, noise_src = self.draw(f0)
        if noise_src is None:
            noise_src = torch.randn(B, L, 1, device=f0.device, dtype=f0.dtype) * self.sine_amp / 3
        f0c = f0.reshape(B, L).contiguous().float()
        w = self.l_linear.weight.detach().reshape(-1).float().cpu().numpy().copy()
        b = float(self.l_linear.bias.detach().float().cpu()[0])
        har = torch.empty((B, L), device=f0.device, dtype=torch.float32)
        ri = rand_ini.contiguous().float()
        nz = noise.contiguous().float()
        _lib.call("nsf_source", f0.device, _lib.fptr(f0c), B, L, dim, float(self.sampling_rate), w.ctypes.data_as(C.c_void_p),
                  b, _lib.fptr(ri), _lib.fptr(nz), float(self.sine_amp), float(self.noise_std), float(self.voiced_threshold),
                  _lib.fptr(har))
        uv = (f0 > self.voiced_threshold).to(f0.dtype)
        return har[:, :, None], noise_src, uv


class HifiGanGenerator(nn.Module):
    _h = _lib.engine_handle

    def __init__(self, h, c_out=1):
        super().__init__()
        self.h = h
        self._init_generator(dict(h, activation=0, snake_logscale=0), c_out, specs.hifigan_param_shapes(h, c_out),
                             bool(h.get("use_pitch_embed", False)))
        if self._use_nsf:
            self.harmonic_num = 8
            self.m_source = SourceModuleHnNSF(sampling_rate=h["audio_sample_rate"], harmonic_num=self.harmonic_num)

    def _init_generator(self, hd, c_out, shapes, use_nsf):
        """What HiFi-GAN and BigVGAN share.  ``hd``: the config with HiFi-GAN's keys plus ``activation`` (0 leaky-relu,
        1 snake, 2 snakebeta) and ``snake_logscale`` (0 / 1); ``shapes``: the folded state-dict table."""
        self._hd, self.c_out, self._shapes, self._use_nsf = hd, c_out, shapes, use_nsf
        self.num_kernels = len(hd["resblock_kernel_sizes"])
        self.num_upsamples = len(hd["upsample_rates"])
        self.hop = int(np.prod(hd["upsample_rates"]))
        self._weight_norm = True
        self._engine = _lib.Engine("agpt_hifigan_create")
        g = torch.Generator().manual_seed(0)
        for key, shape in shapes.items():
            if key.startswith("m_source."):
                continue
            if _wn_key(key):
                v = torch.randn(shape, generator=g) * 0.01
                n = v.reshape(shape[0], -1).norm(dim=1).reshape(-1, *([1] * (len(shape) - 1)))
                paramtree.add_param(self, key + "_g", n.clone())
                paramtree.add_param(self, key + "_v", v)
            else:
                paramtree.add_param(self, key, self._initial_value(key, shape))

    def _initial_value(self, key, shape):
        return torch.zeros(shape)

    # ------------------------------------------------------------------ weight-norm
    def remove_weight_norm(self):
        if not self._weight_norm:
            return
        print("Removing weight norm...")
        for key in self._shapes:
            if key.startswith("m_source.") or not _wn_key(key):
                continue
            g, v = paramtree.get_param(self, key + "_g"), paramtree.get_param(self, key + "_v")
            w = fold_weight_norm(g.data, v.data)
            paramtree.del_param(self, key + "_g")
            paramtree.del_param(self, key + "_v")
            paramtree.add_param(self, key, w)
        self._weight_norm = False

    def load_state_dict(self, state_dict, strict=True, **kw):
        has_wn = any(k.endswith(".weight_g") for k in state_dict)
        if not has_wn and self._weight_norm:
            # checkpoint saved after remove_weight_norm(): switch this module to the folded layout
            self.remove_weight_norm()
        elif has_wn and not self._weight_norm:
            sd = {}
            for k, v in state_dict.items():
                if k.endswith(".weight_g"):
                    sd[k[:-2]] = fold_weight_norm(v, state_dict[k[:-2] + "_v"])
                elif not k.endswith(".weight_v"):
                    sd[k] = v
            state_dict = sd
        return super().load_state_dict(state_dict, strict=strict, **kw)

    def folded_weights(self):
        """fp32 tensors in specs.hifigan_param_shapes order, weight-norm folded."""
        out = []
        for key in self._shapes:
            if self._weight_norm and _wn_key(key):
                out.append(fold_weight_norm(paramtree.get_param(self, key + "_g").data,
                                            paramtree.get_param(self, key + "_v").data))
            else:
                out.append(paramtree.get_param(self, key).data)
        return out

    # ------------------------------------------------------------------ engine
    def _cfg(self):
        hd = self._hd
        c = _lib.HifiganCfg()
        # the reference hard-codes Conv1d(80, ...) for conv_pre (hifigan.py:118); take it from the parameter table
        c.n_mels, c.c_out = int(self._shapes["conv_pre.weight"][1]), self.c_out
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
        c.use_nsf = int(self._use_nsf)
        c.activation, c.snake_logscale = hd["activation"], hd["snake_logscale"]
        return c

    def _build_engine(self, device):
        # the weight-norm layout changes the keys, so the engine is signed by the whole state dict
        self._engine.ensure(device, self.state_dict(keep_vars=True).values(),
                            lambda: ((C.byref(self._cfg()),), self.folded_weights()))

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, x, f0=None):
        """x: [B, 80, T] fp32 CUDA -> [B, c_out, T*hop]   (hifigan.py:144-169)"""
        if not x.is_cuda:
            raise RuntimeError("audiogpt_b200.HifiGanGenerator runs on CUDA only (no CPU fallback); "
                               "move the model and input to a CUDA device (H100)")
        x = x.contiguous().float()
        B, M, T = x.shape
        self._build_engine(x.device)
        har = None
        if f0 is not None:
            if not self._use_nsf:
                raise RuntimeError("f0 given but the generator was built without use_pitch_embed")
            f0u = torch.repeat_interleave(f0[:, None].float(), self.hop, dim=2).transpose(1, 2)  # nearest x hop
            har, _, _ = self.m_source(f0u)
            har = har.transpose(1, 2).contiguous()
        wav = torch.empty((B, self.c_out, T * self.hop), device=x.device, dtype=torch.float32)
        self._engine.call("hifigan_forward", x.device, _lib.fptr(x), _lib.fptr(har) if har is not None else None,
                          B, T, _lib.fptr(wav))
        return wav

    @torch.no_grad()
    def vocode_host(self, mel: np.ndarray, har: np.ndarray = None, device=None) -> np.ndarray:
        """Host-buffer entry (numpy [B,80,T] -> numpy [B,c_out,T*hop]); H2D/D2H inside the call."""
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self._build_engine(dev)
        mel = np.ascontiguousarray(mel, dtype=np.float32)
        B, M, T = mel.shape
        wav = np.empty((B, self.c_out, T * self.hop), dtype=np.float32)
        hp = None
        if har is not None:
            har = np.ascontiguousarray(har, dtype=np.float32)
            hp = har.ctypes.data_as(C.c_void_p)
        _lib.check(_lib.lib().agpt_hifigan_vocode_host(
            self._h, mel.ctypes.data_as(C.c_void_p), hp, B, T, wav.ctypes.data_as(C.c_void_p)))
        return wav
