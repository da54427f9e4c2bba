"""Drop-in for ``modules.diff.net.DiffNet`` (the WaveNet-style epsilon predictor).

Reference: /root/reference/NeuralSeq/modules/diff/net.py:81-130 (DiffNet), :58-78
(ResidualBlock), :32-44 (SinusoidalPosEmb).  Same constructor (reads the global
``hparams`` for hidden_size / residual_layers / residual_channels /
dilation_cycle_length), same ``forward(spec, diffusion_step, cond)``, same
state-dict keys (``input_projection.*``, ``mlp.{0,2}.*``,
``residual_layers.{i}.{dilated_conv,diffusion_projection,conditioner_projection,
output_projection}.*``, ``skip_projection.*``, ``output_projection.*``).

Arithmetic: libagpt_b200.so (csrc/diffnet.cu).  The step-invariant
``conditioner_projection(cond)`` of all layers is hoisted into one GEMM and cached
per ``cond`` tensor.  CUDA only.
"""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from ... import _lib, paramtree, specs
from ...utils import hparams as _hp


class DiffNet(nn.Module):
    _h = _lib.engine_handle

    def __init__(self, in_dims=80, **overrides):
        super().__init__()
        hp = dict(_hp.resolve())
        hp.update(overrides)
        self.cfg = dict(in_dims=in_dims, hidden_size=hp["hidden_size"],
                        residual_layers=hp["residual_layers"],
                        residual_channels=hp["residual_channels"],
                        dilation_cycle_length=hp["dilation_cycle_length"])
        self._shapes = specs.diffnet_param_shapes(self.cfg)
        paramtree.build(self, self._shapes)
        self._engine = _lib.Engine("agpt_diffnet_create")
        self._cond_key = None

    def set_cond(self, cond: torch.Tensor):
        """cond [B, hidden, T]; cached until a different tensor (or an in-place change) arrives."""
        if not cond.is_cuda:
            raise RuntimeError("audiogpt_b200.DiffNet runs on CUDA only (no CPU fallback)")
        ws = [paramtree.get_tensor(self, k) for k in self._shapes]
        if self._engine.ensure(cond.device, ws, lambda: ((C.byref(_lib.DiffnetCfg(**self.cfg)),), ws)):
            self._cond_key = None
        key = (cond.data_ptr(), cond._version, tuple(cond.shape))
        if key == self._cond_key:
            return
        c = cond.contiguous().float()
        self._engine.call("diffnet_set_cond", cond.device, _lib.fptr(c), c.shape[0], c.shape[2])
        self._cond_key = key
        # hold the keyed tensor: while it is alive the caching allocator cannot hand its block to the next
        # utterance's decoder_inp (same B/T/H, version 0), which would make the key match a different cond
        self._cond_keep = (cond, c)
        self._cond_shape = tuple(c.shape)

    @torch.no_grad()
    def forward(self, spec, diffusion_step, cond):
        """spec [B,1,M,T], diffusion_step [B] (tensor or list of ints), cond [B,H,T] -> [B,1,M,T]"""
        self.set_cond(cond)
        x = spec.contiguous().float()
        B = x.shape[0]
        t = diffusion_step.tolist() if torch.is_tensor(diffusion_step) else list(diffusion_step)
        assert len(t) == B
        tt = (C.c_int * B)(*[int(v) for v in t])
        out = torch.empty_like(x)
        self._engine.call("diffnet_eps", x.device, _lib.fptr(x), tt, _lib.fptr(out))
        return out
