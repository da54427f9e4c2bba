"""Drop-in for ``src.models.BinauralNetwork``: the mono-to-binaural network of the Binaural tool (audio-chatgpt.py:713-773).

Reference: mono2binaural/src/models.py (BinauralNetwork, Warpnet, GeometricWarper), warping.py and utils.py (Net).  Same
constructor ``(view_dim=7, warpnet_layers=4, warpnet_channels=64, model_name='binaural_network', use_cuda=True)`` --
``view_dim`` is ignored as it is there, and ``use_cuda`` moves the module to the GPU in ``__init__`` -- the same ``Net``
methods (``load_from_file``, ``load``, ``save``, ``num_trainable_parameters``) and the same state-dict keys, so the
shipped ``binaural_network.net`` loads strictly.  Arithmetic: libagpt_b200.so (csrc/binaural.cu).  CUDA only, eval only.

``binauralize(mono, view)`` is the tool's whole chunk loop (trims, chunks, kept tails, cat, clamp) as one engine call."""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from ... import _lib, paramtree, specs

__all__ = ["BinauralNetwork"]


class BinauralNetwork(nn.Module):
    _h = _lib.engine_handle

    def __init__(self, view_dim=7, warpnet_layers=4, warpnet_channels=64, model_name="binaural_network", use_cuda=True):
        super().__init__()
        self.use_cuda = use_cuda
        self.model_name = model_name
        self.cfg = dict(layers=int(warpnet_layers), channels=int(warpnet_channels))
        self._keys = list(specs.binaural_param_shapes(self.cfg))
        g = torch.Generator().manual_seed(0)
        for key, shape in specs.binaural_param_shapes(self.cfg).items():
            paramtree.add_param(self, key, torch.zeros(shape) if len(shape) == 1 else 0.02 * torch.randn(shape, generator=g))
        self._engine = _lib.Engine("agpt_binaural_create")
        if self.use_cuda:
            self.cuda()

    # ---- utils.Net
    def save(self, model_dir, suffix=""):
        if self.use_cuda:
            self.cpu()
        fname = f"{model_dir}/{self.model_name}.net" if suffix == "" else f"{model_dir}/{self.model_name}.{suffix}.net"
        torch.save(self.state_dict(), fname)
        if self.use_cuda:
            self.cuda()

    def load_from_file(self, model_file):
        if self.use_cuda:
            self.cpu()
        self.load_state_dict(torch.load(model_file))
        if self.use_cuda:
            self.cuda()
        print(f"Loaded: {model_file}")

    def load(self, model_dir, suffix=""):
        self.load_from_file(f"{model_dir}/{self.model_name}.net" if suffix == "" else f"{model_dir}/{self.model_name}.{suffix}.net")

    def num_trainable_parameters(self):
        """The reference's count (every warpnet parameter trains there); the drop-in's own copies are frozen."""
        return sum(p.numel() for p in self.parameters())

    # ---- the engine
    def _ensure(self, dev):
        srcs = [paramtree.get_tensor(self, k) for k in self._keys]
        cc = _lib.BinauralConfig(layers=self.cfg["layers"], channels=self.cfg["channels"])
        self._engine.ensure(dev, srcs, lambda: ((C.byref(cc),), srcs))

    def _check(self, *ts):
        if self.training:
            raise RuntimeError("audiogpt_b200.BinauralNetwork is inference only: call .eval() first (the tool does)")
        for t in ts:
            if not torch.is_tensor(t) or not t.is_cuda:
                raise RuntimeError("audiogpt_b200.BinauralNetwork runs on CUDA only (no CPU fallback)")
        if any(t.device != ts[0].device for t in ts):
            raise ValueError("mono and view must be on the same device")

    def _run(self, mono, view, rows, out, clamp):
        dev = mono.device
        self._ensure(dev)
        arr = (_lib.BinauralRow * len(rows))(*[_lib.BinauralRow(*r) for r in rows])
        self._engine.call("binaural_forward", dev, _lib.fptr(mono), _lib.fptr(view), arr, len(rows), _lib.fptr(out), int(clamp))
        return out

    @torch.no_grad()
    def forward(self, mono, view):
        """mono [B, 1, T], view [B, 7, K] (CUDA) -> the warped left / right ear signals [B, 2, T]."""
        self._check(mono, view)
        if mono.dim() != 3 or mono.shape[1] != 1 or mono.shape[0] < 1 or mono.shape[2] < 1:
            raise ValueError(f"mono must be (batch, 1, samples), got {tuple(mono.shape)}")
        if view.dim() != 3 or view.shape[1] != specs.BINAURAL_VIEW_DIM or view.shape[0] != mono.shape[0]:
            raise ValueError(f"view must be (batch, 7, frames) with mono's batch, got {tuple(view.shape)}")
        if view.shape[2] == 0:
            raise ValueError("view has no frames (the reference's F.interpolate refuses an empty input)")
        B, _, T = mono.shape
        K = view.shape[2]
        m = mono.to(torch.float32).contiguous()
        v = view.to(torch.float32).contiguous()
        out = torch.empty((B, 2, T), device=mono.device, dtype=torch.float32)
        rows = [(b * T, T, b * 7 * K, K, K, 0, b * 2 * T, T) for b in range(B)]
        return self._run(m, v, rows, out, False)

    @torch.no_grad()
    def binauralize(self, mono, view, chunk_size=48000, rec_field=800):
        """The Binaural tool's loop (audio-chatgpt.py:729-766) in one engine call: mono [1, L] and view [7, Kv] (CUDA) ->
        the clamped [2, L'] it saves, every chunk of every ear from the same three launches (specs.binaural_chunks)."""
        self._check(mono, view)
        if mono.dim() != 2 or mono.shape[0] != 1:
            raise ValueError(f"mono must be (1, samples), got {tuple(mono.shape)}")
        if view.dim() != 2 or view.shape[0] != specs.BINAURAL_VIEW_DIM:
            raise ValueError(f"view must be (7, frames), got {tuple(view.shape)}")
        Kv = view.shape[1]
        L_out, plan = specs.binaural_chunks(mono.shape[1], Kv, chunk_size, rec_field)
        if not plan:
            raise ValueError("clip shorter than one 400-sample view frame: nothing to binauralize")
        if any(r["K"] == 0 for r in plan):
            raise ValueError("a chunk's view slice is empty: the view is too short for the clip (the reference's F.interpolate "
                             "refuses it too)")
        m = mono.to(torch.float32).contiguous()
        v = view.to(torch.float32).contiguous()
        out = torch.empty((2, L_out), device=mono.device, dtype=torch.float32)
        rows = [(r["mono_off"], r["T"], r["view_off"], Kv, r["K"], r["keep"], r["out_off"], L_out) for r in plan]
        return self._run(m, v, rows, out, True)
