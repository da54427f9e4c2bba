"""Drop-ins for ``ldm.models.autoencoder.AutoencoderKL`` (SURVEY.md 8f row 1).

Reference: /root/reference/text_to_audio/Make_An_Audio/ldm/models/autoencoder.py:304-362
(``encode(x) = DiagonalGaussianDistribution(quant_conv(encoder(x)))``, ``decode(z) = decoder(post_quant_conv(z))``)
with ``Encoder`` / ``Decoder`` from ldm/modules/diffusionmodules/model.py:368-568.  Both classes take the
constructor keywords of the reference's ``first_stage_config`` (``ddconfig``, ``lossconfig``, ``embed_dim``,
``ckpt_path``, ``ignore_keys``, ``image_key``, ``colorize_nlabels``, ``monitor``); checkpoints load with
``strict=False`` exactly like ``init_from_ckpt`` does.

* ``AutoencoderKL`` -- the DECODE side: owns ``post_quant_conv.*`` and ``decoder.*`` (``encoder.*``,
  ``quant_conv.*``, ``loss.*`` checkpoint entries are ignored).  What the text-to-audio and image-to-audio tools
  need; ``bench.py`` times it.
* ``AutoencoderKLWithEncoder`` -- the whole first stage: also owns ``encoder.*`` and ``quant_conv.*`` (its keys are
  the reference class's), adds ``encode(x)`` and ``forward(input, sample_posterior)``.  ``install(first_stage=True)``
  grafts it as the reference's ``AutoencoderKL``.  The decoder and the encoder are separate engines, each built
  lazily from its own parameters: a tool that only decodes never uploads the encoder.

Arithmetic: libagpt_b200.so (csrc/vae.cu).  CUDA only, inference only.
"""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from ... import _lib, paramtree, specs
from ..modules.distributions.distributions import DiagonalGaussianDistribution


class AutoencoderKL(nn.Module):
    _h = _lib.engine_handle

    def __init__(self, ddconfig, lossconfig=None, embed_dim=4, ckpt_path=None, ignore_keys=(), image_key="image",
                 colorize_nlabels=None, monitor=None):
        super().__init__()
        dd = dict(ddconfig)
        assert dd.get("double_z", True), "AutoencoderKL needs double_z (autoencoder.py:320)"
        if dd.get("attn_type", "vanilla") != "vanilla" or dd.get("use_linear_attn", False):
            raise NotImplementedError("audiogpt_b200.AutoencoderKL supports attn_type='vanilla' only")
        if not dd.get("resamp_with_conv", True) or dd.get("tanh_out", False) or dd.get("give_pre_end", False):
            raise NotImplementedError("audiogpt_b200.AutoencoderKL: resamp_with_conv / tanh_out / give_pre_end variants")
        self.image_key = image_key
        self.embed_dim = int(embed_dim)
        self.cfg = dict(embed_dim=int(embed_dim), z_channels=int(dd["z_channels"]), resolution=int(dd["resolution"]),
                        in_channels=int(dd.get("in_channels", 1)), out_ch=int(dd["out_ch"]), ch=int(dd["ch"]),
                        ch_mult=[int(v) for v in dd["ch_mult"]], num_res_blocks=int(dd["num_res_blocks"]),
                        attn_resolutions=[int(v) for v in dd["attn_resolutions"]], dropout=0.0, double_z=True)
        self._shapes = specs.vae_decoder_param_shapes(self.cfg)
        paramtree.build(self, self._shapes)
        self._engine = _lib.Engine("agpt_vae_create")
        if monitor is not None:
            self.monitor = monitor
        if ckpt_path is not None:
            self.init_from_ckpt(ckpt_path, ignore_keys=ignore_keys)

    def init_from_ckpt(self, path, ignore_keys=()):
        sd = torch.load(path, map_location="cpu")["state_dict"]
        for k in list(sd.keys()):
            if any(k.startswith(ik) for ik in ignore_keys):
                del sd[k]
        self.load_state_dict(sd, strict=False)
        print(f"Restored from {path}")

    # ------------------------------------------------------------------ engine
    def _cfg_struct(self):
        c = _lib.VaeCfg()
        cfg = self.cfg
        c.embed_dim, c.z_channels, c.ch, c.out_ch = cfg["embed_dim"], cfg["z_channels"], cfg["ch"], cfg["out_ch"]
        c.num_levels, c.num_res_blocks = len(cfg["ch_mult"]), cfg["num_res_blocks"]
        for i, m in enumerate(cfg["ch_mult"]):
            c.ch_mult[i] = m
            # the decoder walks the levels top-down starting at resolution / 2^(levels-1) (model.py:481,517-518)
            c.attn_at_level[i] = 1 if (cfg["resolution"] // 2 ** i) in cfg["attn_resolutions"] else 0
        return c

    def _build(self, engine, shapes, device, *args):
        """Build ``engine`` from the parameters named in ``shapes``; ``args``: the create call's arguments after the cfg."""
        ws = [paramtree.get_tensor(self, k) for k in shapes]
        engine.ensure(device, ws, lambda: ((C.byref(self._cfg_struct()),) + args, ws))

    @torch.no_grad()
    def decode(self, z):
        """z [B, embed_dim, H, W] -> [B, out_ch, H * 2^(levels-1), W * 2^(levels-1)]  (autoencoder.py:351-354)"""
        if not z.is_cuda:
            raise RuntimeError("audiogpt_b200.AutoencoderKL runs on CUDA only (no CPU fallback)")
        self._build(self._engine, self._shapes, z.device)
        z = z.contiguous().float()
        B, _, H, W = z.shape
        f = 2 ** (len(self.cfg["ch_mult"]) - 1)
        out = torch.empty((B, self.cfg["out_ch"], H * f, W * f), device=z.device, dtype=torch.float32)
        self._engine.call("vae_decode", z.device, _lib.fptr(z), B, H, W, _lib.fptr(out))
        return out

    def encode(self, x):
        raise NotImplementedError("audiogpt_b200.AutoencoderKL accelerates decode() only; "
                                  "audiogpt_b200.ldm.models.autoencoder.AutoencoderKLWithEncoder also runs encode()")

    def forward(self, input, sample_posterior=True):
        raise NotImplementedError("training forward is out of scope; call decode(z)")

    def get_last_layer(self):
        return paramtree.get_param(self, "decoder.conv_out.weight")


class AutoencoderKLWithEncoder(AutoencoderKL):
    """The whole first stage: decode() as AutoencoderKL, plus encode() and forward() on the encoder engine."""

    # install(first_stage=True) records the reference's DiagonalGaussianDistribution here, so that encode() returns
    # what LatentDiffusion.get_first_stage_encoding (ddpm_audio.py:157-164) accepts; None = the drop-in class
    _posterior_cls = None

    def __init__(self, ddconfig, lossconfig=None, embed_dim=4, ckpt_path=None, ignore_keys=(), image_key="image",
                 colorize_nlabels=None, monitor=None):
        super().__init__(ddconfig, lossconfig=lossconfig, embed_dim=embed_dim, ckpt_path=None, ignore_keys=ignore_keys,
                         image_key=image_key, colorize_nlabels=colorize_nlabels, monitor=monitor)
        self._enc_shapes = specs.vae_encoder_param_shapes(self.cfg)
        paramtree.build(self, self._enc_shapes)
        self._enc_engine = _lib.Engine("agpt_vae_encoder_create")
        if ckpt_path is not None:
            self.init_from_ckpt(ckpt_path, ignore_keys=ignore_keys)

    @torch.no_grad()
    def encode(self, x):
        """x [B, in_channels, H, W] -> posterior over z [B, embed_dim, H // 2^(levels-1), W // 2^(levels-1)]
        (autoencoder.py:345-349).  H and W must be at least 2^(levels-1)."""
        if not x.is_cuda:
            raise RuntimeError("audiogpt_b200.AutoencoderKLWithEncoder runs on CUDA only (no CPU fallback)")
        if x.dim() != 4 or x.shape[1] != self.cfg["in_channels"]:
            raise ValueError(f"expected x of shape [B, {self.cfg['in_channels']}, H, W], got {tuple(x.shape)}")
        self._build(self._enc_engine, self._enc_shapes, x.device, self.cfg["in_channels"])
        x = x.contiguous().float()
        B, _, H, W = x.shape
        f = 2 ** (len(self.cfg["ch_mult"]) - 1)
        moments = torch.empty((B, 2 * self.embed_dim, H // f, W // f), device=x.device, dtype=torch.float32)
        self._enc_engine.call("vae_encode", x.device, _lib.fptr(x), B, H, W, _lib.fptr(moments))
        return (self._posterior_cls or DiagonalGaussianDistribution)(moments)

    def forward(self, input, sample_posterior=True):
        """(decode(z), posterior) with z drawn from the posterior or its mode (autoencoder.py:355-362)"""
        posterior = self.encode(input)
        z = posterior.sample() if sample_posterior else posterior.mode()
        return self.decode(z), posterior
