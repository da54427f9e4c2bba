"""Drop-in for ``ldm.modules.diffusionmodules.openaimodel.UNetModel``.

Reference: /root/reference/text_to_audio/Make_An_Audio/ldm/modules/diffusionmodules/openaimodel.py:413-744
(with ResBlock :163-275, Down/Upsample :91-160, SpatialTransformer ldm/modules/attention.py:218-261).

Module path and class name are kept because the reference instantiates it reflectively
from YAML ``target:`` strings (ldm/util.py:111-118); constructor keywords are the ones
``unet_config.params`` carries; ``state_dict`` keys are the reference's
(``time_embed.{0,2}.*``, ``input_blocks.{i}.{j}...``, ``middle_block.{j}...``,
``output_blocks.{i}.{j}...``, ``out.{0,2}.*``), so LDM checkpoints load with the usual
``model.diffusion_model.`` prefix.

Supported options = what the shipped configs use: dims=2, conv_resample,
use_spatial_transformer=True, no class labels, no scale-shift norm, no resblock_updown.
Anything else raises at construction.  ``use_checkpoint`` (gradient checkpointing invoked
even at inference, util.py:102-148) is accepted and ignored.  CUDA only.
"""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from .... import _lib, paramtree, specs


def _common_unsupported(kw):
    bad = []
    if kw.get("dims", 2) != 2: bad.append("dims != 2")
    if not kw.get("conv_resample", True): bad.append("conv_resample=False")
    if kw.get("num_classes") is not None: bad.append("class-conditional (num_classes)")
    if kw.get("use_fp16", False): bad.append("use_fp16")
    if kw.get("use_scale_shift_norm", False): bad.append("use_scale_shift_norm")
    if kw.get("n_embed") is not None: bad.append("n_embed / predict_codebook_ids")
    if kw.get("num_heads", -1) == -1 and kw.get("num_head_channels", -1) == -1: bad.append("neither num_heads nor num_head_channels")
    return bad


def _unsupported(kw):
    """Constructor options outside what the shipped txt2audio config uses (SURVEY.md 8a-20)."""
    bad = _common_unsupported(kw)
    if kw.get("resblock_updown", False): bad.append("resblock_updown")
    if not kw.get("use_spatial_transformer", False): bad.append("use_spatial_transformer=False (AttentionBlock UNets)")
    if kw.get("context_dim") is None: bad.append("context_dim=None")
    return bad


def _attention_unsupported(kw):
    """Constructor options outside what AttentionUNetModel covers (the Inpaint tool's config and its relatives)."""
    bad = _common_unsupported(kw)
    if kw.get("use_spatial_transformer", False): bad.append("use_spatial_transformer=True (UNetModel covers it)")
    if kw.get("context_dim") is not None: bad.append("context_dim (cross-attention)")
    nhu = kw.get("num_heads_upsample", -1)
    if kw.get("legacy", True) and kw.get("num_head_channels", -1) == -1 and nhu not in (-1, kw.get("num_heads", -1)):
        bad.append("num_heads_upsample != num_heads")
    return bad


class UNetModel(nn.Module):
    # Set by audiogpt_b200.install(): the reference's own UNetModel class.  AudioGPT also builds UNets this back-end
    # does not cover (the inpainting model's AttentionBlock UNet, openaimodel.py:278-410); since install() replaces the
    # class object inside the reference module, constructing one of THOSE configs returns an instance of the
    # reference's class instead of failing -- those tools keep working exactly as before, un-accelerated.
    # This is a routing of unsupported model VARIANTS, not a fallback of the accelerated path: a supported config
    # never leaves the CUDA engine, and without install() (no reference class known) unsupported configs raise.
    _reference_cls = None
    # Set by audiogpt_b200.install(inpaint=True): AttentionUNetModel, which then takes the configs it covers.
    _attention_cls = None
    _h = _lib.engine_handle

    def __new__(cls, *args, **kwargs):
        if cls is UNetModel and not args and _unsupported(kwargs):
            if cls._attention_cls is not None and not _attention_unsupported(kwargs):
                # an uninitialised subclass instance: Python runs its __init__ (once) on return
                return super().__new__(cls._attention_cls)
            if cls._reference_cls is not None:
                return cls._reference_cls(**kwargs)
        return super().__new__(cls)

    def __init__(self, image_size=None, in_channels=4, model_channels=320, out_channels=4, num_res_blocks=2,
                 attention_resolutions=(1, 2), dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2,
                 num_classes=None, use_checkpoint=False, use_fp16=False, num_heads=-1, num_head_channels=-1,
                 num_heads_upsample=-1, use_scale_shift_norm=False, resblock_updown=False,
                 use_new_attention_order=False, use_spatial_transformer=False, transformer_depth=1,
                 context_dim=None, n_embed=None, legacy=True):
        nn.Module.__init__(self)
        unsupported = _unsupported(dict(dims=dims, conv_resample=conv_resample, num_classes=num_classes, use_fp16=use_fp16,
                                        use_scale_shift_norm=use_scale_shift_norm, resblock_updown=resblock_updown,
                                        use_spatial_transformer=use_spatial_transformer, n_embed=n_embed,
                                        context_dim=context_dim, num_heads=num_heads, num_head_channels=num_head_channels))
        if unsupported:
            raise NotImplementedError("audiogpt_b200.UNetModel does not support: " + ", ".join(unsupported))
        if isinstance(context_dim, (list, tuple)) or type(context_dim).__name__ == "ListConfig":
            context_dim = list(context_dim)[0]
        self.image_size, self.in_channels, self.model_channels = image_size, in_channels, model_channels
        self.out_channels, self.num_res_blocks = out_channels, num_res_blocks
        self.attention_resolutions = list(attention_resolutions)
        self.channel_mult = list(channel_mult)
        self.num_heads, self.num_head_channels = num_heads, num_head_channels
        self.transformer_depth, self.context_dim = transformer_depth, int(context_dim)
        self.dtype = torch.float32
        self.cfg = dict(in_channels=in_channels, out_channels=out_channels, model_channels=model_channels,
                        attention_resolutions=self.attention_resolutions, num_res_blocks=num_res_blocks,
                        channel_mult=self.channel_mult, num_heads=num_heads, num_head_channels=num_head_channels,
                        use_spatial_transformer=True, transformer_depth=transformer_depth,
                        context_dim=self.context_dim, legacy=legacy)
        self._shapes = specs.unet_param_shapes(self.cfg)
        paramtree.build(self, self._shapes)
        self._engine = _lib.Engine("agpt_unet_create")
        self._ctx_key = None

    # ------------------------------------------------------------------ engine
    def _cfg_struct(self):
        c = _lib.UnetCfg()
        c.in_channels, c.out_channels, c.model_channels = self.in_channels, self.out_channels, self.model_channels
        c.num_res_blocks, c.num_levels = self.num_res_blocks, len(self.channel_mult)
        for i, m in enumerate(self.channel_mult):
            c.channel_mult[i] = int(m)
            c.attn_at_level[i] = 1 if (2 ** i) in self.attention_resolutions else 0
        c.num_heads, c.num_head_channels = self.num_heads, self.num_head_channels
        c.transformer_depth, c.context_dim = self.transformer_depth, self.context_dim or 0
        c.use_spatial_transformer = int(self.cfg["use_spatial_transformer"])
        c.resblock_updown = int(self.cfg.get("resblock_updown", False))
        c.attention_order = int(self.cfg.get("use_new_attention_order", False))
        return c

    def _ensure_engine(self, t: torch.Tensor) -> bool:
        """Build the engine on t's device from the current weights; True when it was (re)built."""
        if not t.is_cuda:
            raise RuntimeError(f"audiogpt_b200.{type(self).__name__} runs on CUDA only (no CPU fallback)")
        ws = [paramtree.get_tensor(self, k) for k in self._shapes]
        return self._engine.ensure(t.device, ws, lambda: ((C.byref(self._cfg_struct()),), ws))

    def set_context(self, context: torch.Tensor):
        """context [N, S, context_dim]: hoists to_k/to_v(context) of all cross-attentions; cached per tensor."""
        if self._ensure_engine(context):
            self._ctx_key = None
        key = (context.data_ptr(), context._version, tuple(context.shape))
        if key == self._ctx_key:
            return
        c = context.contiguous().float()
        assert c.dim() == 3 and c.shape[2] == self.context_dim, "context must be [N, S, context_dim]"
        self._engine.call("unet_set_context", c.device, _lib.fptr(c), c.shape[0], c.shape[1])
        self._ctx_key = key
        # keep BOTH tensors alive while the key is live: `c` is what the engine read, `context` is what the key
        # was computed from (when they differ -- fp16 / non-contiguous input -- a freed `context` could hand its
        # address to another prompt's embedding of the same shape and the stale K/V would be reused)
        self._ctx_keep = (context, c)

    @torch.no_grad()
    def forward(self, x, timesteps=None, context=None, y=None, **kwargs):
        """x [N,C,H,W], timesteps [N] (tensor or ints), context [N,S,context_dim] -> [N,C_out,H,W]"""
        assert y is None, "must specify y if and only if the model is class-conditional"
        assert context is not None, "cross-attention UNet needs a context"
        self.set_context(context)
        return self._eps(x, timesteps)

    def _eps(self, x, timesteps):
        x = x.contiguous().float()
        N, _, H, W = x.shape
        t = timesteps.tolist() if torch.is_tensor(timesteps) else [int(v) for v in timesteps]
        tt = (C.c_int * N)(*[int(v) for v in t])
        out = torch.empty((N, self.out_channels, H, W), device=x.device, dtype=torch.float32)
        self._engine.call("unet_forward", x.device, _lib.fptr(x), tt, N, H, W, _lib.fptr(out))
        return out

    def convert_to_fp16(self):  # API parity; the engine computes in fp32
        pass

    def convert_to_fp32(self):
        pass


class AttentionUNetModel(UNetModel):
    """The reference UNetModel with AttentionBlock self-attention (use_spatial_transformer=False, no context): the
    denoiser of Make-An-Audio's Inpaint tool (configs/inpaint/txt2audio_args.yaml: 9 input channels, resblock_updown,
    legacy per-head qkv order).  Same constructor keywords, state-dict keys (AttentionBlock ``norm`` / ``qkv`` /
    ``proj_out``, openaimodel.py:278-324) and ``forward(x, timesteps, context=None)``; the context is ignored, as the
    reference's AttentionBlocks ignore it.  ``install(inpaint=True)`` makes ``UNetModel(...)`` build this class for the
    configs it covers.  CUDA only."""

    def __init__(self, image_size=None, in_channels=9, model_channels=320, out_channels=4, num_res_blocks=2,
                 attention_resolutions=(1, 2), dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2,
                 num_classes=None, use_checkpoint=False, use_fp16=False, num_heads=-1, num_head_channels=-1,
                 num_heads_upsample=-1, use_scale_shift_norm=False, resblock_updown=False,
                 use_new_attention_order=False, use_spatial_transformer=False, transformer_depth=1,
                 context_dim=None, n_embed=None, legacy=True):
        nn.Module.__init__(self)
        unsupported = _attention_unsupported(dict(
            dims=dims, conv_resample=conv_resample, num_classes=num_classes, use_fp16=use_fp16,
            use_scale_shift_norm=use_scale_shift_norm, use_spatial_transformer=use_spatial_transformer, n_embed=n_embed,
            context_dim=context_dim, num_heads=num_heads, num_head_channels=num_head_channels,
            num_heads_upsample=num_heads_upsample, legacy=legacy))
        if unsupported:
            raise NotImplementedError("audiogpt_b200.AttentionUNetModel does not support: " + ", ".join(unsupported))
        self.image_size, self.in_channels, self.model_channels = image_size, in_channels, model_channels
        self.out_channels, self.num_res_blocks = out_channels, num_res_blocks
        self.attention_resolutions = list(attention_resolutions)
        self.channel_mult = list(channel_mult)
        self.num_heads, self.num_head_channels = num_heads, num_head_channels
        self.num_heads_upsample = num_heads if num_heads_upsample == -1 else num_heads_upsample
        self.transformer_depth, self.context_dim = transformer_depth, None
        self.dtype = torch.float32
        self.cfg = dict(in_channels=in_channels, out_channels=out_channels, model_channels=model_channels,
                        attention_resolutions=self.attention_resolutions, num_res_blocks=num_res_blocks,
                        channel_mult=self.channel_mult, num_heads=num_heads, num_head_channels=num_head_channels,
                        num_heads_upsample=num_heads_upsample, use_spatial_transformer=False,
                        resblock_updown=bool(resblock_updown), use_new_attention_order=bool(use_new_attention_order),
                        legacy=legacy)
        self._shapes = specs.unet_param_shapes(self.cfg)
        paramtree.build(self, self._shapes)
        self._engine = _lib.Engine("agpt_unet_create")

    def set_concat(self, c: torch.Tensor):
        """c [B, in_channels - out_channels, H, W]: the conditioning channels the on-device DDIM loop appends to the
        latent at every step (DiffusionWrapper 'concat'); copied into the engine's layout once."""
        self._ensure_engine(c)
        c = c.contiguous().float()
        assert c.dim() == 4 and c.shape[1] == self.in_channels - self.out_channels, \
            f"concat conditioning must be [B, {self.in_channels - self.out_channels}, H, W]"
        self._engine.call("unet_set_concat", c.device, _lib.fptr(c), *c.shape)

    @torch.no_grad()
    def forward(self, x, timesteps=None, context=None, y=None, **kwargs):
        """x [N,C_in,H,W], timesteps [N] (tensor or ints) -> [N,C_out,H,W]"""
        assert y is None, "must specify y if and only if the model is class-conditional"
        self._ensure_engine(x)
        return self._eps(x, timesteps)
