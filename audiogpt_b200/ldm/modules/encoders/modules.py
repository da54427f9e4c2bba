"""Drop-in for ``ldm.modules.encoders.modules.FrozenCLAPEmbedder``: the CLAP text encoder that turns every
Make-An-Audio text prompt into the UNet's cross-attention context (LatentDiffusion.get_learned_conditioning).

Reference: text_to_audio/Make_An_Audio/ldm/modules/encoders/modules.py:173-212, with TextEncoder / Projection of
ldm/modules/encoders/CLAP/clap.py:8-52 and HF transformers' BertModel.  Same constructor
``(weights_path, freeze=True, device="cuda", max_length=77)``, same ``caption_encoder.base`` /
``caption_encoder.projection`` state-dict keys, same ``tokenizer``, ``max_length`` and ``device`` attributes and
``freeze()``; ``encode(text)`` returns ``[N, max_length, d_proj]`` on ``self.device``.  The module only stores the
weights: tokenization stays on the host (transformers), the arithmetic runs in libagpt_b200.so (csrc/clap.cu).  CUDA
only, inference only.

Differences from the reference:
- the constructor copies the ``bert-base-uncased`` weights of ``AutoModel.from_pretrained`` into its own parameters
  and keeps no torch model;
- it does not read ``weights_path``: the reference loads that file and discards what it loads (the LDM checkpoint
  later overwrites every weight);
- ``from_config`` builds it without any file or hub access, and ``encode_ids`` is the tokenizer-free entry.
"""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from .... import _lib, paramtree, specs

_TEXT_MODEL = "bert-base-uncased"   # CLAP/config.yml text_model


def clap_config_of(bert_config, d_proj: int = 1024):
    """The engine configuration (specs.clap_param_shapes / agpt_clap_cfg) of a transformers BertConfig."""
    if getattr(bert_config, "hidden_act", "gelu") != "gelu":
        raise NotImplementedError(f"audiogpt_b200.FrozenCLAPEmbedder: hidden_act={bert_config.hidden_act!r} (only 'gelu')")
    if getattr(bert_config, "position_embedding_type", "absolute") != "absolute":
        raise NotImplementedError("audiogpt_b200.FrozenCLAPEmbedder: only absolute position embeddings")
    return dict(vocab_size=int(bert_config.vocab_size), max_position_embeddings=int(bert_config.max_position_embeddings),
                type_vocab_size=int(bert_config.type_vocab_size), hidden_size=int(bert_config.hidden_size),
                num_layers=int(bert_config.num_hidden_layers), num_heads=int(bert_config.num_attention_heads),
                intermediate_size=int(bert_config.intermediate_size), d_proj=int(d_proj),
                layer_norm_eps=float(bert_config.layer_norm_eps), proj_layer_norm_eps=1e-5)


class FrozenCLAPEmbedder(nn.Module):
    _h = _lib.engine_handle

    def __init__(self, weights_path, freeze=True, device="cuda", max_length=77):
        super().__init__()
        from transformers import AutoModel, AutoTokenizer
        tokenizer = AutoTokenizer.from_pretrained(_TEXT_MODEL)
        bert = AutoModel.from_pretrained(_TEXT_MODEL)
        self._setup(clap_config_of(bert.config), tokenizer, device, max_length)
        base = bert.state_dict()
        with torch.no_grad():
            for key in self._shapes:
                if key.startswith("caption_encoder.base."):
                    paramtree.get_tensor(self, key).copy_(base[key[len("caption_encoder.base."):]])
        del bert
        if freeze:
            self.freeze()

    def _setup(self, cfg, tokenizer, device, max_length):
        self.cfg = {k: cfg[k] for k in specs.CLAP_ENGINE_KEYS}
        self.tokenizer = tokenizer
        self.max_length = int(max_length)
        self.device = device
        self._shapes = specs.clap_param_shapes(self.cfg)
        D = self.cfg["d_proj"]
        for key, shape in self._shapes.items():
            paramtree.add_param(self, key, torch.zeros(shape))
        # the reference's Projection as constructed (nn.Linear / nn.LayerNorm initialisation) until a checkpoint loads
        with torch.no_grad():
            q = "caption_encoder.projection."
            paramtree.get_tensor(self, q + "linear1.weight").copy_(nn.Linear(self.cfg["hidden_size"], D, bias=False).weight)
            paramtree.get_tensor(self, q + "linear2.weight").copy_(nn.Linear(D, D, bias=False).weight)
            paramtree.get_tensor(self, q + "layer_norm.weight").fill_(1.0)
        self._engine = _lib.Engine("agpt_clap_create")

    @classmethod
    def from_config(cls, cfg, tokenizer=None, max_length=77, device="cuda"):
        """Built from an engine config (specs.CLAP_BASE / CLAP_SMALL) with no file or hub access; the weights are zero
        (the projection as the reference initialises it) until load_state_dict."""
        self = cls.__new__(cls)
        nn.Module.__init__(self)
        self._setup(cfg, tokenizer, device, max_length)
        return self

    def freeze(self):
        self.caption_encoder.base = self.caption_encoder.base.eval()
        for param in self.caption_encoder.base.parameters():
            param.requires_grad = False

    @torch.no_grad()
    def encode(self, text):
        """text (a string or a list of them) -> z [N, max_length, d_proj] (modules.py:205-212)"""
        if self.tokenizer is None:
            raise RuntimeError("audiogpt_b200.FrozenCLAPEmbedder: no tokenizer (use encode_ids)")
        batch_encoding = self.tokenizer(text, truncation=True, max_length=self.max_length, return_length=True,
                                        return_overflowing_tokens=False, padding="max_length", return_tensors="pt")
        dev = torch.device(self.device)
        if dev.type != "cuda":
            raise RuntimeError("audiogpt_b200.FrozenCLAPEmbedder runs on CUDA only (no CPU fallback)")
        return self.encode_ids(batch_encoding["input_ids"].to(dev))

    @torch.no_grad()
    def encode_ids(self, input_ids):
        """input_ids [N, L] (CUDA, integer) -> z [N, L, d_proj] on the same device: BERT's last_hidden_state through
        the projection, every position attending to every position (the reference passes no attention mask)."""
        if not input_ids.is_cuda:
            raise RuntimeError("audiogpt_b200.FrozenCLAPEmbedder runs on CUDA only (no CPU fallback)")
        if input_ids.dim() != 2 or input_ids.is_floating_point() or input_ids.is_complex():
            raise ValueError(f"input_ids must be an integer [N, L] tensor, got {input_ids.dtype} {tuple(input_ids.shape)}")
        N, L = input_ids.shape
        if N < 1 or L < 1:
            raise ValueError(f"empty input_ids {tuple(input_ids.shape)}")
        if L > self.cfg["max_position_embeddings"]:
            raise ValueError(f"sequence length {L} > max_position_embeddings {self.cfg['max_position_embeddings']}")
        lo, hi = (int(v) for v in torch.aminmax(input_ids))
        if lo < 0 or hi >= self.cfg["vocab_size"]:
            raise ValueError(f"token ids must lie in [0, {self.cfg['vocab_size']}), got [{lo}, {hi}]")
        dev = input_ids.device
        ids = input_ids.to(torch.int32).contiguous()
        ws = [paramtree.get_tensor(self, k) for k in self._shapes]
        self._engine.ensure(dev, ws, lambda: ((C.byref(_lib.ClapConfig(**self.cfg)),), ws))
        z = torch.empty((N, L, self.cfg["d_proj"]), device=dev, dtype=torch.float32)
        self._engine.call("clap_encode", dev, _lib.fptr(ids), N, L, _lib.fptr(z))
        return z
