"""Drop-in for ``sound_extraction.model.LASSNet.LASSNet``: the text-queried separation network of the SoundExtraction
tool (audio-chatgpt.py:675-710), which predicts a magnitude mask from a spectrogram and a caption.

Reference: sound_extraction/model/LASSNet.py, text_encoder.py (prajjwal1/bert-mini, [CLS] row -> Linear(256, 256) ->
ReLU), resunet_film.py (UNetRes_FiLM), modules.py (ConvBlockResCond, EncoderBlockRes2BCond, DecoderBlockRes2BCond),
film.py.  Same constructor ``(device='cuda')``, same ``forward(x, caption)`` and ``get_tokenizer()``, same state-dict
keys (BatchNorm running statistics and ``num_batches_tracked`` included), so a reference checkpoint loads strictly,
inside ``nn.DataParallel`` too.  Arithmetic: libagpt_b200.so (csrc/lass.cu).  CUDA only, inference only (BatchNorm in
eval mode).

Differences from the reference:
- the constructor builds bert-mini's architecture from a built-in config instead of ``BertModel.from_pretrained``,
  whose weights the checkpoint overwrites; the tokenizer still comes from ``BertTokenizer.from_pretrained``, as in the
  reference.  ``from_config(cfg, tokenizer)`` touches neither;
- an old checkpoint's ``text_embedder.bert_layer.embeddings.position_ids`` is accepted and ignored;
- ``forward_ids(x, input_ids, attention_mask)`` is the tokenizer-free entry;
- a frequency axis the UNet's skips cannot close on (F - 2 not 63 mod 64, or F < 129) raises ValueError where the
  reference fails inside ``torch.cat``.
"""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from ... import _lib, paramtree, specs

_TEXT_MODEL = "prajjwal1/bert-mini"
_POSITION_IDS = "text_embedder.bert_layer.embeddings.position_ids"


def _tensor(root: nn.Module, key: str) -> torch.Tensor:
    """The parameter or buffer at ``key``, also on a ``torch.nn.parallel.replicate`` replica, whose tensors are plain
    attributes."""
    node = root
    for p in key.split("."):
        node = getattr(node, p)
    return node


class LASSNet(nn.Module):
    _h = _lib.engine_handle

    def __init__(self, device="cuda"):
        super().__init__()
        self._setup(specs.LASS, device)
        from transformers import BertTokenizer
        self.text_embedder.tokenizer = BertTokenizer.from_pretrained(_TEXT_MODEL)

    @classmethod
    def from_config(cls, cfg=None, tokenizer=None, device="cuda"):
        """Built from a specs.LASS-style config with no file or hub access; ``tokenizer`` may be None (then only
        forward_ids works)."""
        self = cls.__new__(cls)
        nn.Module.__init__(self)
        self._setup(specs.LASS if cfg is None else cfg, device)
        self.text_embedder.tokenizer = tokenizer
        return self

    def _setup(self, cfg, device):
        self.cfg = dict(cfg)
        self.device = device
        self._keys = specs.lass_engine_keys(self.cfg)
        for key, shape in specs.lass_param_shapes(self.cfg).items():
            if key.endswith("num_batches_tracked"):
                paramtree.add_buffer(self, key, torch.zeros((), dtype=torch.long))
            elif key.endswith(("running_mean", "running_var")):
                paramtree.add_buffer(self, key, torch.zeros(shape))
            else:
                paramtree.add_param(self, key, torch.zeros(shape))
        self._engine = _lib.Engine("agpt_lass_create")

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        state_dict.pop(prefix + _POSITION_IDS, None)   # a buffer transformers no longer saves
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)

    def get_tokenizer(self):
        return self.text_embedder.tokenizer

    def tokenize(self, caption):
        """Text_Encoder.tokenize: no special tokens added, padded to the longest caption."""
        tok = self.get_tokenizer()
        if tok is None:
            raise RuntimeError("audiogpt_b200.LASSNet: no tokenizer (use forward_ids)")
        t = tok(caption, add_special_tokens=False, padding=True, return_tensors="pt")
        return t["input_ids"], t["attention_mask"]

    def _ensure(self, dev):
        srcs = [_tensor(self, k) for k in self._keys]
        cfg = _lib.LassConfig(**{k: self.cfg[k] for k in ("vocab_size", "max_position_embeddings", "type_vocab_size",
                                                          "hidden_size", "num_layers", "num_heads", "intermediate_size",
                                                          "layer_norm_eps")})
        self._engine.ensure(dev, srcs, lambda: ((C.byref(cfg),), srcs))

    def forward(self, x, caption):
        input_ids, attns_mask = self.tokenize(caption)
        return self.forward_ids(x, input_ids.to(x.device), attns_mask.to(x.device))

    @torch.no_grad()
    def forward_ids(self, x, input_ids, attention_mask, return_all=False):
        """x [B, 1, T, F] CUDA magnitude (any strides), input_ids / attention_mask [N, L] (N = B, or 1 for one query
        shared by the batch) -> the mask sigmoid(UNet(x, cond, cond)) [B, 1, T, F].  return_all: (mask, logits, cond)."""
        if not x.is_cuda:
            raise RuntimeError("audiogpt_b200.LASSNet runs on CUDA only (no CPU fallback)")
        if x.dim() != 4 or x.shape[1] != 1 or x.shape[0] < 1 or x.shape[2] < 1:
            raise ValueError(f"x must be [B, 1, T, F], got {tuple(x.shape)}")
        B, _, T, F = x.shape
        if F < 129 or (F - 2) % 64 != 63:
            raise ValueError(f"LASSNet: F = {F} frequency bins do not fit UNetRes_FiLM (F - 2 must be 63 mod 64 and F >= 129; "
                             "a 1024-point STFT gives 513)")
        if input_ids.dim() != 2 or input_ids.is_floating_point() or input_ids.shape[0] < 1 or input_ids.shape[1] < 1:
            raise ValueError(f"input_ids must be an integer [N, L] tensor, got {input_ids.dtype} {tuple(input_ids.shape)}")
        N, L = input_ids.shape
        if N not in (1, B):
            raise ValueError(f"{N} captions for a batch of {B}")
        if attention_mask.shape != input_ids.shape:
            raise ValueError(f"attention_mask must have shape {tuple(input_ids.shape)}, got {tuple(attention_mask.shape)}")
        if L > self.cfg["max_position_embeddings"]:
            raise ValueError(f"caption length {L} > max_position_embeddings {self.cfg['max_position_embeddings']}")
        lo, hi = (int(v) for v in torch.aminmax(input_ids))
        if lo < 0 or hi >= self.cfg["vocab_size"]:
            raise ValueError(f"token ids must lie in [0, {self.cfg['vocab_size']}), got [{lo}, {hi}]")
        dev = x.device
        self._ensure(dev)
        ids = input_ids.to(dev, torch.int32).contiguous()
        msk = attention_mask.to(dev, torch.int32).contiguous()
        cond = torch.empty((N, specs.LASS_COND), device=dev, dtype=torch.float32)
        self._engine.call("lass_text", dev, _lib.fptr(ids), _lib.fptr(msk), N, L, _lib.fptr(cond))
        c = cond.expand(B, -1).contiguous() if N != B else cond
        xf = x if x.dtype == torch.float32 else x.float()
        mask = torch.empty((B, 1, T, F), device=dev, dtype=torch.float32)
        logits = torch.empty_like(mask) if return_all else None
        self._engine.call("lass_mask", dev, _lib.fptr(xf), B, T, F, xf.stride(0), xf.stride(2), xf.stride(3), _lib.fptr(c),
                          _lib.fptr(mask), _lib.fptr(logits) if return_all else None)
        return (mask, logits, cond) if return_all else mask
