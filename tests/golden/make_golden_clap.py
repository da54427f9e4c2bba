#!/usr/bin/env python
"""Generate the CLAP text-encoder fixtures (clap_small.npz, clap_base.npz) by running the REFERENCE's own
FrozenCLAPEmbedder.__init__ and .encode (text_to_audio/Make_An_Audio/ldm/modules/encoders/modules.py:173-212) on CPU
fp32, with the helpers of make_golden.py.

Run in the build container only (needs the reference tree, which does not travel to the GPU box):

    python tests/golden/make_golden_clap.py

Nothing reaches the model hub: the constructor's three downloads are stubbed.
- AutoModel.from_pretrained returns a BertModel(BertConfig(...)) of the config, loaded with specs.synth_clap weights.
- AutoTokenizer.from_pretrained returns a stub that maps each prompt to a fixed id row: [CLS] ids [SEP], truncated to
  max_length and zero-padded to it, as the bert-base-uncased tokenizer lays out its rows.
- torch.load (the discarded weights_path read) returns {"model": {}}.
- read_config_as_args returns the config's text_model / d_proj / transformer_embed_dim.
- open_clip and torchlibrosa (imported by the module, unused by this class) are mocks; importlib_resources is
  importlib.resources.
Weights are not stored: the tests regenerate them from the seed.
"""
import os
import sys
import types
from unittest import mock
from unittest.mock import MagicMock

os.environ["HF_HUB_OFFLINE"] = "1"
os.environ["TRANSFORMERS_OFFLINE"] = "1"

import importlib.resources  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import ROOT, import_ldm, save, specs  # noqa: E402

CLS, SEP = 101, 102
SEED = 7070


def prompt_ids(cfg):
    """The fixtures' prompts and the token ids the stub tokenizer gives them (between [CLS] and [SEP])."""
    g = torch.Generator().manual_seed(99)
    V = int(cfg["vocab_size"])
    word = lambda n: torch.randint(103, V - 1, (n,), generator=g).tolist()   # noqa: E731
    return {"": [],
            "a dog barks while birds sing": word(6),
            "rain on a tin roof, " * 20: word(120),            # longer than max_length: truncated
            "the last word of the vocabulary": [V - 1, 7, V - 1, 250]}


class StubTokenizer:
    def __init__(self, table):
        self.table = table

    def __call__(self, text, truncation=True, max_length=77, return_length=True, return_overflowing_tokens=False,
                 padding="max_length", return_tensors="pt"):
        rows = []
        for t in [text] if isinstance(text, str) else text:
            body = self.table[t][:max_length - 2]
            rows.append([CLS] + body + [SEP] + [0] * (max_length - 2 - len(body)))
        return {"input_ids": torch.tensor(rows, dtype=torch.long)}


def reference_embedder(cfg, sd, table):
    """The reference FrozenCLAPEmbedder built offline by its own __init__ (see the module docstring)."""
    import_ldm()
    for m in ("open_clip", "torchlibrosa", "torchlibrosa.stft"):
        sys.modules.setdefault(m, MagicMock())
    sys.modules.setdefault("importlib_resources", importlib.resources)
    import transformers
    import ldm.modules.encoders.CLAP.clap as clap_mod
    import ldm.modules.encoders.modules as mods

    bert_cfg = transformers.BertConfig(vocab_size=cfg["vocab_size"], hidden_size=cfg["hidden_size"],
                                       num_hidden_layers=cfg["num_layers"], num_attention_heads=cfg["num_heads"],
                                       intermediate_size=cfg["intermediate_size"],
                                       max_position_embeddings=cfg["max_position_embeddings"],
                                       type_vocab_size=cfg["type_vocab_size"], layer_norm_eps=cfg["layer_norm_eps"])
    pre = "caption_encoder.base."

    def bert(name):
        assert name == "bert-base-uncased", name
        m = transformers.BertModel(bert_cfg)
        m.load_state_dict({k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}, strict=True)
        return m

    args = types.SimpleNamespace(text_model="bert-base-uncased", d_proj=cfg["d_proj"],
                                 transformer_embed_dim=cfg["hidden_size"])
    with mock.patch.object(clap_mod, "AutoModel", types.SimpleNamespace(from_pretrained=bert)), \
            mock.patch.object(mods, "AutoTokenizer", types.SimpleNamespace(from_pretrained=lambda n: StubTokenizer(table))), \
            mock.patch.object(mods, "read_config_as_args", lambda *a, **k: args), \
            mock.patch("torch.load", return_value={"model": {}}):
        model = mods.FrozenCLAPEmbedder("unread.ckpt", device="cpu", max_length=cfg["max_length"])
    print(model.load_state_dict(sd, strict=True))      # the projection's weights (the LDM checkpoint's role)
    return model.eval(), transformers.__version__


def layout(model):
    ref_sd = model.state_dict()
    return dict(ref_keys=np.array(list(ref_sd.keys())),
                ref_shapes=np.array([",".join(str(v) for v in t.shape) for t in ref_sd.values()]),
                ref_params=np.array(sum(p.numel() for p in model.caption_encoder.parameters())))


def golden_small():
    from oracle import clap_ref
    cfg = specs.CLAP_SMALL
    sd = specs.synth_clap(cfg, SEED)
    table = prompt_ids(cfg)
    model, ver = reference_embedder(cfg, sd, table)
    texts = list(table)
    out = dict(texts=np.array(texts), transformers_version=np.array(ver), **layout(model))
    for L in (77, 20):
        model.max_length = L
        with torch.no_grad():
            z = model.encode(texts)
        ids = StubTokenizer(table)(texts, max_length=L)["input_ids"]
        e = (clap_ref.clap_encode(sd, cfg, ids) - z).abs().max().item()
        print(f"clap_small L={L}: z {tuple(z.shape)} rms {z.pow(2).mean().sqrt().item():.3f}, oracle max |diff| {e:.2e}")
        out[f"ids{L}"] = ids.int()
        out[f"z{L}"] = z
    save("clap_small", **out)


def golden_base():
    """T2A's two calls (audio-chatgpt.py:163-164): 3 x [""] and 3 x [prompt]; only the distinct rows are stored."""
    cfg = specs.CLAP_BASE
    sd = specs.synth_clap(cfg, SEED)
    table = prompt_ids(cfg)
    prompt = "a dog barks while birds sing"
    model, ver = reference_embedder(cfg, sd, table)
    with torch.no_grad():
        uc = model.encode(3 * [""])
        c = model.encode(3 * [prompt])
    assert uc.shape == c.shape == (3, 77, 1024)
    for z in (uc, c):
        assert torch.equal(z[0], z[1]) and torch.equal(z[0], z[2])
    ids = StubTokenizer(table)([""] + [prompt], max_length=77)["input_ids"]
    print(f"clap_base: {model.caption_encoder.__class__.__name__} "
          f"{sum(p.numel() for p in model.caption_encoder.parameters()) * 1e-6:.2f} M params, "
          f"{len(model.state_dict())} keys, z rms {c.pow(2).mean().sqrt().item():.3f}")
    save("clap_base", texts=np.array(["", prompt]), ids=ids.int(), z=torch.stack([uc[0], c[0]]),
         transformers_version=np.array(ver), **layout(model))


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    golden_small()
    golden_base()
