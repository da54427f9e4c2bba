"""CLAP text encoder (FrozenCLAPEmbedder) without a GPU: the CPU oracle against the reference fixtures
(tests/golden/make_golden_clap.py), the drop-in's state-dict layout, the C ABI of agpt_clap_*, install(text_encoder=True)
and the reference-style constructor."""
import ctypes
import os
import re
import subprocess
import sys

os.environ.setdefault("HF_HUB_OFFLINE", "1")          # nothing here may reach the model hub
os.environ.setdefault("TRANSFORMERS_OFFLINE", "1")

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

from audiogpt_b200 import specs  # noqa: E402
from conftest import load_golden, rel_rmse  # noqa: E402
from oracle import clap_ref  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 7070


def test_oracle_small_vs_reference():
    g = load_golden("clap_small")
    sd = specs.synth_clap(specs.CLAP_SMALL, SEED)
    for L in (77, 20):
        ids = torch.tensor(g[f"ids{L}"])
        assert ids.shape == (4, L) and int(ids[0, 0]) == 101 and int(ids[0, 1]) == 102 and int(ids[0, 2:].abs().sum()) == 0
        assert int((ids[2] != 0).sum()) == L                                  # the truncated row fills the whole length
        z = clap_ref.clap_encode(sd, specs.CLAP_SMALL, ids)
        assert z.shape == (4, L, 48)
        assert rel_rmse(z, g[f"z{L}"]) < 1e-5, L
    assert int(g["ids77"].max()) == specs.CLAP_SMALL["vocab_size"] - 1


def test_oracle_base_vs_reference():
    """T2A's two conditioning calls at the shipped shape: the rows of 3 x [""] and of 3 x [prompt]"""
    g = load_golden("clap_base")
    z = clap_ref.clap_encode(specs.synth_clap(specs.CLAP_BASE, SEED), specs.CLAP_BASE, torch.tensor(g["ids"]))
    assert z.shape == (2, 77, 1024)
    assert rel_rmse(z, g["z"]) < 1e-5


@pytest.mark.parametrize("name,cfg", [("clap_small", specs.CLAP_SMALL), ("clap_base", specs.CLAP_BASE)])
def test_drop_in_layout_matches_reference(name, cfg):
    from audiogpt_b200.ldm.modules.encoders.modules import FrozenCLAPEmbedder
    g = load_golden(name)
    sd = FrozenCLAPEmbedder.from_config(cfg).state_dict()
    assert list(sd) == list(g["ref_keys"]) == list(specs.clap_param_shapes(cfg))
    assert [",".join(str(v) for v in t.shape) for t in sd.values()] == list(g["ref_shapes"])


def test_base_parameter_count():
    shapes = specs.clap_param_shapes(specs.CLAP_BASE)
    n = sum(int(np.prod(s)) for s in shapes.values())
    assert len(shapes) == 203
    assert n == int(load_golden("clap_base")["ref_params"])
    assert f"{n * 1e-6:.2f}" == "111.32"


def test_abi_exported_and_config_mirrors_header():
    """agpt_clap_create / agpt_clap_encode are exported with the declared prototypes, and _lib.ClapConfig mirrors the
    agpt_clap_cfg fields (names, order, int / float types)."""
    from audiogpt_b200 import _lib
    from audiogpt_b200.build import build
    L = ctypes.CDLL(build())
    for n in ("agpt_clap_create", "agpt_clap_encode"):
        assert hasattr(L, n)
    hdr = re.sub(r"/\*.*?\*/", " ", open(os.path.join(ROOT, "include", "agpt_b200.h")).read(), flags=re.S)
    body = re.search(r"typedef struct agpt_clap_cfg \{(.*?)\}\s*agpt_clap_cfg\s*;", hdr, re.S).group(1)
    fields = [(d.split()[1], d.split()[0]) for d in filter(str.strip, body.split(";"))]
    ctype = {"int": ctypes.c_int, "float": ctypes.c_float}
    assert [(n, t) for n, t in _lib.ClapConfig._fields_] == [(n, ctype[t]) for n, t in fields]
    assert tuple(n for n, _ in fields) == specs.CLAP_ENGINE_KEYS
    assert re.search(r"int agpt_clap_create\(const agpt_clap_cfg\* cfg, const float\* const\* host_weights, int n_weights, "
                     r"int device, agpt_handle\* out\);", hdr)
    assert re.search(r"int agpt_clap_encode\(agpt_handle h, const int\* input_ids, int N, int L, float\* z, void\* stream\);", hdr)
    P, W = ctypes.c_void_p, ctypes.POINTER(ctypes.POINTER(ctypes.c_float))
    assert _lib.PROTOTYPES["agpt_clap_create"] == (ctypes.c_int, [P, W, ctypes.c_int, ctypes.c_int, ctypes.POINTER(P)])
    assert _lib.PROTOTYPES["agpt_clap_encode"] == (ctypes.c_int, [P, P, ctypes.c_int, ctypes.c_int, P, P])


def _run(code):
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=240)
    assert r.returncode == 0, r.stderr
    return r.stdout.strip()


def test_install_text_encoder_grafts_the_class(tmp_path):
    """install(text_encoder=True) replaces FrozenCLAPEmbedder inside the reference's module (a stub stands in for it);
    the plain install() leaves it alone and patches the same eight modules as before."""
    d = tmp_path / "ldm" / "modules" / "encoders"
    d.mkdir(parents=True)
    for p in (tmp_path / "ldm", tmp_path / "ldm" / "modules", d):
        (p / "__init__.py").write_text("")
    (d / "modules.py").write_text("class FrozenCLAPEmbedder:\n    pass\n\nclass FrozenT5Embedder:\n    pass\n")
    head = "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import audiogpt_b200 as a; " % (str(tmp_path), ROOT)
    check = "import ldm.modules.encoders.modules as m; print(len(p), m.FrozenCLAPEmbedder.__module__, m.FrozenT5Embedder.__module__)"
    plain = _run(head + "p = a.install(); " + check)
    assert plain == "8 ldm.modules.encoders.modules ldm.modules.encoders.modules"
    names = "print(sorted(x.split(' ')[0] for x in p))"
    assert _run(head + "p = a.install(); " + names) == str(sorted(__import__("audiogpt_b200")._INSTALL_MAP))
    assert _run(head + "p = a.install(text_encoder=True); " + check) == \
        "9 audiogpt_b200.ldm.modules.encoders.modules ldm.modules.encoders.modules"
    # not importable and not strict: aliased to ours
    code = ("import sys; sys.path.insert(0, %r); import audiogpt_b200 as a; p = a.install(text_encoder=True); "
            "m = sys.modules['ldm.modules.encoders.modules']; print(p[-1], m.FrozenCLAPEmbedder.__module__)") % ROOT
    assert _run(code) == "ldm.modules.encoders.modules (aliased) audiogpt_b200.ldm.modules.encoders.modules"


def test_reference_style_constructor_copies_bert_and_skips_weights_path(tmp_path, monkeypatch):
    """FrozenCLAPEmbedder(weights_path) takes the tokenizer and the BERT weights from transformers' from_pretrained
    (monkeypatched here: no hub access), copies the weights exactly, keeps no torch model and never opens
    weights_path."""
    transformers = pytest.importorskip("transformers")
    from audiogpt_b200.ldm.modules.encoders.modules import FrozenCLAPEmbedder
    cfg = specs.CLAP_SMALL
    sd = specs.synth_clap(cfg, SEED)
    pre = "caption_encoder.base."
    bert = transformers.BertModel(transformers.BertConfig(
        vocab_size=cfg["vocab_size"], hidden_size=cfg["hidden_size"], num_hidden_layers=cfg["num_layers"],
        num_attention_heads=cfg["num_heads"], intermediate_size=cfg["intermediate_size"],
        max_position_embeddings=cfg["max_position_embeddings"], type_vocab_size=cfg["type_vocab_size"]))
    bert.load_state_dict({k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}, strict=True)
    tok = object()
    names = []
    monkeypatch.setattr(transformers.AutoModel, "from_pretrained", lambda n, *a, **k: names.append(n) or bert)
    monkeypatch.setattr(transformers.AutoTokenizer, "from_pretrained", lambda n, *a, **k: names.append(n) or tok)
    monkeypatch.setattr(torch, "load", lambda *a, **k: pytest.fail("weights_path was read"))
    path = tmp_path / "never_created.ckpt"
    m = FrozenCLAPEmbedder(str(path), freeze=True, device="cuda", max_length=20)
    assert not path.exists() and sorted(names) == ["bert-base-uncased", "bert-base-uncased"]
    assert m.tokenizer is tok and m.max_length == 20 and m.device == "cuda"
    assert m.cfg["hidden_size"] == cfg["hidden_size"] and m.cfg["d_proj"] == 1024
    got = m.state_dict()
    for k, v in sd.items():
        if k.startswith(pre):
            assert torch.equal(got[k], v), k
    assert not any(isinstance(x, torch.nn.Module) and type(x).__name__ == "BertModel" for x in m.modules())
    assert not any(p.requires_grad for p in m.caption_encoder.base.parameters())
    assert list(got) == list(specs.clap_param_shapes(dict(cfg, d_proj=1024)))
