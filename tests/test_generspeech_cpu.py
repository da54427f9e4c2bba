"""GenerSpeech host side without a GPU: the CPU oracle pinned to the fixtures made by the reference module
(tests/golden/make_golden_generspeech.py), the state-dict layout (shared WN layers, weight norm), the settings that raise,
the opt-in graft of install(tts_ood=True), and the C ABI symbols."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from audiogpt_b200 import paramtree, specs
from audiogpt_b200.utils.hparams import set_hparams_from_dict
from conftest import ROOT, load_golden, rel_rmse

CASES = [("generspeech_small", specs.GS_SMALL), ("generspeech_c2", specs.GS_C2)]
INPUTS = ("txt_tokens", "ref_mels", "ref_mel2ph", "ref_mel2word", "spk_embed", "emo_embed")
INT_KEYS = ("dur_choice", "mel2ph", "coarse", "vq_idx_utter", "vq_idx_ph", "vq_idx_word")


def fixture_args(g):
    return [torch.from_numpy(g[k]) for k in INPUTS]


def fixture_view(key, t):
    """the channel subsample the fixture stores"""
    if key in ("mel_out", "mel_pre_flow"):
        return t[..., ::4]
    if key in ("decoder_inp", "ref_prosody") or key.startswith(("prosody_", "aligned_")):
        return t[..., ::8]
    return t


def oracle_outputs(g, cfg, tag):
    from oracle import generspeech_ref as gr
    sd = specs.synth_generspeech(cfg)
    m2p = torch.from_numpy(g["mel2ph_given"]) if tag == "given" else None
    r, coarse, mid, _ = gr.generspeech_forward(sd, cfg, *fixture_args(g), torch.from_numpy(g[tag + "_z"]), mel2ph=m2p)
    r.update(mid, coarse=coarse)
    return r


@pytest.mark.parametrize("name,cfg", CASES)
def test_oracle_matches_reference_fixture(name, cfg):
    g = load_golden(name)
    assert float(g["margins"].min()) >= 1e-3
    for tag in ("pred", "given"):
        r = oracle_outputs(g, cfg, tag)
        keys = [k[len(tag) + 1:] for k in g.files if k.startswith(tag + "_") and k != tag + "_z"]
        assert {"mel_out", "mel_pre_flow", "decoder_inp", "ref_prosody", "vq_idx_ph"} <= set(keys)
        for k in keys:
            got, want = fixture_view(k, r[k]), g[f"{tag}_{k}"]
            if k in INT_KEYS:
                assert np.array_equal(got.numpy(), want), (tag, k)
            else:
                assert rel_rmse(got, want) < 1e-5, (tag, k, rel_rmse(got, want))
    # not vacuous: several frames per token, an odd teacher-forced length, varied pitch bins and VQ codes, an empty segment
    assert g["pred_mel2ph"].shape[1] >= 4 * g["txt_tokens"].shape[1]
    assert g["mel2ph_given"].shape[1] % 2 == 1 and g["given_mel_out"].shape[1] == g["mel2ph_given"].shape[1] - 1
    assert len(np.unique(g["pred_coarse"])) > 5
    assert any(len(np.unique(g["pred_vq_idx_" + lvl])) > 1 for lvl in specs.GS_LEVELS)
    m2p = g["ref_mel2ph"]
    assert any(len(set(range(1, int(m2p.max()) + 1)) - set(np.unique(row).tolist())) for row in m2p)


@pytest.mark.parametrize("name,cfg", CASES)
def test_strict_load_of_reference_state_dict(name, cfg):
    """The drop-in's keys and shapes are the reference's (as recorded from the reference module); a state dict with that
    layout loads strictly, with the token embedding and the shared WN layers of the coupling blocks held once under every
    name, and the weight-norm layout (weight_g / weight_v) kept."""
    from audiogpt_b200.modules.GenerSpeech.model.generspeech import GenerSpeech
    g = load_golden(name)
    ref = {k: tuple(int(v) for v in s.split(",") if v) for k, s in zip(g["ref_keys"].tolist(), g["ref_shapes"].tolist())}
    set_hparams_from_dict(specs.generspeech_hparams(cfg))
    m = GenerSpeech(specs.TokenDictionary(cfg["n_tokens"]))
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == ref
    assert any(k.endswith("wn.in_layers.0.weight_g") for k in ref) and not any(k.endswith("in_layers.0.weight") for k in ref)
    sd = specs.synth_generspeech(cfg)
    sd = {k: sd[k] for k in g["ref_keys"].tolist()}
    m.load_state_dict(sd, strict=True)
    assert m.encoder.embed_tokens.weight is m.encoder_embed_tokens.weight
    share = cfg["share_wn_layers"]
    t = lambda b, k: paramtree.get_tensor(m, f"post_flow.flows.{3 * b + 2}.wn.{k}")   # noqa: E731
    assert t(1, "in_layers.0.weight_v") is t(0, "in_layers.0.weight_v")
    assert t(share - 1, "res_skip_layers.0.weight_g") is t(0, "res_skip_layers.0.weight_g")
    assert t(share, "in_layers.0.weight_v") is not t(0, "in_layers.0.weight_v")
    assert t(1, "cond_layer.weight_v") is not t(0, "cond_layer.weight_v")
    assert torch.equal(t(share + 1, "res_skip_layers.0.weight_g"), sd[f"post_flow.flows.{3 * share + 2}.wn.res_skip_layers.0.weight_g"])
    # the engine's weight list folds weight norm and inverts every InvConvNear
    from oracle import generspeech_ref as gr
    w = m.engine_weights()
    assert any(t.shape == (4, 4) and torch.allclose(t, gr.invconv_inverse(sd, "post_flow.flows.1")) for t in w)
    assert any(t.shape == gr.fold_wn(sd, "post_flow.flows.2.start").shape and
               torch.allclose(t, gr.fold_wn(sd, "post_flow.flows.2.start")) for t in w)


@pytest.mark.parametrize("hp,what", [(dict(use_spk_embed=False), "speaker conditioning"), (dict(use_spk_id=True), "speaker"),
                                     (dict(post_share_cond_layers=True), "post_share_cond_layers"),
                                     (dict(sigmoid_scale=True), "sigmoid_scale"), (dict(use_txt_cond=False), "use_txt_cond"),
                                     (dict(pitch_type="ph"), "pitch"), (dict(use_energy_embed=True), "use_energy_embed"),
                                     (dict(rel_pos=True), "rel_pos"), (dict(ffn_act="relu"), "ffn_act")])
def test_unsupported_settings_raise(hp, what):
    from audiogpt_b200.modules.GenerSpeech.model.generspeech import GenerSpeech
    set_hparams_from_dict(dict(specs.generspeech_hparams(specs.GS_SMALL), **hp))
    with pytest.raises(NotImplementedError, match=what):
        GenerSpeech(specs.TokenDictionary(40))


@pytest.mark.parametrize("kw,what", [(dict(infer=False, global_steps=300000), "infer=False"),
                                     (dict(infer=True, global_steps=100), "forcing"),
                                     (dict(infer=True, global_steps=300000, f0=torch.zeros(1, 4)), "f0")])
def test_unsupported_calls_raise(kw, what):
    from audiogpt_b200.modules.GenerSpeech.model.generspeech import GenerSpeech
    set_hparams_from_dict(specs.generspeech_hparams(specs.GS_SMALL))
    m = GenerSpeech(specs.TokenDictionary(40))
    with pytest.raises(NotImplementedError, match=what):
        m(torch.ones(1, 4, dtype=torch.long), **kw)


def _run(code):
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=240)
    assert r.returncode == 0, r.stderr
    return r.stdout.strip()


def test_install_tts_ood_grafts_generspeech(tmp_path):
    """install(tts_ood=True) replaces GenerSpeech inside the reference's module (where inference/tts/GenerSpeech.py
    imports it from); the default install() leaves it alone."""
    d = tmp_path / "modules" / "GenerSpeech" / "model"
    d.mkdir(parents=True)
    (d / "generspeech.py").write_text("class GenerSpeech:\n    pass\n")
    for p in (d, d.parent, d.parent.parent):
        (p / "__init__.py").write_text("")
    head = "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import audiogpt_b200 as a; " % (str(tmp_path), ROOT)
    check = "from modules.GenerSpeech.model.generspeech import GenerSpeech as G; print(G.__module__)"
    assert _run(head + "a.install(); " + check) == "modules.GenerSpeech.model.generspeech"
    assert _run(head + "a.install(tts_ood=True); " + check) == "audiogpt_b200.modules.GenerSpeech.model.generspeech"


def test_abi_symbols_exist():
    from audiogpt_b200 import _lib
    L = _lib.lib()
    for name in ("agpt_gs_create", "agpt_gs_encode", "agpt_gs_forward"):
        assert isinstance(getattr(L, name), ctypes._CFuncPtr)
        assert name in _lib.PROTOTYPES
    assert ctypes.sizeof(_lib.GsConfig) == ctypes.sizeof(_lib.Fs2Cfg) + 6 * ctypes.sizeof(ctypes.c_int)
    assert os.path.exists(_lib.LIB_PATH)
