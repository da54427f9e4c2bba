"""FastSpeech2 / FastSpeech2MIDI host side without a GPU: the CPU oracle pinned to the fixtures made by the reference
modules (tests/golden/make_golden_fs2.py), the state-dict layout, and the opt-in graft of install(front_end=True)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from audiogpt_b200 import specs
from audiogpt_b200.utils.hparams import set_hparams_from_dict
from conftest import ROOT, load_golden, rel_rmse

CASES = [("fs2_small", specs.FS2_SMALL), ("fs2_c2", specs.FS2_C2), ("fs2_ph", specs.FS2_PH), ("fs2_ds1000", specs.FS2_DS1000)]
INT_KEYS = ("dur_choice", "mel2ph", "coarse")


def fixture_inputs(g, cfg):
    """(txt_tokens, MIDI kwargs, teacher-forced mel2ph, teacher-forced f0 / uv / energy) of a fixture"""
    kw = {k: torch.from_numpy(g[k]) for k in ("pitch_midi", "midi_dur", "is_slur") if k in g}
    tf = {k: torch.from_numpy(g[k]) for k in ("f0", "uv", "energy") if k in g}
    return torch.from_numpy(g["txt_tokens"]), kw, torch.from_numpy(g["mel2ph_given"]), tf


def hp_kwargs(cfg):
    hp = specs.fs2_hparams(cfg)
    return dict(use_uv=hp["use_uv"], pitch_norm=hp["pitch_norm"], f0_mean=hp["f0_mean"], f0_std=hp["f0_std"])


def fixture_view(tag, key, t):
    """the channel subsample the fixture stores"""
    if key == "decoder_inp":
        return t[..., ::8]
    if key == "mel_out":
        return t[..., ::4]
    return t


@pytest.mark.parametrize("name,cfg", CASES)
def test_oracle_matches_reference_fixture(name, cfg):
    from oracle import fs2_ref
    g = load_golden(name)
    assert float(g["margins"].min()) >= 1e-3
    sd = specs.synth_fs2(cfg)
    tok, kw, m2p, tf = fixture_inputs(g, cfg)
    for tag, mel2ph, t in (("pred", None, {}), ("given", m2p, tf)):
        r, coarse, _ = fs2_ref.fs2_forward(sd, cfg, tok, mel2ph=mel2ph, **{k: v.clone() for k, v in t.items()}, **kw,
                                           **hp_kwargs(cfg))
        if coarse is not None:
            r["coarse"] = coarse
        keys = [k[len(tag) + 1:] for k in g.files if k.startswith(tag + "_")]
        assert "mel_out" in keys and "decoder_inp" in keys
        for k in keys:
            got, want = fixture_view(tag, k, r[k]), g[f"{tag}_{k}"]
            if k in INT_KEYS:
                assert np.array_equal(got.numpy(), want), (tag, k)
            else:
                assert rel_rmse(got, want) < 1e-5, (tag, k, rel_rmse(got, want))
    # the fixtures are not vacuous: several frames per token, voiced and varied pitch bins
    assert g["pred_mel2ph"].shape[1] >= 4 * g["txt_tokens"].shape[1]
    if "pred_coarse" in g:
        assert len(np.unique(g["pred_coarse"])) > 5


@pytest.mark.parametrize("name,cfg", CASES)
def test_strict_load_of_reference_state_dict(name, cfg):
    """The drop-in's state-dict keys and shapes are the reference's (as recorded from the reference module), and a state
    dict with that layout loads strictly, the shared token embedding under both of its names."""
    from audiogpt_b200.modules.diffsinger_midi.fs2 import FastSpeech2MIDI
    from audiogpt_b200.modules.fastspeech.fs2 import FastSpeech2
    g = load_golden(name)
    ref = {k: tuple(int(v) for v in s.split(",") if v) for k, s in zip(g["ref_keys"].tolist(), g["ref_shapes"].tolist())}
    set_hparams_from_dict(specs.fs2_hparams(cfg))
    m = (FastSpeech2MIDI if cfg["use_midi"] else FastSpeech2)(specs.TokenDictionary(cfg["n_tokens"]))
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == ref
    sd = specs.synth_fs2(cfg)
    sd = {k: sd[k] for k in g["ref_keys"].tolist()}
    m.load_state_dict(sd, strict=True)
    assert m.encoder.embed_tokens.weight is m.encoder_embed_tokens.weight
    assert torch.equal(m.encoder_embed_tokens.weight, sd["encoder_embed_tokens.weight"])


@pytest.mark.parametrize("hp,what", [(dict(pitch_type="cwt"), "cwt"), (dict(use_spk_id=True), "use_spk_id"),
                                     (dict(ffn_act="relu"), "ffn_act"), (dict(ffn_padding="LEFT"), "ffn_padding"),
                                     (dict(use_bert=True), "use_bert"), (dict(pitch_ar=True), "pitch_ar")])
def test_unsupported_settings_raise(hp, what):
    from audiogpt_b200.modules.fastspeech.fs2 import FastSpeech2
    set_hparams_from_dict(dict(specs.fs2_hparams(specs.FS2_SMALL), **hp))
    with pytest.raises(NotImplementedError, match=what):
        FastSpeech2(specs.TokenDictionary(40))


def _run(code):
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=240)
    assert r.returncode == 0, r.stderr
    return r.stdout.strip()


def test_install_front_end_grafts_both_classes(tmp_path):
    """install(front_end=True) replaces FastSpeech2 / FastSpeech2MIDI inside the reference's modules; the default
    install() leaves them alone and still patches its eight modules."""
    for pkg, cls in (("fastspeech", "FastSpeech2"), ("diffsinger_midi", "FastSpeech2MIDI")):
        d = tmp_path / "modules" / pkg
        d.mkdir(parents=True)
        (d / "fs2.py").write_text(f"class {cls}:\n    pass\n")
        (d / "__init__.py").write_text("")
    (tmp_path / "modules" / "__init__.py").write_text("")
    head = "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import audiogpt_b200 as a; " % (str(tmp_path), ROOT)
    check = ("import modules.fastspeech.fs2 as f, modules.diffsinger_midi.fs2 as m; "
             "print(len(p), f.FastSpeech2.__module__, m.FastSpeech2MIDI.__module__)")
    assert _run(head + "p = a.install(); " + check) == "8 modules.fastspeech.fs2 modules.diffsinger_midi.fs2"
    assert _run(head + "p = a.install(front_end=True); " + check) == \
        "10 audiogpt_b200.modules.fastspeech.fs2 audiogpt_b200.modules.diffsinger_midi.fs2"


def test_gaussian_diffusion_picks_up_front_end():
    """After the opt-in, the drop-in GaussianDiffusion built with use_midi holds our FastSpeech2MIDI (its _fs2_factory
    imports the class from the reference's module name)."""
    code = ("import sys; sys.path.insert(0, %r); import audiogpt_b200 as a; a.install(front_end=True); "
            "from audiogpt_b200 import specs; from audiogpt_b200.utils.hparams import set_hparams_from_dict; "
            "set_hparams_from_dict(dict(specs.fs2_hparams(specs.FS2_DS1000), use_midi=True)); "
            "from modules.diff.shallow_diffusion_tts import GaussianDiffusion; "
            "gd = GaussianDiffusion(specs.TokenDictionary(80), 80, None, timesteps=10, K_step=10, "
            "spec_min=[-5.0] * 80, spec_max=[0.0] * 80); "
            "print(type(gd.fs2).__module__, type(gd.fs2).__name__)") % ROOT
    assert _run(code) == "audiogpt_b200.modules.diffsinger_midi.fs2 FastSpeech2MIDI"
