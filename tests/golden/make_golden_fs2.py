#!/usr/bin/env python
"""Generate the FastSpeech2 / FastSpeech2MIDI golden fixtures (fs2_*.npz) by running the REFERENCE's own modules on
CPU fp32, with the shims and helpers of make_golden.py.

Run in the build container only (needs /root/reference, which does not travel to the GPU box):

    python tests/golden/make_golden_fs2.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF, ROOT, import_neuralseq, save, specs  # noqa: E402


def golden_fs2():
    """FastSpeech2 (NeuralSeq/modules/fastspeech/fs2.py:22-226) and FastSpeech2MIDI (modules/diffsinger_midi/fs2.py) on a
    ragged token batch with a padded tail, with predicted and with teacher-forced mel2ph (the small config also forces f0,
    uv and energy).  Rounding makes mel2ph, the coarse pitch and the energy bucket discontinuous: input seeds are drawn
    until every rounded quantity is >= 1e-3 from its boundary, so that fp32 vs fp16x3 differences cannot flip one.
    decoder_inp / mel_out are stored on a channel subsample to keep the files small."""
    sys.path.insert(0, ROOT)
    from oracle import fs2_ref
    from utils.hparams import hparams
    from modules.fastspeech.fs2 import FastSpeech2
    from modules.diffsinger_midi.fs2 import FastSpeech2MIDI
    for name, cfg, B, T in (("fs2_small", specs.FS2_SMALL, 3, 16), ("fs2_c2", specs.FS2_C2, 3, 12),
                            ("fs2_ph", specs.FS2_PH, 3, 12), ("fs2_ds1000", specs.FS2_DS1000, 3, 12)):
        hparams.clear()
        hparams.update(specs.fs2_hparams(cfg))
        cls = FastSpeech2MIDI if cfg["use_midi"] else FastSpeech2
        model = cls(specs.TokenDictionary(cfg["n_tokens"]))
        sd = specs.synth_fs2(cfg)
        print(name, "load:", model.load_state_dict(sd, strict=True))
        assert set(model.state_dict().keys()) == set(specs.fs2_param_shapes(cfg).keys())
        model.eval()
        for seed in range(1000, 1200):
            inp = specs.synth_fs2_inputs(cfg, B, T, seed)
            kw = {k: v for k, v in inp.items() if k != "txt_tokens"}
            with torch.no_grad():
                r1 = model(inp["txt_tokens"], **kw)
            # teacher-forced durations: one extra frame on every third token
            d2 = (r1["dur_choice"] + (torch.arange(T)[None] % 3 == 0).long()) * (inp["txt_tokens"] > 0).long()
            cum = torch.cumsum(d2, 1)
            pos = torch.arange(int(cum[:, -1].max()))[None, None]
            mel2ph = ((pos >= (cum - d2)[:, :, None]) & (pos < cum[:, :, None])).long()
            mel2ph = (torch.arange(1, T + 1)[None, :, None] * mel2ph).sum(1)
            g = torch.Generator().manual_seed(seed)
            tf = {}
            if cfg is specs.FS2_SMALL:
                shp = mel2ph.shape
                tf = dict(f0=0.5 * torch.randn(shp, generator=g), uv=(torch.rand(shp, generator=g) > 0.6).float(),
                          energy=2.0 + 0.2 * torch.randn(shp, generator=g))
            with torch.no_grad():
                r2 = model(inp["txt_tokens"], mel2ph=mel2ph, **{k: v.clone() for k, v in tf.items()}, **kw)
            e = r1["dur"][..., 0].double().exp() - 1
            m = [float((e - e.floor() - 0.5).abs()[inp["txt_tokens"] > 0].min())]
            for r, t in ((r1, {}), (r2, tf)):
                if "f0_denorm" in r:
                    m.append(fs2_ref.coarse_margin(r["f0_denorm"]))
                if "energy_pred" in r:
                    ee = (t.get("energy", r["energy_pred"])).double() * 64
                    m.append(float((ee - ee.round()).abs().min()))
            if min(m) >= 1e-3:
                break
        print(name, "seed", seed, "margins", ["%.1e" % v for v in m], "frames", r1["mel2ph"].shape[1], mel2ph.shape[1])
        out = dict(seed=np.array(seed), margins=np.array(m), txt_tokens=inp["txt_tokens"], **kw, mel2ph_given=mel2ph, **tf)
        # the reference's state-dict layout, for the strict-load test on machines without the reference tree
        ref_sd = model.state_dict()
        out["ref_keys"] = np.array(list(ref_sd.keys()))
        out["ref_shapes"] = np.array([",".join(str(v) for v in t.shape) for t in ref_sd.values()])
        hp = dict(use_uv=True, pitch_norm=hparams["pitch_norm"], f0_mean=220.0, f0_std=60.0)
        for tag, r, t, m2p in (("pred", r1, {}, None), ("given", r2, tf, mel2ph)):
            ro, coarse, _ = fs2_ref.fs2_forward(sd, cfg, inp["txt_tokens"], mel2ph=m2p, **t, **kw, **hp)
            for k in r:
                if r[k].is_floating_point():
                    print(f"  {tag} oracle {k}: max |diff| {(ro[k] - r[k]).abs().max().item():.2e}")
                else:
                    assert torch.equal(ro[k], r[k]), (tag, k)
            if coarse is not None:
                out[tag + "_coarse"] = coarse
            for k in ("dur", "dur_choice", "mel2ph", "pitch_pred", "f0_denorm", "energy_pred"):
                if k in r and not (tag == "given" and k == "mel2ph"):
                    out[f"{tag}_{k}"] = r[k]
            out[tag + "_decoder_inp"] = r["decoder_inp"][..., ::8]
            out[tag + "_mel_out"] = r["mel_out"][..., ::4]
        save(name, **out)


if __name__ == "__main__":
    import_neuralseq()
    cwd = os.getcwd()
    os.chdir(os.path.join(REF, "NeuralSeq"))
    try:
        golden_fs2()
    finally:
        os.chdir(cwd)
