#!/usr/bin/env python
"""Generate the GenerSpeech golden fixtures (generspeech_*.npz) by running the REFERENCE's own module on CPU fp32, with
the shims and helpers of make_golden.py.

Run in the build container only (needs /root/reference, which does not travel to the GPU box):

    python tests/golden/make_golden_generspeech.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF, ROOT, import_neuralseq, save, specs  # noqa: E402


def golden_generspeech():
    """GenerSpeech (NeuralSeq/modules/GenerSpeech/model/generspeech.py) called as GenerSpeechInfer.forward_model calls it
    (infer=True, global_steps=300000) on a ragged B = 3 batch with padded ref_mels and an empty phoneme segment, once with
    predicted durations and once with a teacher-forced mel2ph of odd length.  The post-flow noise is the reference's own
    draw (dist.Normal(0, 1).sample on the CPU generator after torch.manual_seed(seed), x noise_scale), stored as z_*.
    Input seeds are drawn until every rounded or argmin quantity has a margin against fp16x3 error: the duration rounding
    and the coarse pitch >= 1e-3 from their boundaries, each VQ choice's best and second-best distances >= 1e-3 apart
    (relative).  Intermediates (quantised prosody and code indices per level, aligner outputs, the pre-flow mel) are kept
    so a failure points to a stage; wide tensors are stored on a channel subsample."""
    sys.path.insert(0, ROOT)
    from oracle import generspeech_ref as gr
    from utils.hparams import hparams
    from modules.GenerSpeech.model.generspeech import GenerSpeech
    for name, cfg, B, T, T_ref in (("generspeech_small", specs.GS_SMALL, 3, 16, 40),
                                   ("generspeech_c2", specs.GS_C2, 3, 12, 48)):
        hparams.clear()
        hparams.update(specs.generspeech_hparams(cfg))
        model = GenerSpeech(specs.TokenDictionary(cfg["n_tokens"]))
        sd = specs.synth_generspeech(cfg)
        print(name, "load:", model.load_state_dict(sd, strict=True))
        assert set(model.state_dict().keys()) == set(specs.generspeech_param_shapes(cfg).keys())
        model.eval()
        ns = hparams["noise_scale"]
        for seed in range(2000, 2400):
            inp = specs.synth_generspeech_inputs(cfg, B, T, T_ref, seed)
            args = [inp[k] for k in ("txt_tokens", "ref_mels", "ref_mel2ph", "ref_mel2word", "spk_embed", "emo_embed")]
            # screen the margins on the oracle (the noise only enters after the last rounded quantity)
            with torch.no_grad():
                o1 = gr.generspeech_forward(sd, cfg, *args, None)
            m = [o1[3]["dur_margin"], o1[3]["f0_margin"], o1[3]["vq_margin"]]
            if min(m) < 1e-3:
                continue
            kw = dict(ref_mel2ph=inp["ref_mel2ph"], ref_mel2word=inp["ref_mel2word"], ref_mels=inp["ref_mels"],
                      spk_embed=inp["spk_embed"], emo_embed=inp["emo_embed"], global_steps=300000, infer=True)
            torch.manual_seed(seed)
            with torch.no_grad():
                r1 = model(inp["txt_tokens"], **kw)
            torch.manual_seed(seed)
            z1 = torch.distributions.Normal(0, 1).sample((B, 80, r1["mel2ph"].shape[1])) * ns
            # teacher-forced durations: one extra frame on every third token, and an odd frame count
            d2 = (r1["dur_choice"] + (torch.arange(T)[None] % 3 == 0).long()) * (inp["txt_tokens"] > 0).long()
            cum = torch.cumsum(d2, 1)
            n_fr = int(cum[:, -1].max())
            n_fr += 1 - n_fr % 2
            pos = torch.arange(n_fr)[None, None]
            mel2ph = ((pos >= (cum - d2)[:, :, None]) & (pos < cum[:, :, None])).long()
            mel2ph = (torch.arange(1, T + 1)[None, :, None] * mel2ph).sum(1)
            torch.manual_seed(seed + 1)
            with torch.no_grad():
                r2 = model(inp["txt_tokens"], mel2ph=mel2ph, **kw)
            torch.manual_seed(seed + 1)
            z2 = torch.distributions.Normal(0, 1).sample((B, 80, n_fr)) * ns
            with torch.no_grad():
                o1 = gr.generspeech_forward(sd, cfg, *args, z1)
                o2 = gr.generspeech_forward(sd, cfg, *args, z2, mel2ph=mel2ph)
            m = [o1[3]["dur_margin"], o1[3]["f0_margin"], o2[3]["f0_margin"], o1[3]["vq_margin"]]
            if min(m) >= 1e-3:
                break
        print(name, "seed", seed, "margins", ["%.1e" % v for v in m], "frames", r1["mel2ph"].shape[1], n_fr)
        out = dict(seed=np.array(seed), margins=np.array(m), mel2ph_given=mel2ph, **inp)
        ref_sd = model.state_dict()
        out["ref_keys"] = np.array(list(ref_sd.keys()))
        out["ref_shapes"] = np.array([",".join(str(v) for v in t.shape) for t in ref_sd.values()])
        for tag, r, z, (ro, coarse, mid, _) in (("pred", r1, z1, o1), ("given", r2, z2, o2)):
            for k in ("mel_out", "decoder_inp", "dur", "pitch_pred", "f0_denorm", "f0_denorm_pred", "ref_prosody",
                      "spk_embed", "emo_embed", "x_mask", "mel2ph", "dur_choice"):
                if k not in r:
                    continue
                if r[k].is_floating_point():
                    print(f"  {tag} oracle {k}: max |diff| {(ro[k] - r[k]).abs().max().item():.2e}")
                else:
                    assert torch.equal(ro[k], r[k]), (tag, k)
            out[tag + "_z"] = z
            out[tag + "_coarse"] = coarse
            for k in ("dur", "dur_choice", "mel2ph", "pitch_pred", "f0_denorm", "f0_denorm_pred", "spk_embed", "emo_embed"):
                if k in r and not (tag == "given" and k == "mel2ph"):
                    out[f"{tag}_{k}"] = r[k]
            out[tag + "_decoder_inp"] = r["decoder_inp"][..., ::8]
            out[tag + "_ref_prosody"] = r["ref_prosody"][..., ::8]
            out[tag + "_mel_out"] = r["mel_out"][..., ::4]
            out[tag + "_mel_pre_flow"] = mid["mel_pre_flow"][..., ::4]
            for lvl in specs.GS_LEVELS:
                out[f"{tag}_prosody_{lvl}"] = mid[f"prosody_{lvl}"][..., ::8]
                out[f"{tag}_vq_idx_{lvl}"] = mid[f"vq_idx_{lvl}"]
                out[f"{tag}_aligned_{lvl}"] = mid[f"aligned_{lvl}"][..., ::8]
        save(name, **out)


if __name__ == "__main__":
    import_neuralseq()
    cwd = os.getcwd()
    os.chdir(os.path.join(REF, "NeuralSeq"))
    try:
        golden_generspeech()
    finally:
        os.chdir(cwd)
