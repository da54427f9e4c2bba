"""GenerSpeech on the GPU (through the C ABI) vs the fixtures made by the reference module
(tests/golden/make_golden_generspeech.py) and vs the CPU oracle.  Stated tolerance: rel-RMSE <= 1e-4 on every float output
and stored intermediate (the gate of the other drivers: fp16x3 tensor-core GEMMs); mel2ph, dur_choice, the coarse pitch
bins and every VQ code index must be equal (the fixtures' seeds keep each rounded or argmin quantity >= 1e-3 from its
boundary)."""
import numpy as np
import pytest
import torch

from audiogpt_b200 import _lib, specs
from audiogpt_b200.modules.GenerSpeech.model.generspeech import GenerSpeech
from audiogpt_b200.utils.hparams import set_hparams_from_dict
from conftest import load_golden, rel_rmse
from test_generspeech_cpu import CASES, INPUTS, INT_KEYS, fixture_view, oracle_outputs

pytestmark = pytest.mark.gpu
CALL = dict(global_steps=300000, infer=True)


def build(cfg, **hp):
    set_hparams_from_dict(dict(specs.generspeech_hparams(cfg), **hp))
    m = GenerSpeech(specs.TokenDictionary(cfg["n_tokens"]))
    m.load_state_dict(specs.synth_generspeech(cfg), strict=True)
    return m.eval().to("cuda")


def inputs(g, rows=slice(None)):
    d = {k: torch.from_numpy(g[k])[rows].cuda() for k in INPUTS}
    return d.pop("txt_tokens"), d


def run(m, g, tag, rows=slice(None), **kw):
    tok, d = inputs(g, rows)
    m2p = torch.from_numpy(g["mel2ph_given"])[rows].cuda() if tag == "given" else None
    taps = {}
    r = m(tok, mel2ph=m2p, z_post=torch.from_numpy(g[tag + "_z"])[rows].cuda(), taps=taps, **d, **CALL, **kw)
    r = {k: v.cpu() for k, v in r.items()}
    r["coarse"] = taps.pop("pitch_coarse").cpu()
    r.update({k: v.cpu().long() if k.startswith("vq_idx") else v.cpu() for k, v in taps.items()})
    return r


def check_case(name, cfg):
    g = load_golden(name)
    m = build(cfg)
    for tag in ("pred", "given"):
        r = run(m, g, tag)
        ro = oracle_outputs(g, cfg, tag)
        keys = [k[len(tag) + 1:] for k in g.files if k.startswith(tag + "_") and k != tag + "_z"]
        assert {"mel_out", "mel_pre_flow", "prosody_utter", "vq_idx_word", "ref_prosody"} <= set(keys)
        for k in keys:
            if k.startswith("aligned_"):
                continue                      # the engine adds the aligner outputs straight into ref_prosody
            got, want = fixture_view(k, r[k]), g[f"{tag}_{k}"]
            assert tuple(got.shape) == want.shape, (tag, k, tuple(got.shape), want.shape)
            if k in INT_KEYS:
                assert np.array_equal(got.numpy(), want), (name, tag, k)
            else:
                e1, e2 = rel_rmse(got, want), rel_rmse(r[k], ro[k])
                print(f"{name} {tag} {k}: rel-RMSE vs reference {e1:.2e}, vs oracle {e2:.2e}")
                assert e1 < 1e-4 and e2 < 1e-4, (name, tag, k, e1, e2)
        for k in ("x_mask", "spk_embed", "emo_embed"):
            assert rel_rmse(r[k], ro[k]) < 1e-5, k
        assert r["mel_out"].shape[1] == 2 * (r["mel2ph"].shape[1] // 2)


@pytest.mark.parametrize("name,cfg", CASES)
def test_generspeech_vs_reference(name, cfg):
    check_case(name, cfg)


def test_generspeech_fp32_gemms():
    """the small config again with every GEMM on the fp32-FMA kernel"""
    L = _lib.lib()
    _lib.check(L.agpt_set_tensor_cores(0))
    try:
        check_case("generspeech_small", specs.GS_SMALL)
    finally:
        _lib.check(L.agpt_set_tensor_cores(1))


def test_odd_frames_and_batch_independence():
    """the teacher-forced case has an odd T_mel: the post-flow returns 2 floor(T / 2) frames; each row of the ragged batch
    equals its own B = 1 run (every row reaches the batch's largest segment ids, so the segment grids agree)"""
    name, cfg = CASES[0]
    g = load_golden(name)
    m = build(cfg)
    full = run(m, g, "given")
    T = g["mel2ph_given"].shape[1]
    assert T % 2 == 1 and full["mel_out"].shape[1] == T - 1
    for i in range(full["mel_out"].shape[0]):
        one = run(m, g, "given", rows=slice(i, i + 1))
        for k in ("mel_out", "decoder_inp", "ref_prosody", "pitch_pred"):
            assert rel_rmse(one[k][0], full[k][i]) < 1e-5, (i, k)
        assert torch.equal(one["coarse"][0], full["coarse"][i])


def test_noise_draw_and_zero_noise():
    """the drop-in draws the post-flow noise as the reference does (same seed -> same tensor); noise_scale = 0 gives the
    reverse flow of zeros"""
    from oracle import generspeech_ref as gr
    name, cfg = CASES[0]
    g = load_golden(name)
    m = build(cfg)
    shape = (3, 80, 11)
    torch.manual_seed(7)
    a = m.draw_noise(shape, "cuda")
    torch.manual_seed(7)
    b = torch.distributions.Normal(0, 1).sample(shape) * 0.8
    assert torch.equal(a.cpu(), b)
    tok, d = inputs(g)
    m2p = torch.from_numpy(g["mel2ph_given"]).cuda()
    torch.manual_seed(11)
    r1 = m(tok, mel2ph=m2p, **d, **CALL)
    torch.manual_seed(11)
    z = m.draw_noise((3, 80, m2p.shape[1]), "cuda")
    r2 = m(tok, mel2ph=m2p, z_post=z, **d, **CALL)
    assert torch.equal(r1["mel_out"], r2["mel_out"])
    m0 = build(cfg, noise_scale=0.0)
    r0 = {k: v.cpu() for k, v in m0(tok, mel2ph=m2p, **d, **CALL).items()}
    sd = specs.synth_generspeech(cfg)
    args = [torch.from_numpy(g[k]) for k in INPUTS]
    ro = gr.generspeech_forward(sd, cfg, *args, torch.zeros(3, 80, m2p.shape[1]), mel2ph=m2p.cpu())[0]
    assert rel_rmse(r0["mel_out"], ro["mel_out"]) < 1e-4


def test_errors_raise():
    name, cfg = CASES[0]
    g = load_golden(name)
    m = build(cfg)
    tok, d = inputs(g)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(tok.cpu(), **{k: v.cpu() for k, v in d.items()}, **CALL)
    with pytest.raises(ValueError):
        m(tok, **dict(d, ref_mel2ph=d["ref_mel2ph"][:, :-1]), **CALL)
    with pytest.raises(ValueError):
        m(tok, **dict(d, spk_embed=d["spk_embed"][:, :128]), **CALL)
    with pytest.raises(ValueError, match="z_post"):
        m(tok, mel2ph=torch.from_numpy(g["mel2ph_given"]).cuda(), z_post=torch.zeros(3, 80, 5, device="cuda"), **d, **CALL)


def test_tts_ood_chain_matches_oracles():
    """GenerSpeech -> HiFi-GAN (the TTS_OOD tool's vocoder; 16 kHz, hop 256) vs the two oracles"""
    from audiogpt_b200.modules.hifigan.hifigan import HifiGanGenerator
    from oracle import hifigan_ref as hr
    name, cfg = CASES[1]
    g = load_golden(name)
    m = build(cfg)
    h = dict(specs.HIFIGAN_SMALL, audio_sample_rate=16000)
    assert int(np.prod(h["upsample_rates"])) == 256
    sdh = specs.synth_hifigan(h, 1234)
    voc = HifiGanGenerator(h)
    voc.load_state_dict(sdh, strict=True)
    voc = voc.eval().to("cuda")
    tok, d = inputs(g)
    r = m(tok, mel2ph=torch.from_numpy(g["mel2ph_given"]).cuda(), z_post=torch.from_numpy(g["given_z"]).cuda(), **d, **CALL)
    wav = voc(r["mel_out"].transpose(1, 2).contiguous()).cpu()
    ro = oracle_outputs(g, cfg, "given")
    wo = hr.hifigan_forward(sdh, h, ro["mel_out"].transpose(1, 2).contiguous())
    assert wav.shape == wo.shape
    assert rel_rmse(wav, wo) < 1e-3, rel_rmse(wav, wo)
