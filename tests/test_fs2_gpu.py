"""FastSpeech2 / FastSpeech2MIDI on the GPU (through the C ABI) vs the fixtures made by the reference modules
(tests/golden/make_golden_fs2.py) and vs the CPU oracle, plus the masked attention it runs on.  Stated tolerance:
rel-RMSE <= 1e-4 on every float output (8 FFT layers of attention + k=9 FFN on the fp16x3 tensor-core GEMMs; the gate of
the other drivers); the rounded quantities -- mel2ph, dur_choice, the coarse pitch bins -- must be equal (the fixtures'
seeds keep each one >= 1e-3 from its rounding boundary)."""
import ctypes as C

import numpy as np
import pytest
import torch

from audiogpt_b200 import _lib, specs
from audiogpt_b200.modules.diffsinger_midi.fs2 import FastSpeech2MIDI
from audiogpt_b200.modules.fastspeech.fs2 import FastSpeech2
from audiogpt_b200.utils.hparams import set_hparams_from_dict
from conftest import load_golden, rel_rmse
from test_fs2_cpu import CASES, INT_KEYS, fixture_inputs, fixture_view, hp_kwargs

pytestmark = pytest.mark.gpu


def build(cfg):
    set_hparams_from_dict(specs.fs2_hparams(cfg))
    m = (FastSpeech2MIDI if cfg["use_midi"] else FastSpeech2)(specs.TokenDictionary(cfg["n_tokens"]))
    sd = specs.synth_fs2(cfg)
    m.load_state_dict(sd, strict=True)
    return m.eval().to("cuda"), sd


def cuda(d):
    return {k: v.cuda() for k, v in d.items()}


def check_case(name, cfg):
    from oracle import fs2_ref
    g = load_golden(name)
    m, sd = build(cfg)
    tok, kw, m2p, tf = fixture_inputs(g, cfg)
    for tag, mel2ph, t in (("pred", None, {}), ("given", m2p, tf)):
        r, coarse = m.run(tok.cuda(), mel2ph=None if mel2ph is None else mel2ph.cuda(), **cuda(t), **cuda(kw))
        r = {k: v.cpu() for k, v in r.items()}
        if coarse is not None:
            r["coarse"] = coarse.cpu()
        ro, co, _ = fs2_ref.fs2_forward(sd, cfg, tok, mel2ph=mel2ph, **{k: v.clone() for k, v in t.items()}, **kw, **hp_kwargs(cfg))
        if co is not None:
            ro["coarse"] = co
        assert set(r) - {"coarse"} == set(ro) - {"coarse"}
        for k in [k[len(tag) + 1:] for k in g.files if k.startswith(tag + "_")]:
            got, want = fixture_view(tag, k, r[k]), g[f"{tag}_{k}"]
            assert tuple(got.shape) == want.shape, (tag, k)
            if k in INT_KEYS:
                assert np.array_equal(got.numpy(), want), (name, tag, k)
                assert torch.equal(r[k], ro[k]), (name, tag, k)
            else:
                e1, e2 = rel_rmse(got, want), rel_rmse(r[k], ro[k])
                print(f"{name} {tag} {k}: rel-RMSE vs reference {e1:.2e}, vs oracle {e2:.2e}")
                assert e1 < 1e-4 and e2 < 1e-4, (name, tag, k)
        if tag == "pred":
            assert r["dur"].shape == (*tok.shape, 1)
    return m, g


@pytest.mark.parametrize("name,cfg", CASES)
def test_fs2_vs_reference(name, cfg):
    check_case(name, cfg)


def test_fs2_c2_fp32_gemms():
    """the C2 config again with every GEMM on the fp32-FMA kernel"""
    L = _lib.lib()
    _lib.check(L.agpt_set_tensor_cores(0))
    try:
        check_case("fs2_c2", specs.FS2_C2)
    finally:
        _lib.check(L.agpt_set_tensor_cores(1))


@pytest.mark.parametrize("name,cfg", [("fs2_small", specs.FS2_SMALL), ("fs2_ds1000", specs.FS2_DS1000)])
def test_batch_independence(name, cfg):
    """One utterance run alone equals its row of the ragged batch: no sample reads another's rows (attention masks,
    GEMM tiles, conv boundaries).  The utterance keeps the batch's padded lengths, because the reference's values on
    valid frames depend on the padding length itself (LayerNorm turns a zero padding row into its bias, and the k=9 FFN
    conv and the unmasked pitch / energy predictors read it across the boundary)."""
    g = load_golden(name)
    m, _ = build(cfg)
    tok, kw, _, _ = fixture_inputs(g, cfg)
    rb, _ = m.run(tok.cuda(), **cuda(kw))
    b = 1
    one = {k: v[b:b + 1].cuda() for k, v in kw.items()}
    r1, _ = m.run(tok[b:b + 1].cuda(), **one)
    f = r1["mel2ph"].shape[1]
    assert torch.equal(r1["mel2ph"][0], rb["mel2ph"][b, :f]) and int((rb["mel2ph"][b] > 0).sum()) == f
    assert rel_rmse(r1["dur"][0].cpu(), rb["dur"][b].cpu()) < 1e-5
    r2, _ = m.run(tok[b:b + 1].cuda(), mel2ph=rb["mel2ph"][b:b + 1], **one)
    for k in ("decoder_inp", "mel_out"):
        assert rel_rmse(r2[k][0, :f].cpu(), rb[k][b, :f].cpu()) < 1e-5, k


def test_skip_decoder():
    m, _ = build(specs.FS2_SMALL)
    g = load_golden("fs2_small")
    r = m(torch.from_numpy(g["txt_tokens"]).cuda(), skip_decoder=True)
    assert "mel_out" not in r and rel_rmse(r["decoder_inp"][..., ::8].cpu(), g["pred_decoder_inp"]) < 1e-4


def test_cpu_tensor_raises():
    m, _ = build(specs.FS2_SMALL)
    with pytest.raises(RuntimeError, match="CUDA only"):
        m(torch.ones(1, 4, dtype=torch.long))


def _masked_attention(ptrs, mask, N, heads, d, Lq, Lk):
    qp, q_pitch, kp, vp, kv_pitch = ptrs
    L = _lib.lib()
    C_ = heads * d
    o = torch.full((N, Lq, C_), float("nan"), device="cuda")
    _lib.check(L.agpt_attention_masked(qp, q_pitch, kp, kv_pitch, vp, kv_pitch, _lib.fptr(mask), _lib.fptr(o), C_, N, heads,
                                       d, Lq, Lk, _lib.cur_stream()))
    torch.cuda.synchronize()
    return o.cpu()


# kind -> (Lq, Lk, operand layout of test_ldm_gpu.attention_operands)
MASK_KINDS = {"suffix": (150, 150, "kv"), "scattered": (150, 150, "kv"), "prefix": (150, 150, "kv"),
              "packed": (150, 150, "packed"), "peaky": (150, 150, "peaky"), "lq1": (1, 150, "kv"), "lk1": (70, 1, "kv"),
              "lk65": (65, 65, "packed")}


@pytest.mark.parametrize("d", [40, 128])
@pytest.mark.parametrize("kind", list(MASK_KINDS))
def test_masked_attention_vs_fp64(d, kind):
    """agpt_attention_masked against the fp64 masked softmax, on the wgmma kernel and on the fp32 kernel
    (AGPT_ATTN_TC=0); sample 2 has every key masked and must come out as zeros.  Suffix, scattered and prefix masks
    (the whole first 64-key block, then live keys), packed q | k | v rows, peaky scores, Lq = 1, Lk = 1, Lk = 65.
    rel-RMSE <= 1e-5."""
    from test_ldm_gpu import attention_operands
    N, heads = 3, 2
    Lq, Lk, layout = MASK_KINDS[kind]
    C_ = heads * d
    ptrs, (qh, kh, vh), _keep = attention_operands(N, heads, d, Lq, Lk, layout, 11)
    mask = torch.zeros(N, Lk, dtype=torch.uint8)
    if kind == "scattered":
        g = torch.Generator().manual_seed(5)
        mask[:2] = (torch.rand(2, Lk, generator=g) < 0.4).to(torch.uint8)
        mask[0, 64:128] = 1                                   # a whole 64-key block masked
    elif kind == "prefix":
        mask[:2, :64] = 1
        mask[1, 64:70] = 1
    elif Lk > 1:
        mask[0, Lk * 2 // 3:] = 1
        mask[1, 7:] = 1
    mask[2] = 1
    s = (qh @ kh.transpose(-1, -2) * d ** -0.5).masked_fill(mask.bool()[:, None, None, :], float("-inf"))
    ref = (torch.softmax(s, dim=-1) @ vh).permute(0, 2, 1, 3).reshape(N, Lq, C_)
    L = _lib.lib()
    for tc in (1, 0):
        _lib.check(L.agpt_set_attention_tc(tc))
        try:
            o = _masked_attention(ptrs, mask.cuda(), N, heads, d, Lq, Lk)
        finally:
            _lib.check(L.agpt_set_attention_tc(-1))
        assert torch.equal(o[2], torch.zeros_like(o[2])), tc
        e = rel_rmse(o[:2], ref[:2])
        print(f"masked attention d={d} {kind} tc={tc}: rel-RMSE {e:.2e}")
        assert e < 1e-5, tc
