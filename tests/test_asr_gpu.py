"""The TTS_OOD tool's reference-audio ASR (wav2vec2 CTC) on the engine against transformers' Wav2Vec2ForCTC in fp32 with
TF32 off, on the same seeded weights: the conv feature encoder, the positional conv, whole-model logits and argmax ids,
batch independence, the rebuild after a weight edit, and the AGPT_TENSOR_CORES=0 arm."""
import os
import sys

import pytest
import torch
from transformers import Wav2Vec2Config
from transformers import Wav2Vec2ForCTC as HFWav2Vec2ForCTC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from audiogpt_b200 import _lib, specs  # noqa: E402
from audiogpt_b200.inference.tts.base_tts_infer import Wav2Vec2ForCTC  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt()).item()


@pytest.fixture(scope="module", autouse=True)
def no_tf32():
    m, c = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = m, c


def _pair(cfg_dict, seed):
    cfg = Wav2Vec2Config(**cfg_dict)
    sd = specs.synth_w2v(cfg_dict, seed)
    ours, ref = Wav2Vec2ForCTC(cfg), HFWav2Vec2ForCTC(cfg)
    ours.load_state_dict(sd, strict=True)
    ref.load_state_dict(sd, strict=True)
    return ours.eval().to(DEV), ref.eval().to(DEV)


@pytest.fixture(scope="module")
def base():
    return _pair(specs.W2V_BASE, 2626)


@pytest.fixture(scope="module")
def small():
    return _pair(specs.W2V_SMALL, 2727)


def check_logits(got, want):
    assert got.shape == want.shape
    e = rel(got, want)
    assert e <= 1e-4, e
    w = want.double().cpu()
    top2 = w.topk(2, dim=-1).values
    sure = (top2[..., 0] - top2[..., 1]) > 1e-3 * w.abs().amax(dim=-1)
    ids_g, ids_w = got.argmax(-1).cpu(), w.argmax(-1)
    assert sure.float().mean() > 0.9
    assert torch.equal(ids_g[sure], ids_w[sure])


# Error budget against transformers fp32, measured against an fp64 run of the same module on an H100: the fp32
# reference sits ~3e-7 from fp64 per conv; each 3xfp16 tap-GEMM conv of the feature encoder adds ~6e-6 (fp16 hi / lo
# products with the tensor cores' truncating fp32 accumulation), so the seven-conv encoder lands at ~5e-5.  The stem
# alone (conv0 + GroupNorm + GELU, fp32 FMA) stays at ~1e-7.
STEM = dict(specs.W2V_SMALL, conv_dim=(512,), conv_kernel=(10,), conv_stride=(5,))


@pytest.fixture(scope="module")
def stem():
    return _pair(STEM, 2828)


@pytest.mark.parametrize("S,offset", [(400, 0.0), (401, 0.0), (16003, 0.0), (24011, 0.0), (320000, 0.0), (16000, 10.0)])
def test_stem(stem, S, offset):
    """conv0 + GroupNorm + GELU: the DC offset of 10 puts a mean ~10x the spread into every channel, where a cancelling
    E[x^2] - E[x]^2 in fp32 would miss this bound"""
    ours, ref = stem
    x = specs.synth_w2v_wav(S, seed=S, offset=offset).to(DEV)
    with torch.no_grad():
        want = ref.wav2vec2.feature_extractor(x)
    got = ours.engine_features(x)
    assert got.shape == want.shape
    e = rel(got, want)
    assert e <= 1e-6, e


@pytest.mark.parametrize("S,offset", [(400, 0.0), (401, 0.0), (16003, 0.0), (24011, 0.0), (320000, 0.0), (16000, 10.0)])
def test_feature_encoder(base, S, offset):
    ours, ref = base
    x = specs.synth_w2v_wav(S, seed=S, offset=offset).to(DEV)
    with torch.no_grad():
        want = ref.wav2vec2.feature_extractor(x)
    got = ours.engine_features(x)
    assert got.shape == want.shape
    e = rel(got, want)
    assert e <= 1e-4, e


@pytest.mark.parametrize("T", [1, 49, 64, 65, 499, 999])
def test_positional_conv(base, T):
    """pos_conv_embed's output alone (the engine's fused residual taken back off) on both arms"""
    ours, ref = base
    g = torch.Generator().manual_seed(T)
    h = torch.randn(2, T, 768, generator=g).to(DEV)
    with torch.no_grad():
        want = ref.wav2vec2.encoder.pos_conv_embed(h)
    for tc in (1, 0):
        _lib.check(_lib.lib().agpt_set_tensor_cores(tc))
        try:
            got = ours.engine_pos_conv(h) - h
            torch.cuda.synchronize()
        finally:
            _lib.check(_lib.lib().agpt_set_tensor_cores(1))
        e = rel(got, want)
        assert e <= 1e-5, (tc, e)


def test_small_config_logits(small):
    ours, ref = small
    x = specs.synth_w2v_wav(16000, seed=5).to(DEV)
    with torch.no_grad():
        want = ref(x).logits
    out = ours(x)
    check_logits(out.logits, want)


@pytest.mark.parametrize("sec", [3, 10, 20])
def test_base_config_logits(base, sec):
    ours, ref = base
    x = specs.synth_w2v_wav(sec * specs.W2V_SR, seed=100 + sec).to(DEV)
    with torch.no_grad():
        want = ref(x).logits
    check_logits(ours(x).logits, want)


def test_batch_rows_equal_single_rows(base):
    ours, _ = base
    x = specs.synth_w2v_wav(24011, seed=7, B=3).to(DEV)
    both = ours(x).logits
    for b in range(3):
        one = ours(x[b:b + 1]).logits
        assert rel(both[b:b + 1], one) <= 1e-6


def test_rebuild_after_weight_edit(small):
    ours, ref = small
    x = specs.synth_w2v_wav(16000, seed=9).to(DEV)
    ours(x)
    sig0 = ours._engine.sig
    with torch.no_grad():
        for m in (ours, ref):
            m.lm_head.bias[3] += 5.0
            m.wav2vec2.encoder.layers[0].attention.q_proj.weight.mul_(1.25)
    try:
        with torch.no_grad():
            want = ref(x).logits
        got = ours(x).logits
        assert ours._engine.sig != sig0
        check_logits(got, want)
    finally:
        with torch.no_grad():
            for m in (ours, ref):
                m.lm_head.bias[3] -= 5.0
                m.wav2vec2.encoder.layers[0].attention.q_proj.weight.div_(1.25)


def test_fp32_arm(base):
    ours, ref = base
    x = specs.synth_w2v_wav(10 * specs.W2V_SR, seed=11).to(DEV)
    with torch.no_grad():
        want = ref(x).logits
    _lib.check(_lib.lib().agpt_set_tensor_cores(0))
    try:
        got = ours(x).logits
        torch.cuda.synchronize()
    finally:
        _lib.check(_lib.lib().agpt_set_tensor_cores(1))
    check_logits(got, want)
