"""CPU checks of the TTS_OOD tool's reference-audio ASR (wav2vec2 CTC): the parameter order against transformers'
Wav2Vec2ForCTC, the super-row packing of the strided convs (fp64, with the engine's padding rule), the folded positional
weight, the frame count, install(asr=True), the drop-in's refusals and the C ABI's declarations."""
import ctypes as C
import importlib
import os
import sys
import types

import pytest
import torch
import torch.nn.functional as F
from transformers import Wav2Vec2Config
from transformers import Wav2Vec2ForCTC as HFWav2Vec2ForCTC
from transformers.models.wav2vec2.modeling_wav2vec2 import Wav2Vec2FeatureEncoder

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from audiogpt_b200 import specs  # noqa: E402

LENGTHS = (400, 401, 16003, 24011, 320000)


@pytest.fixture(scope="module")
def small():
    cfg = Wav2Vec2Config(**specs.W2V_SMALL)
    m = HFWav2Vec2ForCTC(cfg).eval()
    m.load_state_dict(specs.synth_w2v(specs.W2V_SMALL), strict=True)
    return cfg, m


@pytest.mark.parametrize("name", ["W2V_SMALL", "W2V_BASE"])
def test_param_order_is_the_state_dict_order(name):
    cfg = getattr(specs, name)
    with torch.device("meta"):
        m = HFWav2Vec2ForCTC(Wav2Vec2Config(**cfg))
    sd = m.state_dict()
    shapes = specs.w2v_param_shapes(cfg)
    assert list(shapes) == list(sd)
    assert all(tuple(sd[k].shape) == v for k, v in shapes.items())


def test_engine_order_reorders_k_v_q_into_q_k_v(small):
    cfg, m = small
    sd = m.state_dict()
    got = specs.w2v_engine_weights(cfg, sd)
    p = "wav2vec2.encoder.layers.1."
    names = [p + "attention." + n for n in ("q_proj", "k_proj", "v_proj")]
    ids = [id(t) for t in got]
    # q, k, v weight / bias pairs are consecutive in that order
    i = ids.index(id(sd[names[0] + ".weight"]))
    assert ids[i:i + 6] == [id(sd[n + s]) for n in names for s in (".weight", ".bias")]
    assert ids[i + 6] == id(sd[p + "attention.out_proj.weight"])
    assert id(sd["wav2vec2.masked_spec_embed"]) not in ids
    nconv = len(cfg.conv_dim)
    assert len(got) == 3 + (nconv - 1) + 4 + 2 + 2 + 16 * cfg.num_hidden_layers + 2


def _superrow_conv(x, w, s, L):
    """The tap-GEMM the engine runs: x [R][Ci] (rows past the input zero) read as super-rows, output rows 0 .. L - 1 of
    the stride-1 conv over them with the packed weight; super-rows at or past L read as zero."""
    wp = specs.w2v_superrow_weight(w, s)
    Co, SC, nt = wp.shape
    sup = x[: (x.shape[0] // s) * s].reshape(-1, SC)[:L]
    sup = torch.cat([sup, sup.new_zeros((nt, SC))])
    return sum(sup[t:t + L] @ wp[:, :, t].T for t in range(nt))


@pytest.mark.parametrize("T", [49, 50, 97, 98, 101, 1000, 1001])
@pytest.mark.parametrize("k,s", [(3, 2), (2, 2), (4, 2), (5, 3)])
def test_superrow_packing_is_a_strided_conv(T, k, s):
    g = torch.Generator().manual_seed(T * 31 + k * 7 + s)
    Ci, Co = 8, 6
    x = torch.randn(T, Ci, generator=g, dtype=torch.float64)
    w = torch.randn(Co, Ci, k, generator=g, dtype=torch.float64)
    ref = F.conv1d(x.T[None], w, stride=s)[0].T
    Lin = -(-T // s)                                  # the GEMM runs over the input's super-rows ...
    buf = torch.cat([x, x.new_zeros((s, Ci))])        # ... padded to whole super-rows with zeros
    out = _superrow_conv(buf, w, s, Lin)
    assert out.shape[0] >= ref.shape[0]
    torch.testing.assert_close(out[: ref.shape[0]], ref, rtol=0, atol=1e-12)
    if -(-k // s) > 1 and T % s:
        # over the output length instead, the last frame would lose its last tap
        short = _superrow_conv(buf, w, s, ref.shape[0])
        assert (short[-1] - ref[-1]).abs().max() > 1e-6


@pytest.mark.parametrize("S", [16000, 16001, 16003, 24011])
def test_superrow_stack_matches_the_feature_encoder(small, S):
    """Conv 1.. chained as the engine runs them: rows past each output's length are zeroed before the next super-row
    view reads them (they hold partial sums of the padding)."""
    cfg, m = small
    fe = m.wav2vec2.feature_extractor.double()
    try:
        x = specs.synth_w2v_wav(S, seed=S)[0].double()
        with torch.no_grad():
            h = fe.conv_layers[0](x[None, None])[0].T               # [T0][C] after conv0 + GroupNorm + GELU
            want = fe(x[None])[0].T
            T = h.shape[0]
            for i in range(1, len(cfg.conv_dim)):
                s, w = cfg.conv_stride[i], fe.conv_layers[i].conv.weight
                Tout = (T - cfg.conv_kernel[i]) // s + 1
                buf = torch.cat([h[:T], h.new_zeros((s, h.shape[1]))])
                out = F.gelu(_superrow_conv(buf, w, s, -(-T // s)))
                out[Tout:] = 0.0
                h, T = out, Tout
        torch.testing.assert_close(h[:T], want, rtol=0, atol=1e-12)
    finally:
        fe.float()


def test_folded_positional_weight_is_the_parametrised_weight(small):
    _, m = small
    conv = m.wav2vec2.encoder.pos_conv_embed.conv
    p = conv.parametrizations.weight
    got = specs.w2v_fold_pos_weight(p.original0, p.original1)
    assert torch.equal(got, conv.weight)


@pytest.mark.parametrize("S", LENGTHS + (399,))
def test_frame_count_matches_the_feature_encoder(S):
    cfg = Wav2Vec2Config(**specs.W2V_BASE)
    with torch.device("meta"):
        fe = Wav2Vec2FeatureEncoder(cfg)
        if S >= 400:
            T = fe(torch.empty(1, S)).shape[-1]
        else:
            T = 0
    assert specs.w2v_lengths(specs.W2V_BASE, S)[-1] == T


def test_abi_frames_matches_python_twin():
    from audiogpt_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libagpt_b200.so is not built")
    ec = specs.w2v_engine_cfg(specs.W2V_BASE)
    cc = _lib.W2vConfig()
    for k, v in ec.items():
        if k in ("conv_kernel", "conv_stride"):
            getattr(cc, k)[:len(v)] = v
        else:
            setattr(cc, k, v)
    n = C.c_int()
    for S in LENGTHS + (399, 1):
        assert _lib.lib().agpt_w2v_frames(C.byref(cc), S, C.byref(n)) == 0
        assert n.value == specs.w2v_lengths(specs.W2V_BASE, S)[-1]


@pytest.mark.parametrize("change,what", [
    (dict(feat_extract_norm="layer", do_stable_layer_norm=True), "feat_extract_norm"),   # the large / lv60 layout
    (dict(do_stable_layer_norm=True), "do_stable_layer_norm"),
    (dict(hidden_act="relu"), "gelu"),
    (dict(conv_bias=True), "conv_bias"),
    (dict(conv_dim=(512,) * 6 + (256,)), "equal"),
    (dict(num_attention_heads=7, hidden_size=768), "head dim"),
    (dict(num_conv_pos_embedding_groups=8), "48"),
])
def test_unsupported_configs_are_refused(change, what):
    with pytest.raises(ValueError, match=what):
        specs.w2v_check(Wav2Vec2Config(**dict(specs.W2V_BASE, **change)))


def test_dropin_refusals():
    from audiogpt_b200.inference.tts.base_tts_infer import Wav2Vec2ForCTC
    m = Wav2Vec2ForCTC(Wav2Vec2Config(**dict(specs.W2V_SMALL, num_hidden_layers=1))).eval()
    x = torch.zeros(1, 16000)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(x)
    with pytest.raises(TypeError, match="float32"):
        m(x.double())
    with pytest.raises(ValueError, match="no frame"):
        m(torch.zeros(1, 399))
    with pytest.raises(NotImplementedError, match="attention_mask"):
        m(x, attention_mask=torch.ones(1, 16000, dtype=torch.long))
    with pytest.raises(NotImplementedError, match="labels"):
        m(x, labels=torch.zeros(1, 3, dtype=torch.long))
    with pytest.raises(NotImplementedError, match="attentions"):
        m(x, output_attentions=True)
    with pytest.raises(NotImplementedError, match="hidden states"):
        m(x, output_hidden_states=True)
    m.train()
    with pytest.raises(RuntimeError, match="inference only"):
        m(x)


def _stub(monkeypatch):
    for n in ("inference", "inference.tts", "inference.tts.base_tts_infer"):
        monkeypatch.delitem(sys.modules, n, raising=False)
    pkg, tts, mod = types.ModuleType("inference"), types.ModuleType("inference.tts"), types.ModuleType("inference.tts.base_tts_infer")
    pkg.__path__, tts.__path__ = [], []
    pkg.tts, tts.base_tts_infer = tts, mod
    mod.Wav2Vec2ForCTC = HFWav2Vec2ForCTC

    class BaseTTSInfer:
        pass
    mod.BaseTTSInfer = BaseTTSInfer
    for n, v in (("inference", pkg), ("inference.tts", tts), ("inference.tts.base_tts_infer", mod)):
        monkeypatch.setitem(sys.modules, n, v)
    return mod


def test_install_asr_patches_the_module_in_place(monkeypatch):
    import audiogpt_b200
    from audiogpt_b200.inference.tts.base_tts_infer import Wav2Vec2ForCTC
    mod = _stub(monkeypatch)
    keep = mod.BaseTTSInfer
    patched = audiogpt_b200.install(asr=True)
    assert "inference.tts.base_tts_infer" in patched
    assert sys.modules["inference.tts.base_tts_infer"] is mod
    assert mod.Wav2Vec2ForCTC is Wav2Vec2ForCTC and mod.BaseTTSInfer is keep


def test_install_without_the_flag_leaves_it_alone(monkeypatch):
    import audiogpt_b200
    mod = _stub(monkeypatch)
    patched = audiogpt_b200.install()
    assert not any("base_tts_infer" in p for p in patched)
    assert mod.Wav2Vec2ForCTC is HFWav2Vec2ForCTC


def test_install_asr_skips_a_missing_module(monkeypatch):
    import audiogpt_b200
    for n in ("inference", "inference.tts", "inference.tts.base_tts_infer"):
        monkeypatch.delitem(sys.modules, n, raising=False)
    real = importlib.import_module

    def fake(name, *a, **k):
        if name.startswith("inference"):
            raise ImportError(name)
        return real(name, *a, **k)
    monkeypatch.setattr(importlib, "import_module", fake)
    patched = audiogpt_b200.install(asr=True)
    assert "inference.tts.base_tts_infer (skipped: not importable)" in patched
    assert "inference.tts.base_tts_infer" not in sys.modules
    with pytest.raises(ImportError):
        audiogpt_b200.install(asr=True, strict=True)


def test_abi_symbols_declared():
    with open(os.path.join(ROOT, "include", "agpt_b200.h")) as f:
        hdr = f.read()
    from audiogpt_b200 import _lib
    for sym in ("agpt_w2v_create", "agpt_w2v_frames", "agpt_w2v_logits", "agpt_w2v_features", "agpt_w2v_pos_conv"):
        assert sym + "(" in hdr
        assert sym in _lib.PROTOTYPES
    assert "agpt_w2v_cfg" in hdr
    body = hdr[hdr.index("typedef struct agpt_w2v_cfg"):hdr.index("} agpt_w2v_cfg;")]
    fields = [ln.split(";")[0].split()[-1].split("[")[0] for ln in body.splitlines()[1:] if ";" in ln]
    assert fields == [f[0] for f in _lib.W2vConfig._fields_]
    assert list(specs.w2v_engine_cfg(specs.W2V_BASE)) == fields
