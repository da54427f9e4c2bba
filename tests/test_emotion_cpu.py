"""CPU checks of the TTS_OOD tool's emotion encoder (data_gen.tts.emotion): the parameter order against the reference's
state_dict() keys, the partial slices of specs and of the C ABI against the reference's, the oracle against the
reference's own embed_utterance / EmotionEncoder (tests/golden/emotion.npz, make_golden_emotion.py), the seeded
weights' gate range, the config and drop-in refusals, install(emotion=True) and the C ABI's declarations."""
import ctypes as C
import importlib
import os
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from audiogpt_b200 import specs  # noqa: E402
from oracle import emotion_ref as ref  # noqa: E402

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "emotion.npz"))
CASES = list(range(len(GOLDEN["lengths"])))
# the oracle and the reference both run fp32 on the CPU with the same nn.LSTM; they differ in the DFT's rounding
ORACLE_TOL = 1e-5


@pytest.fixture(scope="module")
def reference_keys():
    """The reference EmotionEncoder's state_dict() keys and shapes, as make_golden_emotion.py recorded them."""
    return list(GOLDEN["keys"]), [tuple(int(v) for v in s.split(",")) for s in GOLDEN["shapes"]]


@pytest.fixture(scope="module")
def weights():
    return specs.synth_emotion(specs.EMO, int(GOLDEN["weight_seed"]))


def test_param_order_is_the_reference_state_dict_order(reference_keys):
    keys, shapes = reference_keys
    got = specs.emo_param_shapes(specs.EMO)
    assert list(got) == keys
    assert list(got.values()) == shapes


def test_dropin_has_the_reference_keys(reference_keys):
    from audiogpt_b200.data_gen.tts.emotion.model import EmotionEncoder
    sd = EmotionEncoder(torch.device("cpu"), torch.device("cpu")).state_dict()
    assert list(sd) == reference_keys[0]
    assert [tuple(v.shape) for v in sd.values()] == reference_keys[1]


def test_engine_weights_fold_the_biases(weights):
    ws = specs.emo_engine_weights(specs.EMO, weights)
    assert len(ws) == 3 * 3 + 2 + 3
    torch.testing.assert_close(ws[2], weights["lstm.bias_ih_l0"] + weights["lstm.bias_hh_l0"], rtol=0, atol=0)
    assert ws[0] is weights["lstm.weight_ih_l0"] and ws[4] is weights["lstm.weight_hh_l1"]
    assert tuple(ws[-3].shape) == (201, 400) and tuple(ws[-1].shape) == (201, 40)


SWEEP = [0, 1, 200, 201, 12799, 12800, 16000, 25439, 25440, 25599, 25600, 25601, 31999, 32000, 32001, 38399, 38400, 40000,
         44799, 44800, 160000, 283200, 960000, 960001]
KWARGS = [dict(), dict(partial_utterance_n_frames=80), dict(min_pad_coverage=1.0), dict(overlap=0.0), dict(overlap=0.75),
          dict(partial_utterance_n_frames=101, overlap=0.5)]   # 101 * 0.5 = 50.5: np.round takes the even 50


def _abi_partials(n, kw):
    from audiogpt_b200 import _lib
    a = dict(dict(partial_utterance_n_frames=160, min_pad_coverage=0.75, overlap=0.5), **kw)
    N, step, padded = C.c_int(), C.c_int(), C.c_long()
    _lib.check(_lib.lib().agpt_emo_partials(n, a["partial_utterance_n_frames"], a["min_pad_coverage"], a["overlap"],
                                            C.byref(N), C.byref(step), C.byref(padded)))
    return N.value, step.value, padded.value


@pytest.mark.parametrize("kw", KWARGS)
def test_abi_partials_match_python_twin(kw):
    from audiogpt_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libagpt_b200.so is not built")
    for n in SWEEP:
        wav_slices, mel_slices = specs.emo_partials(n, **kw)
        N, step, padded = _abi_partials(n, kw)
        assert N == len(wav_slices), n
        assert [s.start for s in mel_slices] == [i * step for i in range(N)], n
        assert all(s.stop - s.start == kw.get("partial_utterance_n_frames", 160) for s in mel_slices)
        assert padded == specs.emo_padded_length(n, wav_slices), n


@pytest.mark.parametrize("i", CASES)
def test_partials_match_the_reference(i):
    n = int(GOLDEN["lengths"][i])
    wav_slices, _ = specs.emo_partials(n)
    assert [[s.start, s.stop] for s in wav_slices] == GOLDEN[f"c{i}_slices"].tolist()


def _clip(i):
    wav = specs.synth_emotion_wav(int(GOLDEN["lengths"][i]), int(GOLDEN[f"c{i}_seed"]))
    assert abs(float(np.sum(wav, dtype=np.float64)) - float(GOLDEN[f"c{i}_wav_sum"])) <= 1e-6
    return wav


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("i", CASES)
def test_oracle_matches_the_reference(weights, i, dtype):
    wav = _clip(i)
    got = ref.embed_utterance(weights, wav, dtype=dtype)
    tol = ORACLE_TOL if dtype == torch.float32 else 2e-5
    np.testing.assert_allclose(got["partials"].numpy(), GOLDEN[f"c{i}_partials"], rtol=0, atol=tol)
    np.testing.assert_allclose(got["embed"].numpy(), GOLDEN[f"c{i}_embed"], rtol=0, atol=tol)
    frames = torch.stack([got["mel"][s] for s in specs.emo_partials(len(wav))[1]])
    np.testing.assert_allclose(ref.forward(weights, frames, dtype=dtype).numpy(), GOLDEN[f"c{i}_forward"], rtol=0, atol=tol)


def test_oracle_whole_utterance_matches_the_reference(weights):
    wav = specs.synth_emotion_wav(int(GOLDEN["whole_length"]), int(GOLDEN["whole_seed"]))
    got = ref.embed_utterance(weights, wav, using_partials=False, dtype=torch.float32)
    np.testing.assert_allclose(got["embed"].numpy(), GOLDEN["whole_embed"], rtol=0, atol=ORACLE_TOL)


def test_golden_is_not_trivial():
    """The partial embeddings vary between partials and clips by far more than the tolerances"""
    p = GOLDEN["c5_partials"]
    assert p.std(axis=0).mean() > 0.05
    assert np.abs(GOLDEN["c5_embed"] - GOLDEN["c6_embed"]).max() > 0.05


def test_seeded_weights_drive_the_gates_nonlinear(weights):
    """Every layer's gate pre-activations W_ih x + b + W_hh h pass |z| > 1 for a real fraction of them on a seeded clip."""
    wav = specs.synth_emotion_wav(48000, seed=7)
    x = ref.mel(wav)[None, :160]
    for k in range(3):
        one = torch.nn.LSTM(x.shape[-1], 256, 1, batch_first=True).double()
        one.load_state_dict({n.replace(f"_l{k}", "_l0"): weights[f"lstm.{n}"] for n in
                             (f"weight_ih_l{k}", f"weight_hh_l{k}", f"bias_ih_l{k}", f"bias_hh_l{k}")})
        with torch.no_grad():
            out, _ = one(x)
            hprev = torch.cat([torch.zeros_like(out[:, :1]), out[:, :-1]], 1)
            z = x @ one.weight_ih_l0.T + hprev @ one.weight_hh_l0.T + one.bias_ih_l0 + one.bias_hh_l0
        frac = (z.abs() > 1).double().mean().item()
        assert frac > (0.25 if k == 0 else 0.08), (k, frac)
        x = out


@pytest.mark.parametrize("change,what", [
    (dict(hidden_size=128), "hidden_size"),
    (dict(num_layers=0), "num_layers"),
    (dict(input_size=80), "input_size"),
    (dict(embedding_size=0), "embedding_size"),
])
def test_unsupported_configs_are_refused(change, what):
    with pytest.raises(ValueError, match=what):
        specs.emo_check(dict(specs.EMO, **change))


def test_dropin_refusals():
    from audiogpt_b200.data_gen.tts.emotion.model import EmotionEncoder
    m = EmotionEncoder(torch.device("cpu"), torch.device("cpu")).eval()
    x = torch.zeros(2, 160, 40)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.inference(x)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(x)
    with pytest.raises(TypeError, match="float32"):
        m.inference(x.double())
    with pytest.raises(ValueError, match="40"):
        m.inference(torch.zeros(2, 160, 41))
    with pytest.raises(NotImplementedError, match="hidden_init"):
        m.inference(x, hidden_init=(torch.zeros(3, 2, 256), torch.zeros(3, 2, 256)))
    with pytest.raises(ValueError, match="1-D float32 CUDA"):
        m.engine_embed(torch.zeros(16000))
    m.train()
    with pytest.raises(RuntimeError, match="inference only"):
        m.inference(x)
    m.eval()
    m.lstm = torch.nn.LSTM(40, 128, 3, batch_first=True)
    with pytest.raises(ValueError, match="hidden_size"):
        m.engine_cfg()


def test_embed_utterance_needs_a_loaded_dropin(monkeypatch):
    from audiogpt_b200.data_gen.tts.emotion import inference
    monkeypatch.setattr(inference, "_model", None)
    with pytest.raises(Exception, match="load_model"):
        inference.embed_utterance(np.zeros(16000, np.float32))
    monkeypatch.setattr(inference, "_model", torch.nn.LSTM(40, 256, 3, batch_first=True))
    with pytest.raises(TypeError, match="install"):
        inference.embed_utterance(np.zeros(16000, np.float32))


def test_compute_partial_slices_signature():
    from audiogpt_b200.data_gen.tts.emotion import inference
    a = inference.compute_partial_slices(40000, partial_utterance_n_frames=80, min_pad_coverage=0.5, overlap=0.25)
    assert a == specs.emo_partials(40000, 80, 0.5, 0.25)


NAMES = ("data_gen", "data_gen.tts", "data_gen.tts.emotion", "data_gen.tts.emotion.model", "data_gen.tts.emotion.inference",
         "inference", "inference.tts", "inference.tts.GenerSpeech")


def _stub(monkeypatch, with_tool=False):
    for n in NAMES:
        monkeypatch.delitem(sys.modules, n, raising=False)
    mods = {n: types.ModuleType(n) for n in NAMES[:5]}
    for n in NAMES[:3]:
        mods[n].__path__ = []
    model, inf = mods["data_gen.tts.emotion.model"], mods["data_gen.tts.emotion.inference"]

    class RefEmotionEncoder(torch.nn.Module):
        pass
    model.EmotionEncoder = inf.EmotionEncoder = RefEmotionEncoder
    inf._model, inf._device = None, None

    def embed_utterance(wav, using_partials=True, return_partials=False, **kwargs):
        return "reference"

    def embed_frames_batch(frames_batch):
        return "reference"

    def preprocess_wav(fpath_or_wav, source_sr=None):
        return fpath_or_wav
    inf.embed_utterance, inf.embed_frames_batch, inf.preprocess_wav = embed_utterance, embed_frames_batch, preprocess_wav
    if with_tool:
        for n in NAMES[5:7]:
            mods[n] = types.ModuleType(n)
            mods[n].__path__ = []
        mods["inference.tts.GenerSpeech"] = tool = types.ModuleType("inference.tts.GenerSpeech")
        tool.EmotionEncoder, tool.Embed_utterance = inf, embed_utterance
    for n, v in mods.items():
        monkeypatch.setitem(sys.modules, n, v)
    return mods


def test_install_emotion_patches_the_modules_in_place(monkeypatch):
    import audiogpt_b200
    from audiogpt_b200.data_gen.tts.emotion import inference as ours
    from audiogpt_b200.data_gen.tts.emotion.model import EmotionEncoder
    mods = _stub(monkeypatch, with_tool=True)
    monkeypatch.setattr(ours, "_state", ours)
    keep = mods["data_gen.tts.emotion.inference"].preprocess_wav
    patched = audiogpt_b200.install(emotion=True)
    inf = mods["data_gen.tts.emotion.inference"]
    assert "data_gen.tts.emotion.inference" in patched and "data_gen.tts.emotion.model" in patched
    assert sys.modules["data_gen.tts.emotion.inference"] is inf
    assert inf.EmotionEncoder is EmotionEncoder and mods["data_gen.tts.emotion.model"].EmotionEncoder is EmotionEncoder
    assert inf.embed_utterance is ours.embed_utterance and inf.embed_frames_batch is ours.embed_frames_batch
    assert inf.preprocess_wav is keep
    assert ours._state is inf
    assert mods["inference.tts.GenerSpeech"].Embed_utterance is ours.embed_utterance


def test_install_without_the_flag_leaves_it_alone(monkeypatch):
    import audiogpt_b200
    mods = _stub(monkeypatch, with_tool=True)
    inf = mods["data_gen.tts.emotion.inference"]
    before = dict(vars(inf))
    patched = audiogpt_b200.install()
    assert not any("emotion" in p for p in patched)
    assert dict(vars(inf)) == before
    assert mods["inference.tts.GenerSpeech"].Embed_utterance is before["embed_utterance"]


def test_install_emotion_skips_a_missing_module(monkeypatch):
    import audiogpt_b200
    for n in NAMES:
        monkeypatch.delitem(sys.modules, n, raising=False)
    real = importlib.import_module

    def fake(name, *a, **k):
        if name.startswith("data_gen"):
            raise ImportError(name)
        return real(name, *a, **k)
    monkeypatch.setattr(importlib, "import_module", fake)
    patched = audiogpt_b200.install(emotion=True)
    assert "data_gen.tts.emotion.inference (skipped: not importable)" in patched
    assert "data_gen.tts.emotion.model (skipped: not importable)" in patched
    assert "data_gen.tts.emotion.inference" not in sys.modules
    with pytest.raises(ImportError):
        audiogpt_b200.install(emotion=True, strict=True)


def test_abi_symbols_declared():
    with open(os.path.join(ROOT, "include", "agpt_b200.h")) as f:
        hdr = f.read()
    from audiogpt_b200 import _lib
    for sym in ("agpt_emo_create", "agpt_emo_partials", "agpt_emo_embed", "agpt_emo_hidden", "agpt_emo_forward", "agpt_emo_mel",
                "agpt_emo_lstm"):
        assert sym + "(" in hdr
        assert sym in _lib.PROTOTYPES
    body = hdr[hdr.index("typedef struct agpt_emo_cfg"):hdr.index("} agpt_emo_cfg;")]
    fields = [ln.split(";")[0].split()[-1] for ln in body.splitlines()[1:] if ";" in ln]
    assert fields == [f[0] for f in _lib.EmoConfig._fields_]
    assert list(specs.EMO) == fields
