"""The TTS_OOD tool's emotion encoder on the engine: the power-mel stage against the fp64 oracle, one LSTM layer's
recurrence (agpt_emo_lstm) and the whole stack against fp64, hidden[-1], forward and embed_utterance against the
reference's own outputs (tests/golden/emotion.npz) and the fp64 oracle, the AGPT_TENSOR_CORES=0 arm, batch rows, the
rebuild after a weight edit, the refused inputs, and the installed tool's load_model -> Embed_utterance."""
import os
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from audiogpt_b200 import _lib, specs  # noqa: E402
from audiogpt_b200.data_gen.tts.emotion import inference as emo_inference  # noqa: E402
from audiogpt_b200.data_gen.tts.emotion.model import EmotionEncoder  # noqa: E402
from oracle import emotion_ref as ref  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "emotion.npz"))
CASES = list(range(len(GOLDEN["lengths"])))

# Tolerances, set from one run on an H100 80GB HBM3; the worst value measured over the golden clips and the stage grids
# is given for each.  The golden itself (the reference in fp32 on the CPU) is within 1.7e-7 of fp64 on the embedding
# and 6.1e-7 on the partials.
MEL_TOL = 1e-5          # power mel rel-RMSE against fp64 (the DFT on the 3xfp16 tap-GEMM): 4.1e-6
STEP_TOL = 5e-6         # one layer's h (|h| < 1) max abs against fp64, T up to 1001, N up to 74: 3.8e-7
HIDDEN_TOL = 1e-4       # hidden[-1] rel-RMSE against fp64 and the golden: 1.3e-5 (the 3xfp16 input projections), 2.1e-6
                        # with AGPT_TENSOR_CORES=0
EMBED_TOL = 1e-5        # max abs on the unit-norm embedding: 4.4e-6, 7.7e-7 with AGPT_TENSOR_CORES=0


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt()).item()


def mx(a, b):
    return (torch.as_tensor(a).double().cpu() - torch.as_tensor(b).double().cpu()).abs().max().item()


@pytest.fixture(scope="module", autouse=True)
def no_tf32():
    m, c = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = m, c


def _model(sd, layers=3):
    m = EmotionEncoder(DEV, torch.device("cpu"))
    if layers != 3:
        m.lstm = torch.nn.LSTM(40, 256, layers, batch_first=True).to(DEV)
    m.load_state_dict(sd, strict=True)
    return m.eval()


@pytest.fixture(scope="module")
def weights():
    return specs.synth_emotion(specs.EMO, int(GOLDEN["weight_seed"]))


@pytest.fixture(scope="module")
def model(weights):
    return _model(weights)


@pytest.fixture()
def loaded(model, monkeypatch):
    monkeypatch.setattr(emo_inference, "_state", emo_inference)
    monkeypatch.setattr(emo_inference, "_model", model)
    monkeypatch.setattr(emo_inference, "_device", DEV)
    return emo_inference


@pytest.mark.parametrize("n", [201, 202, 16001, 25600, 40003, 160007])
def test_mel_stage(model, n):
    wav = specs.synth_emotion_wav(n, seed=n)
    got = model.engine_mel(torch.from_numpy(wav).to(DEV))
    want = ref.mel(wav, torch.float64)
    assert got.shape == want.shape
    e = rel(got, want)
    assert e <= MEL_TOL, e


def _lstm64(whh, xp, N, T, stride):
    """One layer's recurrence in fp64 on the device: rows n * stride + t of xp [.][1024]."""
    idx = (torch.arange(N, device=DEV)[:, None] * stride + torch.arange(T, device=DEV)[None, :])
    x = xp.double()[idx]                               # [N][T][1024]
    w = whh.double()
    h = torch.zeros(N, 256, dtype=torch.float64, device=DEV)
    c = torch.zeros_like(h)
    hs = []
    for t in range(T):
        z = x[:, t] + h @ w.T
        i, f, g, o = z.chunk(4, dim=1)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
        h = torch.sigmoid(o) * torch.tanh(c)
        hs.append(h)
    return torch.stack(hs, 1)


@pytest.mark.parametrize("N", [1, 5, 12, 33, 74])
@pytest.mark.parametrize("T", [1, 7, 160, 1001])
def test_lstm_stage(T, N):
    g = torch.Generator().manual_seed(T * 131 + N)
    whh = (torch.randn(1024, 256, generator=g) * (2.0 / 16)).to(DEV)
    stride = T if T < 160 else T // 2                  # T >= 160: overlapping sequences, as layer 0's partials read
    rows = (N - 1) * stride + T
    xp = (torch.randn(rows, 1024, generator=g) * 1.5).to(DEV)
    seq = torch.empty(N, T, 256, device=DEV)
    last = torch.empty(N, 256, device=DEV)
    _lib.call("emo_lstm", DEV, _lib.fptr(whh), _lib.fptr(xp), N, T, stride, _lib.fptr(seq), _lib.fptr(last))
    want = _lstm64(whh, xp, N, T, stride)
    e = mx(seq, want)
    assert e <= STEP_TOL, e
    assert torch.equal(last, seq[:, -1])


@pytest.mark.parametrize("layers", [1, 3])
@pytest.mark.parametrize("N,T", [(1, 1), (5, 7), (12, 160), (74, 160), (1, 1001)])
def test_hidden_against_fp64(weights, layers, N, T):
    sd = specs.synth_emotion(dict(specs.EMO, num_layers=layers), 77 + layers)
    m = _model(sd, layers)
    wav = specs.synth_emotion_wav(160 * (N + T) + 1, seed=N * 7 + T)
    mel = ref.mel(wav, torch.float32)
    frames = torch.stack([mel[n:n + T] for n in range(N)]).to(DEV)
    got = m.inference(frames)
    want = ref.hidden(sd, frames.cpu(), dict(specs.EMO, num_layers=layers), torch.float64)
    e = rel(got, want)
    assert e <= HIDDEN_TOL, e


@pytest.mark.parametrize("i", CASES)
def test_embed_utterance_against_the_reference(loaded, weights, i):
    wav = specs.synth_emotion_wav(int(GOLDEN["lengths"][i]), int(GOLDEN[f"c{i}_seed"]))
    embed, partials, slices = loaded.embed_utterance(wav, return_partials=True)
    assert embed.dtype == np.float32 and embed.shape == (256,)
    assert [[s.start, s.stop] for s in slices] == GOLDEN[f"c{i}_slices"].tolist()
    e_p, e_e = rel(partials, GOLDEN[f"c{i}_partials"]), mx(embed, GOLDEN[f"c{i}_embed"])
    assert e_p <= HIDDEN_TOL and e_e <= EMBED_TOL, (e_p, e_e)
    want = ref.embed_utterance(weights, wav, dtype=torch.float64)
    e_p, e_e = rel(partials, want["partials"]), mx(embed, want["embed"])
    assert e_p <= HIDDEN_TOL and e_e <= EMBED_TOL, (e_p, e_e)


@pytest.mark.parametrize("i", [0, 5, 6])
def test_hidden_and_forward_against_the_reference(loaded, model, i):
    wav = specs.synth_emotion_wav(int(GOLDEN["lengths"][i]), int(GOLDEN[f"c{i}_seed"]))
    slices, mel_slices = specs.emo_partials(len(wav))
    x = np.pad(wav, (0, specs.emo_padded_length(len(wav), slices) - len(wav)))
    mel = model.engine_mel(torch.from_numpy(x).to(DEV)).cpu().numpy()
    frames = np.array([mel[s] for s in mel_slices])
    e = rel(loaded.embed_frames_batch(frames), GOLDEN[f"c{i}_partials"])
    assert e <= HIDDEN_TOL, e
    e = mx(model(torch.from_numpy(frames).to(DEV)), GOLDEN[f"c{i}_forward"])
    assert e <= EMBED_TOL, e


def test_whole_utterance(loaded, weights):
    wav = specs.synth_emotion_wav(int(GOLDEN["whole_length"]), int(GOLDEN["whole_seed"]))
    embed, p, s = loaded.embed_utterance(wav, using_partials=False, return_partials=True)
    assert p is None and s is None
    e = rel(embed, GOLDEN["whole_embed"])
    assert e <= HIDDEN_TOL, e
    e = rel(embed, ref.embed_utterance(weights, wav, using_partials=False)["embed"])
    assert e <= HIDDEN_TOL, e


def test_slicer_kwargs(loaded, weights):
    wav = specs.synth_emotion_wav(70001, seed=3)
    kw = dict(partial_utterance_n_frames=101, min_pad_coverage=0.5, overlap=0.3)
    embed, partials, slices = loaded.embed_utterance(wav, return_partials=True, **kw)
    want = ref.embed_utterance(weights, wav, **kw)
    assert len(slices) == len(want["wav_slices"]) == partials.shape[0]
    assert mx(embed, want["embed"]) <= EMBED_TOL


def test_fp32_arm(loaded, weights):
    wav = specs.synth_emotion_wav(160000, seed=11)
    want = ref.embed_utterance(weights, wav, dtype=torch.float64)
    _lib.check(_lib.lib().agpt_set_tensor_cores(0))
    try:
        embed, partials, _ = loaded.embed_utterance(wav, return_partials=True)
        torch.cuda.synchronize()
    finally:
        _lib.check(_lib.lib().agpt_set_tensor_cores(1))
    e_p, e_e = rel(partials, want["partials"]), mx(embed, want["embed"])
    assert e_p <= HIDDEN_TOL and e_e <= EMBED_TOL, (e_p, e_e)


def test_batch_rows_equal_single_rows(model):
    g = torch.Generator().manual_seed(5)
    frames = (torch.rand(5, 160, 40, generator=g) * 0.05).to(DEV)
    both = model.inference(frames)
    for n in range(5):
        assert rel(both[n:n + 1], model.inference(frames[n:n + 1])) <= 1e-6


def test_rebuild_after_weight_edit(weights):
    m = _model(weights)
    wav = specs.synth_emotion_wav(40000, seed=13)
    x = torch.from_numpy(wav).to(DEV)
    m.engine_embed(x)
    sig0 = m._engine.sig
    sd = {k: v.clone() for k, v in weights.items()}
    with torch.no_grad():
        for w in (m.lstm.weight_hh_l1, sd["lstm.weight_hh_l1"]):
            w.mul_(1.5)
        for b in (m.lstm.bias_hh_l2, sd["lstm.bias_hh_l2"]):
            b[:256] += 1.0
    embed, _ = m.engine_embed(x)
    assert m._engine.sig != sig0
    assert torch.equal(embed, _model(sd).engine_embed(x)[0])     # what a model built from the edited weights gives
    assert mx(embed, ref.embed_utterance(weights, wav)["embed"]) > 100 * EMBED_TOL


def test_refused_inputs(model):
    with pytest.raises(RuntimeError, match="201"):
        model.engine_embed(torch.zeros(200, device=DEV), 0)
    with pytest.raises(RuntimeError, match="201"):
        model.engine_mel(torch.zeros(200, device=DEV))
    with pytest.raises(TypeError, match="float32"):
        model.inference(torch.zeros(1, 10, 40, device=DEV, dtype=torch.float64))
    with pytest.raises(ValueError, match="40"):
        model.inference(torch.zeros(1, 10, 41, device=DEV))
    with pytest.raises(NotImplementedError, match="hidden_init"):
        model.inference(torch.zeros(1, 10, 40, device=DEV), hidden_init=torch.zeros(3, 1, 256, device=DEV))
    with pytest.raises(RuntimeError, match="CUDA"):
        model.inference(torch.zeros(1, 10, 40))


def _reference_like_modules(monkeypatch):
    """Stand-ins for data_gen.tts.emotion.{model, inference} and inference.tts.GenerSpeech with the reference's
    structure: load_model builds whatever EmotionEncoder its module's globals hold, and the tool module binds
    embed_utterance by name."""
    names = ("data_gen", "data_gen.tts", "data_gen.tts.emotion", "data_gen.tts.emotion.model", "data_gen.tts.emotion.inference",
             "inference", "inference.tts", "inference.tts.GenerSpeech")
    mods = {n: types.ModuleType(n) for n in names}
    for n in ("data_gen", "data_gen.tts", "data_gen.tts.emotion", "inference", "inference.tts"):
        mods[n].__path__ = []
    inf = mods["data_gen.tts.emotion.inference"]

    class RefEmotionEncoder(torch.nn.Module):
        pass
    mods["data_gen.tts.emotion.model"].EmotionEncoder = RefEmotionEncoder
    src = (
        "import torch\n"
        "_model = None\n"
        "_device = None\n"
        "def load_model(weights_fpath, device=None):\n"
        "    global _model, _device\n"
        "    _device = torch.device('cuda') if device is None else torch.device(device)\n"
        "    _model = EmotionEncoder(_device, torch.device('cpu'))\n"
        "    _model.load_state_dict(torch.load(weights_fpath)['model_state'])\n"
        "    _model.eval()\n"
        "def embed_utterance(wav, using_partials=True, return_partials=False, **kwargs):\n"
        "    raise AssertionError('the reference embed_utterance ran')\n"
        "embed_frames_batch = embed_utterance\n")
    inf.EmotionEncoder = RefEmotionEncoder
    exec(src, inf.__dict__)
    tool = mods["inference.tts.GenerSpeech"]
    tool.EmotionEncoder, tool.Embed_utterance = inf, inf.embed_utterance
    for n in names:
        monkeypatch.setitem(sys.modules, n, mods[n])
    return inf, tool


def test_installed_tool_call(monkeypatch, weights, tmp_path):
    """GenerSpeech.py:37,58 after install(emotion=True): EmotionEncoder.load_model(path), then Embed_utterance(wav)"""
    import audiogpt_b200
    inf, tool = _reference_like_modules(monkeypatch)
    monkeypatch.setattr(emo_inference, "_state", emo_inference)
    patched = audiogpt_b200.install(emotion=True)
    assert "data_gen.tts.emotion.inference" in patched
    path = tmp_path / "encoder.pt"
    torch.save({"model_state": weights, "step": 1}, path)
    tool.EmotionEncoder.load_model(path)
    assert isinstance(inf._model, EmotionEncoder)
    i = 5
    wav = specs.synth_emotion_wav(int(GOLDEN["lengths"][i]), int(GOLDEN[f"c{i}_seed"]))
    embed = tool.Embed_utterance(wav)
    assert mx(embed, GOLDEN[f"c{i}_embed"]) <= EMBED_TOL
