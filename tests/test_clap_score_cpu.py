"""CPU checks of the CLAP candidate scorer (wav_evaluation CLAPWrapper, T2A.select_best_audio): the oracle against the
reference's own CLAPWrapper (tests/golden/clap_score.npz, make_golden_clap_score.py), the restated resampling filter,
the conv-STFT, the checkpoint layout, the checkpoint-key filter of the drop-in and install(scorer=True)."""
import math
import os
import random
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audiogpt_b200 import specs  # noqa: E402
from oracle import clap_score_ref as ref  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "clap_score.npz")
CFG = specs.CLAP_SCORER_SMALL


def _rel_rmse(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt()).item()


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope="module")
def sd(golden):
    return specs.synth_clap_scorer(CFG, int(golden["weight_seed"]))


def golden_clips(g):
    return [torch.from_numpy(x) for x in specs.synth_scorer_clips(tuple(g["clip_lens"]), int(g["sr"]), int(g["clip_seed"]))]


def test_regenerated_clips_match_the_fixture(golden):
    for x, want in zip(golden_clips(golden), golden["clip_stats"]):
        xd = x.double()
        got = np.array([xd.sum().item(), xd.abs().sum().item(), (xd * xd).sum().item()])
        assert np.allclose(got, want, rtol=1e-9, atol=1e-6)


def test_oracle_matches_reference_fixture(golden, sd):
    rng = random.Random(int(golden["py_seed"]))
    sr = int(golden["sr"])
    clips, starts = [], []
    for x in golden_clips(golden):
        c, s = ref.prepare_clip(x, sr, CFG, rng)
        clips.append(c)
        if s is not None:
            starts.append(s)
    assert starts == golden["crop_starts"].tolist()
    assert all(c.shape[0] == int(CFG["duration"]) * sr for c in clips)
    with torch.no_grad():
        a = ref.audio_embeddings(sd, CFG, torch.stack(clips))
        t = ref.text_embeddings(sd, CFG, torch.from_numpy(golden["ids"][:1]), torch.from_numpy(golden["type_ids"][:1]),
                                torch.from_numpy(golden["mask"][:1]))
        tl = ref.text_embeddings(sd, CFG, torch.from_numpy(golden["long_ids"]), torch.from_numpy(golden["long_type_ids"]),
                                 torch.from_numpy(golden["long_mask"]))
        tp = ref.text_embeddings(sd, CFG, torch.from_numpy(golden["ids"]), torch.from_numpy(golden["type_ids"]),
                                 torch.from_numpy(golden["mask"]))
    assert _rel_rmse(a, golden["audio_emb"]) <= 1e-5
    assert _rel_rmse(t, golden["text_emb"]) <= 1e-5
    assert _rel_rmse(tl, golden["text_emb_long"]) <= 1e-5
    assert _rel_rmse(tp, golden["text_emb_pair"]) <= 1e-5
    s = ref.similarity(a, t)[:, 0]
    assert _rel_rmse(s, golden["scores"]) <= 1e-5
    assert int(s.argmax()) == int(golden["best"])


def test_specs_layout_matches_reference_keys(golden):
    shapes = specs.clap_scorer_param_shapes(CFG)
    assert list(shapes) == golden["ref_keys"].tolist()
    assert [",".join(str(v) for v in s) for s in shapes.values()] == golden["ref_shapes"].tolist()
    full = specs.clap_scorer_param_shapes(specs.CLAP_SCORER)
    conv = sum(math.prod(s) for k, s in full.items() if ".conv_block" in k and k.endswith("conv1.weight") or k.endswith("conv2.weight"))
    assert abs(conv / 1e6 - 75.5) < 0.1
    assert math.prod(full["audio_encoder.base.fc1.weight"]) == 2048 * 2048


def test_resample_kernel_matches_torchaudio():
    ta = pytest.importorskip("torchaudio")
    g = torch.Generator().manual_seed(3)
    for L in (159744, 40000, 1001):
        x = torch.randn(L, generator=g) * 0.3
        want = ta.transforms.Resample(16000, 44100)(x)
        got = ref.resample(x, 16000, 44100)
        assert got.shape == want.shape == (math.ceil(441 * L / 160),)
        assert _rel_rmse(got, want) <= 1e-6
    k, width, o, n = specs.sinc_resample_kernel(16000, 44100)
    assert (k.shape, width, o, n) == ((441, 174), 7, 160, 441)


def test_conv_stft_power_equals_torch_stft():
    re, im = specs.stft_dft_weights(1024)
    x = torch.randn(2, 144000, generator=torch.Generator().manual_seed(4)).double() * 0.2
    xp = torch.nn.functional.pad(x[:, None], (512, 512), mode="reflect")
    p = (torch.nn.functional.conv1d(xp, re.double(), stride=320) ** 2 +
         torch.nn.functional.conv1d(xp, im.double(), stride=320) ** 2)
    S = torch.stft(x, 1024, hop_length=320, window=torch.hann_window(1024, dtype=torch.float64), center=True,
                   pad_mode="reflect", return_complex=True)
    assert p.shape == S.shape == (2, 513, 451)
    assert _rel_rmse(p, S.abs() ** 2) <= 1e-6


def test_slaney_mel_shape_and_normalisation():
    m = specs.slaney_mel(44100, 1024, 64, 50, 14000)
    assert m.shape == (64, 513) and (m >= 0).all()
    f = np.fft.rfftfreq(1024, 1 / 44100)
    assert (m[:, f > 14000] == 0).all() and (m[:, f < 50] == 0).all()
    # Slaney area normalisation: each triangle integrates (in Hz) to 1
    area = m.sum(axis=1) * (44100 / 1024)
    assert abs(np.median(area) - 1.0) < 0.02   # (per triangle only approximately: the low ones span a few FFT bins)


def test_checkpoint_key_filter_accepts_2022_checkpoint():
    from audiogpt_b200.wav_evaluation.models.CLAPWrapper import engine_weights
    sd = specs.synth_clap_scorer(CFG, 1)
    sd["caption_encoder.base.embeddings.position_ids"] = torch.arange(CFG["bert"]["max_position_embeddings"])[None]
    audio, text = engine_weights(sd, CFG)
    assert len(audio) == len(specs.cnn14_engine_keys(CFG))
    assert len(text) == len(specs.clap_param_shapes(specs.clap_scorer_bert_cfg(CFG)))
    del sd["audio_encoder.base.fc1.bias"]
    with pytest.raises(KeyError, match="fc1.bias"):
        engine_weights(sd, CFG)


def test_read_config_as_args_matches_reference_yaml(golden):
    from audiogpt_b200.wav_evaluation.models.CLAPWrapper import read_config_as_args
    args = read_config_as_args(str(golden["config_yml"]), is_config_str=True)
    assert args.text_len == 100 and args.duration == 9 and args.sampling_rate == 44100
    assert args.transformer_embed_dim == CFG["transformer_embed_dim"] and args.d_proj == 1024


def test_install_scorer_aliases_wav_evaluation():
    import importlib

    import audiogpt_b200
    saved = {k: sys.modules.get(k) for k in ("wav_evaluation.models.CLAPWrapper",)}
    try:
        patched = audiogpt_b200.install(scorer=True)
        assert "wav_evaluation.models.CLAPWrapper (aliased)" in patched
        mod = importlib.import_module("wav_evaluation.models.CLAPWrapper")
        from audiogpt_b200.wav_evaluation.models.CLAPWrapper import CLAPWrapper
        assert mod.CLAPWrapper is CLAPWrapper
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def test_constructor_refuses_cpu(tmp_path, golden):
    from audiogpt_b200.wav_evaluation.models.CLAPWrapper import CLAPWrapper
    cfg = tmp_path / "config.yml"
    cfg.write_text(str(golden["config_yml"]))
    with pytest.raises(RuntimeError, match="CUDA"):
        CLAPWrapper(str(tmp_path / "missing.pth"), str(cfg), use_cuda=False)
