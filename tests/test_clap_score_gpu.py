"""GPU tests of the CLAP candidate scorer (audiogpt_b200.wav_evaluation.models.CLAPWrapper on csrc/clap_score.cu and
csrc/clap.cu's masked [CLS] path) against the reference's own CLAPWrapper (tests/golden/clap_score.npz, weights
specs.synth_clap_scorer(CLAP_SCORER_SMALL): Cnn14 at full size, a CLAP_SMALL-sized BERT) and the CPU oracle.

Gates (set from the first measured run on an NVIDIA H100 80GB HBM3, 400 W power limit):
- audio embeddings rel-RMSE <= 1e-4: measured 2.4e-5 on the tensor cores (error-compensated fp16 parts, fp32
  accumulation, through the DFT, 12 convs and the log), 1.3e-6 on the fp32-FMA path;
- text embeddings rel-RMSE <= 2e-5: measured 2.0e-6 to 2.1e-6 (fp32-FMA 4.6e-7);
- scores abs <= 1e-5: measured 8.3e-7 (the score margin of the fixture is 2.95e-3);
- identical argmax and crop windows; B = 3 against one clip at a time: measured bit-identical, gate 1e-5.
"""
import os
import random
import sys
from unittest import mock

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audiogpt_b200 import _lib, specs  # noqa: E402
from oracle import clap_score_ref as ref  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(ROOT, "tests", "golden", "clap_score.npz")
CFG = specs.CLAP_SCORER_SMALL


def _rel_rmse(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt()).item()


def bert_config():
    import transformers
    b = CFG["bert"]
    return transformers.BertConfig(vocab_size=b["vocab_size"], hidden_size=b["hidden_size"], num_hidden_layers=b["num_layers"],
                                   num_attention_heads=b["num_heads"], intermediate_size=b["intermediate_size"],
                                   max_position_embeddings=b["max_position_embeddings"], type_vocab_size=b["type_vocab_size"],
                                   layer_norm_eps=b["layer_norm_eps"])


def hub_stubs(tokenizer):
    """The two from_pretrained calls of the constructor, answered without the hub."""
    return mock.patch("transformers.AutoTokenizer.from_pretrained", lambda name: tokenizer), \
        mock.patch("transformers.AutoConfig.from_pretrained", lambda name: bert_config())


class FixtureTokenizer:
    """encode_plus from the fixture's rows (the stub tokenizer make_golden_clap_score.py gave the reference)."""

    def __init__(self, g):
        t = g["texts"].tolist()
        self.rows = {t[0]: (g["ids"][0], g["type_ids"][0], g["mask"][0]),
                     t[1]: (g["long_ids"][0], g["long_type_ids"][0], g["long_mask"][0]),
                     t[2]: (g["ids"][1], g["type_ids"][1], g["mask"][1])}

    def encode_plus(self, text, add_special_tokens=True, max_length=100, padding="max_length", return_tensors="pt"):
        i, ty, m = (torch.from_numpy(np.asarray(v)).long()[None] for v in self.rows[text])
        return {"input_ids": i, "token_type_ids": ty, "attention_mask": m}


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope="module")
def sd(golden):
    return specs.synth_clap_scorer(CFG, int(golden["weight_seed"]))


@pytest.fixture(scope="module")
def scorer(golden, sd):
    from audiogpt_b200.wav_evaluation.models.CLAPWrapper import CLAPWrapper
    return CLAPWrapper.from_config(CFG, sd, tokenizer=FixtureTokenizer(golden))


@pytest.fixture(scope="module")
def ckpt(tmp_path_factory, golden, sd):
    d = tmp_path_factory.mktemp("clap_ckpt")
    sd_2022 = dict(sd)
    sd_2022["caption_encoder.base.embeddings.position_ids"] = torch.arange(CFG["bert"]["max_position_embeddings"])[None]
    torch.save({"model": sd_2022}, d / "CLAP_weights_2022.pth")
    (d / "config.yml").write_text(str(golden["config_yml"]))
    return d


def golden_clips(g):
    """The fixture's clips, regenerated from their seed (tests/test_clap_score_cpu.py checks them against the
    fixture's per-clip sums)."""
    return specs.synth_scorer_clips(tuple(g["clip_lens"]), int(g["sr"]), int(g["clip_seed"]))


def select_best_audio(CLAPWrapper, ckpt, prompt, wav_list, tokenizer):
    """T2A.select_best_audio (audio-chatgpt.py:185-199) with the checkpoint paths of the test."""
    p1, p2 = hub_stubs(tokenizer)
    with p1, p2:
        clap_model = CLAPWrapper(str(ckpt / "CLAP_weights_2022.pth"), str(ckpt / "config.yml"),
                                 use_cuda=torch.cuda.is_available())
    text_embeddings = clap_model.get_text_embeddings([prompt])
    score_list, audio = [], []
    for sr, wav in wav_list:
        audio_embeddings = clap_model.get_audio_embeddings([(torch.FloatTensor(wav), sr)], resample=True)
        audio.append(audio_embeddings[0])
        score = clap_model.compute_similarity(audio_embeddings, text_embeddings, use_logit_scale=False).squeeze().cpu().numpy()
        score_list.append(score)
    max_index = np.array(score_list).argmax()
    return clap_model, text_embeddings, torch.stack(audio), np.array(score_list), int(max_index)


def test_select_best_audio_through_installed_dropin(golden, ckpt):
    import audiogpt_b200
    audiogpt_b200.install(scorer=True)
    from wav_evaluation.models.CLAPWrapper import CLAPWrapper
    sr = int(golden["sr"])
    starts = []
    orig = random.randrange

    def rec(*a):
        starts.append(orig(*a))
        return starts[-1]

    # the fixture seeded Python's random after the reference's constructor had run (torch.load and the transformers
    # imports of a first construction may draw from it); the constructor inside select_best_audio is then a cache hit
    p1, p2 = hub_stubs(FixtureTokenizer(golden))
    with p1, p2:
        CLAPWrapper(str(ckpt / "CLAP_weights_2022.pth"), str(ckpt / "config.yml"), use_cuda=True)
    random.seed(int(golden["py_seed"]))
    with mock.patch.object(random, "randrange", rec):
        _, t, a, scores, best = select_best_audio(CLAPWrapper, ckpt, str(golden["texts"][0]),
                                                  [(sr, w) for w in golden_clips(golden)], FixtureTokenizer(golden))
    ea, et = _rel_rmse(a, golden["audio_emb"]), _rel_rmse(t, golden["text_emb"])
    es = float(np.abs(scores - golden["scores"]).max())
    print(f"\nclap_score: select_best_audio audio rel-RMSE {ea:.2e}, text {et:.2e}, scores max abs {es:.2e}, "
          f"best {best}, starts {starts}")
    assert starts == golden["crop_starts"].tolist()
    assert ea <= 1e-4 and et <= 2e-5 and es <= 1e-5
    assert best == int(golden["best"])


def test_engine_cache_reuses_and_rebuilds(golden, ckpt):
    from audiogpt_b200.wav_evaluation.models import CLAPWrapper as W
    p1, p2 = hub_stubs(FixtureTokenizer(golden))
    with p1, p2:
        a = W.CLAPWrapper(str(ckpt / "CLAP_weights_2022.pth"), str(ckpt / "config.yml"), use_cuda=True)
        b = W.CLAPWrapper(str(ckpt / "CLAP_weights_2022.pth"), str(ckpt / "config.yml"), use_cuda=True)
        assert a.clap is b.clap and len(W._CACHE) == 1
        p = ckpt / "CLAP_weights_2022.pth"
        st = os.stat(p)
        os.utime(p, ns=(st.st_atime_ns, st.st_mtime_ns + 1_000_000_000))
        c = W.CLAPWrapper(str(p), str(ckpt / "config.yml"), use_cuda=True)
        assert c.clap is not a.clap and len(W._CACHE) == 1
    t = c.get_text_embeddings([str(golden["texts"][0])])
    assert _rel_rmse(t, golden["text_emb"]) <= 2e-5


def test_masked_text_fixture_rows_and_oracle(golden, sd, scorer):
    t_long = scorer.get_text_embeddings([str(golden["texts"][1])])
    t_pair = scorer.get_text_embeddings([str(golden["texts"][0]), str(golden["texts"][2])])
    assert golden["long_ids"].shape[1] > 100 and golden["ids"].shape[1] == 100
    e1, e2 = _rel_rmse(t_long, golden["text_emb_long"]), _rel_rmse(t_pair, golden["text_emb_pair"])
    # token types 1 and padding inside the row: only the oracle covers them
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(0, CFG["bert"]["vocab_size"], (3, 100), generator=g)
    ty = torch.randint(0, 2, (3, 100), generator=g)
    mask = (torch.rand(3, 100, generator=g) > 0.4).long()
    mask[:, 0] = 1
    want = ref.text_embeddings(sd, CFG, ids, ty, mask)
    got = scorer.encode_text_ids(ids.cuda(), ty.cuda(), mask.cuda())
    e3 = _rel_rmse(got, want)
    print(f"\nclap_score: text long {e1:.2e}, pair {e2:.2e}, typed + holed mask vs oracle {e3:.2e}")
    assert e1 <= 2e-5 and e2 <= 2e-5 and e3 <= 2e-5


def test_batch_of_three_equals_one_by_one(golden, scorer):
    rng = random.Random(7)
    c = golden_clips(golden)
    clips = [torch.from_numpy(c[0]), torch.from_numpy(c[2]), torch.from_numpy(c[0] * 0.5)]
    scorer.clap.set_rate(16000, True)
    R = scorer.clap.resampled_len(159744)
    starts = [rng.randrange(R - scorer.clap.clip) for _ in clips]
    batch = scorer.embed_audio(torch.stack(clips).cuda(), 16000, starts)
    one = torch.cat([scorer.embed_audio(c[None].cuda(), 16000, [s]) for c, s in zip(clips, starts)])
    e = _rel_rmse(batch, one)
    print(f"\nclap_score: B=3 vs B=1 rel-RMSE {e:.2e}")
    assert e <= 1e-5


def test_fp32_fma_path(golden, scorer):
    sr = int(golden["sr"])
    clips = golden_clips(golden)
    starts = golden["crop_starts"].tolist()
    st = [starts[0], -1, starts[1]]   # clips 0 and 2 are cropped, clip 1 (40000 samples) is tiled
    lib = _lib.lib()
    _lib.check(lib.agpt_set_tensor_cores(0))
    try:
        a = torch.cat([scorer.embed_audio(torch.from_numpy(c)[None].cuda(), sr, [s]) for c, s in zip(clips, st)])
        t = scorer.get_text_embeddings([str(golden["texts"][0])])
    finally:
        _lib.check(lib.agpt_set_tensor_cores(1))
    ea, et = _rel_rmse(a, golden["audio_emb"]), _rel_rmse(t, golden["text_emb"])
    print(f"\nclap_score: fp32-FMA audio {ea:.2e}, text {et:.2e}")
    assert ea <= 1e-5 and et <= 2e-5
    s = scorer.compute_similarity(a, t, use_logit_scale=False)[:, 0].cpu().numpy()
    assert np.abs(s - golden["scores"]).max() <= 1e-5 and int(s.argmax()) == int(golden["best"])


def test_logit_scale_similarity(golden, scorer):
    a = torch.from_numpy(golden["audio_emb"]).cuda()
    t = torch.from_numpy(golden["text_emb_pair"]).cuda()
    got = scorer.compute_similarity(a, t)
    want = float(np.exp(np.log(1 / 0.07))) * (t.double() @ a.double().T).T
    assert got.shape == (3, 2) and torch.allclose(got.double(), want, rtol=1e-5, atol=1e-6)


def test_errors(golden, ckpt, scorer):
    from audiogpt_b200.wav_evaluation.models.CLAPWrapper import CLAPWrapper
    with pytest.raises(RuntimeError, match="CUDA"):
        CLAPWrapper(str(ckpt / "CLAP_weights_2022.pth"), str(ckpt / "config.yml"), use_cuda=False)
    with pytest.raises(RuntimeError, match="CUDA"):
        scorer.encode_text_ids(torch.zeros(1, 10, dtype=torch.long))
    with pytest.raises(RuntimeError, match="CUDA"):
        scorer.embed_audio(torch.zeros(1, 16000), 16000, [-1])
    with pytest.raises(ValueError, match="token ids"):
        scorer.encode_text_ids(torch.full((1, 10), CFG["bert"]["vocab_size"], device="cuda"))
    with pytest.raises(ValueError, match="token type ids"):
        scorer.encode_text_ids(torch.zeros(1, 10, dtype=torch.long, device="cuda"),
                               torch.full((1, 10), 2, dtype=torch.long, device="cuda"))
    with pytest.raises(ValueError, match="max_position_embeddings"):
        scorer.encode_text_ids(torch.zeros(1, CFG["bert"]["max_position_embeddings"] + 1, dtype=torch.long, device="cuda"))
    with pytest.raises(RuntimeError, match="crop start"):        # a cropped clip needs a start inside the window
        scorer.embed_audio(torch.zeros(1, 159744, device="cuda"), 16000, [-1])
    with pytest.raises(RuntimeError, match="tiled"):             # a tiled clip takes -1
        scorer.embed_audio(torch.zeros(1, 16000, device="cuda"), 16000, [0])
    with pytest.raises(ValueError, match="mono"):
        scorer.get_audio_embeddings([(torch.zeros(2, 16000), 16000)], resample=True)
