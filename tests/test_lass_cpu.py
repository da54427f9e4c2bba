"""CPU checks of the sound-extraction tool (LASSNet, STFT): the oracle against the reference's own modules
(tests/golden/lass_small.npz and lass_shipped.npz, made by make_golden_lass.py), the STFT buffers and window sum, the
state-dict layout, strict loading, hub-free construction, install(extraction=True) and the C ABI symbols."""
import ctypes
import os
import subprocess
import sys
from unittest import mock

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audiogpt_b200 import specs  # noqa: E402
from oracle import lass_ref as ref  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def _rel_rmse(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt()).item()


@pytest.fixture(scope="module")
def small():
    return dict(np.load(os.path.join(GOLDEN, "lass_small.npz")))


@pytest.fixture(scope="module")
def shipped():
    return dict(np.load(os.path.join(GOLDEN, "lass_shipped.npz")))


def _small_wav(g):
    n, s = int(g["n"]), int(g["seed_wav"])
    return torch.stack([specs.synth_lass_wav(n, s), specs.synth_lass_wav(n, s + 1)])


def test_oracle_matches_reference_small(small):
    """STFT, text condition, logits, mask and the whole tool chain of the oracle against the reference modules at
    n_fft 256, B = 2, T = 91, captions of 9 and 5 tokens (both fp32 on the CPU: rel-RMSE <= 1e-5)."""
    g = small
    sd = specs.synth_lass(specs.LASS_SMALL, int(g["seed_w"]))
    n_fft = int(g["n_fft"])
    fb, ib = specs.stft_bases(n_fft, n_fft // 2)
    wav = _small_wav(g)
    mag, phase = ref.stft_transform(wav, fb, n_fft // 2)
    assert _rel_rmse(mag, g["mag"]) < 1e-6
    assert _rel_rmse(mag * torch.cos(phase), g["mag"] * np.cos(g["phase"])) < 1e-5
    ids, msk = torch.from_numpy(g["ids"]), torch.from_numpy(g["mask"])
    mask, logits, cond = ref.lass_forward(sd, specs.LASS_SMALL, mag.transpose(2, 1).unsqueeze(1), ids, msk)
    assert _rel_rmse(cond, g["cond"]) < 1e-5
    assert _rel_rmse(logits, g["logits"]) < 1e-5
    assert _rel_rmse(mask, g["mask_out"]) < 1e-5
    assert torch.all(mask[..., -2:] == 0.5)
    est = (mask * mag.transpose(2, 1).unsqueeze(1)).squeeze(1).permute(0, 2, 1)
    out = ref.stft_inverse(est, phase, ib, n_fft // 2)
    assert out.shape == g["wav_out"].shape
    assert _rel_rmse(out, g["wav_out"]) < 1e-5


def test_oracle_matches_reference_shipped(shipped):
    """The tool's shape (one 10 s 32 kHz clip: T = 626, F = 513) against the reference's cond, per-frame sums and
    strided samples."""
    g = shipped
    sd = specs.synth_lass(specs.LASS, int(g["seed_w"]))
    fb, ib = specs.stft_bases()
    wav = specs.synth_lass_wav(int(g["n"]), int(g["seed_wav"]))[None]
    s = int(g["sample_stride"])
    ids, msk = torch.from_numpy(g["ids"]), torch.from_numpy(g["mask"])
    mag, phase = ref.stft_transform(wav, fb, specs.LASS_HOP)
    assert _rel_rmse(mag.reshape(-1)[::s], g["mag_sample"]) < 1e-6
    with torch.no_grad():
        mask, logits, cond = ref.lass_forward(sd, specs.LASS, mag.transpose(2, 1).unsqueeze(0), ids, msk)
    assert mask.shape == (1, 1, 626, 513)
    assert _rel_rmse(cond, g["cond"]) < 1e-5
    assert _rel_rmse(logits.double().sum(-1).reshape(-1), g["logits_rows"]) < 1e-5
    assert _rel_rmse(mask.double().sum(-1).reshape(-1), g["mask_rows"]) < 1e-6
    assert _rel_rmse(logits.reshape(-1)[::s], g["logits_sample"]) < 1e-5


def test_stft_buffers_and_window_sum(small, shipped):
    """specs.stft_bases / stft_window_sum reproduce the reference STFT's buffers and window_sumsquare."""
    fb, ib = specs.stft_bases()
    g, s = shipped, int(shipped["sample_stride"])
    assert fb.shape == ib.shape == (1026, 1, 1024)
    np.testing.assert_array_equal(fb.reshape(-1)[::s].numpy(), g["fwd_sample"])
    np.testing.assert_allclose(ib.reshape(-1)[::s].numpy(), g["inv_sample"], rtol=1e-5, atol=1e-9)
    np.testing.assert_allclose([fb.double().sum().item(), fb.double().abs().sum().item()], g["fwd_sum"], rtol=1e-7)
    np.testing.assert_allclose([ib.double().sum().item(), ib.double().abs().sum().item()], g["inv_sum"], rtol=1e-5)
    np.testing.assert_array_equal(specs.stft_window_sum(626)[::s], g["ws_sample"])
    np.testing.assert_array_equal(specs.stft_window_sum(small["mag"].shape[-1], 256, 128), small["ws"])


def test_param_shapes_match_reference_key_order(small):
    assert list(specs.lass_param_shapes(specs.LASS_SMALL)) == list(small["keys"])
    shapes = specs.lass_param_shapes(specs.LASS)
    n_unet = sum(int(np.prod(v)) for k, v in shapes.items() if k.startswith("UNet.") and "running" not in k
                 and not k.endswith("num_batches_tracked"))
    assert n_unet == 52_228_323   # UNetRes_FiLM(1, 256)'s parameters (52.23 M)
    assert sum(1 for k in shapes if k.endswith(".linear.2.weight")) == 63
    assert len(specs.lass_blocks()) == 26


def test_strict_load_ignores_position_ids():
    from audiogpt_b200.sound_extraction.model.LASSNet import LASSNet
    m = LASSNet.from_config(specs.LASS_SMALL)
    sd = specs.synth_lass(specs.LASS_SMALL, 3)
    sd["text_embedder.bert_layer.embeddings.position_ids"] = torch.arange(64)[None]
    m.load_state_dict(sd, strict=True)
    k = "UNet.decoder_block3.conv_block2.bn1.running_var"
    assert torch.equal(m.state_dict()[k], sd[k])
    assert list(m.state_dict()) == list(specs.lass_param_shapes(specs.LASS_SMALL))
    dp = torch.nn.DataParallel(LASSNet.from_config(specs.LASS_SMALL))
    dp.load_state_dict({"module." + k: v for k, v in sd.items()}, strict=True)
    del sd["UNet.after_conv2.bias"]
    with pytest.raises(RuntimeError, match="after_conv2.bias"):
        m.load_state_dict(sd, strict=True)


def test_from_config_needs_no_hub():
    from transformers import BertModel, BertTokenizer

    from audiogpt_b200.sound_extraction.model.LASSNet import LASSNet

    def boom(*a, **k):
        raise AssertionError("from_pretrained called")

    with mock.patch.object(BertModel, "from_pretrained", boom), mock.patch.object(BertTokenizer, "from_pretrained", boom):
        m = LASSNet.from_config(specs.LASS)
    assert m.get_tokenizer() is None
    assert m.state_dict()["text_embedder.bert_layer.embeddings.word_embeddings.weight"].shape == (30522, 256)


def test_unsupported_stft_geometry_raises():
    from audiogpt_b200.sound_extraction.utils.stft import STFT
    with pytest.raises(NotImplementedError):
        STFT(filter_length=1024, hop_length=256)
    s = STFT()
    fb, ib = specs.stft_bases()
    assert torch.equal(s.forward_basis, fb) and torch.equal(s.inverse_basis, ib)


def _run(code):
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=240)
    assert r.returncode == 0, r.stderr
    return r.stdout.strip()


def test_install_extraction_grafts_lassnet_and_stft(tmp_path):
    """install(extraction=True) replaces LASSNet and STFT inside the reference's modules (where SoundExtraction imports
    them from); the default install() leaves them alone."""
    for sub, src in (("model", "LASSNet.py"), ("utils", "stft.py")):
        d = tmp_path / "sound_extraction" / sub
        d.mkdir(parents=True, exist_ok=True)
        (d / "__init__.py").write_text("")
        (d / src).write_text("class LASSNet:\n    pass\nclass STFT:\n    pass\n")
    (tmp_path / "sound_extraction" / "__init__.py").write_text("")
    head = "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import audiogpt_b200 as a; " % (str(tmp_path), ROOT)
    check = ("from sound_extraction.model.LASSNet import LASSNet as L; from sound_extraction.utils.stft import STFT as S; "
             "print(L.__module__, S.__module__)")
    assert _run(head + "a.install(); " + check) == "sound_extraction.model.LASSNet sound_extraction.utils.stft"
    assert _run(head + "a.install(extraction=True); " + check) == \
        "audiogpt_b200.sound_extraction.model.LASSNet audiogpt_b200.sound_extraction.utils.stft"


def test_abi_symbols_exist():
    from audiogpt_b200 import _lib
    L = _lib.lib()
    for name in ("agpt_lass_create", "agpt_lass_text", "agpt_lass_mask", "agpt_stft_create", "agpt_stft_transform",
                 "agpt_stft_inverse"):
        assert isinstance(getattr(L, name), ctypes._CFuncPtr)
        assert name in _lib.PROTOTYPES
    assert ctypes.sizeof(_lib.LassConfig) == 8 * 4
