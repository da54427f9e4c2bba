"""CPU checks of the sound-event-detection PVT (audio_infer.pytorch.models.PVT, the SoundDetection tool): the oracle
against the reference's own PVT (tests/golden/pvt_small.npz, pvt_shipped.npz, make_golden_pvt.py), the state-dict
layout, the stage-grid arithmetic, install(detection=True) and the C ABI's declarations."""
import ctypes as C
import importlib
import os
import re
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audiogpt_b200 import specs  # noqa: E402
from oracle import pvt_ref as ref  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def _rel_rmse(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt()).item()


def _stats(x):
    x = x.double()
    return np.array([x.sum().item(), x.abs().sum().item(), (x * x).sum().item()])


@pytest.fixture(scope="module")
def small():
    return dict(np.load(os.path.join(GOLDEN, "pvt_small.npz")))


@pytest.fixture(scope="module")
def shipped():
    return dict(np.load(os.path.join(GOLDEN, "pvt_shipped.npz")))


def test_oracle_matches_reference_small(small):
    cfg = specs.PVT_SMALL
    sd = specs.synth_pvt(cfg, int(small["weight_seed"]))
    for k, n in enumerate(small["clip_lens"].tolist()):
        wav = specs.synth_pvt_wav(n, int(small["clip_seed"]) + k)
        assert np.allclose(_stats(wav), small[f"clip_stats{k}"], rtol=1e-9, atol=1e-6)
        with torch.no_grad():
            out = ref.forward(sd, cfg, wav[None])
        assert out["framewise_output"].shape == small[f"framewise{k}"].shape
        assert _rel_rmse(out["logits"], small[f"logits{k}"]) <= 1e-5
        assert np.abs(out["framewise_output"].numpy() - small[f"framewise{k}"]).max() <= 2e-6
        assert np.abs(out["clipwise_output"].numpy() - small[f"clipwise{k}"]).max() <= 2e-6
        if k == 0:
            for i, st in enumerate(out["stages"]):
                assert _rel_rmse(st.flatten(2).transpose(1, 2), small[f"stage{i + 1}"]) <= 1e-5


def test_oracle_matches_reference_shipped(shipped):
    cfg = specs.PVT_SHIPPED
    sd = specs.synth_pvt(cfg, int(shipped["weight_seed"]))
    wav = specs.synth_pvt_wav(int(shipped["clip_len"]), int(shipped["clip_seed"]))
    assert np.allclose(_stats(wav), shipped["clip_stats"], rtol=1e-9, atol=1e-6)
    with torch.no_grad():
        out = ref.forward(sd, cfg, wav[None])
    frame = out["framewise_output"]
    assert list(frame.shape) == shipped["framewise_shape"].tolist() == [1, 1024, 527]
    assert _rel_rmse(out["logits"], shipped["logits"]) <= 1e-5
    assert np.abs(frame[:, ::int(shipped["row_step"])].numpy() - shipped["framewise_rows"]).max() <= 2e-6
    assert np.abs(out["clipwise_output"].numpy() - shipped["clipwise"]).max() <= 2e-6
    top = np.argsort(np.max(frame[0].numpy(), axis=0))[::-1][:10]
    assert top.tolist() == shipped["top10"].tolist()


@pytest.mark.parametrize("name,cfg", [("small", specs.PVT_SMALL), ("shipped", specs.PVT_SHIPPED)])
def test_specs_layout_matches_reference_keys(name, cfg, small, shipped):
    g = small if name == "small" else shipped
    shapes = specs.pvt_param_shapes(cfg)
    assert list(shapes) == g["ref_keys"].tolist()
    assert [",".join(str(v) for v in s) for s in shapes.values()] == g["ref_shapes"].tolist()
    assert len(specs.pvt_engine_keys(cfg)) == len(shapes) - 1
    sd = specs.synth_pvt(cfg, 1)
    # nothing the reference initialises to a constant is left at it
    for k, v in sd.items():
        if v.is_floating_point():
            assert v.std() > 0, k


def test_grid_arithmetic_matches_the_convs():
    """pvt_grids (the twin of agpt_pvt_frames) against the shapes the oracle's convs actually produce"""
    cfg = specs.PVT_SMALL
    sd = specs.synth_pvt(cfg, 2)
    lo = specs.pvt_min_samples(cfg)
    for n in [lo, lo + 1, 3000, 4321, 5040, 8250, 9999, 16000]:
        with torch.no_grad():
            stages = ref.features(sd, cfg, ref.logmel(sd, cfg, torch.zeros(1, n)))
        assert [tuple(s.shape[2:]) for s in stages] == specs.pvt_grids(cfg, n), n
        # Attention.sr's output grid: the rows and columns that do not fill a patch are dropped
        for (H, W), sr in zip(specs.pvt_grids(cfg, n), cfg["sr_ratios"]):
            assert F.conv2d(torch.zeros(1, 1, H, W), torch.zeros(1, 1, sr, sr), stride=sr).shape[2:] == (H // sr, W // sr)
    with pytest.raises(ValueError, match="too short"):
        specs.pvt_grids(cfg, lo - 1)
    assert specs.pvt_min_samples(specs.PVT_SHIPPED) == 9600
    assert specs.pvt_grids(specs.PVT_SHIPPED, 320000) == [(250, 16), (125, 8), (63, 4), (32, 2)]
    assert specs.pvt_grids(specs.PVT_SHIPPED, 60 * 32000)[-1] == (188, 2)
    with pytest.raises(ValueError):
        specs.pvt_grids(specs.PVT_SHIPPED, 512)


def test_abi_frames_matches_python_twin():
    from audiogpt_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libagpt_b200.so is not built")
    from audiogpt_b200.audio_detection.audio_infer.pytorch.models import PVT
    L = _lib.lib()
    for cfg in (specs.PVT_SMALL, specs.PVT_SHIPPED):
        cc = PVT.from_config(cfg)._config()
        lo = specs.pvt_min_samples(cfg)
        for n in (lo, lo + 7, lo + 2640, 3 * lo + 1050, 320000, 320001, 1920000):
            g = ((C.c_int * 2) * 4)()
            assert L.agpt_pvt_frames(C.byref(cc), n, g) == 0, L.agpt_last_error()
            assert [tuple(r) for r in g] == specs.pvt_grids(cfg, n)
        assert L.agpt_pvt_frames(C.byref(cc), lo - 1, ((C.c_int * 2) * 4)()) != 0
        assert b"too short" in L.agpt_last_error()


def test_dropin_state_dict_and_cpu_refusal():
    from audiogpt_b200.audio_detection.audio_infer.pytorch.models import PVT
    m = PVT(sample_rate=32000, window_size=1024, hop_size=320, mel_bins=64, fmin=50, fmax=14000, classes_num=527)
    sd = specs.synth_pvt(specs.PVT_SHIPPED, 5)
    assert list(m.state_dict()) == list(sd)
    # the constructor fills the frozen front end the way torchlibrosa does
    assert torch.equal(m.state_dict()["logmel_extractor.melW"], sd["logmel_extractor.melW"])
    assert torch.equal(m.state_dict()["spectrogram_extractor.stft.conv_imag.weight"], sd["spectrogram_extractor.stft.conv_imag.weight"])
    res = m.load_state_dict({"model": sd}["model"])
    assert not res.missing_keys and not res.unexpected_keys
    assert m.bn0.num_batches_tracked.dtype == torch.long
    with pytest.raises(RuntimeError, match="eval"):
        m(torch.zeros(1, 32000))
    with pytest.raises(RuntimeError, match="CUDA"):
        m.eval()(torch.zeros(1, 32000))
    bad = dict(sd)
    del bad["pvt_transformer.block1.0.attn.sr.weight"]
    with pytest.raises(RuntimeError, match="attn.sr.weight"):
        m.load_state_dict(bad)
    with pytest.raises(ValueError, match="64"):
        PVT(32000, 1024, 320, 128, 50, 14000, 527)


def test_install_detection_aliases_only_the_models_leaf():
    import audiogpt_b200
    names = ("audio_infer", "audio_infer.pytorch", "audio_infer.pytorch.models")
    saved = {k: sys.modules.get(k) for k in names}
    try:
        assert "audio_infer.pytorch.models (aliased)" not in audiogpt_b200.install()
        patched = audiogpt_b200.install(detection=True)
        assert "audio_infer.pytorch.models (aliased)" in patched
        mod = importlib.import_module("audio_infer.pytorch.models")
        from audio_infer.pytorch.models import PVT as grafted
        from audiogpt_b200.audio_detection.audio_infer.pytorch.models import PVT
        assert mod.PVT is PVT and grafted is PVT
        ours = "audiogpt_b200.audio_detection.audio_infer"
        assert all(getattr(sys.modules.get(k), "__name__", k) != ours for k in names[:2])
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def test_abi_symbols_declared():
    with open(os.path.join(ROOT, "include", "agpt_b200.h")) as f:
        header = f.read()
    from audiogpt_b200 import _lib
    for name in ("agpt_pvt_create", "agpt_pvt_forward", "agpt_pvt_frames", "agpt_pvt_dwconv_gelu", "agpt_pvt_patch7",
                 "agpt_pvt_sr_gather", "agpt_pvt_head"):
        assert re.search(r"\bint " + name + r"\(", header), name
        assert name in _lib.PROTOTYPES
    body = header[header.index("typedef struct agpt_pvt_cfg"):header.index("} agpt_pvt_cfg;")]
    fields = re.findall(r"^\s*(?:int|float) (\w+)", body, flags=re.M)
    assert fields == [f[0] for f in _lib.PvtConfig._fields_]
