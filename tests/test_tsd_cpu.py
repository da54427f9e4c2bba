"""CPU checks of the target-sound-detection RaDur_fusion (target_sound_detection.src.models, the TargetSoundDetection
tool): the oracle against the reference's own RaDur_fusion (tests/golden/tsd_tr125.npz, tsd_branches.npz,
make_golden_tsd.py), the state-dict layout, the frame arithmetic, install(target_detection=True) and the C ABI's
declarations."""
import ctypes as C
import os
import re
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audiogpt_b200 import specs  # noqa: E402
from oracle import tsd_ref as ref  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
# the oracle and the reference both run fp32 on the CPU; they differ in BatchNorm's formula and a few summation orders
ORACLE_TOL = 2e-5


def load_cases(name):
    g = dict(np.load(os.path.join(GOLDEN, name)))
    cases = []
    for i in range(int(g["n_cases"])):
        c = {k[len(f"c{i}_"):]: v for k, v in g.items() if k.startswith(f"c{i}_")}
        c["cfg"] = dict(specs.TSD_DEFAULT, time_resolution=int(c["time_resolution"]), att_pool=bool(c["att_pool"]),
                        enhancement=bool(c["enhancement"]), top=int(g["top"]), tao=float(g["tao"]))
        cases.append(c)
    return g, cases


def case_inputs(c):
    return specs.synth_tsd_mel(int(c["T"]), int(c["mel_seed"])), specs.synth_tsd_mel(int(c["Tr"]), int(c["ref_seed"]))


def case_weights(c):
    return specs.synth_tsd(c["cfg"], int(c["weight_seed"]), float(c["out_shift"]))


TR125 = load_cases("tsd_tr125.npz")
BRANCHES = load_cases("tsd_branches.npz")
ALL = [("tr125", i) for i in range(len(TR125[1]))] + [("branches", i) for i in range(len(BRANCHES[1]))]


def _case(which, i):
    return (TR125 if which == "tr125" else BRANCHES)[1][i]


@pytest.mark.parametrize("which,i", ALL)
def test_oracle_matches_reference(which, i):
    c = _case(which, i)
    x, r = case_inputs(c)
    with torch.no_grad():
        out = ref.forward(case_weights(c), c["cfg"], x, r)
    assert out["decision_up"].shape == c["decision_up"].shape
    assert np.abs(out["embedding"].numpy() - c["embedding"]).max() <= ORACLE_TOL * max(1.0, np.abs(c["embedding"]).max())
    assert np.abs(out["decision"].numpy() - c["decision"]).max() <= ORACLE_TOL
    assert np.abs(out["decision_up"].numpy() - c["decision_up"]).max() <= ORACLE_TOL
    if c["cfg"]["enhancement"]:
        assert np.abs(out["decision1"][:, :, 0].numpy() - c["decision1"]).max() <= ORACLE_TOL
        assert out["topk_idx"].numpy().tolist() == c["topk_idx"].tolist()
        assert np.abs(out["topk_val"].numpy() - c["topk_val"]).max() <= ORACLE_TOL
        assert out["wmix"].item() > 0          # the fixture's gate is open: the second pass is mixed in


def test_fixtures_straddle_the_gate():
    """every enhancement fixture has top-k scores on both sides of tao, with the generator's stated margins"""
    g, cases = TR125
    tao = float(g["tao"])
    n = 0
    for c in cases:
        assert np.abs(c["decision_up"][..., 0] - 0.5).min() >= float(g["half_margin"])
        if not c["cfg"]["enhancement"]:
            continue
        v = c["topk_val"][0]
        assert (v > tao).any() and (v < tao).any()
        assert np.abs(v - tao).min() >= float(g["tao_margin"])
        s = np.sort(c["decision1"][0])[::-1][: len(v) + 1]
        assert (s[:-1] - s[1:]).min() >= float(g["gap_margin"])
        if len(s) > len(v):
            assert s[len(v) - 1] - s[len(v)] >= float(g["boundary_margin"])
        n += 1
    assert n == 6
    # the short clip keeps fewer frames than top: every frame is in the top-k
    short = [c for c in cases if int(c["T"]) == 40 and c["cfg"]["enhancement"]]
    assert short and all(c["topk_idx"].shape[1] == c["decision"].shape[1] < int(g["top"]) for c in short)


def test_specs_layout_matches_reference_keys():
    g = TR125[0]
    shapes = specs.tsd_param_shapes(specs.TSD_DEFAULT)
    assert list(shapes) == g["ref_keys"].tolist()
    assert [",".join(str(v) for v in s) for s in shapes.values()] == g["ref_shapes"].tolist()
    keys = specs.tsd_engine_keys(specs.TSD_DEFAULT)
    assert not any(k.startswith(("encoder.spectrogram", "encoder.logmel", "encoder.bn0", "encoder.fc_audioset")) for k in keys)
    assert not any(k.endswith("num_batches_tracked") for k in keys)
    sd = specs.synth_tsd(specs.TSD_DEFAULT, 1)
    for k, v in sd.items():     # nothing the reference initialises to a constant is left at it
        if v.is_floating_point():
            assert v.std() > 0, k


def _meta_shapes(cfg, T, Tr):
    """(T', Tr', Te) from the oracle's own convs and pools, run on meta tensors (shapes only)"""
    sd = {k: torch.empty(v, device="meta") for k, v in specs.tsd_param_shapes(cfg).items()}
    Td = ref.features(sd, cfg, torch.empty(1, T, 64, device="meta")).shape[1]
    Tre = ref.cnn14(sd, torch.empty(1, Tr, 64, device="meta")).shape[1]
    Te = ref.cnn14(sd, torch.empty(1, T, 64, device="meta")).shape[1] if cfg["enhancement"] else 0
    return Td, Tre, Te


@pytest.mark.parametrize("tr", [125, 250, 500, 100])
def test_frame_arithmetic_matches_the_convs(tr):
    cfg = dict(specs.TSD_DEFAULT, time_resolution=tr)
    for T, Tr in [(12, 8), (13, 9), (40, 240), (431, 17), (432, 501), (501, 501), (999, 64), (1002, 80), (1010, 501), (2000, 33)]:
        assert specs.tsd_frames(cfg, T, Tr) == _meta_shapes(cfg, T, Tr), (tr, T, Tr)
    with pytest.raises(ValueError, match="too short"):
        specs.tsd_frames(cfg, 20, 7)
    with pytest.raises(ValueError, match="too short"):
        specs.tsd_frames(cfg, 3, 64)
    assert specs.tsd_frames(specs.TSD_DEFAULT, 501, 501) == (62, 62, 62)
    assert specs.tsd_frames(specs.TSD_DEFAULT, 1010, 501)[0] == 125      # the stem's 500-row crop


def test_abi_frames_matches_python_twin():
    from audiogpt_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libagpt_b200.so is not built")
    L = _lib.lib()
    for tr in (125, 250, 500, 100):
        for enh in (0, 1):
            cfg = dict(specs.TSD_DEFAULT, time_resolution=tr, enhancement=bool(enh))
            cc = _lib.TsdConfig(time_resolution=tr, att_pool=1, enhancement=enh, top=10, tao=0.6, mel_bins=64, outputdim=2)
            for T in range(1, 40):
                for Tr in (1, 7, 8, 9, 501):
                    f = (C.c_int * 3)()
                    rc = L.agpt_tsd_frames(C.byref(cc), T, Tr, f)
                    try:
                        want = specs.tsd_frames(cfg, T, Tr)
                    except ValueError:
                        assert rc != 0 and b"too short" in L.agpt_last_error(), (tr, enh, T, Tr)
                        continue
                    assert rc == 0, L.agpt_last_error()
                    assert tuple(f) == want, (tr, enh, T, Tr)
            for T in (432, 501, 1001, 1002, 1010, 4000):
                f = (C.c_int * 3)()
                assert L.agpt_tsd_frames(C.byref(cc), T, 501, f) == 0
                assert tuple(f) == specs.tsd_frames(cfg, T, 501)


def _dropin(**kw):
    from audiogpt_b200.audio_detection.target_sound_detection.src.models import RaDur_fusion
    conf = dict(att_pool=True, enhancement=True, tao=0.6, top=10, model="RaDur_fusion", thres=0.5)
    conf.update(kw)
    return RaDur_fusion(conf, inputdim=64, outputdim=2, time_resolution=125)


def test_dropin_state_dict_and_cpu_refusal():
    m = _dropin()
    sd = specs.synth_tsd(specs.TSD_DEFAULT, 5)
    assert list(m.state_dict()) == list(sd)
    assert [tuple(v.shape) for v in m.state_dict().values()] == [tuple(v.shape) for v in sd.values()]
    # the constructor fills the encoder's frozen front end the way torchlibrosa does
    assert torch.equal(m.state_dict()["encoder.logmel_extractor.melW"], sd["encoder.logmel_extractor.melW"])
    res = m.load_state_dict(sd)
    assert not res.missing_keys and not res.unexpected_keys
    assert m.bn.num_batches_tracked.dtype == torch.long
    assert (m.att_pool, m.enhancement, m.tao, m.top) == (True, True, 0.6, 10)
    x = specs.synth_tsd_mel(501, 1)
    with pytest.raises(RuntimeError, match="eval"):
        m(x, x)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.eval()(x, x)
    bad = dict(sd)
    del bad["detection.gru.weight_hh_l0_reverse"]
    with pytest.raises(RuntimeError, match="weight_hh_l0_reverse"):
        m.load_state_dict(bad)
    with pytest.raises(ValueError, match="64"):
        from audiogpt_b200.audio_detection.target_sound_detection.src.models import RaDur_fusion
        RaDur_fusion(dict(att_pool=True, enhancement=True, tao=0.6, top=10), inputdim=128, outputdim=2, time_resolution=125)


def test_install_target_detection_patches_in_place_and_never_aliases():
    import audiogpt_b200
    from audiogpt_b200.audio_detection.target_sound_detection.src.models import RaDur_fusion
    names = ("target_sound_detection", "target_sound_detection.src", "target_sound_detection.src.models")
    saved = {k: sys.modules.get(k) for k in names}
    try:
        for k in names:
            sys.modules.pop(k, None)
        # no importable reference module: reported as skipped, nothing registered in its place
        patched = audiogpt_b200.install(target_detection=True)
        assert "target_sound_detection.src.models (skipped: not importable)" in patched
        assert "target_sound_detection.src.models" not in sys.modules
        with pytest.raises(ImportError):
            audiogpt_b200.install(strict=True, target_detection=True)
        assert "target_sound_detection.src.models" not in audiogpt_b200.install()
        # a stand-in of the reference module: RaDur_fusion is replaced, every other name stays
        pkg, src = types.ModuleType("target_sound_detection"), types.ModuleType("target_sound_detection.src")
        pkg.__path__, src.__path__ = [], []
        mod = types.ModuleType("target_sound_detection.src.models")

        class Theirs:
            pass

        labels = ["Alarm", "Bark"]
        mod.RaDur_fusion, mod.event_labels, mod.Cnn14 = Theirs, labels, Theirs
        sys.modules.update({names[0]: pkg, names[1]: src, names[2]: mod})
        src.models = mod
        patched = audiogpt_b200.install(target_detection=True)
        assert "target_sound_detection.src.models" in patched
        from target_sound_detection.src import models as tsd_models
        from target_sound_detection.src.models import event_labels
        assert tsd_models is mod and tsd_models.RaDur_fusion is RaDur_fusion
        assert getattr(tsd_models, "RaDur_fusion") is RaDur_fusion
        assert event_labels is labels and mod.Cnn14 is Theirs
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
    for name in ("agpt_tsd_create", "agpt_tsd_forward", "agpt_tsd_frames", "agpt_tsd_stage_events", "agpt_tsd_stem",
                 "agpt_tsd_avgpool", "agpt_tsd_gru", "agpt_tsd_enhance"):
        assert re.search(r"\bint " + name + r"\(", header), name
        assert name in _lib.PROTOTYPES
    body = header[header.index("typedef struct agpt_tsd_cfg"):header.index("} agpt_tsd_cfg;")]
    fields = re.findall(r"^\s*(?:int|float) (\w+)", body, flags=re.M)
    assert fields == [f[0] for f in _lib.TsdConfig._fields_]
