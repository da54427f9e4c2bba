"""GPU checks of the target-sound-detection RaDur_fusion drop-in (csrc/tsd.cu) against the reference's own outputs
(tests/golden/tsd_tr125.npz, tsd_branches.npz), the fp64 oracle, torch.nn.GRU and the reference's parts, on an H100.

Tolerances: decision and decision_up (probabilities) by max-abs error, about 3x the worst case an H100 80GB HBM3
(700 W power limit) showed over the fixtures: 2.2e-4 on the tensor-core arm (TOL_PROB; 1.6e-4 against the fp64
oracle), 5.0e-6 on the fp32-FMA arm (TOL_FMA).  The binary segments the tool derives (median_filter with window 1 and threshold 0.5) must be identical;
every fixture keeps its values at least 1e-3 from 0.5 and its top-k boundary at least 1e-3 wide.
"""
import ctypes as C
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audiogpt_b200 import _lib, specs  # noqa: E402
from oracle import tsd_ref as ref  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(ROOT, "tests", "golden")
TOL_PROB = 8e-4
TOL_FMA = 2e-5
TOL_GRU = 2e-6      # the recurrence alone, fp32 against fp64: 3.9e-7 worst on the H100


def _maxabs(a, b):
    return (torch.as_tensor(a).double().cpu() - torch.as_tensor(b).double().cpu()).abs().max().item()


def _segments(up):
    """the tool's median_filter(window_size=1, threshold=0.5) on decision_up[:, :, 0], then the contiguous regions"""
    on = torch.as_tensor(up)[..., 0].cpu().numpy() > 0.5
    out = []
    for row in on:
        d = np.diff(np.r_[0, row.astype(np.int8), 0])
        out.append(list(zip(np.nonzero(d == 1)[0].tolist(), np.nonzero(d == -1)[0].tolist())))
    return out


@pytest.fixture(scope="module", autouse=True)
def no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def load_cases(name):
    g = dict(np.load(os.path.join(GOLDEN, name)))
    cases = []
    for i in range(int(g["n_cases"])):
        c = {k[len(f"c{i}_"):]: v for k, v in g.items() if k.startswith(f"c{i}_")}
        c["cfg"] = dict(specs.TSD_DEFAULT, time_resolution=int(c["time_resolution"]), att_pool=bool(c["att_pool"]),
                        enhancement=bool(c["enhancement"]), top=int(g["top"]), tao=float(g["tao"]))
        cases.append(c)
    return cases


CASES = [("tsd_tr125.npz", i) for i in range(len(load_cases("tsd_tr125.npz")))] + \
        [("tsd_branches.npz", i) for i in range(len(load_cases("tsd_branches.npz")))]


def _model(cfg, seed, shift=0.0):
    from audiogpt_b200.audio_detection.target_sound_detection.src.models import RaDur_fusion
    m = RaDur_fusion(dict(att_pool=cfg["att_pool"], enhancement=cfg["enhancement"], tao=cfg["tao"], top=cfg["top"]),
                     inputdim=64, outputdim=cfg["outputdim"], time_resolution=cfg["time_resolution"])
    m.load_state_dict(specs.synth_tsd(cfg, seed, shift), strict=True)
    return m.to(DEV).eval()


def _run_case(c):
    m = _model(c["cfg"], int(c["weight_seed"]), float(c["out_shift"]))
    x = specs.synth_tsd_mel(int(c["T"]), int(c["mel_seed"])).to(DEV)
    r = specs.synth_tsd_mel(int(c["Tr"]), int(c["ref_seed"])).to(DEV)
    decision, up, logit = m(x, r)
    torch.cuda.synchronize()
    return decision, up, logit


def _check_case(c, tag, tol=TOL_PROB):
    decision, up, logit = _run_case(c)
    e_up, e_dec = _maxabs(up, c["decision_up"]), _maxabs(decision, c["decision"])
    print(f"[{tag}] T {int(c['T'])} Tr {int(c['Tr'])} tr {int(c['time_resolution'])} att {int(c['att_pool'])} "
          f"enh {int(c['enhancement'])}: decision_up {e_up:.2e}, decision {e_dec:.2e}")
    assert up.shape == c["decision_up"].shape and decision.shape == c["decision"].shape
    assert logit.shape == (1,) and logit.device.type == "cuda"
    assert e_up <= tol and e_dec <= tol
    assert _segments(up) == _segments(c["decision_up"])


@pytest.mark.parametrize("name,i", CASES)
def test_matches_reference(name, i):
    _check_case(load_cases(name)[i], "tc")


@pytest.mark.parametrize("name,i", [("tsd_tr125.npz", 0), ("tsd_tr125.npz", 3), ("tsd_branches.npz", 2)])
def test_fp32_fma_arm(name, i):
    L = _lib.lib()
    _lib.check(L.agpt_set_tensor_cores(0))
    try:
        _check_case(load_cases(name)[i], "fma", TOL_FMA)
    finally:
        _lib.check(L.agpt_set_tensor_cores(1))


@pytest.mark.parametrize("tr,att,enh,T,Tr", [(125, 1, 1, 617, 333), (125, 0, 1, 1003, 96), (250, 1, 0, 357, 120),
                                              (500, 0, 0, 203, 64), (7, 1, 0, 149, 80)])
def test_matches_fp64_oracle(tr, att, enh, T, Tr):
    """lengths and configs the fixtures do not have, against the oracle in fp64 (on the GPU)"""
    cfg = dict(specs.TSD_DEFAULT, time_resolution=tr, att_pool=bool(att), enhancement=bool(enh))
    sd = specs.synth_tsd(cfg, 9000 + T)
    m = _model(cfg, 9000 + T)
    x, r = specs.synth_tsd_mel(T, T), specs.synth_tsd_mel(Tr, T + 1)
    decision, up, _ = m(x.to(DEV), r.to(DEV))
    with torch.no_grad():
        want = ref.forward({k: v.to(DEV) for k, v in sd.items()}, cfg, x.to(DEV), r.to(DEV), dtype=torch.float64)
    e = _maxabs(up, want["decision_up"])
    print(f"[fp64] tr {tr} att {att} enh {enh} T {T} Tr {Tr}: decision_up {e:.2e}")
    assert e <= TOL_PROB and _maxabs(decision, want["decision"]) <= TOL_PROB


def test_batch_equals_one_row_at_a_time():
    cfg = specs.TSD_DEFAULT
    m = _model(cfg, 4242)
    x = specs.synth_tsd_mel(501, 1, B=2).to(DEV)
    r = specs.synth_tsd_mel(240, 2, B=2).to(DEV)
    d, up, _ = m(x, r)
    for b in range(2):
        db, ub, _ = m(x[b:b + 1], r[b:b + 1])
        assert _maxabs(d[b:b + 1], db) <= 1e-6 and _maxabs(up[b:b + 1], ub) <= 1e-6


def test_strict_load_and_rebuild_on_weight_change():
    c = load_cases("tsd_tr125.npz")[4]
    m = _model(c["cfg"], int(c["weight_seed"]), float(c["out_shift"]))
    x = specs.synth_tsd_mel(int(c["T"]), int(c["mel_seed"])).to(DEV)
    r = specs.synth_tsd_mel(int(c["Tr"]), int(c["ref_seed"])).to(DEV)
    _, up, _ = m(x, r)
    assert _maxabs(up, c["decision_up"]) <= TOL_PROB
    with torch.no_grad():
        m.detection.outputlayer.bias[0] += 0.5       # a weight changes: the next call rebuilds the handle
    _, up2, _ = m(x, r)
    assert _maxabs(up2, up) > 1e-3
    m.load_state_dict(specs.synth_tsd(c["cfg"], int(c["weight_seed"]), float(c["out_shift"])), strict=True)
    _, up3, _ = m(x, r)
    assert _maxabs(up3, c["decision_up"]) <= TOL_PROB


def test_rejected_inputs():
    m = _model(specs.TSD_DEFAULT, 1)
    x = torch.zeros(1, 501, 64, device=DEV)
    with pytest.raises(ValueError, match="64"):
        m(torch.zeros(1, 501, 128, device=DEV), x)
    with pytest.raises(ValueError, match="batch"):
        m(torch.zeros(2, 501, 64, device=DEV), x)
    with pytest.raises(ValueError, match="too short"):
        m(torch.zeros(1, 7, 64, device=DEV), x)
    with pytest.raises(ValueError, match="too short"):
        m(x, torch.zeros(1, 7, 64, device=DEV))
    with pytest.raises(RuntimeError, match="CUDA"):
        m(x.cpu(), x.cpu())
    # the engine refuses the same lengths on its own
    cc = m._config()
    f = (C.c_int * 3)()
    assert _lib.lib().agpt_tsd_frames(C.byref(cc), 501, 7, f) != 0


def test_installed_tool_call():
    """TargetSoundDetection.__init__ / inference (audio-chatgpt.py:775-875) on a stand-in of the reference module"""
    import audiogpt_b200
    names = ("target_sound_detection", "target_sound_detection.src", "target_sound_detection.src.models")
    saved = {k: sys.modules.get(k) for k in names}
    try:
        pkg, src, mod = (types.ModuleType(n) for n in names)
        pkg.__path__, src.__path__ = [], []
        mod.RaDur_fusion, mod.event_labels = object, ["Alarm", "Bark", "Speech"]
        src.models = mod
        sys.modules.update(dict(zip(names, (pkg, src, mod))))
        assert "target_sound_detection.src.models" in audiogpt_b200.install(target_detection=True)
        from target_sound_detection.src import models as tsd_models
        config_parameters = dict(model="RaDur_fusion", att_pool=True, enhancement=True, top=10, thres=0.5,
                                 model_args={}, tao=0.6, time_resolution=125)
        model = getattr(tsd_models, config_parameters["model"])(config_parameters, inputdim=64, outputdim=2,
                                                                time_resolution=config_parameters["time_resolution"],
                                                                **config_parameters["model_args"])
        model.load_state_dict(specs.synth_tsd(specs.TSD_DEFAULT, 77))
        model = model.to(DEV).eval()
        embedding = torch.from_numpy(specs.synth_tsd_mel(380, 5)[0].numpy()).unsqueeze(0).to(DEV).float()
        inputs = torch.from_numpy(specs.synth_tsd_mel(501, 6)[0].numpy()).unsqueeze(0).to(DEV).float()
        decision, decision_up, logit = model(inputs, embedding)
        pred = decision_up.detach().cpu().numpy()[:, :, 0]
        assert pred.shape == (1, 501) and np.isfinite(pred).all() and decision.shape == (1, 62)
        assert ((pred >= 0) & (pred <= 1)).all()
        _segments(decision_up)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


# ---------------------------------------------------------------- kernels through their unit entry points
@pytest.mark.parametrize("B", [1, 3, 4, 5, 9])     # 5 and 9: a second and third group of kGruMaxB = 4 over blockIdx.z
@pytest.mark.parametrize("T", [1, 2, 63, 125, 500])
def test_gru_kernel(T, B):
    g = torch.Generator().manual_seed(T * 10 + B)
    gru = torch.nn.GRU(512, 512, bidirectional=True, batch_first=True).double()
    with torch.no_grad():
        for p in gru.parameters():
            p.copy_(0.06 * torch.randn(p.shape, generator=g, dtype=torch.float64))
    gru = gru.to(DEV)
    x = torch.randn(B, T, 512, generator=g, dtype=torch.float64).to(DEV)
    with torch.no_grad():
        want = gru(x)[0]
        xp = torch.cat([F.linear(x, gru.weight_ih_l0, gru.bias_ih_l0), F.linear(x, gru.weight_ih_l0_reverse, gru.bias_ih_l0_reverse)], 2)
    whh = torch.stack([gru.weight_hh_l0, gru.weight_hh_l0_reverse]).float().contiguous()
    bhh = torch.stack([gru.bias_hh_l0, gru.bias_hh_l0_reverse]).float().contiguous()
    xp = xp.float().contiguous()
    out = torch.empty(B, T, 1024, device=DEV)
    _lib.call("tsd_gru", DEV, _lib.fptr(whh), _lib.fptr(bhh), _lib.fptr(xp), B, T, _lib.fptr(out))
    torch.cuda.synchronize()
    e = _maxabs(out, want)
    print(f"[gru] T {T} B {B}: max-abs {e:.2e}")
    assert e <= TOL_GRU


@pytest.mark.parametrize("T,ph", [(501, 2), (432, 2), (1010, 2), (12, 2), (57, 1), (40, 1)])
def test_stem_kernel(T, ph):
    cfg = dict(specs.TSD_DEFAULT, time_resolution=125 if ph == 2 else 0)
    sd = {k: v.double() for k, v in specs.synth_tsd(cfg, 31).items() if v.is_floating_point()}
    mel = specs.synth_tsd_mel(T, 8, B=2)
    want = ref.stem(sd, mel.double().unsqueeze(1), ph).permute(0, 2, 3, 1)       # [B, m, 32, 96]
    w = torch.zeros(3, 64, 25, dtype=torch.float64)
    b = torch.zeros(3, 64, dtype=torch.float64)
    for br, k in enumerate((1, 3, 5)):
        p = f"detection.features.conv_block1_{br + 1}."
        s = sd[p + "bn1.weight"] / torch.sqrt(sd[p + "bn1.running_var"] + 1e-5)
        w[br, :, :k * k] = sd[p + "conv1.weight"].reshape(64, k * k) * s[:, None]
        b[br] = sd[p + "bn1.bias"] - sd[p + "bn1.running_mean"] * s
    out = torch.empty(want.shape, device=DEV)
    w, b, melg = w.float().to(DEV), b.float().to(DEV), mel.to(DEV).contiguous()
    _lib.call("tsd_stem", DEV, _lib.fptr(melg), _lib.fptr(w), _lib.fptr(b), 2, T, ph, _lib.fptr(out))
    torch.cuda.synchronize()
    assert out.shape[1] == specs.tsd_stem_rows(T, ph)[3]
    assert _maxabs(out, want) <= 1e-5 * max(1.0, want.abs().max().item())


@pytest.mark.parametrize("ph,pw", [(2, 2), (1, 2), (2, 4), (1, 4)])
@pytest.mark.parametrize("H,W,C", [(125, 16, 256), (63, 5, 1024), (7, 8, 96)])
def test_avgpool_kernel(ph, pw, H, W, C):
    x = torch.randn(2, H, W, C, device=DEV)
    want = F.avg_pool2d(x.permute(0, 3, 1, 2).double(), (ph, pw)).permute(0, 2, 3, 1)
    out = torch.empty(want.shape, device=DEV)
    _lib.call("tsd_avgpool", DEV, _lib.fptr(x), 2, H, W, C, ph, pw, _lib.fptr(out))
    torch.cuda.synchronize()
    assert _maxabs(out, want) <= 1e-6


def _enhance(p1, emix, emb, top, tao, w):
    B, Td, O = p1.shape
    k = min(top, Td)
    me = torch.empty(B, 128, device=DEV)
    wmix = torch.empty(B, device=DEV)
    idx = torch.empty(B, k, dtype=torch.int32, device=DEV)
    val = torch.empty(B, k, device=DEV)
    ptrs = (C.POINTER(C.c_float) * 8)(*[C.cast(t.data_ptr(), C.POINTER(C.c_float)) for t in w])
    _lib.call("tsd_enhance", DEV, _lib.fptr(p1), B, Td, O, _lib.fptr(emix), emix.shape[1], _lib.fptr(emb), top, tao, ptrs,
              _lib.fptr(me), _lib.fptr(wmix), _lib.fptr(idx), _lib.fptr(val))
    torch.cuda.synchronize()
    return me, wmix, idx, val


@pytest.mark.parametrize("Td,top", [(62, 10), (5, 10), (500, 3)])
def test_enhance_kernel_with_ties(Td, top):
    """the tail of orcal_EE on random inputs whose scores tie across the top-k boundary, against the oracle in fp64"""
    g = torch.Generator().manual_seed(Td + top)
    B = 2
    sd = {k: v.double() for k, v in specs.synth_tsd(specs.TSD_DEFAULT, 5).items() if v.is_floating_point()}
    s = 0.3 + 0.6 * torch.rand(B, Td, generator=g, dtype=torch.float64)
    s = (s * 64).round() / 64                       # exact in fp32, so the ties survive
    k = min(top, Td)
    s[:, 1] = s[:, 0] = s.max(1).values           # the two first frames tie at the top
    s[0, Td - 1] = s[0].sort(descending=True)[0][k - 1]   # a tie across the top-k boundary, later frame loses
    p1 = torch.stack([s, 1 - s], 2)
    emix = torch.randn(B, max(Td, 8), 128, generator=g, dtype=torch.float64)
    emb = torch.randn(B, 128, generator=g, dtype=torch.float64)
    names = ("q_ee.weight", "q_ee.bias", "k_ee.weight", "k_ee.bias", "EE_fusion.fuse_layer1.conv.weight",
             "EE_fusion.fuse_layer1.conv.bias", "EE_fusion.fuse_layer2.conv.weight", "EE_fusion.fuse_layer2.conv.bias")
    w = [sd[n].float().reshape(sd[n].shape[0], -1).contiguous().to(DEV) if sd[n].dim() > 1 else sd[n].float().to(DEV) for n in names]
    me, wmix, idx, val = _enhance(p1.float().to(DEV), emix.float().to(DEV), emb.float().to(DEV), top, 0.6, w)
    v, i = ref.topk(s, top)
    assert idx.cpu().long().tolist() == i.tolist()
    assert _maxabs(val, v) == 0
    sel = torch.gather(emix, 1, i.unsqueeze(2).expand(-1, -1, 128))
    att = ref.get_w(sd, "q_ee", "k_ee", emb, sel).squeeze(1) * (v * (v > 0.6))
    want = ref.fusion(sd, "EE_fusion.", 4, (sel * att.unsqueeze(2)).mean(1).unsqueeze(1), emb.unsqueeze(1))[:, 0]
    m = v.mean(1)
    assert _maxabs(me, want) <= 1e-5 * max(1.0, want.abs().max().item())
    assert _maxabs(wmix, m * (m > 0.6) / 2) <= 1e-6


def test_enhance_refuses_frames_past_the_mixture_encoder():
    """with T' > Te (time_resolution 250 / 500 / other) a top-k frame the mixture encoder lacks is refused, as the
    reference's gather fails"""
    B, Td, Te = 1, 40, 10
    s = torch.full((B, Td), 0.1)
    s[0, 30] = 0.9
    p1 = torch.stack([s, 1 - s], 2).to(DEV)
    w = [torch.zeros(128, 128, device=DEV), torch.zeros(128, device=DEV), torch.zeros(128, 128, device=DEV), torch.zeros(128, device=DEV),
         torch.zeros(512, 128, device=DEV), torch.zeros(512, device=DEV), torch.zeros(512, 128, device=DEV), torch.zeros(512, device=DEV)]
    with pytest.raises(RuntimeError, match="past the mixture encoder"):
        _enhance(p1, torch.zeros(B, Te, 128, device=DEV), torch.zeros(B, 128, device=DEV), 3, 0.6, w)
