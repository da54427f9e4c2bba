"""GPU checks of the sound-event-detection PVT (csrc/pvt.cu, audio_infer.pytorch.models.PVT) against the reference's
own PVT (tests/golden/pvt_small.npz, pvt_shipped.npz) and the oracle (oracle/pvt_ref.py, on the GPU with TF32 off, in
fp64 where a tolerance is set from it).

Tolerances: pre-sigmoid logits by rel-RMSE (TOL_LOGITS), probabilities by absolute error (TOL_PROB), and the top-10
classes of max-over-time -- what the tool plots -- identical.  TOL_LOGITS is three times what an H100 showed through
the shipped network's 16 blocks (1.3e-5 against the reference and against eager fp32; 4.3e-6 against the fp64 oracle on
PVT_SMALL, where eager fp32 itself is at 8e-7): looser than the 2e-5 the 12-layer CLAP encoder holds, well inside the
project's 1e-4."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audiogpt_b200 import _lib, specs  # noqa: E402
from oracle import pvt_ref as ref  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(ROOT, "tests", "golden")
TOL_LOGITS = 4e-5
TOL_PROB = 5e-5


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt()).item()


def _maxabs(a, b):
    return (torch.as_tensor(a).double().cpu() - torch.as_tensor(b).double().cpu()).abs().max().item()


def _top10(frame):
    return np.argsort(np.max(torch.as_tensor(frame).cpu().numpy(), axis=0))[::-1][:10].tolist()


@pytest.fixture(scope="module", autouse=True)
def no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _model(cfg, seed):
    from audiogpt_b200.audio_detection.audio_infer.pytorch.models import PVT
    m = PVT.from_config(cfg)
    m.load_state_dict(specs.synth_pvt(cfg, seed), strict=True)
    return m.to(DEV).eval()


@pytest.fixture(scope="module")
def small():
    return dict(np.load(os.path.join(GOLDEN, "pvt_small.npz")))


@pytest.fixture(scope="module")
def shipped():
    return dict(np.load(os.path.join(GOLDEN, "pvt_shipped.npz")))


@pytest.fixture(scope="module")
def small_model(small):
    return _model(specs.PVT_SMALL, int(small["weight_seed"]))


@pytest.fixture(scope="module")
def shipped_model(shipped):
    return _model(specs.PVT_SHIPPED, int(shipped["weight_seed"]))


@pytest.fixture(scope="module")
def sd64_small(small):
    return {k: v.to(DEV) for k, v in ref.to_double(specs.synth_pvt(specs.PVT_SMALL, int(small["weight_seed"]))).items()}


def _check_small(m, g, what):
    for k, n in enumerate(g["clip_lens"].tolist()):
        wav = specs.synth_pvt_wav(n, int(g["clip_seed"]) + k).to(DEV)[None]
        out = m(wav, None, return_logits=True)
        assert out["framewise_output"].shape == g[f"framewise{k}"].shape and out["clipwise_output"].shape == g[f"clipwise{k}"].shape
        e = _rel(out["logits"], g[f"logits{k}"])
        print(f"\n[pvt {what}] clip {n}: logits rel-RMSE {e:.2e}, framewise max abs err "
              f"{_maxabs(out['framewise_output'], g[f'framewise{k}']):.2e}")
        assert e <= TOL_LOGITS
        assert _maxabs(out["framewise_output"], g[f"framewise{k}"]) <= TOL_PROB
        assert _maxabs(out["clipwise_output"], g[f"clipwise{k}"]) <= TOL_PROB
        assert _top10(out["framewise_output"][0]) == _top10(g[f"framewise{k}"][0])


def test_small_matches_reference(small_model, small):
    """PVT_SMALL on two clips: stage grids with a remainder in every sr gather (26 / 13 / 7 rows) and without"""
    _check_small(small_model, small, "tensor cores")


def test_fp32_fma_arm(small_model, small):
    """The same parity with every tap-GEMM and attention on the fp32-FMA kernels (fc2 then reads fp32, not planes)"""
    L = _lib.lib()
    _lib.check(L.agpt_set_tensor_cores(0))
    _lib.check(L.agpt_set_attention_tc(0))
    try:
        _check_small(small_model, small, "fp32 FMA")
    finally:
        _lib.check(L.agpt_set_tensor_cores(1))
        _lib.check(L.agpt_set_attention_tc(-1))


def test_small_matches_fp64_oracle(small_model, small, sd64_small):
    """Against the oracle in fp64: the engine's own error, with the fp32 oracle's error beside it as the yardstick"""
    n = int(small["clip_lens"][0])
    wav = specs.synth_pvt_wav(n, int(small["clip_seed"])).to(DEV)[None]
    want = ref.forward(sd64_small, specs.PVT_SMALL, wav)
    sd32 = {k: (v.float() if v.is_floating_point() else v) for k, v in sd64_small.items()}
    eager = ref.forward(sd32, specs.PVT_SMALL, wav)
    out = small_model(wav, None, return_logits=True)
    e, e32 = _rel(out["logits"], want["logits"]), _rel(eager["logits"], want["logits"])
    print(f"\n[pvt] logits vs fp64 oracle: engine {e:.2e}, fp32 eager {e32:.2e}")
    assert e <= TOL_LOGITS
    assert _maxabs(out["framewise_output"], want["framewise_output"]) <= TOL_PROB
    assert _maxabs(out["clipwise_output"], want["clipwise_output"]) <= TOL_PROB


def test_shipped_matches_reference_tool_call(shipped_model, shipped):
    """The tool's request: the shipped config on one 10 s clip, read the way SoundDetection.inference reads it"""
    wav = specs.synth_pvt_wav(int(shipped["clip_len"]), int(shipped["clip_seed"])).to(DEV)[None]
    base = _lib.launch_count()
    out = shipped_model(wav, None, return_logits=True)
    launches = _lib.launch_count() - base
    framewise_output = shipped_model(wav, None)["framewise_output"].data.cpu().numpy()[0]
    assert framewise_output.shape == (1024, 527)
    e = _rel(out["logits"], shipped["logits"])
    print(f"\n[pvt shipped] logits rel-RMSE {e:.2e}, {launches} launches per forward")
    assert e <= TOL_LOGITS
    step = int(shipped["row_step"])
    assert np.abs(framewise_output[::step] - shipped["framewise_rows"][0]).max() <= TOL_PROB
    assert _maxabs(out["clipwise_output"], shipped["clipwise"]) <= TOL_PROB
    sorted_indexes = np.argsort(np.max(framewise_output, axis=0))[::-1]
    assert sorted_indexes[:10].tolist() == shipped["top10"].tolist()
    # interpolate(): every framewise row is repeated 32 times
    assert np.array_equal(framewise_output.reshape(32, 32, 527), np.repeat(framewise_output[::32, None], 32, axis=1))
    assert launches == 201


@pytest.mark.parametrize("n", [specs.pvt_min_samples(specs.PVT_SHIPPED), 32000, 320001, 960000])
def test_ragged_lengths_against_oracle(shipped_model, shipped, n):
    """shortest supported clip, 1 s, 10 s + 1 sample, 30 s (10 s is the fixture's) against the fp32 oracle"""
    sd = {k: v.to(DEV) for k, v in specs.synth_pvt(specs.PVT_SHIPPED, int(shipped["weight_seed"])).items()}
    wav = specs.synth_pvt_wav(n, 77).to(DEV)[None]
    want = ref.forward(sd, specs.PVT_SHIPPED, wav)
    out = shipped_model(wav, None, return_logits=True)
    H4 = specs.pvt_grids(specs.PVT_SHIPPED, n)[-1][0]
    assert out["framewise_output"].shape == (1, 32 * H4, 527) == want["framewise_output"].shape
    assert _rel(out["logits"], want["logits"]) <= TOL_LOGITS
    assert _maxabs(out["framewise_output"], want["framewise_output"]) <= TOL_PROB
    assert _maxabs(out["clipwise_output"], want["clipwise_output"]) <= TOL_PROB


def test_batch_equals_one_clip_at_a_time(small_model):
    wav = torch.stack([specs.synth_pvt_wav(8250, 90 + i) for i in range(3)]).to(DEV)
    out = small_model(wav, None, return_logits=True)
    for i in range(3):
        one = small_model(wav[i:i + 1], None, return_logits=True)
        assert _rel(out["logits"][i], one["logits"][0]) <= 2e-6      # tile shapes, not values, depend on the batch
        for k in ("framewise_output", "clipwise_output"):
            assert _maxabs(out[k][i], one[k][0]) <= 2e-6, k


def test_strict_load_and_rebuild_on_weight_change(small):
    cfg = specs.PVT_SMALL
    from audiogpt_b200.audio_detection.audio_infer.pytorch.models import PVT
    m = PVT.from_config(cfg)
    sd = specs.synth_pvt(cfg, int(small["weight_seed"]))
    m.load_state_dict({k: sd[k] for k in small["ref_keys"].tolist()}, strict=True)     # the reference's key order
    m.to(DEV)
    m.eval()
    wav = specs.synth_pvt_wav(5040, 34).to(DEV)[None]
    a = m(wav)["clipwise_output"].clone()
    assert _maxabs(a, small["clipwise1"]) <= TOL_PROB
    h = m._engine.h.value
    assert torch.equal(m(wav)["clipwise_output"], a) and m._engine.h.value == h      # no rebuild without a change
    with torch.no_grad():
        m.fc_audioset.bias.add_(1.0)
    b = m(wav, return_logits=True)
    assert not torch.equal(b["clipwise_output"], a)
    m.load_state_dict(sd)
    assert torch.equal(m(wav)["clipwise_output"], a)


def test_rejected_inputs(small_model):
    lo = specs.pvt_min_samples(specs.PVT_SMALL)
    with pytest.raises(RuntimeError, match="CUDA"):
        small_model(torch.zeros(1, 8000))
    with pytest.raises(ValueError, match="too short"):
        small_model(torch.zeros(1, lo - 1, device=DEV))
    with pytest.raises(ValueError, match="batch_size"):
        small_model(torch.zeros(8000, device=DEV))
    small_model.train()
    try:
        with pytest.raises(RuntimeError, match="eval"):
            small_model(torch.zeros(1, 8000, device=DEV))
    finally:
        small_model.eval()
    out = small_model(torch.zeros(1, lo, device=DEV))          # the shortest clip runs
    assert torch.isfinite(out["framewise_output"]).all()
    # the ABI refuses the same clip by itself
    cc = small_model._config()
    x = torch.zeros(1, lo - 1, device=DEV)
    o = torch.zeros(1, 32, 23, device=DEV)
    rc = _lib.lib().agpt_pvt_forward(small_model._h, _lib.fptr(x), 1, lo - 1, _lib.fptr(o), _lib.fptr(o), None, None)
    assert rc != 0 and b"too short" in _lib.lib().agpt_last_error()
    assert cc.mel_bins == 64


def test_installed_tool_call(shipped):
    """install(detection=True), then the SoundDetection constructor's model lines and inference's forward"""
    import audiogpt_b200
    saved = sys.modules.get("audio_infer.pytorch.models")
    try:
        audiogpt_b200.install(detection=True)
        from audio_infer.pytorch.models import PVT
        model = PVT(sample_rate=32000, window_size=1024, hop_size=320, mel_bins=64, fmin=50, fmax=14000, classes_num=527)
        checkpoint = {"model": specs.synth_pvt(specs.PVT_SHIPPED, int(shipped["weight_seed"]))}
        model.load_state_dict(checkpoint["model"])
        model.to(DEV)
        waveform = specs.synth_pvt_wav(int(shipped["clip_len"]), int(shipped["clip_seed"])).numpy()[None, :]
        waveform = torch.from_numpy(waveform).to(DEV)
        with torch.no_grad():
            model.eval()
            batch_output_dict = model(waveform, None)
        framewise_output = batch_output_dict["framewise_output"].data.cpu().numpy()[0]
        sorted_indexes = np.argsort(np.max(framewise_output, axis=0))[::-1]
        assert sorted_indexes[0:10].tolist() == shipped["top10"].tolist()
        for missing in ("timm", "mmcv", "mmdet", "torchlibrosa"):
            assert missing not in sys.modules
    finally:
        if saved is None:
            sys.modules.pop("audio_infer.pytorch.models", None)
        else:
            sys.modules["audio_infer.pytorch.models"] = saved


# ---------------------------------------------------------------- the new kernels, one launch each
def _call(name, *args):
    _lib.call(name, torch.device(DEV), *args)


def _rand(*shape, seed, scale=1.0):
    return (torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale).to(DEV)


@pytest.mark.parametrize("C,H,W,B", [(512, 250, 16, 1), (1024, 125, 8, 2), (1280, 63, 4, 1), (2048, 32, 2, 2), (72, 5, 3, 1)])
def test_dwconv_gelu_kernel(C, H, W, B):
    """depthwise 3 x 3 + bias + exact GELU at the four Mlp widths (and a width that is not a multiple of 64), as fp32
    and as operand planes: hi + lo is the fp32 result to 2^-22, and hi is its saturated fp16 rounding"""
    x, w, b = _rand(B, H * W, C, seed=C), _rand(C, 1, 3, 3, seed=C + 1, scale=0.4), _rand(C, seed=C + 2, scale=0.2)
    img = x.double().transpose(1, 2).reshape(B, C, H, W)
    want = F.gelu(F.conv2d(img, w.double(), b.double(), padding=1, groups=C)).flatten(2).transpose(1, 2)
    out = torch.full_like(x, float("nan"))
    _call("pvt_dwconv_gelu", _lib.fptr(x), _lib.fptr(w), _lib.fptr(b), B, H, W, C, _lib.fptr(out), None, None)
    assert _rel(out, want) <= 2e-7
    hi = torch.zeros(B, H * W, C, dtype=torch.float16, device=DEV)
    lo = torch.zeros_like(hi)
    _call("pvt_dwconv_gelu", _lib.fptr(x), _lib.fptr(w), _lib.fptr(b), B, H, W, C, None, _lib.fptr(hi), _lib.fptr(lo))
    assert torch.equal(hi, out.half())
    assert torch.equal(lo, (out - hi.float()).half())
    assert _rel(hi.double() + lo.double(), want) <= 5e-7


@pytest.mark.parametrize("C,H,W,B", [(64, 1001, 64, 1), (64, 31, 64, 3), (128, 104, 64, 2), (32, 9, 11, 1)])
def test_patch7_kernel(C, H, W, B):
    """Conv2d(1, C, 7, stride 4, padding 2) + LayerNorm over C"""
    img, w, b = _rand(B, H, W, seed=C + H), _rand(C, 1, 7, 7, seed=1, scale=0.15), _rand(C, seed=2, scale=0.1)
    g, be = 1 + _rand(C, seed=3, scale=0.1), _rand(C, seed=4, scale=0.1)
    y = F.conv2d(img.double()[:, None], w.double(), b.double(), stride=4, padding=2)
    Ho, Wo = y.shape[2:]
    want = F.layer_norm(y.flatten(2).transpose(1, 2), (C,), g.double(), be.double(), 1e-5)
    out = torch.full((B, Ho * Wo, C), float("nan"), device=DEV)
    _call("pvt_patch7", _lib.fptr(img), _lib.fptr(w), _lib.fptr(b), _lib.fptr(g), _lib.fptr(be), 1e-5, B, H, W, C, _lib.fptr(out))
    assert _rel(out, want) <= 1e-6


@pytest.mark.parametrize("sr,H,W,C", [(8, 250, 16, 64), (8, 16, 16, 64), (4, 125, 8, 128), (4, 8, 8, 128), (2, 63, 5, 320),
                                      (2, 4, 4, 320), (1, 3, 2, 8)])
def test_sr_gather_kernel(sr, H, W, C):
    """the sr x sr patch rows, with and without rows / columns that do not fill a patch: a 1-tap GEMM over them with
    the (ky, kx, ci) weight is the strided conv"""
    B = 2
    x = _rand(B, H * W, C, seed=sr + H)
    Hr, Wr = H // sr, W // sr
    out = torch.full((B, Hr * Wr, sr * sr * C), float("nan"), device=DEV)
    _call("pvt_sr_gather", _lib.fptr(x), B, H, W, C, sr, _lib.fptr(out))
    img = x.reshape(B, H, W, C)[:, :Hr * sr, :Wr * sr]
    want = img.reshape(B, Hr, sr, Wr, sr, C).permute(0, 1, 3, 2, 4, 5).reshape(B, Hr * Wr, sr * sr * C)
    assert torch.equal(out, want)
    w = _rand(16, C, sr, sr, seed=9, scale=0.05).double()
    conv = F.conv2d(x.double().transpose(1, 2).reshape(B, C, H, W), w, stride=sr).flatten(2).transpose(1, 2)
    assert _rel(out.double() @ w.permute(0, 2, 3, 1).reshape(16, -1).t(), conv) <= 1e-12


@pytest.mark.parametrize("B,H,W,C,K,ratio", [(1, 32, 2, 512, 527, 32), (3, 7, 2, 128, 23, 32), (2, 188, 2, 512, 527, 32), (1, 1, 3, 64, 5, 4)])
def test_head_kernel(B, H, W, C, K, ratio):
    """mean over the mel axis, fc_audioset, sigmoid, the row repeat and the clipwise mean"""
    x, w, b = _rand(B, H * W, C, seed=H), _rand(K, C, seed=5, scale=0.1), _rand(K, seed=6, scale=0.3)
    z = F.linear(x.double().reshape(B, H, W, C).mean(2), w.double(), b.double())
    p = torch.sigmoid(z)
    frame = torch.full((B, ratio * H, K), float("nan"), device=DEV)
    clip = torch.full((B, K), float("nan"), device=DEV)
    logits = torch.full((B, H, K), float("nan"), device=DEV)
    _call("pvt_head", _lib.fptr(x), _lib.fptr(w), _lib.fptr(b), B, H, W, C, K, ratio, _lib.fptr(frame), _lib.fptr(clip), _lib.fptr(logits))
    assert _rel(logits, z) <= 1e-6
    assert _maxabs(frame, p.repeat_interleave(ratio, dim=1)) <= 1e-6
    assert _maxabs(clip, p.mean(1)) <= 1e-6
    frame2 = torch.empty_like(frame)
    _call("pvt_head", _lib.fptr(x), _lib.fptr(w), _lib.fptr(b), B, H, W, C, K, ratio, _lib.fptr(frame2), _lib.fptr(clip), None)
    assert torch.equal(frame, frame2)


def test_kernel_entry_points_reject_bad_shapes():
    x = torch.zeros(64, device=DEV)
    L = _lib.lib()
    assert L.agpt_pvt_sr_gather(_lib.fptr(x), 1, 4, 4, 4, 8, _lib.fptr(x), None) != 0
    assert L.agpt_pvt_patch7(_lib.fptr(x), _lib.fptr(x), _lib.fptr(x), _lib.fptr(x), _lib.fptr(x), 1e-5, 1, 8, 8, 48, _lib.fptr(x), None) != 0
    assert L.agpt_pvt_dwconv_gelu(_lib.fptr(x), _lib.fptr(x), _lib.fptr(x), 1, 2, 2, 6, _lib.fptr(x), None, None, None) != 0
    assert L.agpt_pvt_dwconv_gelu(_lib.fptr(x), _lib.fptr(x), _lib.fptr(x), 1, 2, 2, 4, None, None, None, None) != 0
