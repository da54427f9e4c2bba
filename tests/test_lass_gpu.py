"""GPU checks of the sound-extraction drop-ins (LASSNet, STFT; csrc/lass.cu) against the reference's own modules
(tests/golden/lass_*.npz) and the fp32 oracle (oracle/lass_ref.py, run on the GPU with TF32 off).

Tolerances: rel-RMSE <= 1e-4 (the project bar) for the mask, logits, text condition, STFT and waveforms, on the
tensor-core and on the fp32-FMA tap-GEMMs alike; the two top frequency bins are exactly 0.5."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audiogpt_b200 import _lib, specs  # noqa: E402
from oracle import lass_ref as ref  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(ROOT, "tests", "golden")
TOL = 1e-4


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt()).item()


@pytest.fixture(scope="module", autouse=True)
def no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _model(cfg, seed=6060, tokenizer=None):
    from audiogpt_b200.sound_extraction.model.LASSNet import LASSNet
    m = LASSNet.from_config(cfg, tokenizer=tokenizer)
    m.load_state_dict(specs.synth_lass(cfg, seed), strict=True)
    return m.to(DEV).eval()


@pytest.fixture(scope="module")
def small_model():
    return _model(specs.LASS_SMALL)


@pytest.fixture(scope="module")
def sd_small_dev():
    return {k: v.to(DEV) for k, v in specs.synth_lass(specs.LASS_SMALL, 6060).items()}


def _stft(n_fft):
    from audiogpt_b200.sound_extraction.utils.stft import STFT
    return STFT(n_fft, n_fft // 2, n_fft)


def _check_small(m, g):
    n_fft = int(g["n_fft"])
    stft = _stft(n_fft)
    n, s = int(g["n"]), int(g["seed_wav"])
    wav = torch.stack([specs.synth_lass_wav(n, s), specs.synth_lass_wav(n, s + 1)]).to(DEV)
    mag, phase = stft.transform(wav)
    assert mag.is_cuda and mag.shape == g["mag"].shape
    assert _rel(mag, g["mag"]) < TOL
    assert _rel(mag * torch.cos(phase), g["mag"] * np.cos(g["phase"])) < TOL
    x = torch.from_numpy(g["mag"]).to(DEV).transpose(2, 1).unsqueeze(1)       # the tool's transposed view
    assert not x.is_contiguous()
    mask, logits, cond = m.forward_ids(x, torch.from_numpy(g["ids"]).to(DEV), torch.from_numpy(g["mask"]).to(DEV), return_all=True)
    assert _rel(cond, g["cond"]) < TOL
    assert _rel(logits, g["logits"]) < TOL
    assert _rel(mask, g["mask_out"]) < TOL
    assert torch.all(mask[..., -2:] == 0.5)
    est = (torch.from_numpy(g["mask_out"]).to(DEV) * x).squeeze(1).permute(0, 2, 1)
    out = stft.inverse(est, torch.from_numpy(g["phase"]).to(DEV))
    assert out.shape == g["wav_out"].shape
    assert _rel(out, g["wav_out"]) < TOL


def test_small_matches_reference(small_model):
    """n_fft 256 (F = 129), B = 2 clips, T = 91, captions of 9 and 5 tokens (padding keys masked): STFT, cond,
    logits, mask and the inverse STFT against the reference modules."""
    _check_small(small_model, dict(np.load(os.path.join(GOLDEN, "lass_small.npz"))))


def test_fp32_fma_arm(small_model):
    """The same parity with every tap-GEMM on the fp32-FMA kernels."""
    L = _lib.lib()
    _lib.check(L.agpt_set_tensor_cores(0))
    try:
        _check_small(small_model, dict(np.load(os.path.join(GOLDEN, "lass_small.npz"))))
    finally:
        _lib.check(L.agpt_set_tensor_cores(1))


def test_shipped_matches_reference():
    """The tool's shape: one 10 s clip at 32 kHz (T = 626, F = 513), LASS (bert-mini), an 11-token query."""
    g = dict(np.load(os.path.join(GOLDEN, "lass_shipped.npz")))
    m = _model(specs.LASS, int(g["seed_w"]))
    stft = _stft(specs.LASS_FFT)
    wav = specs.synth_lass_wav(int(g["n"]), int(g["seed_wav"]))[None].to(DEV)
    mag, phase = stft.transform(wav)
    s = int(g["sample_stride"])
    assert _rel(mag.reshape(-1)[::s], g["mag_sample"]) < TOL
    x = mag.transpose(2, 1).unsqueeze(0)
    mask, logits, cond = m.forward_ids(x, torch.from_numpy(g["ids"]).to(DEV), torch.from_numpy(g["mask"]).to(DEV), return_all=True)
    assert mask.shape == (1, 1, 626, 513)
    assert _rel(cond, g["cond"]) < TOL
    assert _rel(logits.double().sum(-1).reshape(-1), g["logits_rows"]) < TOL
    assert _rel(mask.double().sum(-1).reshape(-1), g["mask_rows"]) < TOL
    assert _rel(logits.reshape(-1)[::s], g["logits_sample"]) < TOL
    assert _rel(mask.reshape(-1)[::s], g["mask_sample"]) < TOL
    out = stft.inverse((mask * x).squeeze(1).permute(0, 2, 1), phase)
    assert out.shape == (1, 1, 625 * 512)
    assert _rel(out.reshape(-1)[::s], g["wav_out_sample"]) < TOL


@pytest.mark.parametrize("T", [1, 63, 64, 65, 626, 1000])
def test_ragged_T_matches_oracle(small_model, sd_small_dev, T):
    """Any frame count, 1000 being the untruncated long clip of the tool's load_wav: the zero-padded rows up to a
    multiple of 64 pass through the first BatchNorm and reach rows < T through the 3x3 receptive field."""
    g = torch.Generator().manual_seed(T)
    x = (2.0 * torch.randn(1, 1, T, 513, generator=g)).abs().to(DEV)
    ids, msk = specs.synth_lass_ids(specs.LASS_SMALL, [7], 5)
    mask, logits, cond = small_model.forward_ids(x, ids.to(DEV), msk.to(DEV), return_all=True)
    with torch.no_grad():
        rm, rl, rc = ref.lass_forward(sd_small_dev, specs.LASS_SMALL, x, ids.to(DEV), msk.to(DEV))
    assert _rel(cond, rc) < TOL
    assert _rel(logits, rl) < TOL
    assert _rel(mask, rm) < TOL
    assert torch.all(mask[..., -2:] == 0.5)


def test_batch_of_three_matches_single_clips(small_model):
    g = torch.Generator().manual_seed(3)
    x = (2.0 * torch.randn(3, 1, 70, 129, generator=g)).abs().to(DEV)
    ids, msk = specs.synth_lass_ids(specs.LASS_SMALL, [4, 9, 6], 8)
    ids, msk = ids.to(DEV), msk.to(DEV)
    full = small_model.forward_ids(x, ids, msk)
    for b in range(3):
        n = int(msk[b].sum())
        one = small_model.forward_ids(x[b:b + 1], ids[b:b + 1, :n], msk[b:b + 1, :n])
        assert _rel(one, full[b:b + 1]) < 1e-6
    shared = small_model.forward_ids(x, ids[:1, :4], msk[:1, :4])        # one caption for the whole batch
    assert _rel(shared[1:2], small_model.forward_ids(x[1:2], ids[:1, :4], msk[:1, :4])) < 1e-6


def test_transposed_view_equals_contiguous(small_model):
    g = torch.Generator().manual_seed(4)
    mag = (2.0 * torch.randn(1, 129, 80, generator=g)).abs().to(DEV)
    ids, msk = specs.synth_lass_ids(specs.LASS_SMALL, [5], 9)
    v = mag.transpose(2, 1).unsqueeze(0)
    a = small_model.forward_ids(v, ids.to(DEV), msk.to(DEV))
    b = small_model.forward_ids(v.contiguous(), ids.to(DEV), msk.to(DEV))
    assert torch.equal(a, b)


def test_stft_cpu_tensors_round_trip_on_gpu():
    """The tool passes CPU tensors: they run on the GPU and come back on the CPU, equal to the CUDA call."""
    stft = _stft(specs.LASS_FFT)
    wav = specs.synth_lass_wav(40000 + 123, 5)[None]
    mag, phase = stft.transform(wav)
    assert not mag.is_cuda and mag.shape == (1, 513, 40123 // 512 + 1)
    mg, pg = stft.transform(wav.to(DEV))
    assert torch.equal(mag, mg.cpu()) and torch.equal(phase, pg.cpu())
    fb, ib = specs.stft_bases()
    rmag, rph = ref.stft_transform(wav.to(DEV), fb.to(DEV), specs.LASS_HOP)
    assert _rel(mag, rmag) < TOL
    out = stft.inverse(mag, phase)
    assert not out.is_cuda and out.shape == (1, 1, (mag.shape[-1] - 1) * 512)
    rout = ref.stft_inverse(rmag, rph, ib.to(DEV), specs.LASS_HOP)
    assert _rel(out, rout) < TOL
    assert _rel(out[0, 0, :39000], wav[0, :39000]) < TOL            # the STFT pair reconstructs the clip
    assert _rel(stft(wav.to(DEV)), rout) < TOL


def test_data_parallel_and_replica(small_model):
    """nn.DataParallel(device_ids=[0]) calls the module directly; with several devices a B = 1 call runs on a
    replicate() replica, whose tensors may be plain attributes: it must give the same mask."""
    g = torch.Generator().manual_seed(6)
    x = (2.0 * torch.randn(1, 1, 64, 129, generator=g)).abs().to(DEV)
    ids, msk = specs.synth_lass_ids(specs.LASS_SMALL, [6], 10)
    ids, msk = ids.to(DEV), msk.to(DEV)
    want = small_model.forward_ids(x, ids, msk)

    class Tok:
        def __call__(self, caption, add_special_tokens=False, padding=True, return_tensors="pt"):
            return {"input_ids": ids.cpu(), "attention_mask": msk.cpu()}

    small_model.text_embedder.tokenizer = Tok()
    try:
        dp = torch.nn.DataParallel(small_model, device_ids=[0])
        assert torch.equal(dp(x, ["[CLS] dog"]), want)
        rep = torch.nn.parallel.replicate(small_model, [0], detach=True)[0]
        assert torch.equal(rep(x, ["[CLS] dog"]), want)
    finally:
        small_model.text_embedder.tokenizer = None


def test_weight_change_rebuilds_engine():
    m = _model(specs.LASS_SMALL, 11)
    g = torch.Generator().manual_seed(7)
    x = (2.0 * torch.randn(1, 1, 64, 129, generator=g)).abs().to(DEV)
    ids, msk = specs.synth_lass_ids(specs.LASS_SMALL, [4], 12)
    ids, msk = ids.to(DEV), msk.to(DEV)
    a = m.forward_ids(x, ids, msk)
    with torch.no_grad():
        m.UNet.encoder_block2.conv_block1.bn1.running_mean.add_(0.5)
        m.UNet.after_conv2.bias.add_(0.25)
    b = m.forward_ids(x, ids, msk)
    sd = {k: v.to(DEV) for k, v in m.state_dict().items()}
    rm, _, _ = ref.lass_forward(sd, specs.LASS_SMALL, x, ids, msk)
    assert _rel(b, rm) < TOL and _rel(a, b) > 1e-3


def test_errors(small_model):
    ids, msk = specs.synth_lass_ids(specs.LASS_SMALL, [4], 13)
    x = torch.rand(1, 1, 16, 129)
    with pytest.raises(RuntimeError, match="CUDA"):
        small_model.forward_ids(x, ids, msk)
    with pytest.raises(ValueError, match="F = 200"):
        small_model.forward_ids(torch.rand(1, 1, 16, 200, device=DEV), ids.to(DEV), msk.to(DEV))
    with pytest.raises(ValueError, match="F = 65"):
        small_model.forward_ids(torch.rand(1, 1, 16, 65, device=DEV), ids.to(DEV), msk.to(DEV))
    bad = ids.clone()
    bad[0, 1] = specs.LASS_SMALL["vocab_size"]
    with pytest.raises(ValueError, match="token ids"):
        small_model.forward_ids(x.to(DEV), bad.to(DEV), msk.to(DEV))
    with pytest.raises(ValueError, match="captions"):
        small_model.forward_ids(torch.rand(3, 1, 16, 129, device=DEV), torch.cat([ids, ids]).to(DEV), torch.cat([msk, msk]).to(DEV))
    stft = _stft(specs.LASS_FFT)
    with pytest.raises(RuntimeError, match="too few"):
        stft.transform(torch.zeros(1, 300, device=DEV))


def test_tool_chain_through_installed_dropins():
    """SoundExtraction.inference after load_wav and tokenization, through install(extraction=True): CPU wav -> STFT
    -> DataParallel(LASSNet) on the GPU -> mask * mag -> CPU inverse STFT, against the oracle chain."""
    import audiogpt_b200
    saved = {k: sys.modules.get(k) for k in ("sound_extraction.model.LASSNet", "sound_extraction.utils.stft")}
    try:
        audiogpt_b200.install(extraction=True)
        from sound_extraction.model.LASSNet import LASSNet
        from sound_extraction.utils.stft import STFT
        ids, msk = specs.synth_lass_ids(specs.LASS_SMALL, [10], 14)

        class Tok:
            def __call__(self, caption, add_special_tokens=False, padding=True, return_tensors="pt"):
                return {"input_ids": ids, "attention_mask": msk}

        sd = specs.synth_lass(specs.LASS_SMALL, 15)
        net = LASSNet.from_config(specs.LASS_SMALL, tokenizer=Tok())
        model = torch.nn.DataParallel(net, device_ids=[0]).to(DEV)
        model.load_state_dict({"module." + k: v for k, v in sd.items()})
        model.eval()
        stft = STFT()
        waveform = specs.synth_lass_wav(32000 * 3, 16)[:, None].transpose(1, 0)          # load_wav(...)[..., None].T
        mixed_mag, mixed_phase = stft.transform(waveform)
        mixed_mag = mixed_mag.transpose(2, 1).unsqueeze(0).to(DEV)
        est_mask = model(mixed_mag, ["[CLS] dog barking"])
        est_mag = (est_mask * mixed_mag).squeeze(1).permute(0, 2, 1)
        est_wav = stft.inverse(est_mag.cpu().detach(), mixed_phase).squeeze(0).squeeze(0).numpy()
        fb, ib = specs.stft_bases()
        want = ref.extract({k: v.to(DEV) for k, v in sd.items()}, specs.LASS_SMALL, waveform.to(DEV), ids.to(DEV), msk.to(DEV),
                           fb.to(DEV), ib.to(DEV), specs.LASS_HOP)
        assert est_wav.shape == tuple(want.shape)
        assert _rel(est_wav, want) < TOL
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
