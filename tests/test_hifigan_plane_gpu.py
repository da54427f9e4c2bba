"""Plane-fed HiFi-GAN tap-GEMMs (tcconv5_pl_kernel / tcconv_pipe_pl_kernel): the leaky-ReLU convs whose input has more
than 128 channels read it as a pre-split fp16 hi / lo operand plane that the producing epilogue wrote, instead of
converting the fp32 tensor themselves.  The plane holds exactly the operands the fp32 transform makes, so an engine
created with AGPT_PLANE_FEED=0 must give the same waveform bit for bit, with the same tap-GEMM launches."""
import ctypes

import numpy as np
import pytest
import torch

from audiogpt_b200 import _lib, specs
from audiogpt_b200.modules.hifigan.hifigan import HifiGanGenerator

pytestmark = pytest.mark.gpu
# C0 = 512: stages of C = 256 (plane-fed) / 128 / 64 / 32 at T rows each (upsample rates of 1), so T places every
# stage's length around the 128-row tile stride of tcconv5 and the 254 / 250 / 246 strides of the fused pairs
H512_FLAT = dict(specs.HIFIGAN_SMALL, upsample_initial_channel=512, upsample_rates=[1, 1, 1, 1],
                 upsample_kernel_sizes=[1, 1, 1, 1])


def engine(make, monkeypatch, plane, fused=True):
    for var, on in (("AGPT_PLANE_FEED", plane), ("AGPT_FUSE_RESBLOCK", fused)):
        if on:
            monkeypatch.delenv(var, raising=False)
        else:
            monkeypatch.setenv(var, "0")
    m = make().eval().to("cuda")
    m(torch.zeros(1, 80, 2, device="cuda"))   # the handle reads both switches when it is created
    return m


def hifigan(h, seed):
    def make():
        m = HifiGanGenerator(h)
        m.load_state_dict(specs.synth_hifigan(h, seed), strict=True)
        return m
    return make


def profiled(run):
    """(waveform, profiled tap-GEMM launches, of those plane-fed, library launches) of one forward."""
    L = _lib.lib()
    _lib.check(L.agpt_profile_enable(1))
    n0 = _lib.launch_count()
    wav = run()
    torch.cuda.synchronize()
    buf = ctypes.create_string_buffer(1 << 20)
    L.agpt_profile_dump(buf, 1 << 20)
    planes = L.agpt_profile_plane_launches()
    _lib.check(L.agpt_profile_enable(0))
    return wav, len(buf.value.decode().splitlines()), planes, _lib.launch_count() - n0


def compare(make, monkeypatch, run, fused=True, splits=1):
    """Plane-fed and transform engines on the same input: identical waveforms and tap-GEMM launches; the plane-fed
    engine adds `splits` plane_split launches.  Returns the plane-fed launch count."""
    ref = engine(make, monkeypatch, plane=False, fused=fused)
    pl = engine(make, monkeypatch, plane=True, fused=fused)
    wr, nr, pr, lr = profiled(lambda: run(ref))
    wp, np_, pp, lp = profiled(lambda: run(pl))
    print(f"fused={fused}: {np_} tap-GEMM launches, {pp} plane-fed; library launches {lr} -> {lp}")
    assert pr == 0 and nr == np_ and lp == lr + splits
    assert torch.isfinite(wp).all()
    assert torch.equal(wp, wr), (wp - wr).abs().max().item()
    return pp


@pytest.mark.parametrize("T", [1, 126, 127, 128, 129, 246, 254, 256, 257])
@pytest.mark.parametrize("fused", [True, False])
def test_plane_bit_identical_ragged(T, fused, monkeypatch):
    """fused=False: AGPT_FUSE_RESBLOCK=0, every C <= 128 conv as its own (transform-path) launch."""
    mel = specs.synth_tensor((3, 80, T), seed=700 + T, scale=2.0, shift=-4.0).cuda()
    # plane-fed: ups[0] (reads conv_pre's output, split) and the 3 x 3 pairs of the C = 256 stage, two launches each
    # (c1's output only as a plane), and ups[1] (reads the completed MRF sum's plane)
    assert compare(hifigan(H512_FLAT, 81), monkeypatch, lambda m: m(mel), fused=fused) == 1 + 18 + 1


def test_plane_v1_full_size(monkeypatch):
    """V1 at 8 x 800.  Plane-fed: ups[0], ups[1] and the 18 unfused C = 256 convs.  The C <= 128 stages (fused pairs,
    256-row tiles, the time-grouped views of the C = 64 / 32 stages) keep the transform path."""
    mel = specs.synth_tensor((8, 80, 800), seed=0, scale=2.0, shift=-4.0).cuda()
    assert compare(hifigan(specs.HIFIGAN_V1, 1234), monkeypatch, lambda m: m(mel)) == 2 + 18


def test_plane_nsf_har_source(monkeypatch):
    """NSF: the excitation is added to X after the upsampler's epilogue, so X's plane comes from a split pass after
    the add (one for the C = 256 stage, plus conv_pre's)."""
    h = dict(specs.HIFIGAN_V1, use_pitch_embed=True, audio_sample_rate=24000)
    B, T = 2, 40
    mel = specs.synth_tensor((B, 80, T), seed=11, scale=2.0, shift=-4.0).cuda()
    har = torch.tensor(np.random.RandomState(3).uniform(-1, 1, (B, T * 256)), dtype=torch.float32).cuda()

    def run(m):
        m._build_engine(mel.device)
        wav = torch.empty((B, 1, T * 256), device="cuda")
        _lib.check(_lib.lib().agpt_hifigan_forward(m._h, _lib.fptr(mel), _lib.fptr(har), B, T, _lib.fptr(wav),
                                                   _lib.cur_stream()))
        return wav

    assert compare(hifigan(h, 5678), monkeypatch, run, splits=2) == 2 + 18


def test_plane_bigvgan_unchanged(monkeypatch):
    """BigVGAN's snake activations have no plane form: the switch changes nothing and no launch is plane-fed."""
    from audiogpt_b200.vocoder.bigvgan.models import BigVGAN

    def make():
        m = BigVGAN(specs.BIGVGAN_BASE)
        m.load_state_dict(specs.synth_bigvgan(specs.BIGVGAN_BASE, 4321), strict=True)
        return m

    mel = specs.synth_tensor((2, 80, 100), seed=7, scale=2.0, shift=-4.0).cuda()
    assert compare(make, monkeypatch, lambda m: m(mel), splits=0) == 0
