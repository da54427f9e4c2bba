"""256-row tap-GEMM tiles (tcconv5_kernel / tcpair_kernel <BN, 256>) on the narrow stages of HiFi-GAN and BigVGAN.
A tall tile accumulates every output row from the same products in the same order as two 128-row tiles, so an engine
created with AGPT_TALL_TILES=0 must give the same waveform bit for bit, with the same launches."""
import ctypes

import pytest
import torch

from audiogpt_b200 import _lib, specs
from audiogpt_b200.modules.hifigan.hifigan import HifiGanGenerator

pytestmark = pytest.mark.gpu
# C0 = 256: stages of C = 128 / 64 / 32 / 16.  Upsample rates of 1 keep every stage at T rows, so T places each stage's
# length below one tile and around the 256-row stride of tcconv5 and the 254 / 250 / 246 strides of the fused pairs
H256_FLAT = dict(specs.HIFIGAN_SMALL, upsample_initial_channel=256, upsample_rates=[1, 1, 1, 1],
                 upsample_kernel_sizes=[1, 1, 1, 1])


def engine(make, monkeypatch, tall, fused=True):
    for var, on in (("AGPT_TALL_TILES", tall), ("AGPT_FUSE_RESBLOCK", fused)):
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


def bigvgan(h, seed):
    def make():
        from audiogpt_b200.vocoder.bigvgan.models import BigVGAN
        m = BigVGAN(h)
        m.load_state_dict(specs.synth_bigvgan(h, seed), strict=True)
        return m
    return make


def profiled(m, mel):
    """(waveform, profiled tap-GEMM launches, of those with 256-row tiles, library launches) of one forward."""
    L = _lib.lib()
    _lib.check(L.agpt_profile_enable(1))
    n0 = _lib.launch_count()
    wav = m(mel)
    torch.cuda.synchronize()
    buf = ctypes.create_string_buffer(1 << 20)
    L.agpt_profile_dump(buf, 1 << 20)
    tall = L.agpt_profile_tall_launches()
    _lib.check(L.agpt_profile_enable(0))
    return wav, len(buf.value.decode().splitlines()), tall, _lib.launch_count() - n0


def compare(make, monkeypatch, mel, fused=True):
    """Tall and 128-row engines on the same input: identical waveforms and launches; returns the tall launch count."""
    short = engine(make, monkeypatch, tall=False, fused=fused)
    tall = engine(make, monkeypatch, tall=True, fused=fused)
    ws, ns, ts, ls = profiled(short, mel)
    wt, nt, tt, lt = profiled(tall, mel)
    print(f"{tuple(mel.shape)} fused={fused}: {nt} tap-GEMM launches, {tt} with 256-row tiles")
    assert ts == 0 and ns == nt and ls == lt
    assert torch.isfinite(wt).all()
    assert torch.equal(wt, ws), (wt - ws).abs().max().item()
    return tt


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("T", [1, 245, 246, 250, 254, 255, 256, 257, 511])
def test_tall_tiles_bit_identical_ragged_fused(T, monkeypatch):
    # a batch of 4 x SMs samples: even a one-tile stage then has a grid the tall tiles are allowed for
    mel = specs.synth_tensor((4 * sms(), 80, T), seed=500 + T, scale=2.0, shift=-4.0).cuda()
    assert compare(hifigan(H256_FLAT, 79), monkeypatch, mel) > 0


@pytest.mark.parametrize("T", [1, 256, 257, 511])
def test_tall_tiles_bit_identical_ragged_unfused(T, monkeypatch):
    """AGPT_FUSE_RESBLOCK=0: every conv through tcconv5_kernel, with the residual and MRF-accumulate epilogues."""
    mel = specs.synth_tensor((4 * sms(), 80, T), seed=600 + T, scale=2.0, shift=-4.0).cuda()
    assert compare(hifigan(H256_FLAT, 80), monkeypatch, mel, fused=False) > 0


def test_tall_tiles_v1_full_size(monkeypatch):
    mel = specs.synth_tensor((8, 80, 800), seed=0, scale=2.0, shift=-4.0).cuda()
    assert compare(hifigan(specs.HIFIGAN_V1, 1234), monkeypatch, mel) > 0


@pytest.mark.parametrize("B,T", [(2, 100), (4, 800)])
def test_tall_tiles_bigvgan_base(B, T, monkeypatch):
    mel = specs.synth_tensor((B, 80, T), seed=7, scale=2.0, shift=-4.0).cuda()
    tall = compare(bigvgan(specs.BIGVGAN_BASE, 4321), monkeypatch, mel)
    # the widest grid is the last stage's (C = 32, 256 T rows per sample): B T tiles of 256 rows.  At 2 x 100 frames that
    # is below the 4 x SMs tiles the tall tiles need, so every launch stays at 128 rows
    assert (tall > 0) == (B * T >= 4 * sms())
