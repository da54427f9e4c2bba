"""Fused ResBlock pairs of the narrow HiFi-GAN stages as two 128-row CTAs per SM (tcpair2_kernel).  The kernel runs
the same tile body as tcpair_kernel<BN, 128>: every output row accumulates the same products in the same order, so
an engine created with AGPT_PAIR_DUAL=0 must give the same waveform bit for bit, with the same launches."""
import ctypes

import numpy as np
import pytest
import torch

from audiogpt_b200 import _lib, specs
from audiogpt_b200.modules.hifigan.hifigan import HifiGanGenerator

pytestmark = pytest.mark.gpu
# C0 = 128: stages of C = 64 / 32 / 16 / 8 at T rows each (upsample rates of 1), so T places every stage's length
# below one tile and around the 126 / 122 / 118-row strides of the 128-row pairs (k = 3 / 7 / 11)
H128_FLAT = dict(specs.HIFIGAN_SMALL, upsample_initial_channel=128, upsample_rates=[1, 1, 1, 1],
                 upsample_kernel_sizes=[1, 1, 1, 1])


def engine(make, monkeypatch, dual, fused=True):
    for var, on in (("AGPT_PAIR_DUAL", dual), ("AGPT_FUSE_RESBLOCK", fused)):
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
    """(waveform, profiled tap-GEMM launches, of those two CTAs per SM, library launches) of one forward."""
    L = _lib.lib()
    _lib.check(L.agpt_profile_enable(1))
    n0 = _lib.launch_count()
    wav = run()
    torch.cuda.synchronize()
    buf = ctypes.create_string_buffer(1 << 20)
    L.agpt_profile_dump(buf, 1 << 20)
    dual = L.agpt_profile_dual_launches()
    _lib.check(L.agpt_profile_enable(0))
    return wav, len(buf.value.decode().splitlines()), dual, _lib.launch_count() - n0


def compare(make, monkeypatch, run, fused=True):
    """Engines with and without two-CTA pairs on the same input: identical waveforms and launches; returns the
    number of two-CTA launches."""
    ref = engine(make, monkeypatch, dual=False, fused=fused)
    du = engine(make, monkeypatch, dual=True, fused=fused)
    wr, nr, dr, lr = profiled(lambda: run(ref))
    wd, nd, dd, ld = profiled(lambda: run(du))
    print(f"fused={fused}: {nd} tap-GEMM launches, {dd} with two CTAs per SM")
    assert dr == 0 and nr == nd and lr == ld
    assert torch.isfinite(wd).all()
    assert torch.equal(wd, wr), (wd - wr).abs().max().item()
    return dd


@pytest.mark.parametrize("T", [1, 117, 118, 119, 122, 126, 127, 128, 244, 300])
def test_dual_bit_identical_ragged_fused(T, monkeypatch):
    mel = specs.synth_tensor((3, 80, T), seed=900 + T, scale=2.0, shift=-4.0).cuda()
    # the 4 stages x 9 pairs, less the time-grouped ones (d = 1: C = 32 at k = 7 / 11 in groups of 4 rows, C = 64 at
    # k = 11 in groups of 2), which are taken where the groups divide the stage length
    grouped = 2 * (T % 4 == 0) + (T % 2 == 0)
    assert compare(hifigan(H128_FLAT, 82), monkeypatch, lambda m: m(mel)) == 4 * 9 - grouped


@pytest.mark.parametrize("T", [1, 127, 300])
def test_dual_unfused_unchanged(T, monkeypatch):
    """AGPT_FUSE_RESBLOCK=0: no pair is fused, so the switch changes nothing."""
    mel = specs.synth_tensor((3, 80, T), seed=950 + T, scale=2.0, shift=-4.0).cuda()
    assert compare(hifigan(H128_FLAT, 83), monkeypatch, lambda m: m(mel), fused=False) == 0


def test_dual_v1_full_size(monkeypatch):
    """V1 at 8 x 800: the ungrouped pairs of the C = 64 and C = 32 stages (2 x 9 less 3 time-grouped)."""
    mel = specs.synth_tensor((8, 80, 800), seed=0, scale=2.0, shift=-4.0).cuda()
    assert compare(hifigan(specs.HIFIGAN_V1, 1234), monkeypatch, lambda m: m(mel)) == 2 * 9 - 3


def test_dual_nsf_har_source(monkeypatch):
    """NSF: the excitation is added to X before the pairs read it."""
    h = dict(specs.HIFIGAN_V1, use_pitch_embed=True, audio_sample_rate=24000)
    B, T = 2, 40
    mel = specs.synth_tensor((B, 80, T), seed=12, scale=2.0, shift=-4.0).cuda()
    har = torch.tensor(np.random.RandomState(4).uniform(-1, 1, (B, T * 256)), dtype=torch.float32).cuda()

    def run(m):
        m._build_engine(mel.device)
        wav = torch.empty((B, 1, T * 256), device="cuda")
        _lib.check(_lib.lib().agpt_hifigan_forward(m._h, _lib.fptr(mel), _lib.fptr(har), B, T, _lib.fptr(wav),
                                                   _lib.cur_stream()))
        return wav

    assert compare(hifigan(h, 5679), monkeypatch, run) == 2 * 9 - 3
