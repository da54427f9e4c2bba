"""Fused ResBlock pairs of 128 -> 128 channels with two tiles in flight per CTA (tcpair_pipe_kernel).  Each output row
sums the same wgmma products in the same order, and runs the same epilogue, as on tcpair_kernel<128, 128>, so an engine
created with AGPT_PAIR_PIPE=0 must give the same waveform bit for bit, with the same launches."""
import ctypes

import numpy as np
import pytest
import torch

from audiogpt_b200 import _lib, specs
from audiogpt_b200.modules.hifigan.hifigan import HifiGanGenerator

pytestmark = pytest.mark.gpu
# C0 = 256: stages of C = 128 / 64 / 32 / 16 at T rows each (upsample rates of 1), so T places the C = 128 stage below
# one tile, around the 126 / 122 / 118-row strides of the k = 3 / 7 / 11 pairs, and at fewer tiles than SMs
H256_FLAT = dict(specs.HIFIGAN_SMALL, upsample_initial_channel=256, upsample_rates=[1, 1, 1, 1],
                 upsample_kernel_sizes=[1, 1, 1, 1])


def engine(make, monkeypatch, pipe, fused=True):
    for var, on in (("AGPT_PAIR_PIPE", pipe), ("AGPT_FUSE_RESBLOCK", fused)):
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
    """(waveform, profiled tap-GEMM launches, of those two tiles per CTA, library launches) of one forward."""
    L = _lib.lib()
    _lib.check(L.agpt_profile_enable(1))
    n0 = _lib.launch_count()
    wav = run()
    torch.cuda.synchronize()
    buf = ctypes.create_string_buffer(1 << 20)
    L.agpt_profile_dump(buf, 1 << 20)
    pipe = L.agpt_profile_pipe_launches()
    _lib.check(L.agpt_profile_enable(0))
    return wav, len(buf.value.decode().splitlines()), pipe, _lib.launch_count() - n0


def compare(make, monkeypatch, run, fused=True):
    """Engines with and without the two-tile pipeline on the same input: identical waveforms and launches; returns the
    number of two-tile launches."""
    ref = engine(make, monkeypatch, pipe=False, fused=fused)
    pi = engine(make, monkeypatch, pipe=True, fused=fused)
    wr, nr, pr, lr = profiled(lambda: run(ref))
    wp, npp, pp, lp = profiled(lambda: run(pi))
    print(f"fused={fused}: {npp} tap-GEMM launches, {pp} with two tiles per CTA")
    assert pr == 0 and nr == npp and lr == lp
    assert torch.isfinite(wp).all()
    assert torch.equal(wp, wr), (wp - wr).abs().max().item()
    return pp


@pytest.mark.parametrize("T", [1, 117, 118, 119, 122, 126, 127, 128, 244, 300, 400])
def test_pipe_bit_identical_ragged_fused(T, monkeypatch):
    mel = specs.synth_tensor((3, 80, T), seed=700 + T, scale=2.0, shift=-4.0).cuda()
    # at least the C = 128 stage's pairs but k = 11 at dilation 5, whose operand sets do not fit shared memory
    assert compare(hifigan(H256_FLAT, 71), monkeypatch, lambda m: m(mel)) >= 8


@pytest.mark.parametrize("T", [1, 127, 300])
def test_pipe_unfused_unchanged(T, monkeypatch):
    """AGPT_FUSE_RESBLOCK=0: no pair is fused, so the switch changes nothing."""
    mel = specs.synth_tensor((3, 80, T), seed=750 + T, scale=2.0, shift=-4.0).cuda()
    assert compare(hifigan(H256_FLAT, 72), monkeypatch, lambda m: m(mel), fused=False) == 0


def test_pipe_v1_full_size(monkeypatch):
    """V1 at 8 x 800: the C = 128 stage's pairs (and the time-grouped 128-channel views of narrower stages)."""
    mel = specs.synth_tensor((8, 80, 800), seed=0, scale=2.0, shift=-4.0).cuda()
    assert compare(hifigan(specs.HIFIGAN_V1, 1234), monkeypatch, lambda m: m(mel)) >= 8


def test_pipe_nsf_har_source(monkeypatch):
    """NSF: the excitation is added to X before the pairs read it."""
    h = dict(specs.HIFIGAN_V1, use_pitch_embed=True, audio_sample_rate=24000)
    B, T = 2, 40
    mel = specs.synth_tensor((B, 80, T), seed=13, scale=2.0, shift=-4.0).cuda()
    har = torch.tensor(np.random.RandomState(5).uniform(-1, 1, (B, T * 256)), dtype=torch.float32).cuda()

    def run(m):
        m._build_engine(mel.device)
        wav = torch.empty((B, 1, T * 256), device="cuda")
        _lib.check(_lib.lib().agpt_hifigan_forward(m._h, _lib.fptr(mel), _lib.fptr(har), B, T, _lib.fptr(wav),
                                                   _lib.cur_stream()))
        return wav

    assert compare(hifigan(h, 5680), monkeypatch, run) >= 8
