"""The C = 128 ResBlock-pair pipeline (tcpair_pipe_kernel) with its input and residual staged by TMA, against the same
pipeline with one data warpgroup loading them per thread (AGPT_PAIR_PIPE_STAGE=0).  Both run the same wgmma products
in the same order and the same epilogue float operations, so the waveforms must be equal bit for bit, with the same
launches."""
import ctypes

import numpy as np
import pytest
import torch

from audiogpt_b200 import _lib, specs
from audiogpt_b200.modules.hifigan.hifigan import HifiGanGenerator

pytestmark = pytest.mark.gpu
# C0 = 256: stages of C = 128 / 64 / 32 / 16 at T rows each (upsample rates of 1), so T sets the C = 128 stage's length
H256_FLAT = dict(specs.HIFIGAN_SMALL, upsample_initial_channel=256, upsample_rates=[1, 1, 1, 1],
                 upsample_kernel_sizes=[1, 1, 1, 1])


def engine(h, seed, monkeypatch, staged):
    if staged:
        monkeypatch.delenv("AGPT_PAIR_PIPE_STAGE", raising=False)
    else:
        monkeypatch.setenv("AGPT_PAIR_PIPE_STAGE", "0")
    monkeypatch.delenv("AGPT_PAIR_PIPE", raising=False)
    monkeypatch.delenv("AGPT_FUSE_RESBLOCK", raising=False)
    m = HifiGanGenerator(h)
    m.load_state_dict(specs.synth_hifigan(h, seed), strict=True)
    m = m.eval().to("cuda")
    m(torch.zeros(1, 80, 2, device="cuda"))   # the handle reads the switches when it is created
    return m


def profiled(run):
    """(waveform, profiled tap-GEMM launches, of those on the pair pipeline, library launches) of one forward."""
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


def compare(ref, new, run):
    wr, nr, pr, lr = profiled(lambda: run(ref))
    wn, nn, pn, ln = profiled(lambda: run(new))
    assert (nr, pr, lr) == (nn, pn, ln)
    assert torch.isfinite(wn).all()
    assert torch.equal(wn, wr), (wn - wr).abs().max().item()
    return pn


@pytest.fixture(scope="module")
def flat_mel():
    return lambda B, T, seed: specs.synth_tensor((B, 80, T), seed=seed, scale=2.0, shift=-4.0).cuda()


@pytest.mark.parametrize("T", [1, 117, 118, 119, 121, 122, 123, 125, 126, 127, 236, 244, 252, 253])
def test_stage_bit_identical_ragged(T, monkeypatch, flat_mel):
    """Stage lengths around the 126 / 122 / 118-row tile strides of the k = 3 / 7 / 11 pairs, all below one wave."""
    mel = flat_mel(3, T, 900 + T)
    ref = engine(H256_FLAT, 81, monkeypatch, staged=False)
    new = engine(H256_FLAT, 81, monkeypatch, staged=True)
    assert compare(ref, new, lambda m: m(mel)) >= 8


@pytest.mark.parametrize("T", [20000, 20130])
def test_stage_many_tiles_per_cta(T, monkeypatch, flat_mel):
    """4 x 20000 rows: 636 / 656 / 680 tiles of the k = 3 / 7 / 11 pairs, so CTAs walk 4 to 6 tiles each, odd and even
    counts in one launch, cycling both operand sets and the residual ring many times."""
    mel = flat_mel(4, T, 960 + T % 7)
    ref = engine(H256_FLAT, 82, monkeypatch, staged=False)
    new = engine(H256_FLAT, 82, monkeypatch, staged=True)
    assert compare(ref, new, lambda m: m(mel)) >= 8


def test_stage_two_shapes_one_handle(monkeypatch, flat_mel):
    """One handle, two shapes in turn: the plan and the tensor maps follow the shape of each forward."""
    ref = engine(H256_FLAT, 83, monkeypatch, staged=False)
    new = engine(H256_FLAT, 83, monkeypatch, staged=True)
    for B, T in ((2, 700), (5, 131), (2, 700)):
        mel = flat_mel(B, T, 970 + T)
        assert compare(ref, new, lambda m: m(mel)) >= 8


def test_stage_fewer_tiles_than_sms(monkeypatch, flat_mel):
    """One sample of 300 rows: 3 tiles per pair, so most CTAs of a launch would have none."""
    mel = flat_mel(1, 300, 990)
    ref = engine(H256_FLAT, 84, monkeypatch, staged=False)
    new = engine(H256_FLAT, 84, monkeypatch, staged=True)
    assert compare(ref, new, lambda m: m(mel)) >= 8


def test_stage_v1_full_size(monkeypatch):
    """V1 at 8 x 800: the C = 128 stage's pairs and the time-grouped 128-channel views of the narrower stages."""
    mel = specs.synth_tensor((8, 80, 800), seed=0, scale=2.0, shift=-4.0).cuda()
    ref = engine(specs.HIFIGAN_V1, 1234, monkeypatch, staged=False)
    new = engine(specs.HIFIGAN_V1, 1234, monkeypatch, staged=True)
    assert compare(ref, new, lambda m: m(mel)) >= 8


def test_stage_nsf_har_source(monkeypatch):
    """NSF: the excitation is added to X before the pairs read it."""
    h = dict(specs.HIFIGAN_V1, use_pitch_embed=True, audio_sample_rate=24000)
    B, T = 2, 40
    mel = specs.synth_tensor((B, 80, T), seed=17, scale=2.0, shift=-4.0).cuda()
    har = torch.tensor(np.random.RandomState(9).uniform(-1, 1, (B, T * 256)), dtype=torch.float32).cuda()

    def run(m):
        m._build_engine(mel.device)
        wav = torch.empty((B, 1, T * 256), device="cuda")
        _lib.check(_lib.lib().agpt_hifigan_forward(m._h, _lib.fptr(mel), _lib.fptr(har), B, T, _lib.fptr(wav),
                                                   _lib.cur_stream()))
        return wav

    ref = engine(h, 5690, monkeypatch, staged=False)
    new = engine(h, 5690, monkeypatch, staged=True)
    assert compare(ref, new, run) >= 8
