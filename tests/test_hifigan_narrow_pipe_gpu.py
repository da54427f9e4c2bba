"""Narrow fused ResBlock pairs (C <= 64) on the persistent, warp-specialised tile pipeline (tcpair_narrow_kernel).
The kernel sums the same wgmma products in the same order as tcpair2_kernel / tcpair_kernel<BN, 128>, and runs the
same hand-off and epilogue arithmetic, so an engine created with AGPT_NARROW_PIPE=0 must give the same waveform bit
for bit, with the same launches."""
import ctypes

import numpy as np
import pytest
import torch

from audiogpt_b200 import _lib, specs
from audiogpt_b200.modules.hifigan.hifigan import HifiGanGenerator

pytestmark = pytest.mark.gpu
# C0 = 128: stages of C = 64 / 32 / 16 / 8 at T rows each (upsample rates of 1)
H128_FLAT = dict(specs.HIFIGAN_SMALL, upsample_initial_channel=128, upsample_rates=[1, 1, 1, 1],
                 upsample_kernel_sizes=[1, 1, 1, 1])


def engine(make, monkeypatch, narrow):
    if narrow:
        monkeypatch.delenv("AGPT_NARROW_PIPE", raising=False)
    else:
        monkeypatch.setenv("AGPT_NARROW_PIPE", "0")
    m = make().eval().to("cuda")
    m(torch.zeros(1, 80, 2, device="cuda"))   # the handle reads the switch when it is created
    return m


def hifigan(h, seed):
    def make():
        m = HifiGanGenerator(h)
        m.load_state_dict(specs.synth_hifigan(h, seed), strict=True)
        return m
    return make


def profiled(run):
    """(waveform, profiled tap-GEMM launches, narrow pairs with overlapped tiles, of those on the pipeline, library
    launches) of one forward."""
    L = _lib.lib()
    _lib.check(L.agpt_profile_enable(1))
    n0 = _lib.launch_count()
    wav = run()
    torch.cuda.synchronize()
    buf = ctypes.create_string_buffer(1 << 20)
    L.agpt_profile_dump(buf, 1 << 20)
    dual = L.agpt_profile_dual_launches()
    narrow = L.agpt_profile_narrow_pipe_launches()
    _lib.check(L.agpt_profile_enable(0))
    return wav, len(buf.value.decode().splitlines()), dual, narrow, _lib.launch_count() - n0


def compare(make, monkeypatch, runs):
    """Engines with and without the narrow pipeline, each forward of `runs` on both: identical waveforms and launches.
    Returns the number of pipeline launches per forward."""
    ref = engine(make, monkeypatch, narrow=False)
    new = engine(make, monkeypatch, narrow=True)
    counts = []
    for run in runs:
        wr, nr, dr, pr, lr = profiled(lambda: run(ref))
        wn, nn, dn, pn, ln = profiled(lambda: run(new))
        print(f"{nn} tap-GEMM launches, {dn} narrow pairs with overlapped tiles, {pn} on the pipeline")
        assert pr == 0 and nr == nn and dr == dn and lr == ln
        assert torch.isfinite(wn).all()
        assert torch.equal(wn, wr), (wn - wr).abs().max().item()
        counts.append(pn)
    return counts


def flat_pipe(T):
    # the ungrouped pairs (as in test_hifigan_dual_gpu.py) less C = 64's k = 11 pairs, which keep tcpair2_kernel: at
    # C = 64 the pipeline takes k = 3 and 7, at C <= 32 every pair (the dilation-1 ones at k = 7 / 11 unless grouped)
    return 6 + 3 * 9 - 2 * (T % 4 == 0)


V1_PIPE = 6 + 9 - 2   # C = 64 at k = 3 / 7, C = 32 less its two time-grouped pairs


@pytest.mark.parametrize("T", [1, 5, 117, 118, 119, 122, 126, 127, 246, 250, 254, 255, 300])
def test_narrow_pipe_bit_identical_ragged(T, monkeypatch):
    """Stage lengths around the 126 / 122 / 118-row strides and two of them; grids of fewer tiles than SMs."""
    mel = specs.synth_tensor((3, 80, T), seed=700 + T, scale=2.0, shift=-4.0).cuda()
    assert compare(hifigan(H128_FLAT, 82), monkeypatch, [lambda m: m(mel)]) == [flat_pipe(T)]


def test_narrow_pipe_many_tiles_per_cta(monkeypatch):
    """3 x 27 715 rows: 660 tiles of the k = 3 pairs (5 per CTA) and 684 / 705 of k = 7 / 11 (5 or 6), so every CTA
    walks more tiles than it has sets, with odd and even counts per wgmma warpgroup, which exercises the set parities,
    the barrier phases and the shared weight ring's unused last pass."""
    T = 27715
    mel = specs.synth_tensor((3, 80, T), seed=71, scale=2.0, shift=-4.0).cuda()
    assert compare(hifigan(H128_FLAT, 84), monkeypatch, [lambda m: m(mel)]) == [flat_pipe(T)]


def test_narrow_pipe_two_shapes_one_handle(monkeypatch):
    """Two forwards of different batch and length on the same handles."""
    a = specs.synth_tensor((2, 80, 333), seed=72, scale=2.0, shift=-4.0).cuda()
    b = specs.synth_tensor((5, 80, 130), seed=73, scale=2.0, shift=-4.0).cuda()
    got = compare(hifigan(H128_FLAT, 85), monkeypatch, [lambda m: m(a), lambda m: m(b)])
    assert got == [flat_pipe(333), flat_pipe(130)]


def test_narrow_pipe_v1_full_size(monkeypatch):
    """V1 at 8 x 800: of the 15 ungrouped pairs of the C = 64 and C = 32 stages, all but C = 64's two k = 11 ones run
    on the pipeline."""
    mel = specs.synth_tensor((8, 80, 800), seed=0, scale=2.0, shift=-4.0).cuda()
    assert compare(hifigan(specs.HIFIGAN_V1, 1234), monkeypatch, [lambda m: m(mel)]) == [V1_PIPE]


def test_narrow_pipe_nsf_har_source(monkeypatch):
    """NSF: the excitation is added to X before the pairs read it."""
    h = dict(specs.HIFIGAN_V1, use_pitch_embed=True, audio_sample_rate=24000)
    B, T = 2, 40
    mel = specs.synth_tensor((B, 80, T), seed=12, scale=2.0, shift=-4.0).cuda()
    har = torch.tensor(np.random.RandomState(5).uniform(-1, 1, (B, T * 256)), dtype=torch.float32).cuda()

    def run(m):
        m._build_engine(mel.device)
        wav = torch.empty((B, 1, T * 256), device="cuda")
        _lib.check(_lib.lib().agpt_hifigan_forward(m._h, _lib.fptr(mel), _lib.fptr(har), B, T, _lib.fptr(wav),
                                                   _lib.cur_stream()))
        return wav

    assert compare(hifigan(h, 5680), monkeypatch, [run]) == [V1_PIPE]
