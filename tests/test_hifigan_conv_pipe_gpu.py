"""HiFi-GAN's plane-fed single convs and upsamplers on the persistent tile pipeline (tcconv_pipe_pl_kernel).
The kernel sums the same wgmma products in the same order as tcconv5_pl_kernel<128, 128> and runs the same epilogue
arithmetic, so an engine created with AGPT_CONV_PIPE=0 must give the same waveform bit for bit, with the same
launches."""
import ctypes
import math

import numpy as np
import pytest
import torch

from audiogpt_b200 import _lib, specs
from audiogpt_b200.modules.hifigan.hifigan import HifiGanGenerator

pytestmark = pytest.mark.gpu


def engine(make, monkeypatch, pipe):
    if pipe:
        monkeypatch.delenv("AGPT_CONV_PIPE", raising=False)
    else:
        monkeypatch.setenv("AGPT_CONV_PIPE", "0")
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
    """(waveform, profiled tap-GEMM launches, plane-fed launches, of those on the pipeline, library launches) of one
    forward."""
    L = _lib.lib()
    _lib.check(L.agpt_profile_enable(1))
    n0 = _lib.launch_count()
    wav = run()
    torch.cuda.synchronize()
    buf = ctypes.create_string_buffer(1 << 20)
    L.agpt_profile_dump(buf, 1 << 20)
    plane = L.agpt_profile_plane_launches()
    pipe = L.agpt_profile_conv_pipe_launches()
    _lib.check(L.agpt_profile_enable(0))
    return wav, len(buf.value.decode().splitlines()), plane, pipe, _lib.launch_count() - n0


def compare(make, monkeypatch, runs):
    """Engines with and without the pipeline, each forward of `runs` on both: identical waveforms and launches.
    Returns the number of pipeline launches per forward."""
    ref = engine(make, monkeypatch, pipe=False)
    new = engine(make, monkeypatch, pipe=True)
    counts = []
    for run in runs:
        wr, nr, plr, pr, lr = profiled(lambda: run(ref))
        wn, nn, pln, pn, ln = profiled(lambda: run(new))
        print(f"{nn} tap-GEMM launches, {pln} plane-fed, {pn} on the pipeline")
        assert pr == 0 and nr == nn and plr == pln and lr == ln
        assert torch.isfinite(wn).all()
        assert torch.equal(wn, wr), (wn - wr).abs().max().item()
        counts.append(pn)
    return counts


def v1_pipe(B, T):
    """Pipeline launches of V1 (upsample rates 8, 8, 2, 2) on B x T frames: ups[0] (512 -> 8 x 256 channels over T rows),
    the 18 convs of the C = 256 stage and ups[1] (256 -> 8 x 128) over 8 T rows, each where pick_h_tile keeps 128-wide
    tiles: the width with the fewest waves x per-tile cost (128: 1.0, 96: 0.82, 64: 0.62) on this GPU's SMs."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cost = {128: 1.0, 64: 0.62, 96: 0.82}

    def wide(rows, cout):
        rt = math.ceil(rows / 128) * B
        score = {bn: math.ceil(rt * math.ceil(cout / bn) / sms) * cost[bn] for bn in cost}
        return all(score[128] <= score[bn] + 1e-9 for bn in (64, 96))
    return int(wide(T, 2048)) + 18 * int(wide(8 * T, 256)) + int(wide(8 * T, 1024))


@pytest.mark.parametrize("B,T", [(1, 1), (3, 5), (2, 131), (1, 1601), (3, 777)])
def test_conv_pipe_bit_identical_ragged(B, T, monkeypatch):
    """Partial last row tiles (8 T rows that are not a multiple of 128) and B = 1.  Launches of fewer units than SMs
    (1 x 1, 3 x 5, 2 x 131) get 64-wide tiles from pick_h_tile and keep tcconv5_pl_kernel.  1 x 1601: 202 units of the
    C = 256 convs, a last round too full to split; 3 x 777: 294 units, 2 per CTA and a last round of 30 units as 60
    half-units (3 per CTA)."""
    mel = specs.synth_tensor((B, 80, T), seed=900 + T, scale=2.0, shift=-4.0).cuda()
    assert compare(hifigan(specs.HIFIGAN_V1, 91), monkeypatch, [lambda m: m(mel)]) == [v1_pipe(B, T)]


def test_conv_pipe_v1_full_size(monkeypatch):
    """V1 at 8 x 800: 800 units of the C = 256 convs (6 per CTA, 8 more run as 16 half-units: odd and even counts per
    CTA), 896 of ups[0] (with its output plane) and 3200 of ups[1] (without); EPI_ACC with and without the old sum."""
    mel = specs.synth_tensor((8, 80, 800), seed=0, scale=2.0, shift=-4.0).cuda()
    assert compare(hifigan(specs.HIFIGAN_V1, 1234), monkeypatch, [lambda m: m(mel)]) == [20]


def test_conv_pipe_two_shapes_one_handle(monkeypatch):
    """Two forwards of different batch and length on the same handles."""
    a = specs.synth_tensor((2, 80, 1000), seed=92, scale=2.0, shift=-4.0).cuda()
    b = specs.synth_tensor((5, 80, 130), seed=93, scale=2.0, shift=-4.0).cuda()
    got = compare(hifigan(specs.HIFIGAN_V1, 94), monkeypatch, [lambda m: m(a), lambda m: m(b)])
    assert got == [v1_pipe(2, 1000), v1_pipe(5, 130)]


def test_conv_pipe_nsf_har_source(monkeypatch):
    """NSF: the upsamplers write no output plane; the excitation is added to X and split before the convs read it."""
    h = dict(specs.HIFIGAN_V1, use_pitch_embed=True, audio_sample_rate=24000)
    B, T = 2, 800
    mel = specs.synth_tensor((B, 80, T), seed=12, scale=2.0, shift=-4.0).cuda()
    har = torch.tensor(np.random.RandomState(5).uniform(-1, 1, (B, T * 256)), dtype=torch.float32).cuda()

    def run(m):
        m._build_engine(mel.device)
        wav = torch.empty((B, 1, T * 256), device="cuda")
        _lib.check(_lib.lib().agpt_hifigan_forward(m._h, _lib.fptr(mel), _lib.fptr(har), B, T, _lib.fptr(wav),
                                                   _lib.cur_stream()))
        return wav

    assert compare(hifigan(h, 5681), monkeypatch, [run]) == [v1_pipe(B, T)]
