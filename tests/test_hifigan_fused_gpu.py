"""Fused ResBlock1 pairs (tcpair_kernel): x + c2(lrelu(c1(lrelu(x)))) as one launch, c1's output kept in shared
memory.  An engine created with AGPT_FUSE_RESBLOCK=0 issues every conv as its own launch; both engines must agree
with each other and with the CPU oracle."""
import ctypes

import pytest
import torch

from audiogpt_b200 import _lib, specs
from audiogpt_b200.modules.hifigan.hifigan import HifiGanGenerator
from conftest import rmse

pytestmark = pytest.mark.gpu
RMSE_TOL = 2e-5
# stages of C = 128 / 64 / 32 / 16 with k in {3, 7, 11}, d in {1, 3, 5}: every pair shape the fused kernel takes
H256 = dict(specs.HIFIGAN_SMALL, upsample_initial_channel=256)


def engine(h, seed, monkeypatch, fused):
    if fused:
        monkeypatch.delenv("AGPT_FUSE_RESBLOCK", raising=False)
    else:
        monkeypatch.setenv("AGPT_FUSE_RESBLOCK", "0")
    m = HifiGanGenerator(h)
    m.load_state_dict(specs.synth_hifigan(h, seed), strict=True)
    m = m.eval().to("cuda")
    m(torch.zeros(1, 80, 2, device="cuda"))   # the handle reads the switch when it is created
    return m


def profiled(m, mel):
    """(waveform, tap-GEMM launches, fused-pair launches) of one forward."""
    L = _lib.lib()
    _lib.check(L.agpt_profile_enable(1))
    n0 = _lib.launch_count()
    wav = m(mel)
    torch.cuda.synchronize()
    buf = ctypes.create_string_buffer(1 << 20)
    L.agpt_profile_dump(buf, 1 << 20)
    _lib.check(L.agpt_profile_enable(0))
    lines = buf.value.decode().splitlines()
    pairs = sum(1 for line in lines if int(line.split()[7]) >= 16)   # record epi code 16 + c2's epilogue
    return wav, len(lines), pairs, _lib.launch_count() - n0


RAGGED = [(1, 1), (1, 7), (3, 33), (2, 129)]   # stage lengths below one tile and off the 118 / 122 / 126 strides


@pytest.mark.parametrize("B,Tn", RAGGED)
def test_fused_pairs_match_unfused_and_oracle(B, Tn, monkeypatch):
    from oracle import hifigan_ref as hr
    unfused = engine(H256, 77, monkeypatch, fused=False)
    fused = engine(H256, 77, monkeypatch, fused=True)
    mel = specs.synth_tensor((B, 80, Tn), seed=200 + Tn, scale=2.0, shift=-4.0)
    wf, nf, pairs, _ = profiled(fused, mel.cuda())
    wu, nu, pairs_u, _ = profiled(unfused, mel.cuda())
    assert pairs > 0 and pairs_u == 0 and nu - nf == pairs
    ref = hr.hifigan_forward(specs.synth_hifigan(H256, 77), H256, mel)
    ef, eu = rmse(wf.cpu(), ref), rmse(wu.cpu(), ref)
    d = (wf - wu).abs().max().item()
    print(f"B={B} T={Tn}: {pairs} fused pairs, RMSE vs oracle fused {ef:.2e} unfused {eu:.2e}, max diff {d:.2e}")
    assert ef < RMSE_TOL and eu < RMSE_TOL
    # the dilated c1 -> time-grouped c2 pairs run c2 ungrouped when fused: a different summation order
    assert d < 1e-5


@pytest.mark.parametrize("B,Tn", RAGGED)
def test_fused_pairs_same_views_bit_identical(B, Tn, monkeypatch):
    """Dilation 1 everywhere for k = 7 / 11: every fused pair runs the views of the launches it replaces (plain rows,
    or both convs time-grouped), so the fused engine multiplies the same operands in the same order."""
    h = dict(H256, resblock_dilation_sizes=[[1, 3, 5], [1, 1, 1], [1, 1, 1]])
    unfused = engine(h, 78, monkeypatch, fused=False)
    fused = engine(h, 78, monkeypatch, fused=True)
    mel = specs.synth_tensor((B, 80, Tn), seed=300 + Tn, scale=2.0, shift=-4.0).cuda()
    wf, nf, pairs, _ = profiled(fused, mel)
    wu, nu, _, _ = profiled(unfused, mel)
    assert pairs > 0 and nu - nf == pairs
    assert torch.equal(wf, wu), (wf - wu).abs().max().item()


def test_v1_full_size_fused_vs_unfused(monkeypatch):
    unfused = engine(specs.HIFIGAN_V1, 1234, monkeypatch, fused=False)
    fused = engine(specs.HIFIGAN_V1, 1234, monkeypatch, fused=True)
    mel = specs.synth_tensor((8, 80, 800), seed=0, scale=2.0, shift=-4.0).cuda()
    wf, nf, pairs, lf = profiled(fused, mel)
    wu, nu, _, lu = profiled(unfused, mel)
    d = (wf - wu).abs().max().item()
    print(f"V1 8x800: {nu} -> {nf} tap-GEMM launches ({pairs} fused pairs), max |fused - unfused| = {d:.3e}")
    assert torch.isfinite(wf).all() and torch.isfinite(wu).all()
    assert pairs > 0 and nu - nf == pairs and lu - lf == pairs
    assert d < 1e-4
