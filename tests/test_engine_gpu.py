"""The engine lifecycle every drop-in shares (audiogpt_b200._lib.Engine): a handle is rebuilt exactly when a weight it
was built from changes, and every agpt_*_create rejects a wrong weight count without handing out a handle."""
import ctypes as C

import pytest
import torch

from audiogpt_b200 import _lib, paramtree, specs

pytestmark = pytest.mark.gpu


def _hifigan():
    from test_hifigan_gpu import build
    m = build(specs.HIFIGAN_SMALL, 1234)
    return m, m._engine, "conv_post.bias", lambda: m(specs.synth_tensor((1, 80, 8), seed=1).cuda())


def _bigvgan():
    from test_bigvgan_gpu import _model
    m = _model(specs.BIGVGAN_SMALL)
    return m, m._engine, "conv_post.bias", lambda: m(specs.synth_tensor((1, 80, 8), seed=1).cuda())


def _diffnet():
    from test_diffusion_gpu import make
    net = make(specs.DIFFNET_SMALL, 2024).denoise_fn
    x = specs.synth_tensor((2, 1, 80, 9), seed=1).cuda()
    cond = specs.synth_tensor((2, specs.DIFFNET_SMALL["hidden_size"], 9), seed=2).cuda()
    return net, net._engine, "output_projection.bias", lambda: net(x, [3, 7], cond)


def _unet():
    from test_ldm_gpu import build
    u = build(specs.UNET_SMALL, 4040)
    x = specs.synth_tensor((2, 4, 6, 10), seed=1).cuda()
    ctx = specs.synth_tensor((2, 7, specs.UNET_SMALL["context_dim"]), seed=2).cuda()
    return u, u._engine, "out.2.bias", lambda: u(x, [5, 900], ctx)


def _vae_decoder():
    from test_vae_gpu import build
    m, _ = build(specs.VAE_SMALL)
    return m, m._engine, "decoder.conv_out.bias", lambda: m.decode(specs.synth_tensor((1, 4, 10, 78), seed=3).cuda())


def _vae_encoder():
    from test_vae_encoder_gpu import build, mel
    m, _ = build(specs.VAE_SMALL)
    return m, m._enc_engine, "quant_conv.bias", lambda: m.encode(mel(1).cuda()).parameters


def _pitch_extractor():
    from test_pe_gpu import build
    pe, _ = build(specs.PE_SMALL)
    mel = specs.synth_tensor((2, 37, 80), seed=71, scale=1.0, shift=-2.5).cuda()
    return pe, pe._engine, "pitch_predictor.linear.bias", lambda: pe(mel)["pitch_pred"]


def _fastspeech2():
    from test_fs2_gpu import build
    m, _ = build(specs.FS2_SMALL)
    tok = torch.tensor([[5, 9, 13, 21, 2, 0]], device="cuda")
    mel2ph = torch.tensor([[1, 1, 2, 3, 3, 3, 4, 5, 0]], device="cuda")
    return m, m._engine, "mel_out.bias", lambda: m(tok, mel2ph=mel2ph)["mel_out"]


ENGINES = [_hifigan, _bigvgan, _diffnet, _unet, _vae_decoder, _vae_encoder, _pitch_extractor, _fastspeech2]


@pytest.mark.parametrize("make", ENGINES, ids=lambda f: f.__name__[1:])
def test_rebuild_policy(make):
    """unchanged weights keep the handle; an in-place edit of one uploaded weight reaches the next output"""
    m, engine, key, run = make()
    y0 = run().clone()
    h0 = engine.h.value
    assert h0
    assert torch.equal(run(), y0) and engine.h.value == h0
    with torch.no_grad():
        paramtree.get_tensor(m, key).add_(0.5)
    assert not torch.equal(run(), y0)


@pytest.mark.parametrize("make", ENGINES, ids=lambda f: f.__name__[1:])
def test_create_rejects_wrong_weight_count(make, monkeypatch):
    """one weight array too few or too many: a non-zero return with the weight cursor's message, and no handle"""
    builds = []
    ensure = _lib.Engine.ensure
    monkeypatch.setattr(_lib.Engine, "ensure", lambda self, device, sources, build: builds.append((self, build)) or
                        ensure(self, device, sources, build))
    _, engine, _, run = make()
    run()
    build = [b for e, b in builds if e is engine][0]
    args, weights = build()
    L = _lib.lib()
    for ws, msg in ((weights[:-1], b"too few weight arrays"),
                    (weights + weights[-1:], b"weight array count does not match the config")):
        arr, keep = _lib.host_weight_array(ws)
        h = C.c_void_p()
        rc = getattr(L, engine.create)(*args, arr, len(keep), torch.cuda.current_device(), C.byref(h))
        assert rc != 0 and msg in L.agpt_last_error(), (engine.create, L.agpt_last_error())
        assert not h.value


def test_hifigan_bad_channel_count_raises():
    """the channel check of the second upsample stage fails before anything is uploaded"""
    from audiogpt_b200.modules.hifigan.hifigan import HifiGanGenerator
    m = HifiGanGenerator(dict(specs.HIFIGAN_SMALL, upsample_initial_channel=72)).cuda()
    with pytest.raises(RuntimeError, match="multiples of 4"):
        m(torch.zeros(1, 80, 8, device="cuda"))
    assert not m._h.value
