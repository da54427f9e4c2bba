"""AutoencoderKL.encode / forward on the GPU (through the C ABI) vs golden vectors made by the reference's own Encoder +
quant_conv and AutoencoderKL (tests/golden/make_golden_vae_enc.py) and vs the CPU oracle.  Stated tolerance: relative
RMSE <= 1e-4 on the moments and on the reconstruction, the decoder's gate (3 x fp16-part tensor-core products with fp32
accumulation; the attention GEMMs are fp32 FMA)."""
import pytest
import torch

from audiogpt_b200 import _lib, specs
from audiogpt_b200.ldm.models.autoencoder import AutoencoderKLWithEncoder
from conftest import load_golden, rel_rmse

pytestmark = pytest.mark.gpu


def build(cfg):
    m = AutoencoderKLWithEncoder(ddconfig={k: v for k, v in cfg.items() if k != "embed_dim"},
                                 lossconfig={"target": "torch.nn.Identity"}, embed_dim=cfg["embed_dim"])
    sd = dict(specs.synth_vae_encoder(cfg), **specs.synth_vae_decoder(cfg))
    m.load_state_dict(sd, strict=True)
    return m.eval().to("cuda"), sd


def mel(B):
    return specs.synth_masked_mel(2, 80, 848, 848)[:B]


@pytest.mark.parametrize("name,cfg,B", [("vae_enc_small", specs.VAE_SMALL, 2), ("vae_enc_txt2audio", specs.VAE_TXT2AUDIO, 1)])
def test_moments_vs_reference_and_oracle(name, cfg, B):
    from oracle import vae_enc_ref
    g = load_golden(name)
    m, sd = build(cfg)
    x = mel(B)
    post = m.encode(x.cuda())
    got = post.parameters.cpu()
    assert got.shape == (B, 2 * cfg["embed_dim"], 10, 106)
    e = rel_rmse(got, g["moments"])
    eo = rel_rmse(got, vae_enc_ref.vae_encode(sd, cfg, x))
    print(f"{name}: moments rel-RMSE vs reference {e:.3e}, vs oracle {eo:.3e}")
    assert e < 1e-4 and eo < 1e-4
    assert torch.equal(post.mode(), post.parameters[:, :cfg["embed_dim"]])


def test_forward_reconstruction_vs_reference():
    """AutoencoderKL.forward(x, sample_posterior=False) = decode(posterior.mode()) of the shipped config"""
    cfg = specs.VAE_TXT2AUDIO
    g = load_golden("vae_enc_txt2audio")
    m, _ = build(cfg)
    rec, post = m(mel(1).cuda(), sample_posterior=False)
    assert rec.shape == (1, 1, 80, 848)
    rec = rec.cpu()
    e = rel_rmse(rec[:, :, ::2, ::3], g["rec"])
    rd = rec.double()
    es = abs(float((rd * rd).sum()) - g["rec_stats"][2]) / g["rec_stats"][2]
    print(f"reconstruction rel-RMSE {e:.3e}  sum-of-squares rel {es:.3e}")
    assert e < 1e-4 and es < 1e-3


@pytest.mark.parametrize("B,H,W,tc", [(1, 9, 13, 1), (2, 40, 130, 1), (1, 80, 845, 1), (2, 40, 130, 0)])
def test_ragged_vs_oracle(B, H, W, tc):
    """odd sizes: one token at the bottom level (9x13), several ragged strips (845 columns), odd sizes at every
    Downsample; the last case runs every conv on the fp32-FMA kernel"""
    from oracle import vae_enc_ref
    cfg = specs.VAE_SMALL
    m, sd = build(cfg)
    x = specs.synth_tensor((B, 1, H, W), seed=200 + W).tanh()
    ref = vae_enc_ref.vae_encode(sd, cfg, x)
    L = _lib.lib()
    _lib.check(L.agpt_set_tensor_cores(tc))
    try:
        got = m.encode(x.cuda()).parameters.cpu()
    finally:
        _lib.check(L.agpt_set_tensor_cores(1))
    assert got.shape == ref.shape == (B, 8, H // 8, W // 8)
    e = rel_rmse(got, ref)
    print(f"vae_enc small {B}x1x{H}x{W} (tc={tc}): rel-RMSE vs oracle {e:.3e}")
    assert e < 1e-4


def test_batch_independence():
    m, _ = build(specs.VAE_SMALL)
    x = mel(2).cuda()
    both = m.encode(x).parameters
    one = m.encode(x[1:2]).parameters
    assert torch.allclose(one[0], both[1], atol=1e-5, rtol=1e-4)


def test_bad_inputs_raise():
    m, _ = build(specs.VAE_SMALL)
    for shape in ((1, 1, 7, 64), (1, 1, 64, 5)):        # would shrink to zero size at the bottom level (needs >= 8)
        with pytest.raises(RuntimeError, match="zero size"):
            m.encode(torch.zeros(shape, device="cuda"))
    with pytest.raises(RuntimeError, match="CUDA only"):
        m.encode(torch.zeros(1, 1, 16, 16))
    with pytest.raises(ValueError, match="in_channels|expected"):
        m.encode(torch.zeros(1, 2, 16, 16, device="cuda"))


def test_recorded_posterior_class():
    """with a posterior class recorded (install(first_stage=True) records the reference's), encode() returns it"""
    class Fake:
        def __init__(self, parameters):
            self.parameters = parameters

    m, _ = build(specs.VAE_SMALL)
    AutoencoderKLWithEncoder._posterior_cls = Fake
    try:
        p = m.encode(mel(1).cuda())
    finally:
        AutoencoderKLWithEncoder._posterior_cls = None
    assert type(p) is Fake and p.parameters.shape == (1, 8, 10, 106)


def test_engines_are_built_from_their_own_parameters():
    """decode() builds no encoder engine; new encoder weights rebuild the encoder engine only"""
    cfg = specs.VAE_SMALL
    m, _ = build(cfg)
    y = m.decode(specs.synth_tensor((1, 4, 10, 78), seed=3).cuda())
    assert y.shape == (1, 1, 80, 624)
    assert m._h.value and not m._enc_engine.h.value
    dec_h = m._h.value
    x = mel(1).cuda()
    a = m.encode(x).parameters
    enc_h = m._enc_engine.h.value
    assert enc_h and m._h.value == dec_h
    with torch.no_grad():
        m.quant_conv.bias.add_(1.0)
    b = m.encode(x).parameters
    assert m._h.value == dec_h and torch.allclose(b, a + 1.0, atol=1e-4)
    m.decode(specs.synth_tensor((1, 4, 10, 78), seed=3).cuda())
    assert m._h.value == dec_h
