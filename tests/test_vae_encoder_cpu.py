"""AutoencoderKL encoder side without a GPU: the CPU oracle pinned to the fixtures made by the reference's Encoder +
quant_conv (tests/golden/make_golden_vae_enc.py), the FLOP count, the full first-stage class's state-dict layout, the
drop-in posterior, and the opt-in graft of install(first_stage=True)."""
import math
import subprocess
import sys

import pytest
import torch

from audiogpt_b200 import specs
from conftest import ROOT, load_golden, rel_rmse

CASES = [("vae_enc_small", specs.VAE_SMALL, 2), ("vae_enc_txt2audio", specs.VAE_TXT2AUDIO, 1)]


def fixture_input(g, B):
    x = specs.synth_masked_mel(2, 80, 848, 848)[:B]
    xd = x.double()
    got = [xd.sum().item(), xd.abs().sum().item(), (xd * xd).sum().item()]
    assert all(abs(a - b) <= 1e-9 * abs(b) for a, b in zip(got, g["x_stats"])), "input generator drifted"
    return x


@pytest.mark.parametrize("name,cfg,B", CASES)
def test_oracle_matches_reference_fixture(name, cfg, B):
    from oracle import vae_enc_ref
    g = load_golden(name)
    x = fixture_input(g, B)
    # the masked band reaches the encoder as -1 (audio-chatgpt.py:440-444)
    assert (x[0, :, :, 254:395] == -1).all() and x.min() == -1 and x.max() <= 1
    m = vae_enc_ref.vae_encode(specs.synth_vae_encoder(cfg), cfg, x)
    assert m.shape == (B, 2 * cfg["embed_dim"], 10, 106) == g["moments"].shape
    e = rel_rmse(m, g["moments"])
    print(f"{name}: oracle moments rel-RMSE {e:.3e}")
    assert e < 1e-5


def test_encode_flops():
    from oracle.vae_enc_ref import vae_encode_flops
    cfg = specs.VAE_TXT2AUDIO
    assert abs(vae_encode_flops(cfg, 80, 848) / 275.3e9 - 1) < 0.01
    assert abs(vae_encode_flops(cfg, 80, 624) / 194.1e9 - 1) < 0.01
    n = sum(math.prod(s) for s in specs.vae_encoder_param_shapes(cfg).values())
    assert abs(n / 27.94e6 - 1) < 0.001


def _full(cfg):
    from audiogpt_b200.ldm.models.autoencoder import AutoencoderKLWithEncoder
    return AutoencoderKLWithEncoder(ddconfig={k: v for k, v in cfg.items() if k != "embed_dim"},
                                    lossconfig={"target": "torch.nn.Identity"}, embed_dim=cfg["embed_dim"])


def test_full_class_has_the_reference_state_dict():
    """AutoencoderKLWithEncoder's keys and shapes are the reference AutoencoderKL's (recorded from the reference
    module), a state dict with that layout loads strictly, and the key set is the union of the encoder and decoder
    tables."""
    cfg = specs.VAE_TXT2AUDIO
    g = load_golden("vae_enc_txt2audio")
    ref = {k: tuple(int(v) for v in s.split(",") if v) for k, s in zip(g["ref_keys"].tolist(), g["ref_shapes"].tolist())}
    m = _full(cfg)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == ref
    tables = dict(specs.vae_encoder_param_shapes(cfg), **specs.vae_decoder_param_shapes(cfg))
    assert set(tables) == set(ref)
    sd = dict(specs.synth_vae_encoder(cfg), **specs.synth_vae_decoder(cfg))
    m.load_state_dict({k: sd[k] for k in g["ref_keys"].tolist()}, strict=True)
    assert torch.equal(m.encoder.conv_in.weight, sd["encoder.conv_in.weight"])
    assert torch.equal(m.decoder.conv_out.weight, sd["decoder.conv_out.weight"])


def test_decode_only_class_is_unchanged():
    from audiogpt_b200.ldm.models.autoencoder import AutoencoderKL
    cfg = specs.VAE_SMALL
    m = AutoencoderKL(ddconfig={k: v for k, v in cfg.items() if k != "embed_dim"}, embed_dim=cfg["embed_dim"])
    assert set(m.state_dict()) == set(specs.vae_decoder_param_shapes(cfg))
    with pytest.raises(NotImplementedError, match="AutoencoderKLWithEncoder"):
        m.encode(torch.zeros(1, 1, 16, 16))


def test_encode_needs_cuda_tensors():
    m = _full(specs.VAE_SMALL)
    with pytest.raises(RuntimeError, match="CUDA only"):
        m.encode(torch.zeros(1, 1, 16, 16))
    with pytest.raises(RuntimeError, match="CUDA only"):
        m(torch.zeros(1, 1, 16, 16))


def test_posterior_matches_reference_formulas():
    """the drop-in DiagonalGaussianDistribution against the reference's formulas (distributions.py:24-59)"""
    from audiogpt_b200.ldm.modules.distributions.distributions import DiagonalGaussianDistribution as D
    mom = specs.synth_tensor((2, 8, 3, 5), seed=9, scale=3.0)
    mom[0, 4, 0, 0], mom[1, 5, 1, 1] = -50.0, 40.0           # logvar entries past both clamp bounds
    p = D(mom)
    mean, logvar = mom[:, :4], mom[:, 4:].clamp(-30.0, 20.0)
    assert p.parameters is mom
    assert torch.equal(p.mean, mean) and torch.equal(p.logvar, logvar)
    assert p.logvar.min() == -30.0 and p.logvar.max() == 20.0
    assert torch.equal(p.std, torch.exp(0.5 * logvar)) and torch.equal(p.var, torch.exp(logvar))
    assert torch.equal(p.mode(), mean)
    # sample(): host noise of the mean's shape, drawn from the global generator
    torch.manual_seed(1234)
    s = p.sample()
    torch.manual_seed(1234)
    assert torch.equal(s, mean + torch.exp(0.5 * logvar) * torch.randn(mean.shape))
    assert torch.allclose(p.kl(), 0.5 * torch.sum(mean ** 2 + logvar.exp() - 1.0 - logvar, dim=[1, 2, 3]))
    q = D(specs.synth_tensor((2, 8, 3, 5), seed=10))
    want = 0.5 * torch.sum((mean - q.mean) ** 2 / q.var + p.var / q.var - 1.0 - logvar + q.logvar, dim=[1, 2, 3])
    assert torch.allclose(p.kl(q), want)
    want = 0.5 * torch.sum(math.log(2 * math.pi) + logvar + (s - mean) ** 2 / logvar.exp(), dim=[1, 2, 3])
    assert torch.allclose(p.nll(s), want)
    d = D(mom, deterministic=True)
    assert torch.equal(d.std, torch.zeros_like(mean)) and torch.equal(d.sample(), mean)
    assert torch.equal(d.kl(), torch.Tensor([0.0])) and torch.equal(d.nll(s), torch.Tensor([0.0]))


def _run(code):
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=240)
    assert r.returncode == 0, r.stderr
    return r.stdout.strip()


def test_install_first_stage_grafts_full_class(tmp_path):
    """install(first_stage=True) puts AutoencoderKLWithEncoder over the reference's AutoencoderKL and records the
    reference's DiagonalGaussianDistribution; the default install() leaves ldm.models.autoencoder alone and still patches
    its eight modules; first_stage and front_end combine."""
    for d in ("ldm", "ldm/models", "ldm/modules", "ldm/modules/distributions"):
        (tmp_path / d).mkdir(parents=True, exist_ok=True)
        (tmp_path / d / "__init__.py").write_text("")
    (tmp_path / "ldm" / "models" / "autoencoder.py").write_text("class AutoencoderKL:\n    pass\n")
    (tmp_path / "ldm" / "modules" / "distributions" / "distributions.py").write_text(
        "class DiagonalGaussianDistribution:\n    def __init__(self, parameters):\n        self.parameters = parameters\n")
    head = "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import audiogpt_b200 as a; " % (str(tmp_path), ROOT)
    check = ("import ldm.models.autoencoder as ae, ldm.modules.distributions.distributions as dd; "
             "from audiogpt_b200.ldm.models.autoencoder import AutoencoderKLWithEncoder as F; "
             "print(len(p), ae.AutoencoderKL.__module__, ae.AutoencoderKL.__name__, "
             "F._posterior_cls is dd.DiagonalGaussianDistribution)")
    assert _run(head + "p = a.install(); " + check) == "8 ldm.models.autoencoder AutoencoderKL False"
    assert _run(head + "p = a.install(first_stage=True); " + check) == \
        "9 audiogpt_b200.ldm.models.autoencoder AutoencoderKLWithEncoder True"
    assert _run(head + "p = a.install(front_end=True, first_stage=True); " + check).startswith("11 ")


def test_install_first_stage_aliases_without_reference():
    """Without the reference tree, install(first_stage=True) registers ldm.models.autoencoder so that
    `from ldm.models.autoencoder import AutoencoderKL` yields the full class, and encode() keeps the drop-in
    posterior."""
    code = ("import sys; sys.path.insert(0, %r); import audiogpt_b200 as a; p = a.install(first_stage=True); "
            "from ldm.models.autoencoder import AutoencoderKL; "
            "from audiogpt_b200.ldm.models import autoencoder as ours; "
            "assert AutoencoderKL is ours.AutoencoderKLWithEncoder and ours.AutoencoderKL is not AutoencoderKL; "
            "assert ours.AutoencoderKLWithEncoder._posterior_cls is None; "
            "print(len(p), p[-1])") % ROOT
    assert _run(code) == "9 ldm.models.autoencoder (aliased)"
