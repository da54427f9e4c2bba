"""End-to-end and cross-cutting GPU tests: diffusion -> mel -> HiFi-GAN -> waveform pipeline against the
CPU oracle, the vocoder wrapper (numpy in / numpy out), and both tap-GEMM kernels against float64 on the layer
shapes of the BASELINE configs."""
import numpy as np
import pytest
import torch

from audiogpt_b200 import specs
from audiogpt_b200.modules.diff import shallow_diffusion_tts as sdt
from audiogpt_b200.modules.diff.net import DiffNet
from audiogpt_b200.modules.hifigan.hifigan import HifiGanGenerator
from audiogpt_b200.utils.hparams import set_hparams_from_dict
from audiogpt_b200.vocoders.hifigan import HifiGAN, get_vocoder_cls
from conftest import rel_rmse, rmse

pytestmark = pytest.mark.gpu


def test_c3_pipeline_small_vs_oracle():
    """BASELINE configs[2] flow at CPU-second size: 20-step ancestral sampling -> denorm -> HiFi-GAN."""
    from oracle import diffusion_ref as dr
    from oracle import hifigan_ref as hr
    cfg, h = specs.DIFFNET_SMALL, specs.HIFIGAN_SMALL
    set_hparams_from_dict(dict(cfg, keep_bins=80, schedule_type="linear", max_beta=0.06))
    net = DiffNet(80)
    sdn = specs.synth_diffnet(cfg, 2024)
    net.load_state_dict(sdn, strict=True)
    steps = 20
    gd = sdt.GaussianDiffusion(None, 80, net, timesteps=steps, K_step=steps, loss_type="l1",
                               betas=sdt.linear_beta_schedule(steps, 0.06), spec_min=specs.SPEC_MIN,
                               spec_max=specs.SPEC_MAX).eval().to("cuda")
    voc = HifiGanGenerator(h)
    sdh = specs.synth_hifigan(h, 1234)
    voc.load_state_dict(sdh, strict=True)
    voc = voc.eval().to("cuda")
    B, T = 2, 18
    x = specs.synth_tensor((B, 1, 80, T), seed=5)
    cond = specs.synth_tensor((B, cfg["hidden_size"], T), seed=6)
    noises = specs.synth_tensor((steps, B, 1, 80, T), seed=7)
    # ---- GPU path
    xg = gd.sample(cond.cuda(), x_start=x.cuda(), noises=noises.cuda())
    mel = gd.denorm_spec(xg[:, 0].transpose(1, 2))               # [B, T, 80]
    wav = voc(mel.transpose(1, 2).contiguous())
    # ---- oracle path
    tab = dr.schedule_tables(dr.linear_betas(steps, 0.06))
    xo = dr.sample_loop(sdn, cfg, tab, x, cond, noises)
    smin, smax = torch.tensor(specs.SPEC_MIN)[None, None], torch.tensor(specs.SPEC_MAX)[None, None]
    melo = dr.denorm_spec(xo[:, 0].transpose(1, 2), smin, smax)
    wavo = hr.hifigan_forward(sdh, h, melo.transpose(1, 2).contiguous())
    assert rel_rmse(mel.cpu(), melo) < 1e-4
    e = rmse(wav.cpu(), wavo)
    print("C3-small pipeline waveform RMSE:", e)
    assert wav.shape == (B, 1, T * 256) and e < 1e-4


def test_vocoder_wrapper_spec2wav():
    from oracle import hifigan_ref as hr
    h = specs.HIFIGAN_SMALL
    m = HifiGanGenerator(h)
    sd = specs.synth_hifigan(h, 1234)
    m.load_state_dict(sd, strict=True)
    m = m.eval().to("cuda")
    v = HifiGAN(model=m, config=h)
    assert get_vocoder_cls({"vocoder": "hifigan"}) is HifiGAN
    set_hparams_from_dict({})
    mel = specs.synth_tensor((31, 80), seed=9, scale=2.0, shift=-4.0).numpy()      # [T, 80] as the reference passes
    wav = v.spec2wav(mel)
    ref = hr.hifigan_forward(sd, h, torch.from_numpy(mel.T.copy())[None]).reshape(-1)
    assert isinstance(wav, np.ndarray) and wav.shape == (31 * 256,)
    assert rmse(wav, ref) < 2e-5


SHAPES = [  # G, L, Cin, Cout, K, dil, Wreal
    (2, 3000, 256, 256, 11, 5, 0), (2, 5000, 128, 128, 3, 3, 0), (2, 9000, 32, 32, 7, 1, 0),
    (3, 400, 256, 512, 3, 2, 0), (1, 777, 320, 320, 1, 1, 0), (2, 780, 320, 320, 3, 1, 78),
    (2, 195, 640, 640, 3, 1, 39), (1, 130, 1280, 320, 1, 1, 0), (2, 4, 64, 96, 3, 1, 0),
    (2, 300, 80, 256, 7, 1, 0), (1, 780, 4, 320, 3, 1, 78), (2, 500, 96, 40, 5, 2, 0),
    (8, 195, 640, 640, 3, 1, 39),   # 16 row tiles x 640 channels: the 96-wide tile (112 tiles, last column tile partial)
]


def _baseline_layer(name, G, Ln, Cin, Cout, K, dil, Wr, epi_res, **kw):
    """one BASELINE layer shape through agpt_tapconv_probe, leaky-ReLU(0.1) prologue, on both kernels, checked
    against float64 (test_tapconv_gpu.py)"""
    from test_tapconv_gpu import EPI_BIAS, EPI_RES, run_case
    stats = {}
    run_case(name, kind=1 if Wr else 0, Cin=Cin, Cout=Cout, K=K, dil=dil, G=G, L=Ln, Wreal=Wr,
             epi=EPI_RES if epi_res else EPI_BIAS, res=bool(epi_res), stats=stats, **kw)
    return stats


def test_baseline_layers_both_kernels_vs_fp64():
    """Each BASELINE layer shape on the wgmma tap-GEMM (tcconv5: tile width picked to fill the SMs) and on the
    fp32-FMA kernel, both against float64 with the per-element bound of test_tapconv_gpu.py.  Also, RELATIVE to the
    output rms: rms error <= 2e-5 and max error <= 2e-4 (the 3 x fp16-part arithmetic truncates at 2^-22 per
    product and drops lo x lo; the error grows with the contraction length taps x C_in, up to 2 816 here)."""
    torch.zeros(1).cuda()
    for G, Ln, Cin, Cout, K, dil, Wr in SHAPES:
        for epi_res in (0, 1):
            st = _baseline_layer(f"baseline {(G, Ln, Cin, Cout, K, dil, Wr)}", G, Ln, Cin, Cout, K, dil, Wr, epi_res,
                                 seed=G * Ln + Cin + epi_res)
            assert st["max"] < 2e-4 and st["rms"] < 2e-5, (G, Ln, Cin, Cout, K, dil, Wr, epi_res, st)


@pytest.mark.parametrize("x_scale,w_spread,tol_max,tol_rms", [
    (1e-4, 1.0, 4e-4, 4e-5),      # tiny activations: the lo part of |x| < 2^-3 is an fp16 subnormal (absolute floor 2^-25)
    (1e-2, 1.0, 2e-4, 2e-5),
    (30.0, 1.0, 2e-4, 2e-5),      # post-GroupNorm-outlier scale
    (3000.0, 1.0, 2e-4, 2e-5),    # near the fp16 range (65504): still finite and split exactly
    (1.0, 1e3, 1e-3, 1e-4),       # weight-norm g spread x1000 across output channels (ONE power-of-two scale per layer:
                                  # the low-gain channels' lo parts go subnormal -- errors relative to the global rms)
    (1e-3, 1e3, 2e-3, 2e-4),      # both at once (documented head-room, DESIGN 2)
])
def test_wgmma_adversarial_ranges_vs_fp64(x_scale, w_spread, tol_max, tol_rms):
    """Large-dynamic-range parity of the 3 x fp16-part arithmetic: activation scales from 1e-4 to 3e3 and a x1000
    gain spread over output channels, on three layer shapes (narrow / wide / 2-D), both kernels against float64 (the
    per-element bound includes the fp16 subnormal floors), and relative to the output rms within the stated
    tolerances."""
    torch.zeros(1).cuda()
    worst = (0.0, 0.0)
    for G, Ln, Cin, Cout, K, dil, Wr in [(2, 9000, 32, 32, 7, 1, 0), (2, 3000, 256, 256, 11, 5, 0), (2, 780, 320, 320, 3, 1, 78)]:
        st = _baseline_layer(f"range x {x_scale:g} w {w_spread:g} {(G, Ln, Cin, Cout)}", G, Ln, Cin, Cout, K, dil, Wr, 1,
                             x_scale=x_scale, w_spread=w_spread, seed=Ln + Cin)
        worst = (max(worst[0], st["max"]), max(worst[1], st["rms"]))
        assert st["max"] < tol_max and st["rms"] < tol_rms, (x_scale, w_spread, G, Ln, Cin, Cout, K, st)
    print(f"x_scale {x_scale:g} w_spread {w_spread:g}: max/rms {worst[0]:.2e}  rms/rms {worst[1]:.2e}")


def test_saturating_and_zero_inputs():
    """All-zero input -> exactly the bias path; inputs beyond the fp16 range saturate (documented), stay finite."""
    from oracle import hifigan_ref as hr
    h = specs.HIFIGAN_SMALL
    sd = specs.synth_hifigan(h, 1234)
    m = HifiGanGenerator(h)
    m.load_state_dict(sd, strict=True)
    m = m.eval().to("cuda")
    z = torch.zeros(2, 80, 40, device="cuda")
    wz = m(z).cpu()
    ref = hr.hifigan_forward(sd, h, torch.zeros(2, 80, 40))
    assert rmse(wz, ref) < 2e-6
    big = torch.full((1, 80, 16), 1e6, device="cuda")
    assert torch.isfinite(m(big)).all()
