"""Conformance of the non-contraction kernels (nn_kernels.cu) against float64 references.

Every GPU case runs ONE production launcher through agpt_nn_probe on caller-owned device tensors and compares it with
torch.nn.functional in float64 (group_norm, layer_norm, softmax, conv2d, avg_pool2d, interpolate) or the formulas of
ldm/modules/diffusionmodules/util.py (timestep_embedding) and ldm/models/diffusion/ddim.py (p_sample_ddim), written on
the reference's own layouts without any of the kernels' indexing.  Every output buffer is NaN-filled and followed by
GUARD canary floats: each case asserts that no NaN is left inside the output and that the guard is untouched.

Error model and gates (u = 2^-24, the fp32 unit roundoff; LAMBDA = 6; g(n) = min(n, LAMBDA sqrt(n)) for a sum of n
terms: the worst case n u, or the probabilistic bound of Higham & Mary (SIAM J. Sci. Comput. 41(5), 2019),
|error| <= LAMBDA sqrt(n) u sum|terms| except with probability 2 exp(-LAMBDA^2 / 2), whichever is smaller -- the worst
case would not catch a wrong term of a long sum):

  * Data movement (transpose / copy pad, concat, upsample, im2col, cf_to_cl_pad, select_row): exact, padding included.
  * avgpool2: the kernel's documented order ((a + b) + d) + e, then / 4, reproduced in fp32: exact.
  * GroupNorm (one CTA per group of n = HW cpg values; m = values per thread = ceil(n / V / 512) V): the mean is
    per-thread fp32 sums with an fp64 block sum, |mu^ - mu| <= u (g(m) A + |mu|) with A = mean |x| of the group; the
    centred second pass adds 2u per square plus g(m) u, so |r^ - r| / r <= u (2 + g(m) / 2); the output
    (x - mu^) r^ gamma + beta rounds three times.  Per element:
        |y - ref| <= u ((5 + g(m) / 2) |x - mu| r |gamma| + (g(m) + 1) A r |gamma| + |beta|)
  * LayerNorm (one warp per row of C; m = ceil(C / 32) values per lane, then a 5-level fp32 butterfly, n = m + 5):
    the same form with the fp32 warp sums and rsqrtf (2 ulp):
        |y - ref| <= u ((8 + g(n) / 2) |x - mu| r |gamma| + (g(n) + 1) A r |gamma| + |beta|)
  * An activation f maps the bound E of its argument v to max |f(v +- E) - f(v)| + 8 u (|f(v)| + |v|); a residual
    added after it adds u |y|.
  * Besides the per-element bound, the rms error of every normalisation must stay below half the rms bound.
  * softmax_rows: relative, per element, with a = x scale and M = max a over the row: the fp32 argument a - M is off
    by d_j = u (|a_j| + |a_j - M|) and expf adds 2 ulp; the row sum (ceil(cols / 256) per thread, a 5-level butterfly,
    8 warps: n terms) and the normalisation add g(n) u + 2u:
        |p_j - ref_j| <= ref_j (d_j + 2u + sum_k ref_k (d_k + 2u) + g(n) u + 2u) + 2^-126
    and columns cols..pitch-1 must be exact zeros.
  * Timestep embedding: the specification is torch's fp32 arithmetic (freqs and t * freqs in fp32, then cos / sin).
    The fp32 argument a is reproduced on the CPU and cos / sin are evaluated in fp64; a device expf may differ from the
    CPU's by 1 ulp, which moves a by up to 2^-22 |a|:
        |y - ref| <= |a| 2^-22 |sin a or cos a| + (|a| 2^-22)^2 / 2 + 2^-22
  * DDIM step (ddim_update_tab): fp64 ddim.py formulas on the table's fp32 coefficients; every fp32 operation adds
    one rounding of its result, propagated to x_prev and pred_x0 (ddim_bound).  conv_out_ddim: the same after the
    fp64 conv2d(3x3, padding 1) + bias, whose bound is g(n) u conv(|h|, |w|) + u |eps| with n = 9 ceil(C / 32) + 5
    (lanes stride the channels, 9 taps, a 5-level butterfly).

Teeth: each gate family has a CPU-emulated mutant that must FAIL the same gate (single-pass fp32 variance on an
offset group, a group index off by one, a softmax tail left unzeroed, a 3x3 border tap dropped, the CFG halves
swapped).  They need no device and run everywhere.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from audiogpt_b200 import _lib, specs

gpu = pytest.mark.gpu

U = 2.0 ** -24
LAMBDA = 6.0
GUARD = 64
CANARY = -7777.25
NAN = float("nan")
DEV = "cuda"
GN_THREADS, GN_CACHE_FLOATS = 512, 48 * 1024
LATENT = (10, 78)       # the text-to-audio latent: 80 mel bins x 624 frames over the first stage's 8x downsampling

EXERCISED = {}          # (kernel, path) -> worst error / bound over the cases that ran it


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    if EXERCISED:
        print("\nnn_kernels paths exercised: worst error / bound")
        for k in sorted(EXERCISED):
            print(f"  {k[0]:14s} {k[1]:24s}: {EXERCISED[k]:.3f}")


def gam(n):
    return min(float(n), LAMBDA * math.sqrt(n))


def f32(v):
    return float(np.float32(v))


# ------------------------------------------------------------------------------------------------ buffers and the probe
def out_buffer(shape, fill=NAN):
    """fp32 device buffer of `shape` (filled with `fill`) followed by GUARD canary floats; returns (flat, view)"""
    n = math.prod(shape)
    flat = torch.full((n + GUARD,), fill, dtype=torch.float32, device=DEV)
    flat[n:] = CANARY
    return flat, flat[:n].view(shape)


def assert_written(tag, flat, n):
    assert torch.equal(flat[n:], torch.full_like(flat[n:], CANARY)), f"{tag}: written past the end of the output"
    assert not torch.isnan(flat[:n]).any(), f"{tag}: {int(torch.isnan(flat[:n]).sum())} output elements not written"


def probe(op, **kw):
    a = _lib.NnProbeArgs()
    a.op = _lib.NN_OPS.index(op)
    for k, v in kw.items():
        if isinstance(v, torch.Tensor):
            v = v.data_ptr()
        setattr(a, k, v)
    _lib.check(_lib.lib().agpt_nn_probe(C.byref(a), _lib.cur_stream()))


def gate(y, ref, bound):
    """(worst |y - ref| / bound, rms(err) / rms(bound)); NaN counts as a failure"""
    err = (y.double() - ref).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    b = bound + 1e-300
    return float((err / b).max()), float(err.pow(2).mean().sqrt() / b.pow(2).mean().sqrt())


def passes(y, ref, bound, rms=True):
    w, r = gate(y, ref, bound)
    return w <= 1.0 and (not rms or r <= 0.5)


def check(tag, key, y, ref, bound, rms=True):
    w, r = gate(y, ref, bound)
    print(f"{tag}: worst err/bound {w:.3f}, rms err/rms bound {r:.3f}")
    EXERCISED[key] = max(EXERCISED.get(key, 0.0), w)
    if w > 1.0:
        err = (y.double() - ref).abs() / (bound + 1e-300)
        idx = np.unravel_index(int(torch.argmax(torch.nan_to_num(err, nan=math.inf)).item()), tuple(y.shape))
        raise AssertionError(f"{tag}: error {w:.3g} x the bound at {idx}: got {float(y[idx])}, want {float(ref[idx])}")
    if rms:
        assert r <= 0.5, f"{tag}: rms error {r:.3g} x the rms bound"


def f_bound(f, v, E):
    fv = f(v)
    return torch.maximum((f(v + E) - fv).abs(), (f(v - E) - fv).abs()) + 8 * U * (fv.abs() + v.abs())


ACTS = {0: lambda v: v, 1: F.silu, 2: F.relu}


# ================================================================================================ normalisations
def gn_threads_values(HW, cpg):
    """(vector width V, values summed by one thread m) of gn_fused_kernel"""
    V = 4 if cpg % 4 == 0 else (2 if cpg % 2 == 0 else 1)
    return V, math.ceil(HW * cpg // V / GN_THREADS) * V


def gn_reference(x, gamma, beta, G, eps, act, res):
    """x [N][HW][C] (any dtype) -> (ref, bound) float64, on x's device"""
    N, HW, Cc = x.shape
    cpg = Cc // G
    x64 = x.double()
    xcf = x64.permute(0, 2, 1)                                          # [N][C][HW], torch's layout
    g64, b64 = gamma.double(), beta.double()
    v = F.group_norm(xcf, G, g64, b64, eps=f32(eps)).permute(0, 2, 1)
    xg = xcf.reshape(N, G, cpg * HW)
    mu = xg.mean(-1)
    var = (xg - mu[..., None]).pow(2).mean(-1)
    r = 1.0 / torch.sqrt(var + f32(eps))
    A = xg.abs().mean(-1)
    per_c = lambda t: t.repeat_interleave(cpg, dim=1)[:, None, :]       # [N][G] -> [N][1][C]
    _, m = gn_threads_values(HW, cpg)
    dev = (x64 - per_c(mu)).abs()
    E = U * ((5 + gam(m) / 2) * dev * per_c(r) * g64.abs() + (gam(m) + 1) * per_c(A * r) * g64.abs() + b64.abs())
    f = ACTS[act]
    ref = f(v)
    E = f_bound(f, v, E) if act else E
    if res is not None:
        ref = ref + res.double()
        E = E + U * ref.abs()
    return ref, E


def ln_reference(x, gamma, beta, eps):
    rows, Cc = x.shape
    x64 = x.double()
    g64, b64 = gamma.double(), beta.double()
    ref = F.layer_norm(x64, (Cc,), g64, b64, eps=f32(eps))
    mu = x64.mean(-1, keepdim=True)
    r = 1.0 / torch.sqrt((x64 - mu).pow(2).mean(-1, keepdim=True) + f32(eps))
    A = x64.abs().mean(-1, keepdim=True)
    n = math.ceil(Cc / 32) + 5
    E = U * ((8 + gam(n) / 2) * (x64 - mu).abs() * r * g64.abs() + (gam(n) + 1) * A * r * g64.abs() + b64.abs())
    return ref, E


def gn_inputs(N, HW, Cc, seed):
    x = specs.synth_tensor((N, HW, Cc), seed, scale=1.5, shift=0.3)
    gamma = specs.synth_tensor((Cc,), seed + 1, scale=0.5, shift=1.0)
    beta = specs.synth_tensor((Cc,), seed + 2, scale=0.3)
    return x, gamma, beta


def offset_group(x, n, g, cpg, ratio=1e3, sigma=0.5):
    """group g of sample n: mean / sigma = ratio"""
    HW = x.shape[1]
    z = specs.synth_tensor((HW, cpg), 77 + g)
    x[n, :, g * cpg:(g + 1) * cpg] = sigma * (ratio + z)


def run_gn(tag, N, HW, Cc, G, eps, act=1, res=False, seed=0, special=False):
    cpg = Cc // G
    x, gamma, beta = gn_inputs(N, HW, Cc, seed)
    if special:   # one constant group (variance 0: r = eps^-1/2) and one with mean / sigma = 1e3
        x[0, :, 0:cpg] = 0.75
        offset_group(x, N - 1, G - 1, cpg)
    r = specs.synth_tensor((N, HW, Cc), seed + 3) if res else None
    xd, gd, bd = x.to(DEV), gamma.to(DEV), beta.to(DEV)
    rd = r.to(DEV) if res else None
    flat, y = out_buffer((N, HW, Cc))
    probe("GROUPNORM", x=xd, x2=rd, y=flat, gamma=gd, beta=bd, N=N, rows=HW, C=Cc, G=G, eps=eps, act=act)
    assert_written(tag, flat, y.numel())
    ref, E = gn_reference(xd, gd, bd, G, eps, act, rd)
    V, _ = gn_threads_values(HW, cpg)
    path = f"V={V} {'cached' if HW * cpg <= GN_CACHE_FLOATS else 'uncached'}"
    check(f"{tag} [{path}]", ("groupnorm", path), y, ref, E)
    if special and act == 0 and not res:
        assert torch.equal(y[0, :, :cpg], bd[:cpg].expand(HW, cpg)), f"{tag}: a constant group is not exactly beta"


def unet_gn_channels():
    """every GroupNorm width of the shipped text-to-audio UNet (ResBlock in / out channels)"""
    plan = specs.unet_plan(specs.UNET_TXT2AUDIO)
    ch = set()
    for blk in plan["input_blocks"] + [plan["middle_block"]] + plan["output_blocks"]:
        for layer in blk:
            if layer[0] == "res":
                ch.update(layer[1:3])
    return sorted(ch)


def vae_gn_shapes():
    """(C, H, W) of every GroupNorm the VAE decoder plan runs, from the latent up to the full mel"""
    cfg = specs.VAE_TXT2AUDIO
    block_in, levels = specs.vae_decoder_plan(cfg)
    H, W = LATENT
    out = {(block_in, H, W)}                         # conv_in -> mid block (two ResBlocks and the attention)
    for _, blocks, up in levels:
        for cin, cout, _ in blocks:
            out.update({(cin, H, W), (cout, H, W)})
        if up:
            H, W = 2 * H, 2 * W
    return sorted(out, key=lambda s: (s[1] * s[2], s[0]))


UNET_GN = [(c, h, w) for c in unet_gn_channels() for (h, w) in (LATENT, (LATENT[0] // 2, LATENT[1] // 2))]


@gpu
@pytest.mark.parametrize("Cc,H,W", UNET_GN)
def test_groupnorm_unet(Cc, H, W):
    """the UNet's GroupNorm32 with classifier-free guidance (N = 8): cpg = 10 / 20 / 30 / 40 (V = 2 / 4)"""
    run_gn(f"gn unet C {Cc} {H}x{W}", 8, H * W, Cc, 32, 1e-5, act=1, seed=Cc + H)


@gpu
@pytest.mark.parametrize("Cc,H,W", vae_gn_shapes())
def test_groupnorm_vae_decoder(Cc, H, W):
    """every (C, HW) of the VAE decoder: cached slabs at 10x78 and 20x156 / C = 256, re-read through L2 beyond"""
    run_gn(f"gn vae C {Cc} {H}x{W}", 1, H * W, Cc, 32, 1e-6, act=1, seed=Cc + H)


@gpu
@pytest.mark.parametrize("act,res", [(2, True), (0, False), (1, True)])
def test_groupnorm_pitch_extractor(act, res):
    """PitchExtractor: G = H / 16, ReLU, then + x (groupnorm_ex's residual)"""
    Hc = specs.PE_BASE["hidden_size"]
    run_gn(f"gn pe act {act} res {res}", 2, 301, Hc, Hc // 16, 1e-5, act=act, res=res, seed=40 + act)


@gpu
@pytest.mark.parametrize("Cc,G,HW", [(96, 32, 500), (36, 4, 333), (4, 4, 77)])
def test_groupnorm_odd_cpg(Cc, G, HW):
    """cpg odd: the scalar (V = 1) kernel; cpg = 1"""
    run_gn(f"gn cpg {Cc // G}", 2, HW, Cc, G, 1e-5, act=1, seed=50 + Cc)


@gpu
@pytest.mark.parametrize("extra", [0, 1])
def test_groupnorm_cache_boundary(extra):
    """a slab of exactly 48 K floats (shared-memory cache) and one row more (re-read through L2)"""
    cpg = 16
    HW = GN_CACHE_FLOATS // cpg + extra
    run_gn(f"gn slab {HW * cpg}", 2, HW, 32 * cpg, 32, 1e-6, act=1, seed=60 + extra)


@gpu
@pytest.mark.parametrize("act", [0, 1])
def test_groupnorm_constant_and_offset_groups(act):
    """a constant group (variance 0: exactly beta without activation) and a group with mean / sigma = 1e3"""
    run_gn(f"gn special act {act}", 2, 780, 320, 32, 1e-5, act=act, seed=70, special=True)


LN_WIDTHS = sorted({  # (C, eps) of the shipped transformers
    (c, specs.PVT_SHIPPED["layer_norm_eps"]) for c in specs.PVT_SHIPPED["embed_dims"]} | {
    (specs.FS2_C2["hidden_size"], 1e-5), (specs.CLAP_BASE["hidden_size"], specs.CLAP_BASE["layer_norm_eps"]),
    (specs.W2V_BASE["hidden_size"], specs.W2V_BASE["layer_norm_eps"])} | {
    (c, 1e-5) for c in unet_gn_channels() if c in (320, 640)})


@gpu
@pytest.mark.parametrize("Cc,eps", LN_WIDTHS + [(100, 1e-5), (20, 1e-5), (1, 1e-5)])
@pytest.mark.parametrize("rows", [1, 203])
def test_layernorm(Cc, eps, rows):
    """C of every shipped transformer, C not a multiple of 32, C < 32; rows not a multiple of the 8 rows per block;
    row 0 constant and row 1 with mean / sigma = 1e3"""
    x = specs.synth_tensor((rows, Cc), Cc + rows, scale=1.2, shift=-0.2)
    if rows > 2:
        x[0] = 0.75
        x[1] = 0.5 * (1e3 + specs.synth_tensor((Cc,), 7))
    gamma = specs.synth_tensor((Cc,), Cc + 1, scale=0.5, shift=1.0)
    beta = specs.synth_tensor((Cc,), Cc + 2, scale=0.3)
    xd, gd, bd = x.to(DEV), gamma.to(DEV), beta.to(DEV)
    flat, y = out_buffer((rows, Cc))
    probe("LAYERNORM", x=xd, y=flat, gamma=gd, beta=bd, rows=rows, C=Cc, eps=eps)
    assert_written(f"ln C {Cc}", flat, y.numel())
    ref, E = ln_reference(xd, gd, bd, eps)
    check(f"ln C {Cc} rows {rows} eps {eps:g}", ("layernorm", f"C%32={'0' if Cc % 32 == 0 else 'r'}"), y, ref, E)
    if rows > 2:
        assert torch.equal(y[0], bd), "a constant row is not exactly beta"


# ------------------------------------------------------------------------------------------------ mutants (CPU)
def emulate_gn_group(xg, V, eps, single_pass):
    """gn_fused_kernel's arithmetic on one group [HW][cpg] in fp32 numpy, with the centred variance or (the mutant) a
    single-pass E[x^2] - E[x]^2 in fp32; returns the normalised values (gamma = 1, beta = 0)"""
    HW, cpg = xg.shape
    vec = xg.reshape(-1, V).astype(np.float32)                          # vector i = r * vpr + c / V, element k
    nvec = vec.shape[0]
    it = math.ceil(nvec / GN_THREADS)
    pad = np.zeros((it * GN_THREADS, V), np.float32)
    pad[:nvec] = vec
    X = pad.reshape(it, GN_THREADS, V)
    n = HW * cpg
    s = np.zeros(GN_THREADS, np.float32)
    for i in range(it):
        for k in range(V):
            s = (s + X[i, :, k]).astype(np.float32)
    mean = np.float32(s.astype(np.float64).sum() / n)
    q = np.zeros(GN_THREADS, np.float32)
    for i in range(it):
        for k in range(V):
            if single_pass:
                v = X[i, :, k].astype(np.float64)
                q = (q + v * v).astype(np.float32)
            else:
                d = (X[i, :, k] - mean).astype(np.float32)
                d[i * GN_THREADS + np.arange(GN_THREADS) >= nvec] = 0.0
                q = (q + d.astype(np.float64) ** 2).astype(np.float32)
    if single_pass:
        var = np.float32(np.float32(q.astype(np.float64).sum() / n) - mean * mean)
        rstd = np.float32(1.0 / math.sqrt(max(float(var), 0.0) + f32(eps)))
    else:
        rstd = np.float32(1.0 / math.sqrt(q.astype(np.float64).sum() / n + f32(eps)))
    return ((xg.astype(np.float32) - mean).astype(np.float32) * rstd).astype(np.float32)


def test_gate_catches_single_pass_variance():
    """on a group with mean / sigma = 1e3, the kernel's two-pass arithmetic (emulated in fp32) passes the GroupNorm
    gate and a single-pass fp32 variance fails it"""
    HW, cpg = 780, 16
    x = torch.zeros(1, HW, cpg)
    offset_group(x, 0, 0, cpg)
    ones, zeros = torch.ones(cpg), torch.zeros(cpg)
    ref, E = gn_reference(x, ones, zeros, 1, 1e-6, 0, None)
    V, _ = gn_threads_values(HW, cpg)
    good = torch.from_numpy(emulate_gn_group(x[0].numpy(), V, 1e-6, False))[None]
    bad = torch.from_numpy(emulate_gn_group(x[0].numpy(), V, 1e-6, True))[None]
    assert passes(good, ref, E), gate(good, ref, E)
    assert not passes(bad, ref, E), gate(bad, ref, E)


def test_gate_catches_group_off_by_one():
    """normalising each group with its neighbour's statistics fails the GroupNorm gate"""
    N, HW, Cc, G = 2, 390, 320, 32
    x, gamma, beta = gn_inputs(N, HW, Cc, 5)
    ref, E = gn_reference(x, gamma, beta, G, 1e-5, 1, None)
    cpg = Cc // G
    xg = x.double().permute(0, 2, 1).reshape(N, G, cpg * HW)
    mu = torch.roll(xg.mean(-1), 1, dims=1).repeat_interleave(cpg, 1)[:, None, :]      # group g - 1's statistics
    sd = torch.roll((xg.var(-1, unbiased=False) + f32(1e-5)).sqrt(), 1, dims=1).repeat_interleave(cpg, 1)[:, None, :]
    mut = F.silu((x.double() - mu) / sd * gamma.double() + beta.double())
    assert passes(ref.float(), ref, E)
    assert not passes(mut, ref, E)


# ================================================================================================ softmax_rows
def softmax_reference(x, cols, scale):
    a = x[:, :cols].double() * f32(scale)
    ref = torch.softmax(a, dim=-1)
    M = a.max(-1, keepdim=True).values
    d = U * (a.abs() + (a - M).abs()) + 2 * U
    n = math.ceil(cols / 256) + 5 + 8
    E = ref * (d + (ref * d).sum(-1, keepdim=True) + gam(n) * U + 2 * U) + 2.0 ** -126
    return ref, E


def vae_attn_shapes():
    """(HW, C) of the VAE decoder's AttnBlocks: the levels at attn_resolutions"""
    cfg = specs.VAE_TXT2AUDIO
    block_in, levels = specs.vae_decoder_plan(cfg)
    H, W = LATENT
    out = [(H * W, block_in)]                        # the mid block's attention
    for _, blocks, up in levels:
        for cin, cout, attn in blocks:
            if attn and (H * W, cout) not in out:
                out.append((H * W, cout))
        if up:
            H, W = 2 * H, 2 * W
    return out


SOFTMAX_CASES = [(hw, hw, -(-hw // 32) * 32, c ** -0.5) for hw, c in vae_attn_shapes()] + [(37, 100, 128, 0.125),
                                                                                           (5, 255, 256, 1.0)]


@gpu
@pytest.mark.parametrize("rows,cols,pitch,scale", SOFTMAX_CASES)
def test_softmax_rows(rows, cols, pitch, scale):
    """the VAE's [HW][round_up(HW, 32)] scores, cols < 256; row 1 spans more than 100 after scaling (exp underflows)"""
    x = specs.synth_tensor((rows, cols), cols, scale=2.0 / scale)
    x[1 % rows] *= 40.0
    assert float((x[1 % rows].max() - x[1 % rows].min()) * f32(scale)) > 100
    flat, y = out_buffer((rows, pitch))
    y[:, :cols] = x.to(DEV)
    probe("SOFTMAX_ROWS", y=flat, rows=rows, cols=cols, pitch=pitch, scale=scale)
    assert_written("softmax", flat, y.numel())
    assert torch.equal(y[:, cols:], torch.zeros_like(y[:, cols:])), "softmax_rows: the tail is not zeroed"
    ref, E = softmax_reference(x.to(DEV), cols, scale)
    check(f"softmax {rows}x{cols} pitch {pitch}", ("softmax_rows", f"cols {'<' if cols < 256 else '>='} 256"),
          y[:, :cols], ref, E, rms=False)


def softmax_tail_ok(y, cols):
    return bool(torch.equal(y[:, cols:], torch.zeros_like(y[:, cols:])))


def test_gate_catches_unzeroed_softmax_tail():
    """the VAE's PV GEMM reads the padding columns: a tail left holding the scores fails the softmax check"""
    rows, cols, pitch = 4, 780, 800
    x = specs.synth_tensor((rows, pitch), 3)
    ref, E = softmax_reference(x, cols, 512 ** -0.5)
    mut = x.clone()
    mut[:, :cols] = ref.float()
    assert passes(mut[:, :cols], ref, E, rms=False)
    assert not softmax_tail_ok(mut, cols)


# ================================================================================================ data movement
@gpu
@pytest.mark.parametrize("rows,cols,pitch,rows_pad", [(780, 512, 3 * 512, 800), (3120, 256, 3 * 256, 3136),
                                                      (37, 40, 45, 64), (1, 1, 1, 32)])
def test_transpose_and_copy_pad(rows, cols, pitch, rows_pad):
    """K^T [C][round_up(HW, 32)] and V [round_up(HW, 32)][C] out of the VAE's qkv rows [HW][3C], zero padded"""
    x = specs.synth_tensor((rows, pitch), rows + cols).to(DEV)
    flat, y = out_buffer((cols, rows_pad))
    probe("TRANSPOSE_PAD", x=x, y=flat, rows=rows, cols=cols, pitch=pitch, rows_pad=rows_pad)
    assert_written("transpose_pad", flat, y.numel())
    assert torch.equal(y, F.pad(x[:, :cols].t(), (0, rows_pad - rows)))
    flat, y = out_buffer((rows_pad, cols))
    probe("COPY_PAD_ROWS", x=x, y=flat, rows=rows, cols=cols, pitch=pitch, rows_pad=rows_pad)
    assert_written("copy_pad_rows", flat, y.numel())
    assert torch.equal(y, F.pad(x[:, :cols], (0, 0, 0, rows_pad - rows)))


@gpu
@pytest.mark.parametrize("Ca,Cb,rows", [(640, 640, 8 * 195), (640, 320, 8 * 780), (4, 4, 3), (4, 320, 7)])
def test_concat(Ca, Cb, rows):
    """the UNet's skip concatenation torch.cat([h, hs.pop()], dim=1) on channels-last rows"""
    a, b = specs.synth_tensor((rows, Ca), 1).to(DEV), specs.synth_tensor((rows, Cb), 2).to(DEV)
    flat, y = out_buffer((rows, Ca + Cb))
    probe("CONCAT", x=a, x2=b, y=flat, rows=rows, C=Ca, C2=Cb)
    assert_written("concat", flat, y.numel())
    assert torch.equal(y, torch.cat([a, b], dim=1))


SPATIAL = [(8, 5, 39, 640), (2, 10, 78, 320), (1, 1, 1, 4), (3, 7, 1, 8), (1, 3, 5, 12)]


@gpu
@pytest.mark.parametrize("N,H,W,Cc", SPATIAL)
def test_upsample2(N, H, W, Cc):
    x = specs.synth_tensor((N, Cc, H, W), H * W)
    want = F.interpolate(x, scale_factor=2, mode="nearest").permute(0, 2, 3, 1).to(DEV)
    flat, y = out_buffer((N, 2 * H, 2 * W, Cc))
    probe("UPSAMPLE2", x=x.permute(0, 2, 3, 1).contiguous().to(DEV), y=flat, N=N, H=H, W=W, C=Cc)
    assert_written("upsample2", flat, y.numel())
    assert torch.equal(y, want)


@gpu
@pytest.mark.parametrize("N,H,W,Cc", [(8, 10, 78, 320), (2, 5, 39, 640), (1, 3, 5, 12), (2, 2, 2, 4), (1, 7, 4, 8)])
def test_avgpool2(N, H, W, Cc):
    """AvgPool2d(2, 2) (floor): the kernel's order ((a + b) + d) + e, then / 4, in fp32 -- exact; and 2 ulp of the fp64
    average"""
    x = specs.synth_tensor((N, Cc, H, W), H + W)
    xe = x[:, :, :H // 2 * 2, :W // 2 * 2]
    a, b, d, e = xe[:, :, 0::2, 0::2], xe[:, :, 0::2, 1::2], xe[:, :, 1::2, 0::2], xe[:, :, 1::2, 1::2]
    want = ((((a + b) + d) + e) / 4.0).permute(0, 2, 3, 1).to(DEV)
    ref64 = F.avg_pool2d(x.double(), 2).permute(0, 2, 3, 1).to(DEV)
    flat, y = out_buffer((N, H // 2, W // 2, Cc))
    probe("AVGPOOL2", x=x.permute(0, 2, 3, 1).contiguous().to(DEV), y=flat, N=N, H=H, W=W, C=Cc)
    assert_written("avgpool2", flat, y.numel())
    assert torch.equal(y, want)
    s = F.avg_pool2d(x.double().abs(), 2).permute(0, 2, 3, 1).to(DEV)
    check(f"avgpool2 {H}x{W}", ("avgpool2", "fp64"), y, ref64, 4 * U * s + 1e-300, rms=False)


IM2COL = [s + (p,) for s in [(8, 10, 78, 320), (2, 5, 39, 8), (2, 80, 624, 4), (1, 3, 2, 4)] for p in (1, 0)] + [
    (1, 1, 1, 4, 1), (1, 4, 1, 4, 1)]     # pad 0 needs H, W >= 2 (Ho = H / 2)


@gpu
@pytest.mark.parametrize("N,H,W,Cc,pad", IM2COL)
def test_im2col_stride2(N, H, W, Cc, pad):
    """3x3 stride-2 taps, H and W odd and even; pad 1: Conv2d(k3, s2, p1); pad 0: F.pad(x, (0, 1, 0, 1)) then a conv
    without padding"""
    x = specs.synth_tensor((N, Cc, H, W), H * W + Cc)
    xp = F.pad(x, (1, 1, 1, 1)) if pad else F.pad(x, (0, 1, 0, 1))
    cols = F.unfold(xp, 3, stride=2)                                      # [N][C * 9][L], channel-major taps
    Ho, Wo = ((H - 1) // 2 + 1, (W - 1) // 2 + 1) if pad else (H // 2, W // 2)
    want = cols.view(N, Cc, 9, Ho, Wo).permute(0, 3, 4, 2, 1).to(DEV)     # [N][Ho][Wo][tap][C]
    flat, y = out_buffer((N, Ho, Wo, 9, Cc))
    probe("IM2COL_S2", x=x.permute(0, 2, 3, 1).contiguous().to(DEV), y=flat, N=N, H=H, W=W, C=Cc, pad=pad)
    assert_written("im2col", flat, y.numel())
    assert torch.equal(y, want)


@gpu
@pytest.mark.parametrize("N,Nsrc,Cc,Cpad,H,W", [(8, 4, 4, 8, 10, 78), (4, 4, 4, 4, 10, 78), (2, 1, 9, 12, 3, 5),
                                                 (3, 3, 1, 4, 1, 7)])
def test_cf_to_cl_pad(N, Nsrc, Cc, Cpad, H, W):
    """[Nsrc][C][HW] -> [N][HW][Cpad], zero channels past C, sample n from n % Nsrc (x_in = cat([x] * 2))"""
    x = specs.synth_tensor((Nsrc, Cc, H * W), Cc + N)
    want = F.pad(torch.cat([x] * (N // Nsrc)).permute(0, 2, 1), (0, Cpad - Cc)).to(DEV)
    flat, y = out_buffer((N, H * W, Cpad))
    probe("CF_TO_CL_PAD", x=x.to(DEV), y=flat, N=N, C=Cc, pitch=Cpad, H=H, W=W, Nsrc=Nsrc)
    assert_written("cf_to_cl_pad", flat, y.numel())
    assert torch.equal(y, want)


# ================================================================================================ timestep embedding
def timestep_reference(t, dim):
    """util.py timestep_embedding: freqs and t * freqs in torch's fp32 (CPU), cos / sin in fp64; (ref, bound)"""
    half = dim // 2
    freqs = torch.exp(-math.log(10000) * torch.arange(0, half, dtype=torch.float32) / half)
    a = (torch.tensor(t, dtype=torch.int64)[:, None].float() * freqs[None]).double()
    ref = torch.cat([torch.cos(a), torch.sin(a)], dim=-1)
    slope = torch.cat([torch.sin(a).abs(), torch.cos(a).abs()], dim=-1)
    aa = torch.cat([a, a], dim=-1).abs()
    E = aa * 2.0 ** -22 * slope + (aa * 2.0 ** -22) ** 2 / 2 + 2.0 ** -22
    if dim % 2:
        ref, E = F.pad(ref, (0, 1)), F.pad(E, (0, 1))
    return ref, E


@gpu
@pytest.mark.parametrize("dim", [specs.UNET_TXT2AUDIO["model_channels"], 64, 33, 7])
@pytest.mark.parametrize("dev", [False, True])
def test_timestep_embedding(dim, dev):
    """t in [0, 999] (999 included), dim even and odd (a zero last column)"""
    ts = [0, 1, 999, 500, 981, 37, 250, 998]
    flat, y = out_buffer((len(ts), dim))
    if dev:
        td = torch.tensor(ts, dtype=torch.int32, device=DEV)
        probe("TIMESTEP_DEV", t=td, y=flat, N=len(ts), C=dim)
    else:
        th = (C.c_int * len(ts))(*ts)
        probe("TIMESTEP", t=C.cast(th, C.c_void_p).value, y=flat, N=len(ts), C=dim)
    assert_written("timestep", flat, y.numel())
    ref, E = timestep_reference(ts, dim)
    check(f"timestep dim {dim} dev {dev}", ("timestep", "device t" if dev else "host t"), y.cpu(), ref, E, rms=False)
    if dim % 2:
        assert torch.equal(y[:, -1], torch.zeros_like(y[:, -1]))


# ================================================================================================ DDIM
def coef_table(steps, seed, cfg_scale):
    """[steps][6] fp32 {sqrt(a_t), sqrt(a_prev), sqrt(1 - a_prev - sigma^2), sigma, sqrt(1 - a_t), s}"""
    rs = np.random.RandomState(seed)
    rows = []
    for _ in range(steps):
        a_t, a_prev = sorted(rs.uniform(0.05, 0.99, 2))
        sg = 0.0
        rows.append([math.sqrt(a_t), math.sqrt(a_prev), math.sqrt(1 - a_prev - sg * sg), sg, math.sqrt(1 - a_t), cfg_scale])
    return torch.tensor(rows, dtype=torch.float32)


def ddim_reference(x, eu, ec, E_eu, E_ec, c):
    """ddim.py:198-225 on the fp32 coefficient row c, from (eu, ec or None) and their bounds; returns
    ((x_prev, pred_x0), (bounds))"""
    sqrt_at, sqrt_aprev, dir_coef, _, sqrt_om, s = (float(v) for v in c)
    x = x.double()
    if ec is None:
        e, E_e = eu, E_eu
    else:
        e = eu + s * (ec - eu)
        E_e = abs(1 - s) * E_eu + abs(s) * E_ec + U * (2 * abs(s) * (ec - eu).abs() + e.abs())
    p0 = (x - sqrt_om * e) / sqrt_at
    E_p0 = (sqrt_om * E_e + 2 * U * (sqrt_om * e.abs() + x.abs())) / sqrt_at + U * p0.abs()
    xp = sqrt_aprev * p0 + dir_coef * e
    E_xp = sqrt_aprev * E_p0 + dir_coef * E_e + 2 * U * (sqrt_aprev * p0.abs() + dir_coef * e.abs())
    return (xp, p0), (E_xp, E_p0)


@gpu
@pytest.mark.parametrize("single", [0, 1])
@pytest.mark.parametrize("with_p0", [True, False])
@pytest.mark.parametrize("alias", [True, False])
def test_ddim_update_tab(single, with_p0, alias):
    """select_row + ddim_update_tab + step_inc, the captured DDIM step's table lookups, at step 3 of 5"""
    B, n, steps, step0 = 4, 4 * LATENT[0] * LATENT[1], 5, 3
    tab = coef_table(steps, 11 + single, 3.0).to(DEV)
    emb = specs.synth_tensor((steps, 1280), 12).to(DEV)
    x = specs.synth_tensor((B, n), 13).to(DEV)
    eps2 = specs.synth_tensor(((1 if single else 2) * B, n), 14).to(DEV)
    step = torch.tensor([step0], dtype=torch.int32, device=DEV)
    sflat, sel = out_buffer((1280,))
    xflat, xv = out_buffer((B, n))
    xv.copy_(x)
    if alias:
        yflat, yv = xflat, xv
    else:
        yflat, yv = out_buffer((B, n))
    pflat, pv = out_buffer((B, n)) if with_p0 else (None, None)
    probe("DDIM_TAB", x=xflat, x2=eps2, y=yflat, y2=pflat, table=tab, step=step, sel_table=emb, sel_out=sflat,
          sel_cols=1280, N=B, rows=n, single=single)
    assert int(step.item()) == step0 + 1, "step_inc"
    assert_written("select_row", sflat, sel.numel())
    assert torch.equal(sel, emb[step0])
    zeros = torch.zeros_like(x, dtype=torch.float64)
    (xp, p0), (E_xp, E_p0) = ddim_reference(x, eps2[:B].double(), None if single else eps2[B:].double(), zeros, zeros,
                                            tab[step0].cpu())
    assert_written("ddim x_prev", yflat, yv.numel())
    path = f"{'single' if single else 'cfg'} {'alias' if alias else 'x_prev'}"
    check(f"ddim_update_tab {path} p0 {with_p0}", ("ddim_update_tab", path), yv, xp, E_xp, rms=False)
    if not alias:
        assert torch.equal(xv, x), "ddim_update_tab wrote x"
    if with_p0:
        assert_written("ddim pred_x0", pflat, pv.numel())
        check(f"ddim_update_tab pred_x0 {path}", ("ddim_update_tab", "pred_x0"), pv, p0, E_p0, rms=False)


def conv_out_reference(hn, w, bias, B, H, W, single, drop_last_col_tap=False):
    """hn [N][HW][C] -> eps halves (eu, ec or None) and their bounds, fp64 conv2d(3x3, padding 1) + bias"""
    N, HW, Cc = hn.shape
    h = hn.double().permute(0, 2, 1).reshape(N, Cc, H, W)
    w64 = w.double()
    if drop_last_col_tap:     # the mutant: the last column misses its own column's taps
        e = F.conv2d(h, w64, bias.double(), padding=1)
        own = F.conv2d(h, w64 * torch.tensor([0.0, 1.0, 0.0], dtype=torch.float64)[None, None, None, :], padding=1)
        e[..., W - 1] -= own[..., W - 1]
    else:
        e = F.conv2d(h, w64, bias.double(), padding=1)
    S = F.conv2d(h.abs(), w64.abs(), padding=1)
    n = 9 * math.ceil(Cc / 32) + 5
    E = gam(n) * U * S + U * e.abs()
    e, E = e.reshape(N, 4, HW), E.reshape(N, 4, HW)
    if single:
        return e[:B], None, E[:B], None
    return e[:B], e[B:], E[:B], E[B:]


def conv_out_inputs(B, H, W, Cc, single, seed):
    N = B if single else 2 * B
    hn = specs.synth_tensor((N, H * W, Cc), seed)
    w = specs.synth_tensor((4, Cc, 3, 3), seed + 1, scale=1.0 / math.sqrt(9 * Cc))
    bias = specs.synth_tensor((4,), seed + 2, scale=0.1)
    x = specs.synth_tensor((B, 4, H * W), seed + 3)
    return hn, w, bias, x


CONV_OUT = [(4, LATENT[0], LATENT[1], specs.UNET_TXT2AUDIO["model_channels"], 0),
            (4, LATENT[0], LATENT[1], specs.UNET_TXT2AUDIO["model_channels"], 1),
            (2, 1, 13, 100, 0), (2, 9, 1, 100, 1), (1, 1, 1, 36, 0), (3, 5, 39, 64, 0)]


@gpu
@pytest.mark.parametrize("B,H,W,Cc,single", CONV_OUT)
@pytest.mark.parametrize("with_p0", [True, False])
def test_conv_out_ddim(B, H, W, Cc, single, with_p0):
    """the UNet's out conv fused with guidance and the DDIM update: 3x3 borders, 1-wide maps, C % 32 != 0, single,
    pred_x0 null; x updated in place with the coefficients at *step"""
    hn, w, bias, x = conv_out_inputs(B, H, W, Cc, single, 20 + Cc)
    steps, step0 = 4, 2
    tab = coef_table(steps, 21, 3.0)
    w9c4 = w.permute(2, 3, 1, 0).reshape(9, Cc, 4).contiguous()
    xflat, xv = out_buffer((B, 4, H * W))
    xv.copy_(x.to(DEV))
    pflat, pv = out_buffer((B, 4, H * W)) if with_p0 else (None, None)
    step = torch.tensor([step0], dtype=torch.int32, device=DEV)
    probe("CONV_OUT_DDIM", x=hn.to(DEV), w=w9c4.to(DEV), b=bias.to(DEV), y=xflat, y2=pflat, table=tab.to(DEV),
          step=step, N=B, H=H, W=W, C=Cc, single=single)
    assert int(step.item()) == step0, "conv_out_ddim changed the step"
    eu, ec, E_eu, E_ec = conv_out_reference(hn.to(DEV), w.to(DEV), bias.to(DEV), B, H, W, single)
    (xp, p0), (E_xp, E_p0) = ddim_reference(x.to(DEV), eu, ec, E_eu, E_ec, tab[step0])
    path = f"{'single' if single else 'cfg'} {'C%32=0' if Cc % 32 == 0 else 'C%32=r'}"
    assert_written("conv_out_ddim x", xflat, xv.numel())
    check(f"conv_out_ddim B {B} {H}x{W} C {Cc} {path}", ("conv_out_ddim", path), xv, xp, E_xp)
    if with_p0:
        assert_written("conv_out_ddim pred_x0", pflat, pv.numel())
        check(f"conv_out_ddim pred_x0 {path}", ("conv_out_ddim", "pred_x0"), pv, p0, E_p0)


def test_gate_catches_dropped_border_tap():
    """the last column without its own column's taps fails the conv_out_ddim gate"""
    B, H, W, Cc = 2, 4, 6, 64
    hn, w, bias, x = conv_out_inputs(B, H, W, Cc, 0, 30)
    tab = coef_table(1, 31, 3.0)
    eu, ec, E_eu, E_ec = conv_out_reference(hn, w, bias, B, H, W, 0)
    (xp, _), (E_xp, _) = ddim_reference(x, eu, ec, E_eu, E_ec, tab[0])
    mu, mc, _, _ = conv_out_reference(hn, w, bias, B, H, W, 0, drop_last_col_tap=True)
    (mxp, _), _ = ddim_reference(x, mu, mc, E_eu, E_ec, tab[0])
    assert passes(xp.float(), xp, E_xp)
    assert not passes(mxp, xp, E_xp)


def test_gate_catches_swapped_cfg_halves():
    """e = e_c + s (e_u - e_c) instead of e_u + s (e_c - e_u) fails the DDIM gate (conv_out_ddim and ddim_update_tab)"""
    B, H, W, Cc = 2, 3, 5, 32
    hn, w, bias, x = conv_out_inputs(B, H, W, Cc, 0, 40)
    tab = coef_table(1, 41, 3.0)
    eu, ec, E_eu, E_ec = conv_out_reference(hn, w, bias, B, H, W, 0)
    (xp, p0), (E_xp, E_p0) = ddim_reference(x, eu, ec, E_eu, E_ec, tab[0])
    (mxp, mp0), _ = ddim_reference(x, ec, eu, E_ec, E_eu, tab[0])
    assert not passes(mxp, xp, E_xp) and not passes(mp0, p0, E_p0)
    zeros = torch.zeros_like(eu)
    (txp, _), (tE, _) = ddim_reference(x, eu, ec, zeros, zeros, tab[0])
    (sxp, _), _ = ddim_reference(x, ec, eu, zeros, zeros, tab[0])
    assert passes(txp.float(), txp, tE, rms=False) and not passes(sxp, txp, tE, rms=False)
