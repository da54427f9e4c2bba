"""Conformance of the small kernels of the vocoder and diffusion-step back end against float64, kernel by kernel:
HiFi-GAN / BigVGAN's channels-last layout (cf_to_cl) and conv_post (both kernels), BigVGAN's anti-aliased Snake /
SnakeBeta, the NSF noise-conv add and harmonic source, DiffNet's step embedding (host and device timesteps), and the
diffusion step arithmetic: p_sample (eager), the graph-replayed p_sample_tab and the PLMS combine axpby5.

Every GPU case runs ONE production launcher (through agpt_voc_probe, or agpt_nsf_source / agpt_gd_p_sample with eps
given / agpt_axpby5, which call theirs directly) on caller-owned device tensors, and compares it with a reference
written from the reference code's formulas on its own layouts, never from the kernels' indexing:
NeuralSeq/modules/hifigan/hifigan.py:144-169 (noise_convs as Conv1d, conv_post, tanh); BigVGAN's Activation1d
(alias_free_torch/act.py, resample.py, filter.py: replicate pad 5, ratio * conv_transpose1d stride 2 cropped 15 / 15,
Snake / SnakeBeta x + 1 / b sin^2(a x) from activations.py, replicate pad (5, 6), stride-2 low-pass conv1d);
parallel_wavegan/models/source.py:311-532 (SineGen, SourceModuleHnNSF); diff/net.py SinusoidalPosEmb; and
shallow_diffusion_tts.py:134-204 (predict_start_from_noise, clamp, q_posterior, the noise term, the PLMS combinations).
Float outputs are NaN-filled and followed by GUARD canaries: every case asserts that the whole output was written and
nothing past it.

Error model and gates (u = 2^-24; ulp(v) = 2^(floor(log2 |v|) - 23); g(n) = min(n, 6 sqrt(n)), the worst case or the
Higham-Mary probabilistic bound for a sum of n terms, as in test_nn_kernels_gpu.py; the device-function figures are the
CUDA math guide's maximum ulp errors: sinf, cosf, tanhf and expf 2 ulp each):

  * CF_TO_CL: data movement, exact.
  * CONV_POST: the leaky-ReLU is reproduced exactly in fp32 (torch's F.leaky_relu rounds x * slope once, as the kernel
    does); the bias plus 7 C products is a (7C + 1)-term fmaf chain, E = g(7C + 1) u (|b| + sum |w h|) against the fp64
    conv; tanh carries it with its slope 1 - tanh^2 taken at the end of [acc - E, acc + E] nearest 0, plus tanhf's
    2 ulp.  conv_post32_kernel must equal the generic kernel bit for bit, channel by channel.
  * AA_SNAKE: the up-FIR is a 6-term fmaf chain times 2 (exact), E_u = 6 u 2 sum |f x|.  The sine's argument follows
    torch's fp32 arithmetic: theta = fl32(fl32(u) a), sin in fp64; the kernel's argument is then off by at most
    |a| (E_u + u |u|) + 2 u |theta|.  sinf adds 2 ulp, the square, the product with inv_b and the sum with u one
    rounding each (a contracted FMA drops one).  The stride-2 low-pass is a 12-term fmaf chain:
    12 u sum |f s| + sum |f| E_s.  Every case runs twice: with the Kaiser-sinc taps of the state dict, and with a
    random asymmetric 12-tap filter, since the symmetric taps cannot tell a reversed filter from the right one.
  * NSF_ADD: a (K + 1)-term fmaf chain (bias, then K taps; taps outside har read 0) against the fp64 Conv1d(1, C, K,
    st, pad), g(K + 1) u (|b| + sum |w har|), plus one rounding u |out| for the in-place +=.
  * NSF_SOURCE: rad = (f0 (h + 1) / sr) mod 1 is reproduced exactly in fp32 (torch's arithmetic and the kernel's are
    the same two roundings and an exact fractional part).  The phase is the fractional part of the prefix sum seeded
    with rand_ini (harmonic 0 unseeded), computed EXACTLY on the host (every rad and rand_ini is a multiple of 2^-40);
    the kernel's fp64 three-level scan is within (chunks + 1) 20 2^-44 cycles of it.  The kernel then rounds the phase
    to fp32 (u), multiplies by fl32(2 pi) (the reference's fp32 `* 2 * np.pi`; one rounding), takes sinf (2 ulp) and
    scales by sine_amp (one rounding).  uv = f0 > thr is exact (f0 == thr is unvoiced), so the voiced term is the sine
    itself; noise_amp is reproduced exactly in fp32 and na * noise and the sum round once each.  The merge is a
    (dim + 1)-term fmaf chain, g(dim + 1) u (|b| + sum |w x|) + sum |w| E_x, and tanh carries it as above.
  * STEP_EMBED / STEP_EMBED_DEV: the specification is torch's fp32 arithmetic (neg_emb = fp32 of the double
    -ln(1e4) / (C/2 - 1), e_i = expf(i neg_emb), a = t e_i in fp32), reproduced on the CPU; sin / cos in fp64.  A device
    expf 1 ulp off the CPU's moves a by at most 2^-22 |a|:  |y - ref| <= |a| 2^-22 |cos a or sin a| + (|a| 2^-22)^2 / 2
    + 2^-22.  At t = 0 the outputs are exactly 0 (sin) and 1 (cos).
  * P_SAMPLE / P_SAMPLE_TAB: the fp64 formula on the fp32 coefficient row {A, Bc, c1, c2, s}:
    x0 = A x - Bc eps, clamped to [-1, 1] when clip; out = c1 x0 + c2 x + s noise.  Each fp32 product and sum adds one
    rounding of its result, carried forward (a contracted FMA drops one, so it stays inside the bound; no exactness is
    claimed).  The clamp is 1-Lipschitz.
  * AXPBY5: out = a0 x + a1 e0 + a2 e1 + a3 e2 + a4 e3 over the non-null e_i: one rounding per product and per sum.

Teeth: CPU-emulated mutants must FAIL the gate the kernel passes: aa_snake with the taps reversed (only the asymmetric
filter catches it), with zero instead of replicate padding, and with down-sample pads (6, 5); conv_post with the taps
reversed and with leaky slope 0.1; the NSF source with rand_ini applied to harmonic 0, with uv = f0 >= thr, and with
the chunk base shifted by one chunk; nsf_add with the pad sign flipped; the step embedding divided by C/2 instead of
C/2 - 1; p_sample without the clamp; p_sample_tab reading noise row k; axpby5 with its coefficients shifted by one.
They need no device.  The launchers' precondition checks (and agpt_nsf_source's 16-harmonic limit) are tested without a
device too: they throw before anything is launched.
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
GUARD = 64
CANARY = -7777.25
DEV = "cuda"
NSF_CHUNK = 1024
TWO_PI_F32 = float(np.float32(2 * np.pi))

# the VC_OPS, then the entries that reach their kernels through their own production launchers
OPS = _lib.VC_OPS + ("NSF_SOURCE", "P_SAMPLE", "AXPBY5")
EXERCISED = {}          # op -> worst error / bound over the cases that ran it (0 for the exact gates)


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    if EXERCISED:
        print("\nvocoder / diffusion-step kernels exercised: worst error / bound (0 = exact)")
        for k in OPS:
            if k in EXERCISED:
                print(f"  {k:14s}: {EXERCISED[k]:.3f}")


def gam(n):
    return min(n, 6.0 * math.sqrt(n))


def seen(op, ratio=0.0):
    EXERCISED[op] = max(EXERCISED.get(op, 0.0), ratio)


def ulp32(v):
    """the fp32 ulp at |v| (fp64 tensor), rounded up across a power of two, at least the subnormal step"""
    a = v.abs().double() * (1 + 2.0 ** -20)
    e = torch.floor(torch.log2(a.clamp(min=2.0 ** -126)))
    return torch.exp2(e - 23).clamp(min=2.0 ** -149)


def tanh_carry(acc, E):
    """the bound of tanhf(acc') for |acc' - acc| <= E: the largest slope on the interval times E, plus tanhf's 2 ulp"""
    near = (acc.abs() - E).clamp(min=0)
    y = torch.tanh(acc)
    return (1 - torch.tanh(near) ** 2) * E + 2 * ulp32(y), y


# ------------------------------------------------------------------------------------------------ buffers and the probe
def out_f(shape):
    n = math.prod(shape)
    flat = torch.full((n + GUARD,), float("nan"), dtype=torch.float32, device=DEV)
    flat[n:] = CANARY
    return flat, flat[:n].view(shape)


def written(tag, flat):
    n = flat.numel() - GUARD
    assert torch.equal(flat[n:], torch.full_like(flat[n:], CANARY)), f"{tag}: written past the end of the output"
    assert not torch.isnan(flat[:n]).any(), f"{tag}: {int(torch.isnan(flat[:n]).sum())} output elements not written"


def probe(op, stream=True, **kw):
    a = _lib.VocProbeArgs()
    a.op = _lib.VC_OPS.index(op)
    keep = []
    for k, v in kw.items():
        if isinstance(v, torch.Tensor):
            assert v.is_cuda, k
            v = v.data_ptr()
        elif isinstance(v, np.ndarray):
            keep.append(v)
            v = v.ctypes.data
        setattr(a, k, v)
    _lib.check(_lib.lib().agpt_voc_probe(C.byref(a), _lib.cur_stream() if stream else None))


def ratio(y, ref, bound):
    err = (y.double().cpu() - ref.double().cpu()).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    return float((err / (bound.double().cpu() + 1e-300)).max()) if err.numel() else 0.0


def passes(y, ref, bound):
    return ratio(y, ref, bound) <= 1.0


def check(tag, op, y, ref, bound):
    y, ref, bound = y.double().cpu(), ref.double().cpu(), bound.double().cpu()
    w = ratio(y, ref, bound)
    print(f"{tag}: worst err/bound {w:.3f}")
    seen(op, w)
    if w > 1.0:
        err = (y - ref).abs() / (bound + 1e-300)
        idx = np.unravel_index(int(torch.argmax(torch.nan_to_num(err, nan=math.inf)).item()), tuple(y.shape))
        raise AssertionError(f"{tag}: error {w:.3g} x the bound at {idx}: got {float(y[idx])}, want {float(ref[idx])}")


def exact(tag, op, y, want):
    y, want = y.float().cpu(), want.float().cpu()
    assert y.shape == want.shape, (tag, y.shape, want.shape)
    bad = y.contiguous().view(torch.int32) != want.contiguous().view(torch.int32)
    if bad.any():
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError(f"{tag}: {int(bad.sum())} elements differ, first at {i}: got {float(y[i])!r}, "
                             f"want {float(want[i])!r}")
    print(f"{tag}: exact")
    seen(op)


def dev(t):
    return t.float().contiguous().to(DEV)


def rnd(shape, seed, scale=1.0, shift=0.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale + shift


# ================================================================================================ CF_TO_CL
@gpu
@pytest.mark.parametrize("B,Cc,T", [(3, 80, 37), (2, 33, 1), (2, 1, 65), (4, 257, 100), (2, 80, 800)])
def test_cf_to_cl(B, Cc, T):
    x = rnd((B, Cc, T), 3 + Cc + T)
    flat, y = out_f((B, T, Cc))
    probe("CF_TO_CL", x=dev(x), y=y, B=B, C=Cc, L=T)
    written("CF_TO_CL", flat)
    exact(f"CF_TO_CL B={B} C={Cc} T={T}", "CF_TO_CL", y, x.transpose(1, 2))


# ================================================================================================ CONV_POST
def conv_post_ref(x, w, b, slope):
    """hifigan.py:165-167: leaky_relu(x, slope) (fp32, as torch) -> Conv1d(C, c_out, 7, padding=3) in fp64 -> tanh.
    x [B][L][C] rows, w [c_out][C][7] (the reference layout); returns (ref [B][c_out][L], bound)."""
    h = F.leaky_relu(x.float(), slope).double().transpose(1, 2)
    w64 = w.double()
    acc = F.conv1d(h, w64, b.double(), padding=3)
    S = F.conv1d(h.abs(), w64.abs(), b.double().abs(), padding=3)
    E = gam(7 * x.shape[2] + 1) * U * S
    bound, y = tanh_carry(acc, E)
    return y, bound * (1 + 1e-6)


def conv_post_inputs(B, L, Cc, c_out, seed):
    x = rnd((B, L, Cc), seed, 1.5)
    w = rnd((c_out, Cc, 7), seed + 1, 1.2 / math.sqrt(7 * Cc))
    b = rnd((c_out,), seed + 2, 0.3)
    return x, w, b


def run_conv_post(x, w, b, slope):
    B, L, Cc = x.shape
    c_out = w.shape[0]
    flat, y = out_f((B, c_out, L))
    ran = np.full(1, -1, dtype=np.int32)
    probe("CONV_POST", x=dev(x), w=dev(w.permute(0, 2, 1)), b=dev(b), y=y, ran=ran, B=B, L=L, C=Cc, c_out=c_out,
          slope=slope)
    written("CONV_POST", flat)
    return y, "conv_post32" if ran[0] == 1 else "conv_post"


CP_LENGTHS = [1, 2, 3, 6, 7, 255, 256, 257, 511, 513, 70001]   # L % 256 != 0, L < 7, and one L > 2^16


@gpu
@pytest.mark.parametrize("slope", [0.01, 1.0])
@pytest.mark.parametrize("Cc", [4, 8, 16, 32, 64, 128])
def test_conv_post(Cc, slope):
    for L in CP_LENGTHS:
        x, w, b = conv_post_inputs(3, L, Cc, 1, 100 + Cc + L)
        y, kern = run_conv_post(x, w, b, slope)
        assert kern == ("conv_post32" if Cc == 32 else "conv_post"), kern
        ref, bound = conv_post_ref(x, w, b, slope)
        check(f"CONV_POST [{kern}] C={Cc} c_out=1 L={L} slope={slope}", "CONV_POST", y, ref, bound)


@gpu
@pytest.mark.parametrize("c_out", [1, 2, 9, 10])
def test_conv_post_c32_outputs(c_out):
    """C = 32: c_out 1, 2, 9 take conv_post32 (c_out 7 32 4 bytes <= 8 KB), c_out 10 the generic kernel"""
    for L in (3, 257, 513):
        x, w, b = conv_post_inputs(3, L, 32, c_out, 300 + c_out + L)
        y, kern = run_conv_post(x, w, b, 0.01)
        assert kern == ("conv_post32" if c_out <= 9 else "conv_post"), kern
        ref, bound = conv_post_ref(x, w, b, 0.01)
        check(f"CONV_POST [{kern}] C=32 c_out={c_out} L={L}", "CONV_POST", y, ref, bound)


@gpu
@pytest.mark.parametrize("slope", [0.01, 1.0])
def test_conv_post32_matches_the_generic_kernel(slope):
    """per output channel, conv_post32 and the generic kernel accumulate in the same order: bit-identical"""
    for L in (1, 6, 255, 257, 70001):
        x, w, b = conv_post_inputs(3, L, 32, 10, 500 + L)
        y10, k10 = run_conv_post(x, w, b, slope)
        y1, k1 = run_conv_post(x, w[:1], b[:1], slope)
        assert (k10, k1) == ("conv_post", "conv_post32")
        assert torch.equal(y10[:, :1], y1), f"L={L}: conv_post32 differs from the generic kernel"


# ================================================================================================ AA_SNAKE
def asym_taps(seed):
    f = rnd((12,), seed, 0.3)
    f[3] += 0.5
    return f.float()


def kaiser_taps():
    return specs.kaiser_sinc_filter12().reshape(12).float()


def aa_snake_ref(x, a, ib, f, pad_mode="replicate", down_pads=(5, 6)):
    """Activation1d(Snake | SnakeBeta) on x [B][L][C] (fp32), a / ib [C] as the engine precomputes them (alpha, exp'd
    when log-scaled; 1 / (beta + 1e-9)), f [12] the filter taps; returns (ref [B][L][C], bound).  pad_mode / down_pads:
    the mutants."""
    B, L, Cc = x.shape
    xc = x.double().transpose(1, 2)
    f64 = f.double()
    a64, ib64 = a.double()[None, :, None], ib.double()[None, :, None]

    def up(v, taps):
        vp = F.pad(v, (5, 5), mode=pad_mode) if pad_mode == "replicate" else F.pad(v, (5, 5))
        return 2 * F.conv_transpose1d(vp, taps.view(1, 1, 12).expand(Cc, 1, 12), stride=2, groups=Cc)[..., 15:-15]

    u = up(xc, f64)
    E_u = 6 * U * up(xc.abs(), f64.abs())
    theta = (u.float() * a.float()[None, :, None]).double()          # torch's fp32 x * alpha
    E_t = a64.abs() * (E_u + U * u.abs()) + 2 * U * theta.abs()
    sn = torch.sin(theta)
    E_sn = torch.cos(theta).abs() * E_t + E_t ** 2 / 2 + 2.0 ** -22 * (sn.abs() + E_t)
    sq = sn * sn
    E_sq = 2 * sn.abs() * E_sn + E_sn ** 2 + U * sq
    t = ib64 * sq
    s = u + t
    E_s = E_u + ib64.abs() * E_sq + U * t.abs() + U * s.abs()

    def down(v, taps):
        vp = F.pad(v, down_pads, mode="replicate")
        return F.conv1d(vp, taps.view(1, 1, 12).expand(Cc, 1, 12), stride=2, groups=Cc)

    y = down(s, f64)
    E = 12 * U * down(s.abs(), f64.abs()) + down(E_s, f64.abs())
    return y.transpose(1, 2), E.transpose(1, 2) * (1 + 1e-5)


def snake_inputs(B, L, Cc, seed):
    """x of rms ~1.5; per-channel alpha spanning 0.05 .. 400 so that |a u| reaches ~10^3, inv_b in [0.2, 5]"""
    x = rnd((B, L, Cc), seed, 1.5)
    g = torch.Generator().manual_seed(seed + 1)
    a = torch.exp(torch.linspace(math.log(0.05), math.log(400.0), Cc)[torch.randperm(Cc, generator=g)])
    ib = 1.0 / (torch.exp(torch.rand(Cc, generator=g) * 3.2 - 1.6) + 1e-9)
    return x.float(), a.float(), ib.float()


AA_LENGTHS = [1, 2, 5, 6, 7, 63, 64, 65, 129, 1000]


@gpu
@pytest.mark.parametrize("taps", ["kaiser", "asymmetric"])
@pytest.mark.parametrize("Cc", [4, 32, 33, 96])
def test_aa_snake(Cc, taps):
    f = kaiser_taps() if taps == "kaiser" else asym_taps(7)
    fh = f.numpy().astype(np.float32)
    for L in AA_LENGTHS:
        x, a, ib = snake_inputs(3, L, Cc, 40 + Cc + L)
        flat, y = out_f((3, L, Cc))
        probe("AA_SNAKE", x=dev(x), y=y, a=dev(a), inv_b=dev(ib), taps=fh, B=3, L=L, C=Cc)
        written("AA_SNAKE", flat)
        ref, bound = aa_snake_ref(x, a, ib, f)
        check(f"AA_SNAKE {taps} C={Cc} L={L}", "AA_SNAKE", y, ref, bound)


# ================================================================================================ NSF_ADD
def nsf_add_ref(x, har, w, b, st, pad, flip_pad=False):
    """x [B][L][C] + Conv1d(1, C, K, stride st, padding pad)(har [B][Lh]) (hifigan.py:155-157); (ref, bound).
    flip_pad: the mutant that reads har[p st + pad + k]."""
    K = w.shape[1]
    h = har.double()[:, None]
    if flip_pad:
        h = torch.cat([h[..., 2 * pad:], torch.zeros_like(h[..., :2 * pad])], dim=-1)
    w64 = w.double()[:, None]
    acc = F.conv1d(h, w64, b.double(), stride=st, padding=pad).transpose(1, 2)
    S = F.conv1d(h.abs(), w64.abs(), b.double().abs(), stride=st, padding=pad).transpose(1, 2)
    out = x.double() + acc
    return out, (gam(K + 1) * U * S + U * out.abs()) * (1 + 1e-6)


NSF_CONVS = [(64, 32, 16), (8, 4, 2), (4, 2, 1), (1, 1, 0)]   # HiFi-GAN V1's noise convs, the last stage's 1x1


@gpu
@pytest.mark.parametrize("K,st,pad", NSF_CONVS)
@pytest.mark.parametrize("L,Cc", [(1, 32), (7, 64), (200, 33), (2048, 256)])
def test_nsf_add(K, st, pad, L, Cc):
    B = 3
    Lh = L * st
    x = rnd((B, L, Cc), K + L + Cc, 0.8)
    har = torch.tanh(rnd((B, Lh), K + L + Cc + 1, 1.0))
    w = rnd((Cc, K), K + L + Cc + 2, 1.0 / math.sqrt(K))
    b = rnd((Cc,), K + L + Cc + 3, 0.1)
    flat, y = out_f((B, L, Cc))
    y.copy_(dev(x))
    probe("NSF_ADD", y=y, x=dev(har), w=dev(w), b=dev(b), B=B, L=L, C=Cc, Lh=Lh, K=K, st=st, pad=pad)
    written("NSF_ADD", flat)
    ref, bound = nsf_add_ref(x, har, w, b, st, pad)
    check(f"NSF_ADD K={K} st={st} pad={pad} L={L} C={Cc}", "NSF_ADD", y, ref, bound)
    if L > 1:        # the first and last rows, where taps fall outside har
        check(f"NSF_ADD K={K} edges", "NSF_ADD", y[:, [0, -1]], ref[:, [0, -1]], bound[:, [0, -1]])


# ================================================================================================ NSF_SOURCE
SR = 22050.0


def nsf_rad(f0, dim, sr=SR):
    """source.py: f0_buf[..., h] = f0 * (h + 1); rad = (f0_buf / sr) % 1 -- in fp32, as torch computes it"""
    f0 = f0.float()
    cols = [f0 if h == 0 else f0 * float(h + 1) for h in range(dim)]
    v = torch.stack(cols, -1)
    return torch.remainder(v / torch.full_like(v, sr), 1.0)


def nsf_source_ref(f0, rand_ini, noise, lw, lb, dim, thr, sine_amp=0.1, noise_std=0.003, mutant=None):
    """SineGen + SourceModuleHnNSF on f0 [B][L] (at the sample rate); (ref har [B][L], bound).  mutant: 'rand0' (rand_ini
    seeds harmonic 0 too), 'uv_ge' (uv = f0 >= thr), 'chunk' (every sample past the first chunk uses the base of the
    chunk before its own)."""
    B, L = f0.shape
    rad = nsf_rad(f0, dim)                                                          # [B][L][dim] fp32
    q = rad.double() * 2.0 ** 40
    assert torch.equal(q, torch.round(q)), "every rad must be a multiple of 2^-40 for the exact phase"
    qi = q.long()
    ini = torch.zeros(B, dim, dtype=torch.long)
    if rand_ini is not None:
        r = rand_ini.double() * 2.0 ** 40
        assert torch.equal(r, torch.round(r))
        ini = r.long()
        if mutant != "rand0":
            ini[:, 0] = 0
    cs = torch.cumsum(qi, dim=1)
    if mutant == "chunk":
        base = torch.zeros_like(cs)
        for c in range(1, -(-L // NSF_CHUNK)):
            lo, hi = c * NSF_CHUNK, min((c + 1) * NSF_CHUNK, L)
            prev = cs[:, (c - 1) * NSF_CHUNK - 1] if c >= 2 else torch.zeros_like(cs[:, 0])
            base[:, lo:hi] = (cs[:, lo - 1] - prev)[:, None]
        cs = cs - base
    ph = torch.remainder(cs + ini[:, None, :], 2 ** 40).double() / 2.0 ** 40     # exact fractional phase
    E_ph = (-(-L // NSF_CHUNK) + 1) * 20 * 2.0 ** -44                               # the kernel's fp64 scan
    theta = ph * TWO_PI_F32
    E_th = TWO_PI_F32 * (E_ph + U * ph) + U * (theta.abs() + TWO_PI_F32 * E_ph)
    sn = torch.sin(theta)
    E_sn = torch.cos(theta).abs() * E_th + E_th ** 2 / 2 + 2.0 ** -22 * (sn.abs() + E_th)
    amp = float(np.float32(sine_amp))                                              # `* self.sine_amp` in fp32
    sines = amp * sn
    E_sines = amp * E_sn + U * sines.abs()
    uv = ((f0 >= thr) if mutant == "uv_ge" else (f0 > thr)).double()[..., None]   # [B][L][1]
    # uv * noise_std + (1 - uv) * sine_amp / 3 in fp32, uv 0 or 1: noise_std or fl32(fl32(sine_amp) / 3)
    na_u = float(np.float32(sine_amp) / np.float32(3))
    na = uv * float(np.float32(noise_std)) + (1 - uv) * na_u
    nz = noise.double() if noise is not None else torch.zeros(B, L, dim, dtype=torch.float64)
    nt = na * nz
    xv = sines * uv + nt
    E_x = E_sines * uv + U * nt.abs() + U * xv.abs()
    w64 = lw.double()
    acc = float(lb) + (xv * w64).sum(-1)
    S = abs(float(lb)) + (xv.abs() * w64.abs()).sum(-1)
    E_acc = gam(dim + 1) * U * S + (E_x * w64.abs()).sum(-1)
    bound, y = tanh_carry(acc, E_acc)
    return y, bound * (1 + 1e-5)


def nsf_inputs(B, L, dim, thr, seed, with_rand, with_noise):
    """f0 [B][L]: voiced runs (up to ~1.9 kHz: with 16 harmonics rad wraps past 1), unvoiced zeros, and samples exactly
    at thr; every f0 a multiple of 2^-8 (so every rad is a multiple of 2^-40)"""
    g = torch.Generator().manual_seed(seed)
    f0 = torch.round((80.0 + 1800.0 * torch.rand(B, L, generator=g)) * 256) / 256
    f0[torch.rand(B, L, generator=g) < 0.2] = 0.0
    f0[torch.rand(B, L, generator=g) < 0.1] = thr
    f0[:, 0] = thr
    rand_ini = torch.rand(B, dim, generator=g) if with_rand else None
    noise = torch.randn(B, L, dim, generator=g) if with_noise else None
    lw = torch.randn(dim, generator=g) * 0.6
    lb = float(torch.randn(1, generator=g)) * 0.1
    return f0.float(), rand_ini, noise, lw.float(), np.float32(lb)


def run_nsf_source(f0, rand_ini, noise, lw, lb, dim, thr, stream=True):
    B, L = f0.shape
    flat, har = out_f((B, L))
    lwh = lw.numpy().astype(np.float32)
    fd = dev(f0)
    rd = dev(rand_ini) if rand_ini is not None else None
    nd = dev(noise) if noise is not None else None
    _lib.check(_lib.lib().agpt_nsf_source(
        fd.data_ptr(), B, L, dim, SR, lwh.ctypes.data, float(lb), rd.data_ptr() if rd is not None else None,
        nd.data_ptr() if nd is not None else None, 0.1, 0.003, thr, har.data_ptr(), _lib.cur_stream()))
    torch.cuda.synchronize()
    written("NSF_SOURCE", flat)
    return har


NSF_LENGTHS = [1, 3, 4, 5, 1023, 1024, 1025, 4097, 100003]


@gpu
@pytest.mark.parametrize("dim", [1, 9, 16])
@pytest.mark.parametrize("L", NSF_LENGTHS)
def test_nsf_source(L, dim):
    thr = 50.0
    for k, (with_rand, with_noise) in enumerate([(True, True), (False, True), (True, False), (False, False)]):
        if L > 5000 and k in (1, 2):
            continue
        f0, ri, nz, lw, lb = nsf_inputs(3, L, dim, thr, 17 * L + dim + k, with_rand, with_noise)
        har = run_nsf_source(f0, ri, nz, lw, lb, dim, thr)
        ref, bound = nsf_source_ref(f0, ri, nz, lw, lb, dim, thr)
        check(f"NSF_SOURCE L={L} dim={dim} rand_ini={with_rand} noise={with_noise}", "NSF_SOURCE", har, ref, bound)


# ================================================================================================ STEP_EMBED(_DEV)
def step_embed_ref(ts, Cc, divisor=None):
    """SinusoidalPosEmb in torch's fp32 arithmetic (module docstring): (ref [B][C], bound).  divisor: the mutant's."""
    half = Cc // 2
    d = half - 1 if divisor is None else divisor
    neg = torch.tensor(-(math.log(10000.0) / d), dtype=torch.float32)
    f = torch.exp(torch.arange(half, dtype=torch.float32) * neg)
    a = (torch.tensor(ts, dtype=torch.int64).float()[:, None] * f[None]).double()
    ref = torch.cat([torch.sin(a), torch.cos(a)], dim=-1)
    slope = torch.cat([torch.cos(a).abs(), torch.sin(a).abs()], dim=-1)
    aa = torch.cat([a, a], dim=-1).abs()
    return ref, aa * 2.0 ** -22 * slope + (aa * 2.0 ** -22) ** 2 / 2 + 2.0 ** -22


def timesteps(B, seed):
    g = torch.Generator().manual_seed(seed)
    ts = [0, 1, 99, 999] + torch.randint(0, 1000, (max(B - 4, 0),), generator=g).tolist()
    return ts[:B]


@gpu
@pytest.mark.parametrize("on_device", [False, True])
@pytest.mark.parametrize("Cc", [8, 32, 256])
@pytest.mark.parametrize("B", [4, 37, 256])
def test_step_embed(Cc, B, on_device):
    ts = timesteps(B, Cc + B)
    flat, y = out_f((B, Cc))
    if on_device:
        op = "STEP_EMBED_DEV"
        probe(op, t=torch.tensor(ts, dtype=torch.int32, device=DEV), y=y, B=B, C=Cc)
    else:
        op = "STEP_EMBED"
        probe(op, t=np.array(ts, dtype=np.int32), y=y, B=B, C=Cc)
    written(op, flat)
    ref, bound = step_embed_ref(ts, Cc)
    check(f"{op} C={Cc} B={B}", op, y, ref, bound)
    half = Cc // 2
    assert torch.equal(y[0, :half].cpu(), torch.zeros(half)) and torch.equal(y[0, half:].cpu(), torch.ones(half)), \
        "t = 0 must give exactly sin 0 = 0 and cos 0 = 1"


# ================================================================================================ P_SAMPLE / P_SAMPLE_TAB
def p_sample_ref(x, eps, noise, coef, clip):
    """shallow_diffusion_tts.py:134-166 on x / eps / noise [B][n] and fp32 coefficient rows coef [B][5] = {A, Bc, c1, c2,
    s}; (ref, bound)"""
    A, Bc, c1, c2, s = (coef.double()[:, i:i + 1] for i in range(5))
    x, e = x.double(), eps.double()
    p1, p2 = A * x, Bc * e
    x0 = p1 - p2
    E0 = U * (p1.abs() + p2.abs() + x0.abs())
    if clip:
        x0 = x0.clamp(-1.0, 1.0)
    q1, q2 = c1 * x0, c2 * x
    o = q1 + q2
    E = c1.abs() * E0 + U * (q1.abs() + q2.abs() + o.abs())
    if noise is not None:
        q3 = s * noise.double()
        o = o + q3
        E = E + U * (q3.abs() + o.abs())
    return o, E * (1 + 1e-6)


def coef_rows(rows, seed):
    """{A, Bc, c1, c2, s} rows: x0 = A x - Bc eps lands on both sides of +-1"""
    g = torch.Generator().manual_seed(seed)
    A = 1.0 + 20.0 * torch.rand(rows, generator=g)
    Bc = 0.1 + 20.0 * torch.rand(rows, generator=g)
    c1, c2 = torch.rand(rows, generator=g), torch.rand(rows, generator=g)
    s = 0.5 * torch.rand(rows, generator=g)
    return torch.stack([A, Bc, c1, c2, s], 1).float()


P_SIZES = [(3, 80 * 37), (3, 1184 * 256 + 1007), (1, 1)]


@gpu
@pytest.mark.parametrize("with_noise", [True, False])
@pytest.mark.parametrize("clip", [1, 0])
@pytest.mark.parametrize("B,n", P_SIZES)
def test_p_sample(B, n, clip, with_noise):
    x = rnd((B, n), n + B, 0.2)
    eps = rnd((B, n), n + B + 1, 0.2)
    noise = rnd((B, n), n + B + 2) if with_noise else None
    coef = coef_rows(B, n + clip)
    flat, y = out_f((B, n))
    ch = np.ascontiguousarray(coef.numpy())
    xd, ed = dev(x), dev(eps)          # (held: a temporary's memory could be handed to the next tensor)
    nd = dev(noise) if with_noise else None
    _lib.check(_lib.lib().agpt_gd_p_sample(None, xd.data_ptr(), ed.data_ptr(), None, ch.ctypes.data,
                                           nd.data_ptr() if nd is not None else None, clip, B, n, y.data_ptr(),
                                           _lib.cur_stream()))
    torch.cuda.synchronize()
    written("P_SAMPLE", flat)
    ref, bound = p_sample_ref(x, eps, noise, coef, clip)
    check(f"P_SAMPLE B={B} n={n} clip={clip} noise={with_noise}", "P_SAMPLE", y, ref, bound)


@gpu
@pytest.mark.parametrize("with_noise", [True, False])
@pytest.mark.parametrize("clip", [1, 0])
@pytest.mark.parametrize("B,n", P_SIZES[:2])
def test_p_sample_tab(B, n, clip, with_noise):
    """k = *ctr at 0, in the middle and at nsteps - 1; noise row nsteps - 1 - k; x updated in place"""
    nsteps = 7
    tab = coef_rows(nsteps, 70 + n)
    noises = rnd((nsteps, B, n), 71 + n) if with_noise else None
    nd = dev(noises) if with_noise else None
    slot = torch.tensor([nd.data_ptr() if with_noise else 0], dtype=torch.int64, device=DEV)
    for k in (0, 3, nsteps - 1):
        x = rnd((B, n), 72 + n + k, 0.2)
        eps = rnd((B, n), 73 + n + k, 0.2)
        flat, xio = out_f((B, n))
        xio.copy_(dev(x))
        ctr = torch.tensor([k], dtype=torch.int32, device=DEV)
        probe("P_SAMPLE_TAB", y=xio, x=dev(eps), w=dev(tab), ctr=ctr, noises_pp=slot, noise_stride=B * n,
              nsteps=nsteps, clip=clip, B=B, n=n)
        written("P_SAMPLE_TAB", flat)
        assert int(ctr.item()) == k, "p_sample_tab must not move the step counter"
        row = tab[k:k + 1].expand(B, 5)
        ref, bound = p_sample_ref(x, eps, noises[nsteps - 1 - k] if with_noise else None, row, clip)
        check(f"P_SAMPLE_TAB B={B} n={n} clip={clip} noise={with_noise} k={k}", "P_SAMPLE_TAB", xio, ref, bound)


# ================================================================================================ AXPBY5
def axpby5_ref(x, es, coef):
    """a0 x + a1 e0 + a2 e1 + a3 e2 + a4 e3 over the non-null e_i, coef [B][5]; (ref, bound)"""
    a = [coef.double()[:, i:i + 1] for i in range(5)]
    o = a[0] * x.double()
    E = U * o.abs()
    for i, e in enumerate(es):
        if e is None:
            continue
        p = a[i + 1] * e.double()
        o = o + p
        E = E + U * (p.abs() + o.abs())
    return o, E * (1 + 1e-6)


@gpu
@pytest.mark.parametrize("mask", range(16))
def test_axpby5(mask):
    B, n = 3, (1184 * 256 + 333 if mask == 15 else 80 * 37)
    x = rnd((B, n), 90 + mask)
    es = [rnd((B, n), 91 + mask + i) if mask >> i & 1 else None for i in range(4)]
    coef = (rnd((B, 5), 95 + mask) * 2).float()
    flat, y = out_f((B, n))
    xd = dev(x)
    ed = [dev(e) if e is not None else None for e in es]
    ch = np.ascontiguousarray(coef.numpy())
    _lib.check(_lib.lib().agpt_axpby5(xd.data_ptr(), *[e.data_ptr() if e is not None else None for e in ed],
                                      ch.ctypes.data, B, n, y.data_ptr(), _lib.cur_stream()))
    torch.cuda.synchronize()
    written("AXPBY5", flat)
    ref, bound = axpby5_ref(x, es, coef)
    check(f"AXPBY5 e_i given {mask:04b} n={n}", "AXPBY5", y, ref, bound)


# ================================================================================================ preconditions (no device)
def _refused(op, match, **kw):
    with pytest.raises(RuntimeError, match=match):
        probe(op, stream=False, **kw)


def test_probe_refuses_conv_post_beyond_its_limits():
    _refused("CONV_POST", "C % 4", B=1, L=100, C=6, c_out=1, slope=0.01)
    _refused("CONV_POST", "48 KB", B=1, L=100, C=1024, c_out=2, slope=0.01)


def test_probe_refuses_an_empty_snake_input():
    _refused("AA_SNAKE", "L >= 1", taps=np.zeros(12, dtype=np.float32), B=1, L=0, C=32)


def test_probe_refuses_an_nsf_add_without_taps_or_stride():
    _refused("NSF_ADD", "K >= 1", B=1, L=10, C=32, Lh=10, K=0, st=1, pad=0)
    _refused("NSF_ADD", "stride >= 1", B=1, L=10, C=32, Lh=10, K=2, st=0, pad=0)


def test_probe_refuses_step_embeddings_it_cannot_index():
    t = np.zeros(257, dtype=np.int32)
    for op in ("STEP_EMBED", "STEP_EMBED_DEV"):
        _refused(op, "even C", t=t, B=4, C=33)
        _refused(op, "C / 2 > 1", t=t, B=4, C=2)
    _refused("STEP_EMBED", "B <= 256", t=t, B=257, C=32)


def test_probe_refuses_a_p_sample_tab_without_steps():
    _refused("P_SAMPLE_TAB", "nsteps >= 1", B=1, n=10, nsteps=0)


def test_nsf_source_refuses_seventeen_harmonics():
    f0, lw, har = (np.zeros(17, dtype=np.float32) for _ in range(3))
    rc = _lib.lib().agpt_nsf_source(f0.ctypes.data, 1, 1, 17, SR, lw.ctypes.data, 0.0, None, None, 0.1, 0.003, 0.0,
                                    har.ctypes.data, None)
    with pytest.raises(RuntimeError, match="at most 16 harmonics"):
        _lib.check(rc)


# ================================================================================================ mutants (CPU)
def test_gate_catches_reversed_snake_taps_only_with_an_asymmetric_filter():
    x, a, ib = snake_inputs(2, 65, 8, 5)
    fk, fa = kaiser_taps(), asym_taps(7)
    ref, bound = aa_snake_ref(x, a, ib, fk)
    assert passes(ref.float(), ref, bound)
    assert passes(aa_snake_ref(x, a, ib, fk.flip(0))[0].float(), ref, bound)     # symmetric taps: invisible
    ref, bound = aa_snake_ref(x, a, ib, fa)
    assert passes(ref.float(), ref, bound)
    assert not passes(aa_snake_ref(x, a, ib, fa.flip(0))[0].float(), ref, bound)


def test_gate_catches_zero_padded_snake():
    x, a, ib = snake_inputs(2, 65, 8, 6)
    x = x + 2.0                          # an offset, so the edges differ from zero padding
    ref, bound = aa_snake_ref(x, a, ib, kaiser_taps())
    assert not passes(aa_snake_ref(x, a, ib, kaiser_taps(), pad_mode="zeros")[0].float(), ref, bound)


def test_gate_catches_swapped_downsample_pads():
    x, a, ib = snake_inputs(2, 65, 8, 8)
    ref, bound = aa_snake_ref(x, a, ib, kaiser_taps())
    assert not passes(aa_snake_ref(x, a, ib, kaiser_taps(), down_pads=(6, 5))[0].float(), ref, bound)


def test_gate_catches_reversed_conv_post_taps_and_a_wrong_slope():
    x, w, b = conv_post_inputs(2, 257, 32, 1, 9)
    ref, bound = conv_post_ref(x, w, b, 0.01)
    assert passes(ref.float(), ref, bound)
    assert not passes(conv_post_ref(x, w.flip(2), b, 0.01)[0].float(), ref, bound)
    assert not passes(conv_post_ref(x, w, b, 0.1)[0].float(), ref, bound)


@pytest.mark.parametrize("mutant", ["rand0", "uv_ge", "chunk"])
def test_gate_catches_nsf_source_mutants(mutant):
    thr, dim = 50.0, 9
    f0, ri, nz, lw, lb = nsf_inputs(2, 4097, dim, thr, 11, True, True)
    ref, bound = nsf_source_ref(f0, ri, nz, lw, lb, dim, thr)
    assert passes(ref.float(), ref, bound)
    assert not passes(nsf_source_ref(f0, ri, nz, lw, lb, dim, thr, mutant=mutant)[0].float(), ref, bound)


def test_gate_catches_flipped_nsf_pad():
    K, st, pad = NSF_CONVS[0]
    L, Cc = 40, 16
    x, har = rnd((2, L, Cc), 1), torch.tanh(rnd((2, L * st), 2))
    w, b = rnd((Cc, K), 3, 1.0 / math.sqrt(K)), rnd((Cc,), 4, 0.1)
    ref, bound = nsf_add_ref(x, har, w, b, st, pad)
    assert passes(ref.float(), ref, bound)
    assert not passes(nsf_add_ref(x, har, w, b, st, pad, flip_pad=True)[0].float(), ref, bound)


def test_gate_catches_step_embedding_divided_by_half():
    ts = timesteps(37, 3)
    ref, bound = step_embed_ref(ts, 32)
    assert passes(ref.float(), ref, bound)
    assert not passes(step_embed_ref(ts, 32, divisor=16)[0].float(), ref, bound)


def test_gate_catches_p_sample_without_the_clamp():
    x, eps, noise = rnd((3, 500), 1, 0.2), rnd((3, 500), 2, 0.2), rnd((3, 500), 3)
    coef = coef_rows(3, 4)
    ref, bound = p_sample_ref(x, eps, noise, coef, 1)
    assert passes(ref.float(), ref, bound)
    assert not passes(p_sample_ref(x, eps, noise, coef, 0)[0].float(), ref, bound)


def test_gate_catches_p_sample_tab_reading_noise_row_k():
    nsteps, k = 7, 2
    tab = coef_rows(nsteps, 5)
    noises = rnd((nsteps, 2, 400), 6)
    x, eps = rnd((2, 400), 7, 0.2), rnd((2, 400), 8, 0.2)
    row = tab[k:k + 1].expand(2, 5)
    ref, bound = p_sample_ref(x, eps, noises[nsteps - 1 - k], row, 1)
    assert not passes(p_sample_ref(x, eps, noises[k], row, 1)[0].float(), ref, bound)


def test_gate_catches_axpby5_coefficients_shifted_by_one():
    x = rnd((3, 300), 1)
    es = [rnd((3, 300), 2 + i) for i in range(4)]
    coef = rnd((3, 5), 9).float()
    ref, bound = axpby5_ref(x, es, coef)
    assert passes(ref.float(), ref, bound)
    assert not passes(axpby5_ref(x, es, coef.roll(-1, dims=1))[0].float(), ref, bound)


@gpu
def test_every_op_exercised():
    """runs last in this module: every AGPT_VC_* selector and the three direct entries have been through a gate"""
    missing = [op for op in OPS if op not in EXERCISED]
    assert not missing, f"not exercised: {missing}"
