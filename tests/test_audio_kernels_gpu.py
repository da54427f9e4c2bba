"""Conformance of the kernels that touch audio samples and spectrogram bins against float64 and torch's fp32, kernel by
kernel: the torchlibrosa log-mel front end (framing, power / mel / log / bn0), the emotion encoder's power mel, the
sound-extraction STFT and its inverse, LASS's mask input and output stores, Cnn14's resampler and pooling tail, the CLAP
scorer's L2 norms and similarity, and wav2vec2's conv stem (conv0 + GroupNorm + GELU).

Every GPU case runs ONE production launcher through agpt_audio_probe on caller-owned device tensors and compares it with
a reference written from the reference code's formulas on its own layouts, never from the kernels' indexing:
torchlibrosa's Spectrogram (center, reflect) / LogmelFilterBank (ref 1, amin 1e-10) and Cnn14's bn0;
sound_extraction/utils/stft.py transform / inverse; librosa's power mel as make_golden_emotion.py restates it;
torchaudio's Resample through specs.sinc_resample_kernel and CLAPWrapper.resample_and_duration's crop / tile; HF
Wav2Vec2GroupNormConvLayer; Cnn14.forward's pooling tail; CLAPWrapper's normalisation and compute_similarity;
UNetRes_FiLM's bn1 on the padded input and after_conv2 -> F.pad(x, (0, 2)) -> crop -> sigmoid.  Float outputs are
NaN-filled and followed by GUARD canaries: every case asserts that the whole output was written and nothing past it.

Error model and gates (u = 2^-24; ulp(v) = 2^(floor(log2 |v|) - 23); device-function ulp figures are the CUDA math
guide's; g(n) = min(n, 6 sqrt(n)), the worst case or the Higham-Mary probabilistic bound for a sum of n terms, as in
test_nn_kernels_gpu.py):

  * FRAMES, STFT_ROWS: data movement, exact (reflect padding is x[-s] / x[2 (N - 1) - s]; STFT rows past N + n are 0).
  * LOGMEL: the power re^2 + im^2 is FMA-contracted (at most 2 u relative); the mel product is a sequential fmaf chain
    of nb non-negative terms, (g(nb) + 2) u relative to the fp64 mel; the 1e-10 clamp is 1-Lipschitz; 10 log10f adds
    10 / ln 10 times that relative error plus log10f's 2 ulp and one rounding; bn0 is one FMA, so |s| times the dB
    error plus u (|s db| + |t|).  CH 4 writes channels 1..3 exactly 0.
  * POWMEL: the same without the log: (g(201) + 2) u relative.
  * MAGPHASE: the magnitude is exact against torch's fp32 re**2 + im**2 and a correctly rounded sqrt (what torch
    computes on the GPU; the fp32 sum's sqrt taken in fp64 and rounded once, since torch's vectorised CPU sqrtf is not
    always correctly rounded); the kernel's __fmul_rn / __fadd_rn keep nvcc from contracting the power.  The phase is within atan2f's 3 ulp of fp64 atan2, and exact (sign of zero included)
    against torch's fp32 atan2 where re or im is +-0.
  * ISTFT_FRAMES: mag cosf(phase) / mag sinf(phase): |mag| 2 ulp(cos) plus one rounding; row T and columns >= 2 nb
    exactly 0.
  * ISTFT_FINISH: exact against torch fp32: divide where ws > FLT_MIN (np.finfo(float32).tiny), then multiply by
    n / hop.
  * RESAMPLE: a fmaf chain over the taps inside the clip, g(taps) u sum |ker x| against the fp64 conv over the
    zero-padded clip.
  * W2V_STEM: conv0 is a k0-term fmaf chain (k0 u sum |w x|); the statistics are fp64 over those fp32 values, so the
    mean moves by at most the mean conv error and sigma by at most the largest (sigma is 1-Lipschitz in the max norm),
    and the mean and rstd are rounded to fp32; the affine is one subtraction and one FMA with gamma rstd rounded; GELU's
    slope is at most 1.13 and gelu_erf's own evaluation adds (4 + |z|) u |z| + 2 u |gelu|.  Rows T0 .. T0 + zpad - 1
    are exactly 0, rows past them are untouched, and cnt is back at 0 (a second call is bit-identical).
  * CNN14_HEAD: sequential fp32 means over F (g(F) u of sum |x| / F plus the division), the max is 1-Lipschitz, the
    mean over T adds g(T) u and a division, the final sum one rounding.
  * L2NORM2: relative, (g(D) + 6) u |ref| (the first norm's scale error cancels in the second division).
  * SIMILARITY: g(D) u |scale| sum |a t| plus the scale's rounding; the argmax over audio candidates per text equals the
    fp64 argmax unless the top two are within the sum of their bounds.
  * LASS_INPUT: channel 0 is one FMA of x with the folded bn1 (s, t rounded to fp32 on the host, as lass_create folds
    them) against the fp64 BatchNorm, so |x| |s - s64| + |t - t64| + u |out|; channel 1 is x exactly; channels 2..3 are
    0; padded rows t >= T hold bn1(0) = t exactly in channel 0 (the reference pads before encoder_block1's bn1) and 0
    in channel 1.
  * LASS_HEAD: the logit is a 32-term fmaf chain plus the bias, 32 u sum |x w| + u |logit|; the mask is sigmoid of it
    within sigma (1 - sigma) times that plus expf's 2 ulp and two roundings; the two padded bins are exactly logit 0 and
    mask 0.5.

Engine behaviour beyond the reference, stated rather than tested: cnn14_head_kernel takes the max with fmaxf, which
drops a NaN where torch.max keeps it.

Teeth: ten CPU-emulated mutants must FAIL the gate the kernel passes: symmetric framing / STFT-row padding (x[-s - 1]),
an FMA-contracted magnitude, the phase from atan(im / re) with a quadrant fix that drops the sign of zero, ISTFT_FINISH
dividing where ws >= FLT_MIN, the resampler's tiling wrapped at clip instead of R, single-pass fp32 E[x^2] - E[x]^2
stem statistics, stem chunks merged with equal weights, the log-mel without the amin clamp, the pooling head's max over
frequency, and LASS's bias applied to the padded bins.  They need no device.  The probe's precondition checks (reflect
padding, two inverse-STFT frames, the stem's k0 and C, crop starts) are tested without a device too: they throw before
anything is launched.
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
UNTOUCHED = -5555.5
DEV = "cuda"
FLT_MIN = float(np.finfo(np.float32).tiny)

EXERCISED = {}          # op -> worst error / bound over the cases that ran it (0 for the exact gates)


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    if EXERCISED:
        print("\naudio kernels exercised: worst error / bound (0 = exact)")
        for k in _lib.AU_OPS:
            if k in EXERCISED:
                print(f"  {k:13s}: {EXERCISED[k]:.3f}")


def gam(n):
    return min(n, 6.0 * math.sqrt(n))


def seen(op, ratio=0.0):
    EXERCISED[op] = max(EXERCISED.get(op, 0.0), ratio)


def ulp32(v):
    """the fp32 ulp at |v| (fp64 tensor), rounded up across a power of two, at least the subnormal step"""
    a = v.abs().double() * (1 + 2.0 ** -20)
    e = torch.floor(torch.log2(a.clamp(min=2.0 ** -126)))
    return torch.exp2(e - 23).clamp(min=2.0 ** -149)


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
    a = _lib.AudioProbeArgs()
    a.op = _lib.AU_OPS.index(op)
    keep = []
    for k, v in kw.items():
        if isinstance(v, torch.Tensor):
            assert v.is_cuda, k
            v = v.data_ptr()
        elif isinstance(v, np.ndarray):
            keep.append(v)
            v = v.ctypes.data
        setattr(a, k, v)
    _lib.check(_lib.lib().agpt_audio_probe(C.byref(a), _lib.cur_stream() if stream else None))


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


def same(y, want):
    """bitwise equality (so -0 != +0 and NaN == NaN)"""
    y, want = y.float().cpu().contiguous(), want.float().cpu().contiguous()
    return y.shape == want.shape and torch.equal(y.view(torch.int32), want.view(torch.int32))


def exact(tag, op, y, want):
    y, want = y.float().cpu(), want.float().cpu()
    assert y.shape == want.shape, (tag, y.shape, want.shape)
    bad = y.view(torch.int32) != want.contiguous().view(torch.int32)
    if bad.any():
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError(f"{tag}: {int(bad.sum())} elements differ, first at {i}: got {float(y[i])!r}, "
                             f"want {float(want[i])!r}")
    print(f"{tag}: exact")
    seen(op)


def dev(t):
    return t.float().contiguous().to(DEV)


# ================================================================================================ FRAMES / STFT_ROWS
def reflect_frames(x, n, hop, mode="reflect"):
    """torchlibrosa Spectrogram's framing: x [B][N] padded by n / 2 each side (center=True, pad_mode='reflect'),
    frames t hop .. t hop + n - 1 for t <= N // hop (what conv1d(stride=hop) reads).  mode 'symmetric': the mutant's
    edge-repeating pad."""
    N = x.shape[1]
    xp = torch.from_numpy(np.pad(x.numpy(), ((0, 0), (n // 2, n // 2)), mode=mode))
    return xp.unfold(1, n, hop)[:, :N // hop + 1]


def stft_rows_ref(x, n, hop, mode="reflect"):
    """stft.py transform's input: F.pad(reflect) [B][N + n], read as rows of hop samples (zero past the end)"""
    B, N = x.shape
    R = -(-(N + n) // hop)
    xp = torch.from_numpy(np.pad(x.numpy(), ((0, 0), (n // 2, n // 2)), mode=mode))
    return F.pad(xp, (0, R * hop - (N + n))).view(B, R, hop)


def signals(B, N, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, N, generator=g) * torch.linspace(0.5, 2.0, B)[:, None]


FRAME_CASES = [  # (n, hop, N, B)
    (1024, 320, 513, 1),              # the minimum clip the drivers accept
    (1024, 320, 320 * 50, 2),         # a multiple of hop
    (1024, 320, 320 * 50 + 1, 3),     # one off it
    (256, 80, 80 * 37 + 17, 3),       # PVT small
    (400, 160, 201, 1),               # the emotion encoder's minimum
    (400, 160, 16000 + 77, 2),
    (1024, 320, 320 * 600, 2),        # above the 4096 x 256 cap
]


@gpu
@pytest.mark.parametrize("n,hop,N,B", FRAME_CASES)
def test_frames(n, hop, N, B):
    x = signals(B, N, 11 + N)
    T = N // hop + 1
    flat, y = out_f((B, T, n))
    probe("FRAMES", x=dev(x), y=y, B=B, N=N, n=n, hop=hop)
    written("FRAMES", flat)
    exact(f"FRAMES n={n} hop={hop} N={N} B={B}", "FRAMES", y, reflect_frames(x, n, hop))


STFT_CASES = [  # (n, hop, N, B)
    (1024, 512, 513, 1),              # N = n / 2 + 1
    (1024, 512, 512 * 40, 3),         # a multiple of hop
    (1024, 512, 512 * 40 + 1, 2),     # one off it: the last row is part padding, part zero
    (1024, 512, 512 * 40 + 300, 2),
    (256, 128, 129, 2),
    (1024, 512, 512 * 2100, 2),       # above the 8192 x 256 cap
]


@gpu
@pytest.mark.parametrize("n,hop,N,B", STFT_CASES)
def test_stft_rows(n, hop, N, B):
    x = signals(B, N, 23 + N)
    R = -(-(N + n) // hop)
    flat, y = out_f((B, R, hop))
    probe("STFT_ROWS", x=dev(x), y=y, B=B, N=N, n=n, hop=hop)
    written("STFT_ROWS", flat)
    want = stft_rows_ref(x, n, hop)
    exact(f"STFT_ROWS n={n} hop={hop} N={N} B={B}", "STFT_ROWS", y, want)
    assert not y.view(B, -1)[:, N + n:].any(), "rows past N + n must be zero"


# ================================================================================================ LOGMEL / POWMEL
def mel_bound(spec, nb, melW):
    """the fp64 mel of the fp32 spectrum [rows][pitch] and its bound (module docstring)"""
    s = spec.double()
    pw = s[:, :nb] ** 2 + s[:, nb:2 * nb] ** 2
    mel = pw @ melW.double()
    return mel, (gam(nb) + 2) * U * mel * (1 + 1e-6)


def logmel_ref(spec, nb, melW, bs, bt, clamp=True):
    """LogmelFilterBank (ref 1, amin 1e-10, no top_db) and bn0 with the folded scale / shift, fp64, and the bound"""
    mel, emel = mel_bound(spec, nb, melW)
    amin = float(np.float32(1e-10))
    mc = mel.clamp(min=amin) if clamp else mel
    lg = torch.log10(mc)
    db = 10.0 * lg
    edb = 10.0 / math.log(10.0) * emel / mc + 10.0 * 4 * U * lg.abs() + U * db.abs()
    s, t = bs.double(), bt.double()
    v = db * s + t
    return v, s.abs() * edb + U * ((s * db).abs() + t.abs()) + U * v.abs()


def spectra(rows, nb, pitch, scale, seed):
    g = torch.Generator().manual_seed(seed)
    spec = torch.full((rows, pitch), 123.0)        # the pitch's tail columns are never read
    spec[:, :2 * nb] = torch.randn(rows, 2 * nb, generator=g) * scale
    return spec


def bn0_params(nm, seed, shift=0.0):
    """eval BatchNorm over the mel axis, folded as LogmelFront::load folds it (fp32 on the host)"""
    g = torch.Generator().manual_seed(seed)
    w = (0.5 + torch.rand(nm, generator=g)).numpy().astype(np.float32)
    b = (0.1 * torch.randn(nm, generator=g)).numpy().astype(np.float32)
    rm = (-30 + 5 * torch.randn(nm, generator=g)).numpy().astype(np.float32) + np.float32(shift)
    rv = (20 + 10 * torch.rand(nm, generator=g)).numpy().astype(np.float32)
    s = (w / np.sqrt(rv + np.float32(1e-5))).astype(np.float32)
    t = (b - rm * s).astype(np.float32)
    return torch.from_numpy(s), torch.from_numpy(t)


LOGMEL_CASES = [  # (n, sr, fmin, fmax, pitch extra, bn0 shift, spectrum scale)
    (1024, 44100, 50, 14000, 6, 0.0, 1.0),      # the CLAP scorer's Cnn14 (nb = 513, 64 mels)
    (1024, 32000, 50, 14000, 0, 0.0, 30.0),     # PVT shipped
    (256, 16000, 50, 8000, 2, 0.0, 0.3),        # PVT small (nb = 129)
    (1024, 44100, 50, 14000, 6, 1e4, 1.0),      # |t| >> |s db|: the folded shift's cancellation
]


@gpu
@pytest.mark.parametrize("ch", [1, 4])
@pytest.mark.parametrize("n,sr,fmin,fmax,extra,shift,scale", LOGMEL_CASES)
def test_logmel(ch, n, sr, fmin, fmax, extra, shift, scale):
    nb, nm = n // 2 + 1, 64
    pitch = 2 * nb + extra
    rows = 97
    spec = spectra(rows, nb, pitch, scale, 31 + n + extra)
    melW = torch.from_numpy(specs.slaney_mel(sr, n, nm, fmin, fmax).T.copy())
    spec[0, :2 * nb] = 0.0                                      # silence: the 1e-10 clamp
    spec[1, :2 * nb] = torch.tensor([0.0, -0.0]).repeat(nb)     # signed zeros
    base = spec[2, :2 * nb].clone()
    mel1 = mel_bound(spec[2:3], nb, melW)[0][0]
    for r, f in zip(range(2, 8), (0.5, 0.999, 0.99999, 1.00001, 1.001, 2.0)):   # a bin sum on either side of the clamp
        spec[r, :2 * nb] = base * math.sqrt(f * 1e-10 / float(mel1[7]))
    bs, bt = bn0_params(nm, 5 + n, shift)
    flat, y = out_f((rows, nm, ch))
    probe("LOGMEL", x=dev(spec), w=dev(melW), g=dev(bs), b=dev(bt), y=y, rows=rows, pitch=pitch, nb=nb, nm=nm, ch=ch)
    written("LOGMEL", flat)
    ref, bound = logmel_ref(spec, nb, melW, bs, bt)
    y = y.cpu()
    check(f"LOGMEL ch={ch} nb={nb} shift={shift}", "LOGMEL", y[..., 0], ref, bound)
    if ch == 4:
        exact(f"LOGMEL ch=4 nb={nb}: channels 1..3", "LOGMEL", y[..., 1:], torch.zeros(rows, nm, 3))


@gpu
@pytest.mark.parametrize("rows,pitch", [(101, 402), (77, 408), (3000, 408)])
def test_powmel(rows, pitch):
    nb = specs.EMO_N_FFT // 2 + 1
    spec = spectra(rows, nb, pitch, 3.0, 41 + rows)
    spec[0, :2 * nb] = 0.0                                      # zero frames (padding) give exactly 0
    spec[rows // 2, :2 * nb] = 0.0
    melW = torch.from_numpy(specs.slaney_mel(specs.EMO_SR, specs.EMO_N_FFT, specs.EMO_MELS, 0.0, specs.EMO_SR / 2.0).T.copy())
    flat, y = out_f((rows, specs.EMO_MELS))
    probe("POWMEL", x=dev(spec), w=dev(melW), y=y, rows=rows, pitch=pitch)
    written("POWMEL", flat)
    ref, bound = mel_bound(spec, nb, melW)
    check(f"POWMEL rows={rows} pitch={pitch}", "POWMEL", y, ref, bound)
    assert not y[0].any() and not y[rows // 2].any()


# ================================================================================================ MAGPHASE
def magphase_inputs(B, R, pitch, nb, seed):
    g = torch.Generator().manual_seed(seed)
    spec = torch.randn(B, R, pitch, generator=g) * torch.exp2(torch.randint(-8, 9, (B, R, pitch), generator=g).float())
    specials = [(0.0, 0.0), (-0.0, 0.0), (0.0, -0.0), (-0.0, -0.0), (1.5, 0.0), (1.5, -0.0), (-1.5, 0.0),
                (-1.5, -0.0), (0.0, 2.5), (-0.0, 2.5), (0.0, -2.5), (-0.0, -2.5), (3e18, 7e17), (-3e18, 1e-20),
                (1e-30, 1e-30), (-1e-25, 3e-26)]
    for i, (re, im) in enumerate(specials):     # at DC, at Nyquist and in between
        for f in (0, nb - 1, nb // 2):
            t = i % R
            spec[i % B, t, f], spec[i % B, t, nb + f] = re, im
    return spec


def sqrt_rn(p):
    """the correctly rounded fp32 sqrt of fp32 p (sqrt in fp64, rounded once: 53 >= 2 * 24 + 2 makes that exact)"""
    return torch.sqrt(p.double()).float()


def magphase_ref(spec, nb, T):
    """stft.py transform's tail on the fp32 spectrum: (torch fp32 magnitude, fp64 phase, torch fp32 phase), [B][nb][T]"""
    re = spec[:, :T, :nb].transpose(1, 2).contiguous()
    im = spec[:, :T, nb:2 * nb].transpose(1, 2).contiguous()
    return sqrt_rn(re ** 2 + im ** 2), torch.atan2(im.double(), re.double()), torch.atan2(im, re), re, im


def magphase_gate(mag, ph, spec, nb, T):
    """(magnitude exact, phase err / bound, axis phases exact) of a [B][nb][T] result"""
    m32, p64, p32, re, im = magphase_ref(spec, nb, T)
    axis = (re == 0) | (im == 0)
    r = ratio(ph, p64, 3 * ulp32(p64))
    return same(mag, m32), r, same(ph[axis], p32[axis]), int(axis.sum())


@gpu
@pytest.mark.parametrize("B,R,pitch,nb,T", [(3, 43, 1026, 513, 41), (2, 12, 136, 65, 12), (2, 2103, 1032, 513, 2101)])
def test_magphase(B, R, pitch, nb, T):
    spec = magphase_inputs(B, R, pitch, nb, 51 + T)
    fm, mag = out_f((B, nb, T))
    fp, ph = out_f((B, nb, T))
    probe("MAGPHASE", x=dev(spec), y=mag, y2=ph, B=B, R=R, pitch=pitch, nb=nb, T=T)
    written("MAGPHASE mag", fm)
    written("MAGPHASE phase", fp)
    m32, p64, p32, re, im = magphase_ref(spec, nb, T)
    exact(f"MAGPHASE B={B} nb={nb} T={T}: magnitude", "MAGPHASE", mag, m32)
    check(f"MAGPHASE B={B} nb={nb} T={T}: phase", "MAGPHASE", ph, p64, 3 * ulp32(p64))
    axis = (re == 0) | (im == 0)
    exact(f"MAGPHASE: {int(axis.sum())} axis phases", "MAGPHASE", ph.cpu()[axis], p32[axis])


# ================================================================================================ ISTFT_FRAMES / FINISH
def istft_frames_ref(mag, phase, pitch):
    """stft.py inverse's input: cat([mag cos(phase), mag sin(phase)], dim=1) [B][2 nb][T] in fp64, laid out as the
    conv_transpose1d rows [B][T + 1][pitch] (row T and the columns past 2 nb zero), and the bound"""
    B, nb, T = mag.shape
    m, p = mag.double(), phase.double()
    c, s = torch.cos(p), torch.sin(p)
    x = torch.cat([m * c, m * s], 1).transpose(1, 2)
    e = torch.cat([2 * m.abs() * ulp32(c) + 2 * U * (m * c).abs(), 2 * m.abs() * ulp32(s) + 2 * U * (m * s).abs()], 1)
    ref = torch.zeros(B, T + 1, pitch, dtype=torch.float64)
    bound = torch.zeros_like(ref)
    ref[:, :T, :2 * nb] = x
    bound[:, :T, :2 * nb] = e.transpose(1, 2)
    return ref, bound


@gpu
@pytest.mark.parametrize("B,nb,T,pitch", [(2, 513, 41, 1026), (3, 513, 17, 1032), (2, 65, 9, 136), (2, 513, 1100, 1032)])
def test_istft_frames(B, nb, T, pitch):
    g = torch.Generator().manual_seed(61 + T)
    mag = torch.rand(B, nb, T, generator=g) * 4
    phase = (torch.rand(B, nb, T, generator=g) * 2 - 1) * math.pi
    pi32 = float(np.float32(math.pi))
    for i, v in enumerate((pi32, -pi32, 0.0, -0.0, pi32 / 2, -pi32 / 2)):   # phases at +-pi, 0 and +-pi / 2
        phase[0, i, :] = v
    flat, X = out_f((B, T + 1, pitch))
    probe("ISTFT_FRAMES", x=dev(mag), x2=dev(phase), y=X, B=B, nb=nb, T=T, pitch=pitch)
    written("ISTFT_FRAMES", flat)
    ref, bound = istft_frames_ref(mag, phase, pitch)
    check(f"ISTFT_FRAMES B={B} nb={nb} T={T} pitch={pitch}", "ISTFT_FRAMES", X, ref, bound)
    Xc = X.cpu()
    exact("ISTFT_FRAMES: row T", "ISTFT_FRAMES", Xc[:, T], torch.zeros(B, pitch))
    exact("ISTFT_FRAMES: columns >= 2 nb", "ISTFT_FRAMES", Xc[:, :, 2 * nb:], torch.zeros(B, T + 1, pitch - 2 * nb))


def istft_finish_ref(y, ws, T, n, hop, strict=True):
    """stft.py inverse's tail in torch fp32: y[:, idx] /= ws[idx] where ws > tiny, y *= n / hop, crop n / 2 each side.
    strict=False: the mutant's ws >= tiny."""
    v = y.clone()
    idx = ws > FLT_MIN if strict else ws >= FLT_MIN
    v[:, idx] = v[:, idx] / ws[idx]
    v *= float(n) / hop
    return v[:, n // 2:][:, :(T - 1) * hop]


def finish_inputs(B, T, n, hop, synthetic, seed):
    g = torch.Generator().manual_seed(seed)
    y = torch.randn(B, (T + 1) * hop, generator=g)
    ws = torch.from_numpy(specs.stft_window_sum(T, n, hop)).float()
    if synthetic:
        sub = float(np.float32(1e-40))
        vals = torch.tensor([0.0, sub, FLT_MIN / 2, FLT_MIN, float(np.nextafter(np.float32(FLT_MIN), np.float32(1))),
                             1e-30, 0.75, 2e-38], dtype=torch.float32)
        pos = torch.randint(0, ws.numel(), (ws.numel() // 4,), generator=g)
        ws[pos] = vals[torch.arange(pos.numel()) % vals.numel()]
        ws[n // 2:n // 2 + vals.numel()] = vals     # the first outputs see every value
    return y, ws


@gpu
@pytest.mark.parametrize("B,T,synthetic", [(2, 40, False), (3, 40, True), (1, 2, False), (2, 2100, True)])
def test_istft_finish(B, T, synthetic):
    n, hop = specs.LASS_FFT, specs.LASS_HOP
    y, ws = finish_inputs(B, T, n, hop, synthetic, 71 + T)
    flat, out = out_f((B, (T - 1) * hop))
    probe("ISTFT_FINISH", x=dev(y), x2=dev(ws), y=out, B=B, T=T, n=n, hop=hop)
    written("ISTFT_FINISH", flat)
    exact(f"ISTFT_FINISH B={B} T={T} synthetic={synthetic}", "ISTFT_FINISH", out, istft_finish_ref(y, ws, T, n, hop))


# ================================================================================================ RESAMPLE
def resample_ref(x, rates, clip, starts):
    """torchaudio Resample (specs.sinc_resample_kernel) per clip in fp64 over the zero-padded clip, then
    resample_and_duration's crop (start >= 0) or tile (start -1); and the bound"""
    ker, width, o, nw = specs.sinc_resample_kernel(*rates)
    B, L = x.shape
    R = -(-nw * L // o)
    xp = F.pad(x.double()[:, None], (width, width + o))
    k = ker.double()[:, None]
    y = F.conv1d(xp, k, stride=o).transpose(1, 2).reshape(B, -1)[:, :R]
    a = F.conv1d(xp.abs(), k.abs(), stride=o).transpose(1, 2).reshape(B, -1)[:, :R]
    idx = torch.stack([(torch.arange(clip) + max(s, 0)) % R for s in starts])
    e = gam(ker.shape[1]) * U * a * (1 + 1e-6)
    return y.gather(1, idx), e.gather(1, idx), y, e


RESAMPLE_CASES = [  # (orig, new, L, clip, starts, B)
    ((16000, 44100), 16037, 44100, "crop", 3),       # the shipped 16 k -> 44.1 k; L not a multiple of orig
    ((16000, 44100), 8000 + 13, 44100, "tile", 2),   # R < clip
    ((16000, 44100), 16000, 44100, "tile", 1),       # R = clip
    ((44100, 16000), 44100 + 13, 16000, "crop", 2),  # down-sampling
    ((16000, 44100), 16000 * 9 + 5, 44100 * 9, "crop", 3),   # above the 4096 x 256 cap
]


def resample_setup(rates, L, clip, mode, B):
    ker, width, o, nw = specs.sinc_resample_kernel(*rates)
    R = -(-nw * L // o)
    if mode == "tile":
        assert R <= clip
        starts = [-1] * B
    else:
        assert R > clip
        starts = ([0, R - clip - 1] + [(R - clip) // 2] * B)[:B]     # the first and the last crop starts
    return ker, width, o, nw, R, np.array(starts, dtype=np.int32)


@gpu
@pytest.mark.parametrize("rates,L,clip,mode,B", RESAMPLE_CASES)
def test_resample(rates, L, clip, mode, B):
    ker, width, o, nw, R, starts = resample_setup(rates, L, clip, mode, B)
    x = signals(B, L, 81 + L)
    flat, y = out_f((B, clip))
    probe("RESAMPLE", x=dev(x), w=dev(ker), starts=starts, y=y, B=B, N=L, orig=o, nw=nw, width=width, clip=clip)
    written("RESAMPLE", flat)
    ref, bound, _, _ = resample_ref(x, rates, clip, starts.tolist())
    check(f"RESAMPLE {rates} L={L} clip={clip} {mode} starts={starts.tolist()}", "RESAMPLE", y, ref, bound)


# ================================================================================================ CNN14_HEAD
def head_ref(x, over_f="mean"):
    """Cnn14.forward after conv_block6 on [B][T][F][C]: mean over F (dim 3 of [B, C, T, F]), max_t + mean_t; the
    bound.  over_f='max': the mutant."""
    xd = x.double()
    B, T, Fq, Cc = x.shape
    m = xd.mean(2) if over_f == "mean" else xd.amax(2)                      # [B][T][C]
    et = gam(Fq) * U * xd.abs().sum(2) / Fq + U * m.abs()
    mean_t = m.mean(1)
    ref = m.amax(1) + mean_t
    E = et.amax(1) + (et.sum(1) + gam(T) * U * m.abs().sum(1)) / T + U * mean_t.abs() + U * ref.abs()
    return ref, E * (1 + 1e-6)


@gpu
@pytest.mark.parametrize("B,T,Fq,Cc", [(2, 38, 2, 2048), (3, 1, 2, 2048), (2, 5, 1, 64), (1, 1, 1, 256), (3, 27, 3, 200)])
def test_cnn14_head(B, T, Fq, Cc):
    g = torch.Generator().manual_seed(91 + T)
    x = torch.relu(torch.randn(B, T, Fq, Cc, generator=g))
    x[0, 0, :, 0] += 50.0           # a row whose max is at t = 0
    x[0, T - 1, :, 1 % Cc] += 50.0  # one at t = T - 1
    x[B - 1, :, :, Cc - 1] = -torch.rand(T, Fq, generator=g)
    flat, y = out_f((B, Cc))
    probe("CNN14_HEAD", x=dev(x), y=y, B=B, T=T, F=Fq, C=Cc)
    written("CNN14_HEAD", flat)
    ref, bound = head_ref(x)
    check(f"CNN14_HEAD B={B} T={T} F={Fq} C={Cc}", "CNN14_HEAD", y, ref, bound)


# ================================================================================================ L2NORM2 / SIMILARITY
def l2_ref(x):
    """CLAPWrapper: _get_audio_embeddings' x / ||x|| and get_audio_embeddings' second division, fp64, and the bound"""
    xd = x.double()
    r = xd / xd.norm(dim=-1, keepdim=True)
    r = r / r.norm(dim=-1, keepdim=True)
    return r, (gam(x.shape[-1]) + 6) * U * r.abs()


@gpu
@pytest.mark.parametrize("rows,D,dominant", [(5, 1024, False), (3, 1007, False), (4, 77, True), (2, 1024, True)])
def test_l2norm2(rows, D, dominant):
    g = torch.Generator().manual_seed(101 + D)
    x = torch.randn(rows, D, generator=g)
    if dominant:
        x[:, 3] = 1e4
    flat, y = out_f((rows, D))
    probe("L2NORM2", x=dev(x), y=y, rows=rows, D=D)
    written("L2NORM2", flat)
    ref, bound = l2_ref(x)
    check(f"L2NORM2 rows={rows} D={D} dominant={dominant}", "L2NORM2", y, ref, bound)


def sim_ref(a, t, scale):
    """compute_similarity: (t @ a.T).T [Na][Nt] times the scale, fp64, and the bound"""
    ref = scale * (a.double() @ t.double().T)
    return ref, gam(a.shape[1]) * U * abs(scale) * (a.double().abs() @ t.double().abs().T) + U * ref.abs()


def argmax_ok(y, ref, bound):
    """per text column: the chosen audio row is the fp64 argmax, or within the bounds of it"""
    y, ref, bound = y.double().cpu(), ref.double().cpu(), bound.double().cpu()
    got, want = y.argmax(0), ref.argmax(0)
    j = torch.arange(y.shape[1])
    return bool(((got == want) | (ref[want, j] - ref[got, j] <= bound[want, j] + bound[got, j])).all())


@gpu
@pytest.mark.parametrize("Na,Nt,D,scale,near", [(1, 1, 1024, 1.0, False), (4, 3, 1024, 1.0, False),
                                                (4, 3, 1024, 1 / 0.07, True), (5, 2, 1007, 1.0, True)])
def test_similarity(Na, Nt, D, scale, near):
    g = torch.Generator().manual_seed(111 + Na + D)
    a = l2_ref(torch.randn(Na, D, generator=g))[0].float()
    t = l2_ref(torch.randn(Nt, D, generator=g))[0].float()
    if near:                                    # near-tied candidates: audio 1 a hair away from audio 0
        a[1] = a[0]
        a[1, 0] = float(np.nextafter(np.float32(a[0, 0]), np.float32(2)))
        a[2] = a[0]
    flat, y = out_f((Na, Nt))
    probe("SIMILARITY", x=dev(a), x2=dev(t), y=y, Na=Na, Nt=Nt, D=D, scale=scale)
    written("SIMILARITY", flat)
    ref, bound = sim_ref(a, t, scale)
    check(f"SIMILARITY {Na}x{Nt} D={D} scale={scale:.3g}", "SIMILARITY", y, ref, bound)
    assert argmax_ok(y, ref, bound), "the chosen audio candidate is not the fp64 argmax"
    if near:
        assert same(y[0], y[2]), "identical candidates must score identically"


# ================================================================================================ LASS_INPUT / LASS_HEAD
def bn1_fold(seed):
    """encoder_block1.conv_block1.bn1 (one channel) and its fp32 fold, as lass_create computes it"""
    g = torch.Generator().manual_seed(seed)
    w, b = np.float32(0.5 + float(torch.rand(1, generator=g))), np.float32(float(torch.randn(1, generator=g)))
    rm, rv = np.float32(1.3 + float(torch.rand(1, generator=g))), np.float32(2.0 + float(torch.rand(1, generator=g)))
    s = np.float32(w / np.sqrt(np.float32(rv + np.float32(1e-5))))
    t = np.float32(b - rm * s)
    s64 = float(w) / math.sqrt(float(rv) + 1e-5)
    return float(s), float(t), s64, float(b) - float(rm) * s64


def lass_input_ref(mag_btf, T, Tp, W, fold):
    """the reference pads the [B, 1, T, F] input to Tp rows before encoder_block1's bn1: ch 0 bn1(x) fp64 (and its
    bound against the folded FMA), ch 1 x; [B][Tp][W][4]"""
    s, t, s64, t64 = fold
    B = mag_btf.shape[0]
    x = F.pad(mag_btf[:, :T, :W].double(), (0, 0, 0, Tp - T))
    ref = torch.zeros(B, Tp, W, 4, dtype=torch.float64)
    ref[..., 0] = x * s64 + t64
    ref[..., 1] = x
    bound = torch.zeros_like(ref)
    bound[..., 0] = (x.abs() * abs(s - s64) + abs(t - t64) + U * (x * s + t).abs()) * (1 + 1e-6)
    return ref, bound


@gpu
@pytest.mark.parametrize("B,T,W,strided", [(2, 100, 511, True), (1, 64, 511, False), (3, 37, 127, True),
                                           (2, 1000, 511, True)])
def test_lass_input(B, T, W, strided):
    Fb = W + 2
    g = torch.Generator().manual_seed(121 + T)
    mag_bft = torch.rand(B, Fb, T, generator=g) * 5          # the STFT's [B][nb][T] magnitude
    fold = bn1_fold(7 + T)
    Tp = -(-T // 64) * 64
    flat, y = out_f((B, Tp, W, 4))
    if strided:     # mask() reads the magnitude in place: sb = nb T, stt = 1, sf = T
        md = dev(mag_bft)
        probe("LASS_INPUT", x=md, y=y, B=B, T=T, W=W, sb=Fb * T, stt=1, sf=T, scale=fold[0], shift=fold[1])
    else:
        md = dev(mag_bft.transpose(1, 2))
        probe("LASS_INPUT", x=md, y=y, B=B, T=T, W=W, sb=T * Fb, stt=Fb, sf=1, scale=fold[0], shift=fold[1])
    written("LASS_INPUT", flat)
    ref, bound = lass_input_ref(mag_bft.transpose(1, 2), T, Tp, W, fold)
    yc = y.cpu()
    check(f"LASS_INPUT B={B} T={T} W={W} strided={strided}", "LASS_INPUT", yc[..., 0], ref[..., 0], bound[..., 0])
    exact("LASS_INPUT: channel 1 (raw x, 0 when padded)", "LASS_INPUT", yc[..., 1], ref[..., 1].float())
    exact("LASS_INPUT: channels 2..3", "LASS_INPUT", yc[..., 2:], torch.zeros(B, Tp, W, 2))
    exact("LASS_INPUT: padded rows hold bn1(0)", "LASS_INPUT", yc[:, T:, :, 0], torch.full((B, Tp - T, W), fold[1]))


def lass_head_ref(x, wb, T, pad_first=False):
    """after_conv2 (1x1 conv + bias) on [B, 32, Tp, W], F.pad(x, (0, 2)), crop to T, sigmoid; fp64 logits / mask and
    their bounds.  pad_first: the mutant that pads before the conv (the bias reaches the padded bins)."""
    xd = x.double().permute(0, 3, 1, 2)
    w = wb[:32].double().view(1, 32, 1, 1)
    b = wb[32:].double()
    if pad_first:
        lg = F.conv2d(F.pad(xd, (0, 2)), w, b)[:, 0, :T]
        el = torch.zeros_like(lg)
    else:
        lg = F.pad(F.conv2d(xd, w, b), (0, 2))[:, 0, :T]
        el = F.pad(F.conv2d(xd.abs(), w.abs()), (0, 2))[:, 0, :T] * 32 * U
        el = el + U * lg.abs()
    sg = torch.sigmoid(lg)
    e = torch.exp(-lg)
    em = sg * (1 - sg) * el + sg * (4 * U * e / (1 + e) + 3 * U)
    return lg, el * (1 + 1e-6), sg, em * (1 + 1e-6)


@gpu
@pytest.mark.parametrize("B,T,W,with_logits", [(2, 100, 511, True), (2, 100, 511, False), (1, 128, 127, True),
                                               (3, 1000, 511, True)])
def test_lass_head(B, T, W, with_logits):
    Tp = -(-T // 64) * 64
    g = torch.Generator().manual_seed(131 + T)
    x = torch.randn(B, Tp, W, 32, generator=g)
    wb = torch.randn(33, generator=g) * 0.3
    wb[32] = 0.7
    fm, mask = out_f((B, T, W + 2))
    fl, logits = out_f((B, T, W + 2))
    probe("LASS_HEAD", x=dev(x), w=dev(wb), y=mask, y2=logits if with_logits else None, B=B, T=T, W=W)
    written("LASS_HEAD mask", fm)
    lg, el, sg, em = lass_head_ref(x, wb, T)
    check(f"LASS_HEAD B={B} T={T} W={W}: mask", "LASS_HEAD", mask, sg, em)
    exact("LASS_HEAD: padded bins' mask", "LASS_HEAD", mask.cpu()[..., W:], torch.full((B, T, 2), 0.5))
    if with_logits:
        written("LASS_HEAD logits", fl)
        check(f"LASS_HEAD B={B} T={T} W={W}: logits", "LASS_HEAD", logits, lg, el)
        exact("LASS_HEAD: padded bins' logits", "LASS_HEAD", logits.cpu()[..., W:], torch.zeros(B, T, 2))
    else:
        assert torch.isnan(fl[:-GUARD]).all(), "logits written although null"


# ================================================================================================ W2V_STEM
def stem_conv(x, w0, s0):
    """Wav2Vec2GroupNormConvLayer.conv: Conv1d(1, C, k0, stride s0, bias=False) in fp64 -> [B][T0][C], and
    sum |w x| per output"""
    xd = x.double()[:, None]
    wd = w0.double()[:, None]
    return F.conv1d(xd, wd, stride=s0).transpose(1, 2), F.conv1d(xd.abs(), wd.abs(), stride=s0).transpose(1, 2)


def stem_ref(x, w0, s0, gamma, beta, eps=1e-5, stats=None):
    """Wav2Vec2GroupNormConvLayer (GroupNorm(C, C) over time, GELU) in fp64, and the propagated bound (module
    docstring).  stats: (mean, var) [B][C] to use instead of the exact ones (the mutants)."""
    k0 = w0.shape[1]
    h, a = stem_conv(x, w0, s0)
    eh = k0 * U * a
    mu, var = (h.mean(1), h.var(1, unbiased=False)) if stats is None else stats
    sig = torch.sqrt(var + eps)
    gm, bt = gamma.double(), beta.double()
    z = (h - mu[:, None]) / sig[:, None] * gm + bt
    ref = F.gelu(z)
    dmu = eh.mean(1) + U * mu.abs()
    drs = eh.amax(1) / sig + 2 * U                                # relative error of rstd and of gamma rstd
    d = (h - mu[:, None]).abs()
    dz = (gm.abs() / sig)[:, None] * (eh + dmu[:, None] + U * d) + d * (gm.abs() / sig)[:, None] * drs[:, None] + U * z.abs()
    bound = 1.13 * dz + (4 + z.abs()) * U * z.abs() + 2 * U * ref.abs()
    return ref, bound * 1.01, h


STEM_CASES = [  # (B, S, k0, s0, C, s1, kind)
    (1, 160000, 10, 5, 512, 2, "noise"),          # the shipped stem at a 10 s clip: T0 = 31999, 250 chunks, 1 zero row
    (3, 505, 10, 5, 512, 2, "noise"),             # T0 = 100 < 128: one chunk
    (3, 1290, 10, 5, 512, 2, "noise"),            # T0 = 257 = 2 * 128 + 1: a one-row last chunk
    (2, 1290, 10, 5, 512, 4, "const"),            # constant input: variance 0; three zero rows
    (3, 6410, 10, 5, 512, 2, "dc"),               # a 1e3 DC offset with unit noise
    (2, 3000, 16, 3, 96, 0, "noise"),             # k0 = 16, no zero rows
]


def stem_inputs(B, S, k0, C, kind, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "const":
        x = torch.full((B, S), 0.37) * torch.arange(1, B + 1)[:, None]
    else:
        x = torch.randn(B, S, generator=g) * torch.linspace(0.3, 1.5, B)[:, None]
        if kind == "dc":
            x = x + 1e3
    w0 = torch.randn(C, k0, generator=g) / math.sqrt(k0)
    gamma = 0.5 + torch.rand(C, generator=g)
    beta = 0.2 * torch.randn(C, generator=g)
    return x, w0, gamma, beta


@gpu
@pytest.mark.parametrize("B,S,k0,s0,C,s1,kind", STEM_CASES)
def test_w2v_stem(B, S, k0, s0, C, s1, kind):
    x, w0, gamma, beta = stem_inputs(B, S, k0, C, kind, 141 + S)
    T0 = (S - k0) // s0 + 1
    zpad = -(-T0 // s1) * s1 - T0 if s1 else 0
    R = T0 + 8
    nch = -(-T0 // 128)
    part = torch.full((B * nch * C * 2,), float("nan"), dtype=torch.float64, device=DEV)
    stat = torch.full((B * C * 2,), float("nan"), dtype=torch.float32, device=DEV)
    cnt = torch.zeros(B, dtype=torch.int32, device=DEV)
    flat = torch.full((B * R * C + GUARD,), CANARY, dtype=torch.float32, device=DEV)
    y = flat[:B * R * C].view(B, R, C)
    y[:, :T0 + zpad] = float("nan")
    y[:, T0 + zpad:] = UNTOUCHED
    args = dict(x=dev(x), w=dev(w0), g=dev(gamma), b=dev(beta), part=part, stat=stat, cnt=cnt, y=y, B=B, N=S, k0=k0,
                s0=s0, C=C, s1=s1, R=R, eps=1e-5)
    probe("W2V_STEM", **args)
    tag = f"W2V_STEM B={B} T0={T0} k0={k0} s0={s0} C={C} zpad={zpad} {kind}"
    assert torch.equal(flat[-GUARD:], torch.full_like(flat[-GUARD:], CANARY)), f"{tag}: written past the end"
    assert not torch.isnan(y[:, :T0 + zpad]).any(), f"{tag}: rows not written"
    assert bool((y[:, T0 + zpad:] == UNTOUCHED).all()), f"{tag}: rows past T0 + zpad written"
    assert not cnt.any(), f"{tag}: the CTA counters are not back at 0"
    ref, bound, _ = stem_ref(x, w0, s0, gamma, beta)
    check(tag, "W2V_STEM", y[:, :T0], ref, bound)
    exact(f"{tag}: zero rows", "W2V_STEM", y[:, T0:T0 + zpad], torch.zeros(B, zpad, C))
    first = y.clone()
    probe("W2V_STEM", **args)                   # the same workspaces again
    assert torch.equal(first, y), f"{tag}: a second call on the same workspaces differs"
    assert not cnt.any()


# ================================================================================================ preconditions (no device)
def _refused(op, match, **kw):
    with pytest.raises(RuntimeError, match=match):
        probe(op, stream=False, **kw)


def test_probe_refuses_a_clip_too_short_to_reflect():
    _refused("FRAMES", "reflect padding", B=1, N=512, n=1024, hop=320)
    _refused("FRAMES", "reflect padding", B=1, N=200, n=400, hop=160)


def test_probe_refuses_an_stft_input_too_short_to_reflect():
    _refused("STFT_ROWS", "reflect padding", B=1, N=512, n=1024, hop=512)


def test_probe_refuses_an_inverse_stft_of_one_frame():
    _refused("ISTFT_FRAMES", "two frames", B=1, nb=513, T=1, pitch=1026)
    _refused("ISTFT_FINISH", "two frames", B=1, T=1, n=1024, hop=512)


def test_probe_refuses_a_stem_beyond_its_limits():
    _refused("W2V_STEM", "k0 must be 1..16", B=1, N=1000, k0=17, s0=5, C=512, s1=2, R=1000)
    _refused("W2V_STEM", "at most 1024 channels", B=1, N=1000, k0=10, s0=5, C=1025, s1=2, R=1000)


def test_probe_refuses_invalid_crop_starts():
    ker, width, o, nw = specs.sinc_resample_kernel(16000, 44100)
    L, clip = 16037, 44100
    R = -(-nw * L // o)
    kw = dict(B=1, N=L, orig=o, nw=nw, width=width, clip=clip)
    _refused("RESAMPLE", "crop start", starts=np.array([R - clip], dtype=np.int32), **kw)     # one past the last
    _refused("RESAMPLE", "crop start", starts=np.array([-1], dtype=np.int32), **kw)          # a tile start on a crop
    kw["N"] = 16000                                                                          # R = clip: tiled
    _refused("RESAMPLE", "tiled", starts=np.array([0], dtype=np.int32), **kw)


# ================================================================================================ mutants (CPU)
def test_gate_catches_symmetric_padding():
    x = signals(2, 320 * 50 + 1, 7)
    good, bad = reflect_frames(x, 1024, 320), reflect_frames(x, 1024, 320, mode="symmetric")
    assert not same(bad, good)
    good, bad = stft_rows_ref(x, 1024, 512), stft_rows_ref(x, 1024, 512, mode="symmetric")
    assert not same(bad, good)


def test_gate_catches_fma_magnitude():
    nb, T = 65, 12
    spec = magphase_inputs(2, 12, 136, nb, 3)
    m32, _, _, re, im = magphase_ref(spec, nb, T)
    # one rounding for re * re + (im * im): the product re * re is exact in fp64
    fma = sqrt_rn((re.double() * re.double() + (im * im).double()).float())
    assert not same(fma, m32)


def test_gate_catches_sign_dropping_phase():
    nb, T = 65, 12
    spec = magphase_inputs(2, 12, 136, nb, 3)
    _, p64, p32, re, im = magphase_ref(spec, nb, T)
    r, i = re.double(), im.double()
    at = torch.atan(i / torch.where(r == 0, torch.ones_like(r), r))
    bad = torch.where(r > 0, at, torch.where(i >= 0, at + math.pi, at - math.pi))
    bad = torch.where(r == 0, torch.where(i > 0, math.pi / 2, torch.where(i < 0, -math.pi / 2, 0.0)), bad).float()
    axis = (re == 0) | (im == 0)
    assert passes(p32, p64, 3 * ulp32(p64))                       # torch's fp32 atan2 passes the gate
    assert not same(bad[axis], p32[axis])


def test_gate_catches_finish_dividing_at_flt_min():
    n, hop, T = specs.LASS_FFT, specs.LASS_HOP, 40
    y, ws = finish_inputs(2, T, n, hop, True, 5)
    assert not same(istft_finish_ref(y, ws, T, n, hop, strict=False), istft_finish_ref(y, ws, T, n, hop))


def test_gate_catches_tiling_wrapped_at_clip():
    rates, L, clip, mode, B = RESAMPLE_CASES[1]
    ker, width, o, nw, R, starts = resample_setup(rates, L, clip, mode, B)
    x = signals(B, L, 9)
    ref, bound, y, _ = resample_ref(x, rates, clip, starts.tolist())
    assert passes(ref.float(), ref, bound)
    xp = F.pad(x.double()[:, None], (width, width + o + clip))    # the conv continued past R with zeros
    ext = F.conv1d(xp, ker.double()[:, None], stride=o).transpose(1, 2).reshape(B, -1)[:, :clip]
    assert not passes(ext.float(), ref, bound)


def _stem_case(S, kind):
    x, w0, gamma, beta = stem_inputs(2, S, 10, 64, kind, 3)
    ref, bound, h = stem_ref(x, w0, 5, gamma, beta)
    return x, w0, gamma, beta, ref, bound, h


def test_gate_catches_single_pass_stem_statistics():
    x, w0, gamma, beta, ref, bound, h = _stem_case(6410, "dc")
    h32 = h.float().numpy()
    T0 = h32.shape[1]
    means, m2s, ns = [], [], []
    for c0 in range(0, T0, 128):     # per chunk: fp32 sequential sums of h and h^2, var = E[h^2] - E[h]^2
        blk = h32[:, c0:c0 + 128]
        n = blk.shape[1]
        s1 = np.add.accumulate(blk, axis=1, dtype=np.float32)[:, -1]
        s2 = np.add.accumulate(blk * blk, axis=1, dtype=np.float32)[:, -1]
        m = s1 / np.float32(n)
        means.append(m.astype(np.float64))
        m2s.append(((s2 / np.float32(n) - m * m) * np.float32(n)).astype(np.float64))
        ns.append(n)
    mu, M2, n = np.zeros_like(means[0]), np.zeros_like(means[0]), 0
    for m, q, nb in zip(means, m2s, ns):                              # the same chunk merge as the kernel
        nn = n + nb
        d = m - mu
        mu, M2, n = mu + d * nb / nn, M2 + q + d * d * n * nb / nn, nn
    bad = stem_ref(x, w0, 5, gamma, beta, stats=(torch.from_numpy(mu), torch.from_numpy(M2 / n)))[0]
    assert passes(ref.float(), ref, bound)
    assert not passes(bad.float(), ref, bound)


def test_gate_catches_equal_weight_chunk_merge():
    x, w0, gamma, beta, ref, bound, h = _stem_case(1290, "noise")    # T0 = 257: a one-row last chunk
    T0 = h.shape[1]
    mu, M2, n = 0.0, 0.0, 0
    for c0 in range(0, T0, 128):
        blk = h[:, c0:c0 + 128]
        m, q, nb = blk.mean(1), ((blk - blk.mean(1, keepdim=True)) ** 2).sum(1), 128   # every chunk weighted 128
        nn = n + nb
        d = m - mu
        mu, M2, n = mu + d * nb / nn, M2 + q + d * d * n * nb / nn, nn
    bad = stem_ref(x, w0, 5, gamma, beta, stats=(mu, M2 / n))[0]
    assert not passes(bad.float(), ref, bound)


def test_gate_catches_logmel_without_the_clamp():
    nb, nm = 513, 64
    spec = spectra(8, nb, 2 * nb, 1.0, 3)
    spec[0] = 0.0
    melW = torch.from_numpy(specs.slaney_mel(44100, 1024, nm, 50, 14000).T.copy())
    bs, bt = bn0_params(nm, 3)
    ref, bound = logmel_ref(spec, nb, melW, bs, bt)
    assert passes(ref.float(), ref, bound)
    bad = logmel_ref(spec, nb, melW, bs, bt, clamp=False)[0]
    assert not passes(bad.float(), ref, bound)


def test_gate_catches_head_max_over_frequency():
    g = torch.Generator().manual_seed(3)
    x = torch.relu(torch.randn(2, 38, 2, 256, generator=g))
    ref, bound = head_ref(x)
    assert passes(ref.float(), ref, bound)
    assert not passes(head_ref(x, over_f="max")[0].float(), ref, bound)


def test_gate_catches_bias_on_padded_bins():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 128, 127, 32, generator=g)
    wb = torch.randn(33, generator=g)
    lg, el, sg, em = lass_head_ref(x, wb, 100)
    bad_lg, _, bad_sg, _ = lass_head_ref(x, wb, 100, pad_first=True)
    assert passes(lg.float(), lg, el)
    assert not passes(bad_lg.float(), lg, el) and not passes(bad_sg.float(), sg, em)


@gpu
def test_every_op_exercised():
    """runs last in this module: every AGPT_AU_* selector has been through at least one gate"""
    missing = [op for op in _lib.AU_OPS if op not in EXERCISED]
    assert not missing, f"not exercised: {missing}"
