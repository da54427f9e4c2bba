"""Conformance of the FastSpeech-family element-wise kernels (fs_layers.cu, fs2.cu, generspeech.cu, pe.cu) against
float64 and torch's fp32, kernel by kernel.

Every GPU case runs ONE production launcher through agpt_fs_probe on caller-owned device tensors and compares it with a
reference written from the NeuralSeq formulas on the reference's own layouts (fs2.py add_dur / add_pitch / add_energy,
tts_modules.py LengthRegulator, utils/__init__.py make_positions, common_layers.py SinusoidalPositionalEmbedding,
espnet_positional_embedding.py RelPositionalEncoding, pitch_utils.py f0_to_coarse / denorm_f0, tts_utils.py
group_hidden_by_segs, GenerSpeech's VQEmbeddingEMA.encode, wavenet.py's gate and glow_modules.py's squeeze,
CouplingBlock, InvConvNear and ActNorm in reverse), never from the kernels' indexing.  Float outputs are NaN-filled,
int outputs hold a sentinel and byte outputs 0xAB, each followed by GUARD canaries: every case asserts that the whole
output was written and nothing past it.

Error model and gates (u = 2^-24, the fp32 unit roundoff; g(n) = min(n, 6 sqrt(n)) as in test_nn_kernels_gpu.py, the
worst case or the Higham-Mary probabilistic bound for a sum of n terms):

  * Exact.  Masks (ROWMASK, PE_MASK, GS_REFMASK, GS_KPM, EMBED_TOKENS' nonpad / kpm); index kernels (POSITIONS,
    LR_SCAN, LR_FILL, GATHER and its tgt); data movement (GS_COND_CAT, GS_SQUEEZE); ENERGY's buckets; the __fadd_rn
    chains against torch fp32 in the same order (GS_SUM, GS_ACCUM, EMBED_ADD, the token embedding without MIDI terms);
    GS_VQ's q = x + (e - x); f0_denorm for the 'standard' norm, f0 * std + mean with the product and the sum rounded
    separately as torch does (an FMA would round once and differ by an ulp).
  * Rounded integers.  dur_choice = round-half-even of fp64 exp(x) - 1, clamped at 0 and 0 on padding tokens; where
    exp(x) - 1 lies within the device expf error (2 ulp of exp(x), plus the subtraction's half ulp) of a .5 boundary
    either neighbour is allowed.  Where torch's own fp32 exp on the same device lands exactly on a tie k + .5, the
    result must be torch.round's, the even neighbour (x = log 1.5 / 2.5 / 3.5 and their fp32 neighbours).  Coarse pitch
    bins equal torch's fp32 f0_to_coarse of the kernel's f0_denorm, except within the logf / exp2f margin of a bin edge
    (the fp64 distance of the scaled f0_mel from .5, coarse_margin's quantity, below 16 u of its magnitude).
  * Bounded.  Sinusoid tables (pos_mode 1 / 2, POSEMB_ADD, GS_CATPOS): the timestep-embedding rule -- the fp32
    argument a reproduced on the CPU, the device expf moving it by up to 2^-22 |a|, plus 2^-22 for sinf / cosf -- and
    u per rounded add.  GS_WN_GATE: tanhf and expf 2 ulp each plus 4 roundings, relative.  GS_SEGMEAN: a sequential
    fp32 sum of cnt terms, g(cnt) u sum|h| / cnt + u |mean|.  GS_FLOW_STEP: the coupling's (x - m) exp(-logs)
    (2 roundings + expf), the 4-term fmaf mix (4 u sum|w v| plus the propagated input bound) and the ActNorm's
    (s - bias) exp(-logs).  AFFINE_MASK with a / b: one FMA, u |ref| (a correctly rounded result reaches 1.0 of it).
    'log' f0_denorm: exp2f's 2 ulp.
  * VQ choice.  The chosen code is the fp64 argmin of (|e|^2 + |x|^2) - 2 dot over the fp32 inputs; another code is
    allowed only when its fp64 distance is within the fp32 rounding bound of both distances.  With exact ties
    (duplicate codebook rows, the dots fed in directly) the lowest index must win, as torch.argmin.

Engine behaviour beyond the reference, stated where it is tested: mel2ph values above T_txt gather the last token
(the reference's gather would fail); negative energies take bucket 0 (the reference's clamp has no lower bound);
segment ids above nseg are ignored (the reference sizes its scatter by the largest id).  The reference's
RelPositionalEncoding keeps the longer table once it has seen T > 5000, so a later short input would read it; the
engine sizes the table per call, max(5000, T), which is what a fresh module computes.  That statefulness is not
emulated.

Teeth: eight CPU-emulated mutants must FAIL the gate the kernel passes: make_positions counting padding, LR_FILL's
search with >=, durations rounded half up, the FMA-contracted denorm, VQ ties to the highest index, segmean divided by
T, InvConvNear's groups transposed (i = 2 r + a) and the squeeze with j and c swapped.  They need no device.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from audiogpt_b200 import _lib, specs
from oracle.fs2_ref import F0_MEL_MAX, F0_MEL_MIN, _denorm, f0_to_coarse, make_positions, rel_pe, sinusoidal
from oracle.generspeech_ref import vq_encode

gpu = pytest.mark.gpu

U = 2.0 ** -24
GUARD = 64
CANARY = -7777.25
ICANARY, ISENT = -987654, -123457
BCANARY, BSENT = 0xCD, 0xAB
DEV = "cuda"
EW_CAP = 2368 * 256     # ew_grid's cap: beyond this many elements the grid-stride loops iterate

EXERCISED = {}          # op -> worst error / bound over the cases that ran it (0 for the exact gates)


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    if EXERCISED:
        print("\nFastSpeech-family kernels exercised: worst error / bound (0 = exact)")
        for k in _lib.FS_OPS:
            if k in EXERCISED:
                print(f"  {k:14s}: {EXERCISED[k]:.3f}")


def gam(n):
    if isinstance(n, torch.Tensor):
        return torch.minimum(n.double(), 6.0 * n.double().sqrt())
    return min(n, 6.0 * math.sqrt(n))


def f32(v):
    return float(np.float32(v))


def seen(op, ratio=0.0):
    EXERCISED[op] = max(EXERCISED.get(op, 0.0), ratio)


# ------------------------------------------------------------------------------------------------ buffers and the probe
def out_f(shape):
    n = math.prod(shape)
    flat = torch.full((n + GUARD,), float("nan"), dtype=torch.float32, device=DEV)
    flat[n:] = CANARY
    return flat, flat[:n].view(shape)


def out_i(shape):
    n = math.prod(shape)
    flat = torch.full((n + GUARD,), ISENT, dtype=torch.int32, device=DEV)
    flat[n:] = ICANARY
    return flat, flat[:n].view(shape)


def out_b(shape):
    n = math.prod(shape)
    flat = torch.full((n + GUARD,), BSENT, dtype=torch.uint8, device=DEV)
    flat[n:] = BCANARY
    return flat, flat[:n].view(shape)


def written(tag, flat):
    n = flat.numel() - GUARD
    if flat.dtype == torch.float32:
        assert torch.equal(flat[n:], torch.full_like(flat[n:], CANARY)), f"{tag}: written past the end of the output"
        assert not torch.isnan(flat[:n]).any(), f"{tag}: {int(torch.isnan(flat[:n]).sum())} output elements not written"
    elif flat.dtype == torch.int32:
        assert bool((flat[n:] == ICANARY).all()), f"{tag}: written past the end of the output"
        unset = int((flat[:n] == ISENT).sum())
        assert not unset, f"{tag}: {unset} output elements not written"
    else:
        assert bool((flat[n:] == BCANARY).all()), f"{tag}: written past the end of the output"
        assert bool(((flat[:n] == 0) | (flat[:n] == 1)).all()), f"{tag}: mask elements not written or not 0 / 1"


def probe(op, **kw):
    a = _lib.FsProbeArgs()
    a.op = _lib.FS_OPS.index(op)
    for k, v in kw.items():
        if isinstance(v, torch.Tensor):
            assert v.is_cuda and v.is_contiguous(), k
            v = v.data_ptr()
        setattr(a, k, v)
    _lib.check(_lib.lib().agpt_fs_probe(C.byref(a), _lib.cur_stream()))


def ratio(y, ref, bound):
    err = (y.double() - ref.double()).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    return float((err / (bound + 1e-300)).max()) if err.numel() else 0.0


def passes(y, ref, bound):
    return ratio(y, ref, bound) <= 1.0


def check(tag, op, y, ref, bound):
    w = ratio(y, ref, bound)
    print(f"{tag}: worst err/bound {w:.3f}")
    seen(op, w)
    if w > 1.0:
        err = (y.double() - ref.double()).abs() / (bound + 1e-300)
        idx = np.unravel_index(int(torch.argmax(torch.nan_to_num(err, nan=math.inf)).item()), tuple(y.shape))
        raise AssertionError(f"{tag}: error {w:.3g} x the bound at {idx}: got {float(y[idx])}, want {float(ref[idx])}")


def exact(tag, op, y, want):
    assert y.shape == want.shape, (tag, y.shape, want.shape)
    bad = y.cpu() != want.to(y.dtype).cpu()
    if bad.any():
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError(f"{tag}: {int(bad.sum())} elements differ, first at {i}: got {y.cpu()[i]}, "
                             f"want {want.cpu()[i]}")
    seen(op)


# ------------------------------------------------------------------------------------------------ reference pieces
def sin_table(pos, dim):
    """fairseq SinusoidalPositionalEmbedding rows for integer positions (0 = zero row), fp64 sin / cos of torch's fp32
    argument, and the timestep-embedding bound of each entry"""
    half = dim // 2
    freq = torch.exp(torch.arange(half, dtype=torch.float32) * -(math.log(10000) / (half - 1)))
    a = (pos.cpu().float()[..., None] * freq).double()
    ref = torch.cat([torch.sin(a), torch.cos(a)], -1)
    slope = torch.cat([torch.cos(a).abs(), torch.sin(a).abs()], -1)
    aa = torch.cat([a, a], -1).abs()
    E = aa * 2.0 ** -22 * slope + (aa * 2.0 ** -22) ** 2 / 2 + 2.0 ** -22
    if dim % 2:
        ref, E = F.pad(ref, (0, 1)), F.pad(E, (0, 1))
    zero = (pos.cpu() == 0)[..., None]
    return ref.masked_fill(zero, 0.0), E.masked_fill(zero, 0.0)


def lr_mel2ph(dur, Tm, chunk=4096):
    """LengthRegulator (tts_modules.py): token_mask form over Tm frames (0 past an utterance's last frame), built
    `chunk` frames at a time"""
    dur = dur.long().cpu()
    cum = torch.cumsum(dur, 1)
    prev = F.pad(cum, [1, -1])
    tok = torch.arange(1, dur.shape[1] + 1)[None, :, None]
    out = []
    for f0 in range(0, Tm, chunk):
        pos_idx = torch.arange(f0, min(f0 + chunk, Tm))[None, None]
        mask = (pos_idx >= prev[:, :, None]) & (pos_idx < cum[:, :, None])
        out.append((tok * mask.long()).sum(1))
    return torch.cat(out, 1)


def dur_gate(x, nonpad, dch, tie_e=None):
    """True when dch [rows] is within the rounded-integer gate for xs = x * nonpad; tie_e = torch's fp32 exp(xs) - 1
    on the same device (the exact-tie rule applies where it is k + .5)"""
    x64 = x.double().cpu()
    e64 = torch.exp(x64)
    v = e64 - 1
    want = torch.round(v).clamp(min=0)
    lo = torch.floor(v)
    ulp_e = torch.exp2(torch.floor(torch.log2(e64.clamp(min=1e-30)))) * 2.0 ** -23
    w = 2.5 * ulp_e
    near = (v - lo - 0.5).abs() <= w
    d = dch.cpu().long().double()
    ok = (d == want) | (near & ((d == lo.clamp(min=0)) | (d == (lo + 1).clamp(min=0))))
    if tie_e is not None:
        te = tie_e.double().cpu()
        tie = (te - torch.floor(te)) == 0.5
        ok &= ~tie | (d == torch.round(te).clamp(min=0))
    ok = torch.where(nonpad.cpu() != 0, ok, d == 0)
    return bool(ok.all())


def coarse_gate(f0d, coarse):
    """coarse [n] against torch's fp32 f0_to_coarse of f0d, except within the margin of a bin edge"""
    f = f0d.float().cpu()
    want = f0_to_coarse(f.clone())
    mel = 1127 * torch.log1p(f.double() / 700)
    m = (mel - F0_MEL_MIN) * 254 / (F0_MEL_MAX - F0_MEL_MIN) + 1
    marg = 16 * U * (mel.abs() * 254 / (F0_MEL_MAX - F0_MEL_MIN) + m.abs())
    edge = (mel > 0) & (m > 1) & (m < 255) & ((m - m.floor() - 0.5).abs() <= marg)
    c = coarse.cpu().long()
    ok = (c == want) | (edge & ((c == m.floor().long()) | (c == m.floor().long() + 1)))
    return ok, int(edge.sum())


def check_coarse(tag, op, f0d, coarse):
    ok, nedge = coarse_gate(f0d, coarse)
    if not bool(ok.all()):
        i = int((~ok).nonzero()[0])
        raise AssertionError(f"{tag}: coarse bin {int(coarse.cpu()[i])} for f0 {float(f0d.cpu()[i])!r}, want "
                             f"{int(f0_to_coarse(f0d.float().cpu()[i:i + 1].clone()))}")
    print(f"{tag}: coarse bins exact ({nedge} within the edge margin)")
    seen(op)


def denorm_ref(f, norm, mean, std):
    """utils/pitch_utils.py denorm_f0 in torch fp32 (standard: product and sum rounded separately) and its bound"""
    f = f.float()
    if norm == 1:
        r = _denorm(f, "standard", mean, std)
        return r, torch.zeros_like(r, dtype=torch.float64)
    r = _denorm(f.double(), "log", mean, std)
    return r, 2.0 ** -22 * r.abs()


def check_denorm(tag, op, y, ref, E, norm):
    if norm == 1:
        exact(tag + " f0_denorm", op, y, ref)
    else:
        check(tag + " f0_denorm", op, y, ref, E)


def f0_edges(n):
    """fp32 f0 values on the first n coarse bin edges inside [50, 1100] Hz (m = k + .5) and their neighbours"""
    k = torch.arange(2, 2 + n, dtype=torch.float64) + 0.5
    mel = (k - 1) * (F0_MEL_MAX - F0_MEL_MIN) / 254 + F0_MEL_MIN
    f = (700 * torch.expm1(mel / 1127)).float()
    nb = torch.stack([torch.nextafter(f, f - 1), f, torch.nextafter(f, f + 1)], 1)
    return nb.reshape(-1)


# ================================================================================================ fs_layers: tokens
def token_batch(B, T, ntok, seed, interior=True):
    """ragged token ids [B][T]: utterance b has T - 3 b tokens, the last one all padding when B >= 3, interior zeros"""
    g = torch.Generator().manual_seed(seed)
    tok = torch.randint(1, ntok, (B, T), generator=g, dtype=torch.int32)
    for b in range(B):
        tok[b, max(T - 3 * b, 0):] = 0
    if B >= 3:
        tok[B - 1] = 0
    if interior and T >= 6:
        tok[0, 2] = 0
        tok[0, T // 2] = 0
    return tok


EMBED_CASES = [  # (cfg name, B, T, pos_mode, midi)
    ("FS2_SMALL", 3, 23, 1, False), ("FS2_C2", 3, 61, 1, False), ("FS2_C2", 1, 1, 1, False),
    ("FS2_C2", 2, 40, 0, False),
    ("FS2_DS1000", 3, 45, 2, True), ("FS2_DS1000", 2, 17, 2, False), ("FS2_SMALL", 3, 19, 1, True),
    ("FS2_DS1000", 1, 5100, 2, True)]


@gpu
@pytest.mark.parametrize("name,B,T,pos_mode,midi", EMBED_CASES)
def test_embed_tokens(name, B, T, pos_mode, midi):
    """token embedding * sqrt(H) (+ MIDI pitch / duration / slur terms), fairseq or rel_pos positions, the source masks;
    T = 1, interior padding tokens, an all-padding utterance, rel_pos past 5000 frames"""
    cfg = getattr(specs, name)
    H, ntok = cfg["hidden_size"], cfg["n_tokens"]
    tok = token_batch(B, T, ntok, T + H)
    E = specs.synth_tensor((ntok, H), 1, scale=0.3)
    escale = f32(math.sqrt(H))
    kw = {}
    xs = escale * E[tok.long()]
    tb = xs.abs().double()
    if midi:
        g = torch.Generator().manual_seed(5)
        pm = torch.randint(0, 300, (B, T), generator=g, dtype=torch.int32)
        md = specs.synth_tensor((B, T), 6).abs()
        sl = torch.randint(0, 2, (B, T), generator=g, dtype=torch.int32)
        E2, w, b, E3 = (specs.synth_tensor(s, 7 + i, scale=0.2) for i, s in enumerate([(300, H), (H,), (H,), (2, H)]))
        lin = md[..., None].double() * w.double() + b.double()
        xs = xs.double() + E2[pm.long()].double() + lin + E3[sl.long()].double()
        tb = (tb + E2[pm.long()].abs().double() + lin.abs() + md[..., None].double() * w.abs().double()
              + E3[sl.long()].abs().double())
        kw = dict(midi=pm.to(DEV), x=md.to(DEV), slur=sl.to(DEV), E2=E2.to(DEV), w=w.to(DEV), b=b.to(DEV),
                  E3=E3.to(DEV))
    xs = xs.double()
    E_x = 4 * U * tb if midi else torch.zeros_like(xs)
    neg_emb = f32(-(math.log(10000.0) / (H / 2 - 1)))
    if pos_mode == 1:
        pref, pE = sin_table(make_positions(tok), H)
        ref, bound = xs + pref, E_x + pE + U * (xs + pref).abs()
    elif pos_mode == 2:
        # RelPositionalEncoding of a fresh module: positions max(5000, T) - 1 - t, torch's fp32 argument, fp64 sin / cos
        div = torch.exp(torch.arange(0, H, 2, dtype=torch.float32) * -(math.log(10000.0) / H))
        a = (torch.arange(max(5000, T) - 1, -1, -1.0, dtype=torch.float32)[:T, None] * div).double()
        pe = torch.stack([torch.sin(a), torch.cos(a)], -1).reshape(T, H)
        assert float((pe - rel_pe(T, H).double()).abs().max()) < 1e-5
        xv = xs * escale
        ref = xv + pe[None]
        bound = E_x * escale + U * xv.abs() + 2.0 ** -22 + U * ref.abs()
        kw["x2"] = div.to(DEV)
    else:
        ref, bound = xs, E_x
    yf, y = out_f((B, T, H))
    nf, npd = out_f((B, T))
    kf, kpm = out_b((B, T))
    probe("EMBED_TOKENS", tok=tok.to(DEV), E=E.to(DEV), ntok=ntok, escale=escale, pos_mode=pos_mode, neg_emb=neg_emb,
          xscale=escale, y=yf, y2=nf, kpm=kf, B=B, T=T, H=H, **kw)
    for t, f in (("x", yf), ("nonpad", nf), ("kpm", kf)):
        written(f"embed {t}", f)
    exact("embed nonpad", "EMBED_TOKENS", npd, (tok != 0).float())
    exact("embed kpm", "EMBED_TOKENS", kpm, (tok == 0).to(torch.uint8))
    tag = f"embed {name} B {B} T {T} pos {pos_mode} midi {midi}"
    if not midi and pos_mode == 0:
        exact(tag, "EMBED_TOKENS", y, (escale * E[tok.long()]))
    else:
        check(tag, "EMBED_TOKENS", y.cpu(), ref, bound)


# ================================================================================================ masks
@gpu
@pytest.mark.parametrize("rows,Cc", [(203, 64), (61, 256), (37, 80), (8, 1), (EW_CAP // 200 + 5, 256)])
def test_row_masks(rows, Cc):
    """fs_rowmask (any(x != 0)), pe_mask (abs-sum != 0), gs_refmask (x[..., 0] != 0 over 80-bin rows), gs_kpm
    (x[..., 0] == 0): zero rows, -0.0 rows, one non-zero in the last column, a subnormal, column 0 alone zero"""
    x = specs.synth_tensor((rows, Cc), rows + Cc)
    x[::3] = 0.0
    x[1::7] = -0.0
    if rows > 10:
        x[4] = 0.0
        x[4, -1] = 2.5
        x[5] = 0.0
        x[5, Cc // 2] = 1e-40
        x[6, 0] = 0.0
    x[2 % rows, 0] = -0.0
    xd = x.to(DEV)
    nf, npd = out_f((rows,))
    kf, kpm = out_b((rows,))
    probe("ROWMASK", x=xd, y=nf, kpm=kf, rows=rows, C=Cc)
    written("rowmask", nf)
    written("rowmask kpm", kf)
    pad = x.abs().sum(-1).eq(0)
    exact(f"rowmask {rows}x{Cc}", "ROWMASK", npd, (~pad).float())
    exact(f"rowmask kpm {rows}x{Cc}", "ROWMASK", kpm, pad.to(torch.uint8))
    mf, m = out_f((rows,))
    probe("PE_MASK", x=xd, y=mf, rows=rows, M=Cc)
    written("pe_mask", mf)
    exact(f"pe_mask {rows}x{Cc}", "PE_MASK", m, (~pad).float())
    kf, kpm = out_b((rows,))
    probe("GS_KPM", x=xd, kpm=kf, rows=rows, H=Cc)
    written("gs_kpm", kf)
    exact(f"gs_kpm {rows}x{Cc}", "GS_KPM", kpm, x[:, 0].eq(0).to(torch.uint8))
    if Cc == 80:
        rf, rm = out_f((rows,))
        probe("GS_REFMASK", x=xd, y=rf, rows=rows)
        written("gs_refmask", rf)
        exact(f"gs_refmask {rows}", "GS_REFMASK", rm, (~x[:, 0].eq(0)).float())


@gpu
def test_refmask_large():
    """gs_refmask over more rows than one grid-stride pass"""
    rows = EW_CAP + 1001
    x = specs.synth_tensor((rows, 80), 3)
    x[::5, 0] = 0.0
    rf, rm = out_f((rows,))
    probe("GS_REFMASK", x=x.to(DEV), y=rf, rows=rows)
    written("gs_refmask", rf)
    exact("gs_refmask large", "GS_REFMASK", rm, (~x[:, 0].eq(0)).float())


# ================================================================================================ durations, LR
def tie_inputs():
    """fp32 x around log 1.5, log 2.5, log 3.5 (exp(x) - 1 near the ties .5, 1.5, 2.5), 8 neighbours each side"""
    out = []
    for t in (1.5, 2.5, 3.5):
        x = torch.tensor([math.log(t)], dtype=torch.float32)
        for _ in range(8):
            x = torch.nextafter(x, torch.tensor([-1.0]))
        for _ in range(17):
            out.append(float(x))
            x = torch.nextafter(x, torch.tensor([9.0]))
    return torch.tensor(out, dtype=torch.float32)


def dur_inputs(rows, seed):
    x = specs.synth_tensor((rows,), seed, scale=1.2, shift=0.8)
    edge = torch.cat([torch.tensor([0.0, -0.0, -50.0, -200.0, 5.0, -1e-6]), tie_inputs()])
    n = min(rows, edge.numel())
    x[:n] = edge[:n]
    nonpad = torch.ones(rows)
    nonpad[n::5] = 0.0
    return x, nonpad


@gpu
@pytest.mark.parametrize("rows", [3 * 61, 67, EW_CAP + 333])
def test_dur(rows):
    """dur = pred * nonpad; dur_choice = clamp(round(exp(dur) - 1), 0), half to even, 0 on padding"""
    x, nonpad = dur_inputs(rows, rows)
    pred4 = specs.synth_tensor((rows, 4), 1)
    pred4[:, 0] = x
    df, dur = out_f((rows,))
    cf, dch = out_i((rows,))
    probe("DUR", x=pred4.to(DEV), x2=nonpad.to(DEV), y=df, iy=cf, rows=rows)
    written("dur", df)
    written("dur_choice", cf)
    xs = x * nonpad
    exact(f"dur {rows}", "DUR", dur, xs)
    tie_e = torch.exp(xs.to(DEV)) - 1
    ntie = int(((tie_e - torch.floor(tie_e)) == 0.5).sum())
    assert ntie >= (3 if rows >= 57 else 0), f"only {ntie} exact ties reached"
    assert dur_gate(xs, nonpad, dch, tie_e), f"dur_choice {rows}: outside the rounding gate"
    print(f"dur {rows}: dur_choice within the gate ({ntie} exact ties)")
    seen("DUR")
    df, _ = out_f((rows,))
    probe("DUR", x=pred4.to(DEV), x2=nonpad.to(DEV), y=df, rows=rows)      # dch null: durations only
    written("dur only", df)


def ragged_durations(B, T, seed, mean=4):
    g = torch.Generator().manual_seed(seed)
    d = torch.randint(0, 2 * mean + 1, (B, T), generator=g, dtype=torch.int32)
    d[0, min(1, T - 1)] = 0
    if B >= 2:
        d[1] = 0                                 # an utterance whose durations sum to 0
    if B >= 3:
        d[2, T // 2:] = 0                        # trailing padding tokens
    return d


LR_CASES = [(3, 23, 4, 0), (3, 61, 4, 7), (3, 61, 4, -9), (1, 1, 3, 0), (4, 100, 2, 1), (3, 1000, 300, 0)]


@gpu
@pytest.mark.parametrize("B,T,mean,dTm", LR_CASES)
def test_length_regulator(B, T, mean, dTm):
    """fs_lr_scan (cumsum, mel_len) then fs_lr_fill (mel2ph) against the LengthRegulator's token_mask form; an utterance
    of total duration 0, zero-duration tokens, Tm above / below the longest mel_len, B Tm past one grid-stride pass"""
    d = ragged_durations(B, T, T + B, mean)
    cf, cum = out_i((B, T))
    lf, mlen = out_i((B,))
    probe("LR_SCAN", idx=d.to(DEV), iy=cf, iy2=lf, B=B, T=T)
    written("lr_scan cum", cf)
    written("lr_scan mel_len", lf)
    exact(f"lr_scan B {B} T {T}", "LR_SCAN", cum, torch.cumsum(d, 1).int())
    exact(f"lr_scan mel_len B {B} T {T}", "LR_SCAN", mlen, d.sum(1).int())
    Tm = max(1, int(d.sum(1).max()) + dTm)
    mf, m2p = out_i((B, Tm))
    probe("LR_FILL", idx=cum, idx2=mlen, iy=mf, B=B, T=T, T2=Tm)
    written("lr_fill", mf)
    exact(f"lr_fill B {B} T {T} Tm {Tm}", "LR_FILL", m2p, lr_mel2ph(d, Tm))


@gpu
@pytest.mark.parametrize("B,Tt,Tm,H", [(3, 23, 97, 64), (3, 61, 250, 256), (1, 1, 7, 256), (3, 40, 1000, 256)])
def test_gather(B, Tt, Tm, H):
    """expand_states: gather(pad(enc, 1 leading zero row), mel2ph), tgt = mel2ph > 0; mel2ph 0 rows, an all-zero
    utterance, and values above T_txt, which the engine clamps to the last token (the reference's gather would fail)"""
    enc = specs.synth_tensor((B, Tt, H), Tm)
    g = torch.Generator().manual_seed(Tm)
    m2p = torch.randint(0, Tt + 1, (B, Tm), generator=g, dtype=torch.int32)
    m2p[0, :5] = Tt + 3
    m2p[:, -3:] = 0
    if B >= 2:
        m2p[1] = 0
    of, out = out_f((B, Tm, H))
    tf, tgt = out_f((B, Tm))
    probe("GATHER", x=enc.to(DEV), mel2ph=m2p.to(DEV), y=of, y2=tf, B=B, T=Tt, T2=Tm, H=H)
    written("gather", of)
    written("gather tgt", tf)
    idx = m2p.clamp(max=Tt).long()
    want = torch.gather(F.pad(enc, [0, 0, 1, 0]), 1, idx[..., None].repeat(1, 1, H))
    exact(f"gather B {B} Tt {Tt} Tm {Tm} H {H}", "GATHER", out, want)
    exact(f"gather tgt B {B} Tm {Tm}", "GATHER", tgt, (m2p > 0).float())


# ================================================================================================ affine, positions
@gpu
@pytest.mark.parametrize("rows,Cc,affine", [(3 * 97, 32, True), (3 * 97, 256, True), (203, 80, False),
                                            (3 * 1000, 256, False), (3 * 1000, 256, True)])
def test_affine_mask(rows, Cc, affine):
    """x * mask and the PitchExtractor's BatchNorm (x a + b) * mask: exact / one FMA"""
    x = specs.synth_tensor((rows, Cc), rows + Cc, scale=2.0)
    mask = (specs.synth_tensor((rows,), 2) > -0.7).float()
    a = specs.synth_tensor((Cc,), 3, scale=0.5, shift=1.0) if affine else None
    b = specs.synth_tensor((Cc,), 4, scale=0.3) if affine else None
    yf, y = out_f((rows, Cc))
    y.copy_(x.to(DEV))
    probe("AFFINE_MASK", y=yf, w=a.to(DEV) if affine else None, b=b.to(DEV) if affine else None, x=mask.to(DEV),
          rows=rows, C=Cc)
    written("affine_mask", yf)
    tag = f"affine_mask {rows}x{Cc} affine {affine}"
    if affine:
        ref = (x.double() * a.double() + b.double()) * mask.double()[:, None]
        check(tag, "AFFINE_MASK", y.cpu(), ref, U * ref.abs() + 1e-45)
    else:
        exact(tag, "AFFINE_MASK", y, x * mask[:, None])


def frame_batch(B, T, Cc, seed):
    """[B][T][C] rows, x[..., 0] zero on padding frames, interior frames and a whole utterance (B >= 3), -0.0 once"""
    x = specs.synth_tensor((B, T, Cc), seed)
    for b in range(B):
        x[b, max(T - 5 * b, 0):, 0] = 0.0
    if B >= 3:
        x[B - 1, :, 0] = 0.0
    if T >= 4:
        x[0, 1, 0] = 0.0
        x[0, 3, 0] = -0.0
    return x


@gpu
@pytest.mark.parametrize("B,T,Cc,alpha,alias", [(3, 97, 64, 1.0, False), (3, 61, 256, 0.73, True),
                                                (1, 1, 256, 1.0, False), (2, 40, 33, 1.3, False),
                                                (3, 1000, 256, 1.0, True)])
def test_positions_and_posemb_add(B, T, Cc, alpha, alias):
    """make_positions on x[..., 0] (padding idx 0: interior zeros, -0.0, an all-zero utterance), then x + alpha *
    SinusoidalPositionalEmbedding(positions) (row 0 zero, an odd C's zero last column), in place or not"""
    x = frame_batch(B, T, Cc, T + Cc)
    xd = x.to(DEV)
    pf, pos = out_i((B, T))
    probe("POSITIONS", x=xd, iy=pf, B=B, T=T, C=Cc)
    written("positions", pf)
    want = make_positions(x[..., 0])
    exact(f"positions B {B} T {T}", "POSITIONS", pos, want)
    tab, E = sin_table(want, Cc)
    ref = x.double() + alpha * tab
    bound = abs(alpha) * E + U * (ref.abs() + abs(alpha) * tab.abs())
    if alias:
        yf, y = out_f((B, T, Cc))
        y.copy_(xd)
        probe("POSEMB_ADD", x=yf, idx=pos, y=yf, alpha=alpha, rows=B * T, C=Cc)
    else:
        yf, y = out_f((B, T, Cc))
        probe("POSEMB_ADD", x=xd, idx=pos, y=yf, alpha=alpha, rows=B * T, C=Cc)
    written("posemb_add", yf)
    check(f"posemb_add B {B} T {T} C {Cc} alias {alias}", "POSEMB_ADD", y.cpu(), ref, bound)


# ================================================================================================ fs2 pitch / energy
NORMS = [(1, 220.0, 60.0), (1, f32(211.37), f32(48.91)), (2, 0.0, 1.0)]


def pitch_inputs(rows, norm, seed):
    pred4 = specs.synth_tensor((rows, 4), seed)
    if norm == 2:
        pred4[:, 0] = specs.synth_tensor((rows,), seed + 1, scale=0.8, shift=7.6)      # log2 f0 around 200 Hz
    return pred4


@gpu
@pytest.mark.parametrize("norm,mean,std", NORMS)
@pytest.mark.parametrize("forced", [False, True])
@pytest.mark.parametrize("use_uv", [1, 0])
@pytest.mark.parametrize("rows", [3 * 197, EW_CAP + 777])
def test_pitch_frame(norm, mean, std, forced, use_uv, rows):
    """add_pitch 'frame': f0_denorm with uv and padding zeroed, pitch_pred (channel 0 zeroed on padding when predicted),
    coarse bins; teacher-forced f0 / uv, f0 on bin edges"""
    pred4 = pitch_inputs(rows, norm, rows + norm)
    g = torch.Generator().manual_seed(rows)
    m2p = torch.randint(0, 30, (rows,), generator=g, dtype=torch.int32)
    kw = {}
    f0 = pred4[:, 0]
    uv = pred4[:, 1] > 0
    if forced:
        f0 = specs.synth_tensor((rows,), 9, scale=1.0)
        if norm == 1:
            ed = f0_edges(60)
            f0[:ed.numel()] = (ed - mean) / std                  # lands near the edges after the denorm
        else:
            f0 = specs.synth_tensor((rows,), 9, scale=0.8, shift=7.6)
        uvf = (specs.synth_tensor((rows,), 10) > 0.3).float()
        uv = uvf > 0
        kw = dict(x2=f0.to(DEV), x3=uvf.to(DEV))
    pf, pp = out_f((rows, 2))
    ff, f0d = out_f((rows,))
    cf, coarse = out_i((rows,))
    probe("PITCH_FRAME", x=pred4.to(DEV), mel2ph=m2p.to(DEV), use_uv=use_uv, norm=norm, mean=mean, std_=std, y=pf,
          y2=ff, iy=cf, rows=rows, **kw)
    for t, f in (("pitch_pred", pf), ("f0d", ff), ("coarse", cf)):
        written(f"pitch_frame {t}", f)
    pad = m2p == 0
    ref, E = denorm_ref(f0, norm, mean, std)
    zero = pad | (uv if use_uv else torch.zeros_like(pad))
    ref, E = ref.masked_fill(zero, 0.0), E.masked_fill(zero, 0.0)
    tag = f"pitch_frame norm {norm} forced {forced} uv {use_uv} rows {rows}"
    check_denorm(tag, "PITCH_FRAME", f0d.cpu(), ref, E, norm)
    want_pp = pred4[:, :2].clone()
    if not forced:
        want_pp[pad, 0] = 0.0
    exact(tag + " pitch_pred", "PITCH_FRAME", pp, want_pp)
    check_coarse(tag, "PITCH_FRAME", f0d, coarse)


@gpu
@pytest.mark.parametrize("norm,mean,std", NORMS)
@pytest.mark.parametrize("forced", [False, True])
def test_pitch_ph(norm, mean, std, forced):
    """add_pitch 'ph': per token, no uv, no padding zeroing"""
    rows = 3 * 61
    pred4 = pitch_inputs(rows, norm, 31)
    f0 = pred4[:, 0]
    kw = {}
    if forced:
        f0 = (f0_edges(61)[:rows] - mean) / std if norm == 1 else specs.synth_tensor((rows,), 9, scale=0.8, shift=7.6)
        kw = dict(x2=f0.contiguous().to(DEV))
    pf, pp = out_f((rows,))
    ff, f0d = out_f((rows,))
    cf, coarse = out_i((rows,))
    probe("PITCH_PH", x=pred4.to(DEV), norm=norm, mean=mean, std_=std, y=pf, y2=ff, iy=cf, rows=rows, **kw)
    for t, f in (("pitch_pred", pf), ("f0d", ff), ("coarse", cf)):
        written(f"pitch_ph {t}", f)
    ref, E = denorm_ref(f0, norm, mean, std)
    tag = f"pitch_ph norm {norm} forced {forced}"
    check_denorm(tag, "PITCH_PH", f0d.cpu(), ref, E, norm)
    exact(tag + " pitch_pred", "PITCH_PH", pp, pred4[:, 0])
    check_coarse(tag, "PITCH_PH", f0d, coarse)


@gpu
@pytest.mark.parametrize("forced", [False, True])
@pytest.mark.parametrize("rows", [3 * 300, EW_CAP + 5])
def test_energy(forced, rows):
    """add_energy: bucket = clamp(e * 256 // 4, max = 255) exactly, on and around every bucket edge k / 64, at 4.0
    and far above; negative energies take bucket 0 (the engine's lower clamp; the reference's embedding would fail)"""
    pred4 = specs.synth_tensor((rows, 4), rows, scale=1.5, shift=1.5)
    e = pred4[:, 0].clone()
    edges = torch.arange(0, 260, dtype=torch.float32) / 64
    special = torch.cat([edges, torch.nextafter(edges, edges - 1), torch.nextafter(edges, edges + 1),
                         torch.tensor([100.0, 1e30, -0.0, -1e-8, -3.0])])
    e[:special.numel()] = special
    kw = {}
    if forced:
        kw = dict(x2=e.to(DEV))
    else:
        pred4[:, 0] = e
    pf, ep = out_f((rows,))
    bf, bkt = out_i((rows,))
    probe("ENERGY", x=pred4.to(DEV), y=pf, iy=bf, rows=rows, **kw)
    written("energy_pred", pf)
    written("energy bucket", bf)
    exact(f"energy_pred forced {forced}", "ENERGY", ep, pred4[:, 0])
    want = torch.clamp(e * 256 // 4, max=255).long()
    want = torch.where(e < 0, torch.zeros_like(want), want)
    exact(f"energy bucket forced {forced} rows {rows}", "ENERGY", bkt, want)


@gpu
@pytest.mark.parametrize("mode", ["frame+energy", "frame", "ph", "energy"])
@pytest.mark.parametrize("B,Tt,Tm,H", [(3, 23, 97, 64), (3, 40, 1000, 256)])
def test_embed_add(mode, B, Tt, Tm, H):
    """decoder_inp = (gathered + pitch_embed[pitch] + energy_embed[energy]) * tgt_nonpad, in torch's fp32 order; 'ph'
    bins through F.pad(coarse, [1, 0]) and mel2ph (values above T_txt clamp to the last token)"""
    rows = B * Tm
    x = specs.synth_tensor((rows, H), Tm)
    g = torch.Generator().manual_seed(H)
    m2p = torch.randint(0, Tt + 1, (B, Tm), generator=g, dtype=torch.int32)
    m2p[0, :3] = Tt + 2
    tgt = (m2p > 0).float().reshape(rows)
    pE = specs.synth_tensor((300, H), 2)
    eE = specs.synth_tensor((256, H), 3)
    pframe = torch.randint(1, 256, (rows,), generator=g, dtype=torch.int32)
    ptok = torch.randint(1, 256, (B, Tt), generator=g, dtype=torch.int32)
    ebkt = torch.randint(0, 256, (rows,), generator=g, dtype=torch.int32)
    kw = {}
    want = x.clone()
    if mode.startswith("frame"):
        kw.update(E=pE.to(DEV), idx=pframe.to(DEV))
        want = want + pE[pframe.long()]
    elif mode == "ph":
        kw.update(E=pE.to(DEV), idx2=ptok.to(DEV))
        bins = torch.gather(F.pad(ptok, [1, 0]), 1, m2p.clamp(max=Tt).long()).reshape(rows)
        want = want + pE[bins.long()]
    if "energy" in mode:
        kw.update(E2=eE.to(DEV), idx3=ebkt.to(DEV))
        want = want + eE[ebkt.long()]
    want = want * tgt[:, None]
    yf, y = out_f((rows, H))
    probe("EMBED_ADD", x=x.to(DEV), x2=tgt.to(DEV), mel2ph=m2p.to(DEV), y=yf, T=Tt, T2=Tm, rows=rows, H=H, **kw)
    written("embed_add", yf)
    exact(f"embed_add {mode} B {B} Tm {Tm} H {H}", "EMBED_ADD", y, want)


# ================================================================================================ GenerSpeech
@gpu
@pytest.mark.parametrize("form", ["dur_inp", "inpainter", "decoder_inp"])
@pytest.mark.parametrize("B,T,H", [(3, 97, 64), (3, 1000, 256)])
def test_gs_sum(form, B, T, H):
    """(x + spk + emo (+ pitch_embed[coarse]) (+ prosody)) * mask, in generspeech.py's fp32 order"""
    rows = B * T
    x, s = specs.synth_tensor((rows, H), 1), specs.synth_tensor((rows, H), 2)
    spk, emo = specs.synth_tensor((B, H), 3), specs.synth_tensor((B, H), 4)
    tab = specs.synth_tensor((300, H), 5)
    idx = torch.randint(1, 256, (rows,), generator=torch.Generator().manual_seed(T), dtype=torch.int32)
    mask = (specs.synth_tensor((rows,), 6) > -0.5).float()
    bi = torch.arange(rows) // T
    want = (x + spk[bi]) + emo[bi]
    kw = {}
    if form == "decoder_inp":
        want = want + tab[idx.long()]
        kw.update(E=tab.to(DEV), idx=idx.to(DEV))
    if form != "dur_inp":
        want = want + s
        kw.update(x4=s.to(DEV))
    want = want * mask[:, None]
    yf, y = out_f((rows, H))
    probe("GS_SUM", x=x.to(DEV), x2=spk.to(DEV), x3=emo.to(DEV), x5=mask.to(DEV), y=yf, T=T, rows=rows, H=H, **kw)
    written("gs_sum", yf)
    exact(f"gs_sum {form} B {B} T {T} H {H}", "GS_SUM", y, want)


@gpu
@pytest.mark.parametrize("n", [3 * 97 * 64, EW_CAP + 4097])
def test_gs_accum(n):
    """the prosody sum: dst = src (first level), then dst + src"""
    a, b = specs.synth_tensor((n,), 1), specs.synth_tensor((n,), 2)
    yf, y = out_f((n,))
    probe("GS_ACCUM", y=yf, x=a.to(DEV), rows=n, first=1)
    written("gs_accum first", yf)
    exact(f"gs_accum first {n}", "GS_ACCUM", y, a)
    probe("GS_ACCUM", y=yf, x=b.to(DEV), rows=n, first=0)
    written("gs_accum", yf)
    exact(f"gs_accum {n}", "GS_ACCUM", y, a + b)


@gpu
@pytest.mark.parametrize("rows,Cc", [(3 * 151, 80), (3 * 61, 32), (3 * 61, 128), (3 * 2700, 80)])
def test_gs_wn_gate(rows, Cc):
    """WN's fused_add_tanh_sigmoid_multiply: tanh(a[:, :C]) * sigmoid(a[:, C:]); saturated arguments included"""
    a = specs.synth_tensor((rows, 2 * Cc), rows + Cc, scale=2.5)
    a[0, :4] = torch.tensor([30.0, -30.0, 1e-20, 0.0])
    a[0, Cc:Cc + 4] = torch.tensor([-100.0, 100.0, 0.0, -0.0])
    yf, y = out_f((rows, Cc))
    probe("GS_WN_GATE", x=a.to(DEV), y=yf, rows=rows, C=Cc)
    written("wn_gate", yf)
    a64 = a.double()
    ref = torch.tanh(a64[:, :Cc]) * torch.sigmoid(a64[:, Cc:])
    check(f"wn_gate {rows}x{Cc}", "GS_WN_GATE", y.cpu(), ref, ref.abs() * (2 * 2.0 ** -22 + 4 * U) + 1e-38)


def segmean_reference(h, seg, nseg):
    """group_hidden_by_segs (utils/tts_utils.py) via scatter_add in fp64, ids above nseg dropped; (ref, bound)"""
    B, T, Cc = h.shape
    n = max(int(seg.max()), nseg)
    idx = seg.long()
    s = torch.zeros(B, n + 1, Cc, dtype=torch.float64).scatter_add_(1, idx[..., None].repeat(1, 1, Cc), h.double())
    a = torch.zeros(B, n + 1, Cc, dtype=torch.float64).scatter_add_(1, idx[..., None].repeat(1, 1, Cc),
                                                                     h.double().abs())
    c = torch.zeros(B, n + 1, dtype=torch.float64).scatter_add_(1, idx, torch.ones(B, T, dtype=torch.float64))
    s, a, c = s[:, 1:nseg + 1], a[:, 1:nseg + 1], c[:, 1:nseg + 1, None]
    ref = s / c.clamp(min=1)
    return ref, gam(c) * U * a / c.clamp(min=1) + U * ref.abs()


def seg_ids(B, T, nseg, seed):
    """ragged segment ids 1..nseg in runs, 0 on padding frames, skipped ids (empty segments), ids above nseg"""
    g = torch.Generator().manual_seed(seed)
    seg = torch.zeros(B, T, dtype=torch.int32)
    for b in range(B):
        n = T - 7 * b
        cuts = torch.sort(torch.randint(0, nseg + 3, (max(n, 0),), generator=g)).values
        seg[b, :max(n, 0)] = cuts.int()
    seg[seg == nseg // 2] = 0                  # segment nseg / 2 is empty
    if B >= 3:
        seg[B - 1] = 0
    return seg


@gpu
@pytest.mark.parametrize("B,T,nseg", [(3, 151, 37), (3, 151, 11), (1, 5, 9), (2, 1000, 120)])
def test_gs_segmean(B, T, nseg):
    """segment means of the WN output over ref_mel2ph / ref_mel2word: empty segments (0), an all-padding utterance, ids
    above nseg ignored"""
    Cc = specs.GS_STYLE_C
    h = specs.synth_tensor((B, T, Cc), T + nseg, shift=0.5)
    seg = seg_ids(B, T, nseg, T)
    yf, y = out_f((B, nseg, Cc))
    probe("GS_SEGMEAN", x=h.to(DEV), idx=seg.to(DEV), y=yf, B=B, T=T, nseg=nseg, C=Cc)
    written("segmean", yf)
    ref, E = segmean_reference(h, seg, nseg)
    check(f"segmean B {B} T {T} nseg {nseg}", "GS_SEGMEAN", y.cpu(), ref, E)


def vq_bound(x, dots, enorm):
    """fp64 distances (|e|^2 + |x|^2) - 2 dot of the fp32 inputs, and the bound of the kernel's fp32 evaluation"""
    H = x.shape[1]
    xn = x.double().pow(2).sum(1, keepdim=True)
    D = (enorm.double()[None] + xn) - 2 * dots.double()
    n = math.ceil(H / 32) + 5
    E = U * ((gam(n) + 1) * xn + (enorm.double()[None] + xn).abs() + D.abs()) + 1e-300
    return D, E


def vq_choice_ok(x, dots, enorm, idx):
    D, E = vq_bound(x, dots, enorm)
    best = D.argmin(1)
    r = torch.arange(D.shape[0])
    i = idx.long().cpu()
    return (i == best) | (D[r, i] - D[r, best] <= E[r, i] + E[r, best])


def vq_tie_ok(dots, enorm, idx, rows):
    """on `rows` (whose fp32 distances tie exactly between duplicate codes) idx is the lowest index of the tie"""
    d = (enorm[None] + 0.0) - 2 * dots           # the tie is exact in any order: duplicate codes give identical terms
    lowest = torch.stack([int(torch.nonzero(d[r] == d[r].min())[0]) * torch.ones((), dtype=torch.long) for r in rows])
    return idx.long().cpu()[rows] == lowest


def vq_inputs(rows, H, M, seed, dup=()):
    emb = specs.synth_tensor((M, H), seed, scale=0.5)
    for lo, hi in dup:
        emb[hi] = emb[lo]
    x = specs.synth_tensor((rows, H), seed + 1, scale=0.5)
    x[1::9] = 0.0                                 # padding rows of the masked ConvBlocks output
    for k, (lo, _) in enumerate(dup):
        x[2 + k] = emb[lo] + 1e-3 * specs.synth_tensor((H,), 50 + k)
    dots = (x.double() @ emb.double().t()).float()
    for k, (lo, hi) in enumerate(dup):
        dots[:, hi] = dots[:, lo]
    enorm = (emb ** 2).sum(1)
    return x, emb, dots, enorm


VQ_CASES = [(3 * 37, 64, 16, ()), (3 * 37, 256, 128, ((3, 35), (7, 40), (64, 127))),
            (3 * 61, 256, 50, ((0, 49), (17, 18))), (203, 64, 16, ((2, 9), (4, 15))), (3 * 1000, 256, 128, ())]


@gpu
@pytest.mark.parametrize("rows,H,M,dup", VQ_CASES)
@pytest.mark.parametrize("alias", [False, True])
def test_gs_vq(rows, H, M, dup, alias):
    """VQEmbeddingEMA.encode + straight-through: argmin over M = 16 / 128 / 50 codes (lanes with no code, two codes per
    lane), exact ties between duplicate codes on the same and on different lanes, q = x + (e - x), q aliasing x"""
    x, emb, dots, enorm = vq_inputs(rows, H, M, rows + M, dup)
    xd = x.to(DEV)
    if alias:
        qf, q = out_f((rows, H))
        q.copy_(xd)
        src = qf
    else:
        qf, q = out_f((rows, H))
        src = xd
    jf, idx = out_i((rows,))
    probe("GS_VQ", x=src, x2=dots.to(DEV), E=emb.to(DEV), x3=enorm.to(DEV), iy=jf, y=qf, rows=rows, H=H, M=M)
    written("vq idx", jf)
    written("vq q", qf)
    ok = vq_choice_ok(x, dots, enorm, idx)
    assert bool(ok.all()), f"vq: row {int((~ok).nonzero()[0])} chose code {int(idx[int((~ok).nonzero()[0])])}"
    if dup:
        tie_rows = list(range(2, 2 + len(dup)))
        assert bool(vq_tie_ok(dots, enorm, idx, tie_rows).all()), f"vq ties: {idx[2:2 + len(dup)].tolist()}"
    _, ref_idx, _ = vq_encode(emb.double(), x.double()[None])
    agree = int((ref_idx[0] == idx.cpu().long()).sum())
    print(f"vq rows {rows} H {H} M {M}: {agree}/{rows} choices equal to the fp64 encode, all within the gate")
    qi = idx.long().cpu()
    exact(f"vq q rows {rows} M {M} alias {alias}", "GS_VQ", q, x + (emb[qi] - x))
    qf, q2 = out_f((rows, H))
    probe("GS_VQ", x=xd, x2=dots.to(DEV), E=emb.to(DEV), x3=enorm.to(DEV), y=qf, rows=rows, H=H, M=M)     # idx null
    written("vq q (no idx)", qf)
    exact("vq q (no idx)", "GS_VQ", q2, q)


@gpu
@pytest.mark.parametrize("B,T,H", [(3, 37, 64), (3, 11, 256), (1, 1, 256), (3, 1000, 256)])
def test_gs_catpos(B, T, H):
    """l1's input cat[prosody, SinusoidalPositionalEmbedding(make_positions(prosody[..., 0]))]"""
    x = frame_batch(B, T, H, T + H)
    pos = make_positions(x[..., 0]).int()
    yf, y = out_f((B, T, 2 * H))
    probe("GS_CATPOS", x=x.to(DEV), idx=pos.to(DEV), y=yf, rows=B * T, H=H)
    written("catpos", yf)
    exact(f"catpos B {B} T {T} H {H} prosody half", "GS_CATPOS", y[..., :H], x)
    ref, E = sin_table(pos, H)
    check(f"catpos B {B} T {T} H {H}", "GS_CATPOS", y[..., H:].cpu(), ref, E)


@gpu
@pytest.mark.parametrize("forced_edges", [False, True])
@pytest.mark.parametrize("rows", [3 * 197, EW_CAP + 3])
def test_gs_pitch(forced_edges, rows):
    """inpaint_pitch: pitch_pred = p1 + p2; f0_denorm = f0_denorm_pred = (pp0 * std + mean), uv and padding zeroed"""
    mean, std = 220.0, 60.0
    p1, p2 = specs.synth_tensor((rows, 4), 1), specs.synth_tensor((rows, 4), 2, scale=0.5)
    if forced_edges:
        ed = f0_edges(60)
        p1[:ed.numel(), 0] = (ed - mean) / std - p2[:ed.numel(), 0]
        p1[:ed.numel(), 1] = -1.0 - p2[:ed.numel(), 1].abs()
    m2p = torch.randint(0, 20, (rows,), generator=torch.Generator().manual_seed(rows), dtype=torch.int32)
    pf, pp = out_f((rows, 2))
    ff, f0d = out_f((rows,))
    gf, f0p = out_f((rows,))
    cf, coarse = out_i((rows,))
    probe("GS_PITCH", x=p1.to(DEV), x2=p2.to(DEV), mel2ph=m2p.to(DEV), mean=mean, std_=std, y=pf, y2=ff, y3=gf, iy=cf,
          rows=rows)
    for t, f in (("pitch_pred", pf), ("f0d", ff), ("f0d_pred", gf), ("coarse", cf)):
        written(f"gs_pitch {t}", f)
    s = p1[:, :2] + p2[:, :2]
    tag = f"gs_pitch rows {rows} edges {forced_edges}"
    exact(tag + " pitch_pred", "GS_PITCH", pp, s)
    ref, _ = denorm_ref(s[:, 0], 1, mean, std)
    ref = ref.masked_fill((s[:, 1] > 0) | (m2p == 0), 0.0)
    exact(tag + " f0_denorm", "GS_PITCH", f0d, ref)
    exact(tag + " f0_denorm_pred", "GS_PITCH", f0p, ref)
    check_coarse(tag, "GS_PITCH", f0d, coarse)


@gpu
@pytest.mark.parametrize("B,T,H", [(3, 97, 64), (2, 61, 256), (3, 700, 256)])
def test_gs_cond_cat(B, T, H):
    """the post-flow's g = cat[mel_out, decoder_inp, spk, emo, ref_prosody] per frame"""
    M = 80
    rows = B * T
    mel, dec, pros = (specs.synth_tensor((B, T, c), i) for i, c in ((1, M), (2, H), (3, H)))
    spk, emo = specs.synth_tensor((B, H), 4), specs.synth_tensor((B, H), 5)
    gf, g = out_f((B, T, M + 4 * H))
    probe("GS_COND_CAT", x=mel.to(DEV), x2=dec.to(DEV), x3=spk.to(DEV), x4=emo.to(DEV), x5=pros.to(DEV), y=gf, T=T,
          rows=rows, M=M, H=H)
    written("cond_cat", gf)
    want = torch.cat([mel, dec, spk[:, None].expand(-1, T, -1), emo[:, None].expand(-1, T, -1), pros], -1)
    exact(f"cond_cat B {B} T {T} H {H}", "GS_COND_CAT", g, want)


def glow_squeeze(z, T2):
    """glow_modules.py squeeze(x, n_sqz = 2) of z [B][M][Tz] over its first 2 T2 frames -> channels-last [B][T2][2M]"""
    b, c, _ = z.shape
    x = z[:, :, :2 * T2]
    return x.reshape(b, c, T2, 2).permute(0, 3, 1, 2).reshape(b, c * 2, T2).transpose(1, 2)


@gpu
@pytest.mark.parametrize("B,M,Tz,T2", [(3, 80, 97, 48), (3, 80, 98, 49), (2, 80, 20, 7), (1, 4, 3, 1),
                                       (3, 80, 3000, 1500)])
def test_gs_squeeze(B, M, Tz, T2):
    """squeeze(z, 2) into the channels-last flow state: odd Tz (the last frame dropped), Tz > 2 T2"""
    z = specs.synth_tensor((B, M, Tz), Tz)
    xf, x = out_f((B, T2, 2 * M))
    probe("GS_SQUEEZE", x=z.to(DEV), y=xf, B=B, T=Tz, T2=T2, M=M)
    written("squeeze", xf)
    exact(f"squeeze B {B} M {M} Tz {Tz} T2 {T2}", "GS_SQUEEZE", x, glow_squeeze(z, T2))


def flow_inputs(rows, C2, seed):
    x = specs.synth_tensor((rows, C2), seed)
    e = specs.synth_tensor((rows, C2), seed + 1, scale=0.5)
    w = torch.linalg.qr(specs.synth_tensor((4, 4), seed + 2).double())[0]
    winv = torch.inverse(w).float()
    bias = specs.synth_tensor((C2,), seed + 3, scale=0.2)
    logs = specs.synth_tensor((C2,), seed + 4, scale=0.3)
    return x, e, winv, bias, logs


def flow_reference(x, e, winv, bias, logs, transposed=False):
    """CouplingBlock, InvConvNear and ActNorm reverse (glow_modules.py) on channels-first views of [rows][C2] in fp64,
    and the bound of the kernel's fp32 evaluation.  transposed: the mutant's group order i = 2 r + a."""
    t, c = x.shape
    X, Em = x.double().t()[None], e.double().t()[None]                          # [1][C2][t]
    x0, x1 = X[:, :c // 2], X[:, c // 2:]
    m, lg = Em[:, :c // 2], Em[:, c // 2:]
    z1 = (x1 - m) * torch.exp(-lg)
    V = torch.cat([x0, z1], 1)
    EV = torch.cat([torch.zeros_like(x0), z1.abs() * (2.0 ** -22 + 2 * U)], 1)
    perm = (0, 3, 1, 2, 4) if transposed else (0, 1, 3, 2, 4)

    def to_groups(a):
        return a.view(1, 2, c // 4, 2, t).permute(*perm).contiguous().view(1, 4, c // 4, t)

    def from_groups(a):
        if transposed:
            return a.view(1, 2, 2, c // 4, t).permute(0, 2, 3, 1, 4).contiguous().view(1, c, t)
        return a.view(1, 2, 2, c // 4, t).permute(0, 1, 3, 2, 4).contiguous().view(1, c, t)
    w = winv.double()
    Y = F.conv2d(to_groups(V), w.view(4, 4, 1, 1))
    wa = w.abs().view(4, 4, 1, 1)
    EY = F.conv2d(to_groups(EV), wa) + 4 * U * F.conv2d(to_groups(V).abs(), wa)
    S, ES = from_groups(Y), from_groups(EY)
    b, l = bias.double()[None, :, None], logs.double()[None, :, None]
    out = (S - b) * torch.exp(-l)
    Eo = (ES + U * (S - b).abs()) * torch.exp(-l) + (2.0 ** -22 + U) * out.abs()
    return out[0].t(), Eo[0].t()


@gpu
@pytest.mark.parametrize("rows,C2", [(3 * 48, 160), (3 * 500, 160), (97, 8), (16001, 160)])
def test_gs_flow_step(rows, C2):
    """one reverse post-flow block step in place: C2 = 160 (80 mel bins squeezed) and C2 = 8 (one channel group)"""
    x, e, winv, bias, logs = flow_inputs(rows, C2, rows + C2)
    blk = torch.cat([winv.reshape(16), bias, logs])
    yf, y = out_f((rows, C2))
    y.copy_(x.to(DEV))
    probe("GS_FLOW_STEP", y=yf, x=e.to(DEV), w=blk.to(DEV), rows=rows, C=C2)
    written("flow_step", yf)
    ref, E = flow_reference(x, e, winv, bias, logs)
    check(f"flow_step rows {rows} C2 {C2}", "GS_FLOW_STEP", y.cpu(), ref, E)


# ================================================================================================ PitchExtractor
@gpu
@pytest.mark.parametrize("norm,mean,std", NORMS)
@pytest.mark.parametrize("use_uv", [1, 0])
@pytest.mark.parametrize("rows", [2 * 301, EW_CAP // 2 * 3 + 11])
def test_pe_denorm(norm, mean, std, use_uv, rows):
    """PitchExtractor: pitch_pred = pred[..., :2]; f0 = denorm_f0(pred[..., 0], uv = pred[..., 1] > 0, padding)"""
    pred4 = pitch_inputs(rows, norm, rows)
    if norm == 1:
        ed = f0_edges(60)
        pred4[:ed.numel(), 0] = (ed - mean) / std
    mask = (specs.synth_tensor((rows,), 5) > -0.8).float()
    pf, pp = out_f((rows, 2))
    ff, f0 = out_f((rows,))
    probe("PE_DENORM", x=pred4.to(DEV), x2=mask.to(DEV), y=pf, y2=ff, rows=rows, use_uv=use_uv, norm=norm, mean=mean,
          std_=std)
    written("pe pitch_pred", pf)
    written("pe f0", ff)
    exact(f"pe pitch_pred rows {rows}", "PE_DENORM", pp, pred4[:, :2])
    ref, E = denorm_ref(pred4[:, 0], norm, mean, std)
    zero = (mask == 0) | ((pred4[:, 1] > 0) if use_uv else torch.zeros(rows, dtype=torch.bool))
    check_denorm(f"pe_denorm norm {norm} uv {use_uv} rows {rows}", "PE_DENORM", f0.cpu(), ref.masked_fill(zero, 0.0),
                 E.masked_fill(zero, 0.0), norm)


# ================================================================================================ mutants (CPU)
def test_gate_catches_positions_counting_padding():
    """make_positions counting padding tokens (cumsum of ones) fails POSITIONS and the sinusoid gate"""
    x = frame_batch(3, 40, 64, 1)
    want = make_positions(x[..., 0])
    mut = torch.cumsum(torch.ones_like(want), 1) * (x[..., 0] != 0).long()
    assert not torch.equal(mut, want)
    ref, E = sin_table(want, 64)
    assert passes(ref.float(), ref, E)
    assert not passes(sin_table(mut, 64)[0].float(), ref, E)


def test_gate_catches_lr_fill_off_by_one():
    """the mel2ph search `first t with cum[t] >= f` (instead of >) fails LR_FILL's exact gate"""
    d = ragged_durations(3, 23, 26)
    Tm = int(d.sum(1).max())
    cum = torch.cumsum(d, 1)
    f = torch.arange(Tm)[None].expand(3, -1).contiguous()
    good = torch.searchsorted(cum, f, right=True) + 1
    bad = torch.searchsorted(cum, f, right=False) + 1
    live = f < cum[:, -1:]
    good, bad = torch.where(live, good, 0), torch.where(live, bad, 0)
    assert torch.equal(good, lr_mel2ph(d, Tm))
    assert not torch.equal(bad, lr_mel2ph(d, Tm))


def test_gate_catches_durations_rounded_half_up():
    """durations rounded half up (floor(v + .5)) fail the tie rule where fp32 exp(x) - 1 is exactly k + .5"""
    x = tie_inputs()
    nonpad = torch.ones_like(x)
    e = torch.exp(x) - 1
    assert int(((e - e.floor()) == 0.5).sum()) >= 3
    good = torch.round(e).clamp(min=0)
    bad = torch.floor(e + 0.5).clamp(min=0)
    assert dur_gate(x, nonpad, good, e)
    assert not dur_gate(x, nonpad, bad, e)


def test_gate_catches_fma_denorm():
    """f0 * std + mean rounded once (an FMA, emulated in fp64 then rounded) fails the f0_denorm exactness gate"""
    f = specs.synth_tensor((4096,), 3)
    for mean, std in ((220.0, 60.0), (f32(211.37), f32(48.91))):
        ref, _ = denorm_ref(f, 1, mean, std)
        fma = (f.double() * std + mean).float()
        assert torch.equal(((f * std) + mean), ref)
        assert not torch.equal(fma, ref), "the emulated FMA matches the two-rounding result everywhere"


def test_gate_catches_vq_ties_to_highest():
    """on exact ties between duplicate codes, the highest index fails the tie gate (both pass the choice gate)"""
    dup = ((3, 35), (7, 40))
    x, emb, dots, enorm = vq_inputs(20, 64, 64, 9, dup)
    D = (enorm[None] + 0.0) - 2 * dots
    lowest = torch.tensor([int(torch.nonzero(D[r] == D[r].min())[0]) for r in range(20)])
    highest = torch.tensor([int(torch.nonzero(D[r] == D[r].min())[-1]) for r in range(20)])
    rows = [2, 3]
    assert bool(vq_choice_ok(x, dots, enorm, lowest).all()) and bool(vq_choice_ok(x, dots, enorm, highest).all())
    assert bool(vq_tie_ok(dots, enorm, lowest, rows).all())
    assert not bool(vq_tie_ok(dots, enorm, highest, rows).all())


def test_gate_catches_segmean_over_t():
    """segment sums divided by T instead of the segment's frame count fail the segmean gate"""
    B, T, nseg = 2, 151, 37
    h = specs.synth_tensor((B, T, 80), 4, shift=0.5)
    seg = seg_ids(B, T, nseg, 5)
    ref, E = segmean_reference(h, seg, nseg)
    c = torch.zeros(B, nseg + 4).scatter_add_(1, seg.long(), torch.ones(B, T))[:, 1:nseg + 1, None]
    assert passes(ref.float(), ref, E)
    assert not passes((ref * c.clamp(min=1) / T).float(), ref, E)


def test_gate_catches_transposed_invconv_groups():
    """InvConvNear's channel groups taken as i = 2 r + a (instead of 2 a + r) fail the flow-step gate"""
    x, e, winv, bias, logs = flow_inputs(64, 160, 7)
    ref, E = flow_reference(x, e, winv, bias, logs)
    mut, _ = flow_reference(x, e, winv, bias, logs, transposed=True)
    assert passes(ref.float(), ref, E)
    assert not passes(mut.float(), ref, E)


def test_gate_catches_squeeze_j_c_swapped():
    """the squeeze writing x[b][t][2 c + j] (instead of j M + c) fails the exact squeeze gate"""
    B, M, Tz, T2 = 2, 80, 21, 10
    z = specs.synth_tensor((B, M, Tz), 1)
    want = glow_squeeze(z, T2)
    bad = z[:, :, :2 * T2].reshape(B, M, T2, 2).permute(0, 2, 1, 3).reshape(B, T2, 2 * M)
    assert not torch.equal(bad, want)
    good = z[:, :, :2 * T2].reshape(B, M, T2, 2).permute(0, 2, 3, 1).reshape(B, T2, 2 * M)
    assert torch.equal(good, want)


# ================================================================================================ coverage
@gpu
def test_every_op_exercised():
    """runs last in this module: every AGPT_FS_* op was run and checked by a case above"""
    missing = [op for op in _lib.FS_OPS if op not in EXERCISED]
    assert not missing, f"not exercised: {missing}"
