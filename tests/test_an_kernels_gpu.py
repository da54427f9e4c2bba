"""Conformance of the analysis models' kernels outside the GEMMs against float64, kernel by kernel: LASSNet's FiLM
ResUNet (the BatchNorm affine and identity residual, the transposed conv's im2col and sub-pixel shuffle, the FiLM
second Linears, and through a LASSNet handle its FiLM vectors and whole decoder up path), RaDur's detection tail (the
4-channel pad, the Fusion product, the reference-embedding attention pool, the fc / softmax head, the two-pass mix and
interpolation), the BERT embeddings (untyped and typed with the key-padding mask), the CLAP Projection's GELU, and the
emotion encoder's tail (the mean-and-normalise and the Linear-ReLU-normalise).

Every GPU case runs ONE production launcher through agpt_an_probe on caller-owned device tensors and compares it with a
reference written from the reference code's formulas on its own layouts, never from the kernels' indexing:
sound_extraction/model/modules.py, film.py and resunet_film.py (oracle/lass_ref.py: _bn, _film, the decoder's
ConvTranspose2d(3, stride 2) pruned by x[:, :, :-1, :]); target_sound_detection/src/models.py:1109-1291 (oracle/
tsd_ref.py: fusion, get_w, interpolate); HF BertEmbeddings; NeuralSeq/data_gen/tts/emotion/model.py:56-59 and
inference.py:150-151.  Float outputs are filled with a sentinel (NaN, or a finite one where NaN is a legitimate output)
and followed by GUARD canaries: every case asserts that the whole output was written, nothing past it, and that every
input is bit-for-bit unchanged.

Error model and gates (u = 2^-24; g(n) = min(n, 6 sqrt(n)), the worst case or the Higham-Mary probabilistic bound for
a sum of n terms, as in test_nn_kernels_gpu.py; the CUDA math guide's maximum errors: expf and erff 2 ulp, sqrtf 1 ulp
(0 with the default -prec-sqrt=true; 1 is allowed)):

  * Exact: TSD_PAD4 and LASS_SHUFFLE (data movement), and every zero LASS_UPCOL writes outside the h x w map.
    CLAP_EMBED / CLAP_EMBED_TYPED must equal torch's fp32 (word + type) + pos, BertEmbeddings' order, bit for bit,
    with ids and type ids clamped into their tables; the key-padding mask must be exactly attention_mask == 0.
  * One correctly rounded FMA: LASS_AFFINE's a and LASS_UPCOL before its ReLU, |y - (x s + t)| <= u |x s + t| (the
    ReLU is 1-Lipschitz); the residual r = x + vec rounds once, u |x + vec|.
  * LASS_FILM: each film output is a lane-strided fmaf chain of nin terms plus a 5-level butterfly and the bias,
    g(nin + 6) u (sum |w h| + |b2|), through the ReLU; fmaf(alpha, ., beta) and the optional + film(jb) add one
    rounding each.
  * TSD_FUSE: a sequential n-term product sum and the division, g(n) u sum |a f| + u |out|.
  * TSD_REFEMB: the sequential mean over Trr, g(Trr) u mean |E| + u |m| (att_pool 0).  With att_pool the attention
    starts from that mean reproduced exactly on the host (a sequential fp32 sum; the att_pool 0 cases gate it against
    fp64): the q Linear (129 terms) and the folded key projection (128 terms, then the 160-term block sum of q . kb),
    the score sum and the 11.3 division, all in fp64 with their propagated rounding bounds; the softmax
    carries a score error E_s into a relative error e^(2 E_s) - 1 of each weight, plus expf's 2 ulp, the Trr-term sum and
    the division; the weighted sum is a Trr-term fmaf chain.
  * TSD_HEAD: 1024 products in 32 lane chains, the butterfly and the bias, g(1030) u (sum |w h| + |b|); the softmax as
    above with an O-term sum.
  * TSD_MIX_INTERP: the mix (1 - w) p1 + w p2 rounds four times; the interpolation rounds l0 = 1 - l1 and its two
    products and sum.  The reference runs ATen's linear interpolation (align_corners=False) in float64; ATen's fp32
    source index scale (t + 0.5) - 0.5, scale = (float)Td / T, may be rounded or contracted either way, so the bound
    adds that index's rounding, 3 u (scale (t + 0.5) + 1), times the largest slope of the two segments around it: no
    particular floor at an exact integer boundary is required.
  * CLAP_GELU: 0.5 x (1 + erff(x fl(1/sqrt 2))) against fp64 erf-GELU: the argument's two roundings through erf's slope,
    erff's 2 ulp, one rounding of 1 + erf, and the products; erff's 2 ulp next to 1 is the absolute term 2^-23 0.5 |x|
    that covers the cancellation in 1 + erf at large negative x.  At +-0, +-inf and NaN the kernel must match torch's
    fp32 F.gelu on the device (NaN matches NaN, the sign of a zero included).  (torch's CPU F.gelu gives NaN at +inf,
    where the kernel and torch on the device give +inf, the limit of x Phi(x).)
  * EMO_MEAN_NORM / EMO_LINEAR_NORM: the mean (or the 256-term Linear and its ReLU) as above, the block sum of squares,
    sqrtf and the division, propagated.  An all-zero ReLU row gives 0 / 0 = NaN in the reference and must in the kernel.
  * LASS_FILM_VEC and LASS_UP run the handle's own tables and packed tap-GEMMs, under the tap-GEMM error model
    test_tapconv_gpu.py states (its c, U, FLOOR and weight pre-scale, tensor-core path), carried through the fp32
    epilogue and the kernels above.  The expected FiLM vector comes from the float64 state dict: the blocks in forward
    order, each [e1: cout][r2: cout], e1 = s2 film1 + t2 (bn2 folded; the engine folds it in fp32: 6 u of |s2 film1|,
    |be| and |rm s2|) and r2 = film2 (+ film_res).  LASS_UP is compared with relu(bn1(y)) -> F.conv_transpose2d(W,
    stride=2)[:, :, :-1, :] (DecoderBlockRes2BCond.prune), concatenated with the skip.

Teeth: CPU-emulated mutants must FAIL the gate the kernel passes: the shuffle with its phase bits swapped, upcol without
its nn < w guard, affine's sample index taken from the row without dividing by C4, the embedding added as
word + (type + pos), the mask stored as mask != 0, mix_interp's i1 not clamped at Td - 1, mix_interp with an
align_corners=True scale, refemb's softmax without the 1 / 11.3, the head normalising over O - 1 outputs,
linear_norm normalising before the ReLU, and the FiLM kernel ignoring jb.  They need no device; neither do the
launchers' precondition checks, which throw before anything is launched.
"""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audiogpt_b200 import _lib, specs  # noqa: E402

gpu = pytest.mark.gpu

U = 2.0 ** -24
GUARD = 64
CANARY = -7777.25
SENT = 1.25e30          # the fill of outputs where NaN is a legitimate value
DEV = "cuda"
TEMP = 11.3
OUTS = ("y", "y2", "scratch", "kpm", "info")
EXERCISED = {}          # op -> worst error / bound over the cases that ran it (0 for the exact gates)


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    if EXERCISED:
        print("\nanalysis-model kernels exercised: worst error / bound (0 = exact)")
        for k in _lib.AN_OPS:
            if k in EXERCISED:
                print(f"  {k:16s}: {EXERCISED[k]:.3f}")


def gam(n):
    return min(n, 6.0 * math.sqrt(n))


def seen(op, ratio=0.0):
    EXERCISED[op] = max(EXERCISED.get(op, 0.0), ratio)


# ------------------------------------------------------------------------------------------------ buffers and the probe
def out_f(shape, fill=float("nan")):
    n = math.prod(shape)
    flat = torch.full((n + GUARD,), fill, dtype=torch.float32, device=DEV)
    flat[n:] = CANARY
    return flat, flat[:n].view(shape)


def written(tag, flat, fill=float("nan")):
    n = flat.numel() - GUARD
    assert torch.equal(flat[n:], torch.full_like(flat[n:], CANARY)), f"{tag}: written past the end of the output"
    left = torch.isnan(flat[:n]) if math.isnan(fill) else flat[:n] == fill
    assert not left.any(), f"{tag}: {int(left.sum())} output elements not written"


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def probe(op, stream=True, **kw):
    """one agpt_an_probe call; every tensor argument that is not an output must come back bit for bit unchanged"""
    a = _lib.AnProbeArgs()
    a.op = _lib.AN_OPS.index(op)
    keep, inputs = [], []
    for k, v in kw.items():
        if isinstance(v, torch.Tensor):
            assert v.is_cuda, k
            if k not in OUTS:
                inputs.append((k, v, _bits(v).clone()))
            v = v.data_ptr()
        elif isinstance(v, np.ndarray):
            keep.append(v)
            v = v.ctypes.data
        setattr(a, k, v)
    _lib.check(_lib.lib().agpt_an_probe(C.byref(a), _lib.cur_stream() if stream else None))
    for k, v, before in inputs:
        assert torch.equal(_bits(v), before), f"{op}: input {k} was modified"


def ratio(y, ref, bound):
    """worst |y - ref| / bound; NaN in both is a match, NaN in one is a failure"""
    y, ref, bound = y.double(), ref.double(), bound.double()
    both = torch.isnan(y) & torch.isnan(ref)
    err = (y - ref).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    r = torch.where(both, torch.zeros_like(err), err / (bound + 1e-300))
    return float(r.max()) if r.numel() else 0.0


def passes(y, ref, bound):
    return ratio(y, ref, bound) <= 1.0


def check(tag, op, y, ref, bound):
    y, ref, bound = y.double(), ref.double().to(y.device), bound.double().to(y.device)
    w = ratio(y, ref, bound)
    print(f"{tag}: worst err/bound {w:.3f}")
    seen(op, w)
    if w > 1.0:
        err = torch.nan_to_num((y - ref).abs() / (bound + 1e-300), nan=math.inf)
        idx = np.unravel_index(int(torch.argmax(err).item()), tuple(y.shape))
        raise AssertionError(f"{tag}: error {w:.3g} x the bound at {idx}: got {float(y[idx])}, want {float(ref[idx])}")


def exact(tag, op, y, want):
    y, want = y.cpu(), want.cpu()
    assert y.shape == want.shape, (tag, y.shape, want.shape)
    bad = _bits(y) != _bits(want.to(y.dtype))
    if bad.any():
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError(f"{tag}: {int(bad.sum())} elements differ, first at {i}: got {y[i].item()!r}, "
                             f"want {want[i].item()!r}")
    print(f"{tag}: exact")
    seen(op)


def dev(t):
    return t.float().contiguous().to(DEV)


def rnd(shape, seed, scale=1.0, shift=0.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale + shift


def softmax_rel(E_s, n):
    """relative error bound of a softmax weight for scores off by at most E_s: e^(2 E_s) - 1, expf's 2 ulp (2^-22
    relative), the n-term sum and the division"""
    return torch.expm1(2 * E_s) + 2.0 ** -22 + gam(n) * U + U


# ================================================================================================ LASS_AFFINE
def affine_ref(x, s, t, vec, vec_off, rps, mutant=False):
    """a = x s + t and r = x + vec[b][vec_off + c] on x [rows][C] (fp64); (a, bound_a, r, bound_r).  mutant: the sample
    index taken from the float4 index without dividing by C4"""
    x64 = x.double()
    a = x64 * s.double() + t.double()
    rows, Cc = x.shape
    row = torch.arange(rows, device=x.device)
    if mutant:
        b = (row * (Cc // 4)).div(rps, rounding_mode="floor").clamp(max=vec.shape[0] - 1)
    else:
        b = row.div(rps, rounding_mode="floor")
    e = vec.double()[b][:, vec_off:vec_off + Cc]
    r = x64 + e
    tiny = 2.0 ** -149
    return a, U * a.abs() + tiny, r, U * r.abs() + tiny


def affine_inputs(rows, Cc, seed):
    x = rnd((rows, Cc), seed, 1.3)
    s = rnd((Cc,), seed + 1, 0.5, 1.0)
    t = rnd((Cc,), seed + 2, 0.3)
    return x, s, t


def lass_affine_shapes(W0):
    """(C, h-divisor, w, identity) of every affine pass the shipped UNet makes on a W0-wide input, per level"""
    enc = [c for _, c in specs.LASS_ENC]
    Ws = [W0]
    for _ in range(6):
        Ws.append(Ws[-1] // 2)
    out = []
    for k in range(6):
        if k > 0:
            out.append((enc[k - 1], 2 ** k, Ws[k], enc[k - 1] == enc[k]))     # encoder block 1 (cin = previous cout)
        out.append((enc[k], 2 ** k, Ws[k], True))                            # encoder block 2
        out.append((2 * enc[k], 2 ** k, Ws[k], False))                       # decoder conv_block2 (the concat)
        out.append((enc[k], 2 ** k, Ws[k], True))                            # decoder conv_block3 / after_conv_block1
    out.append((384, 64, Ws[6], True))                                       # conv_block7
    return sorted(set(out))


@gpu
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("Tp", [64, 128, 640])
def test_lass_affine(Tp, B):
    """every (C, h, w) the shipped LASSNet runs at F = 513 (T in {1, 63, 64} -> Tp 64, T 65 -> 128, T 626 -> 640);
    the residual on the identity blocks, each sample reading its own row of vec"""
    for Cc, div, W, ident in lass_affine_shapes(511):
        H = Tp // div
        rows = B * H * W
        x, s, t = affine_inputs(rows, Cc, Cc + H + W)
        vec_len, vec_off = 2 * Cc + 64, Cc + 32
        vec = rnd((B, vec_len), Cc + 7, 0.7)
        fa, a = out_f((rows, Cc))
        xd, vd = dev(x), dev(vec)
        kw = dict(x=xd, s=dev(s), t=dev(t), y=a, vec=vd, vec_len=vec_len, vec_off=vec_off, rows=rows,
                  rows_per_sample=H * W, C=Cc)
        if ident:
            fr, r = out_f((rows, Cc))
            kw["y2"] = r
        probe("LASS_AFFINE", **kw)
        written("LASS_AFFINE a", fa)
        ra, ba, rr, br = affine_ref(xd, dev(s), dev(t), vd, vec_off, H * W)
        check(f"LASS_AFFINE C={Cc} {H}x{W} B={B}", "LASS_AFFINE", a, ra, ba)
        if ident:
            written("LASS_AFFINE r", fr)
            check(f"LASS_AFFINE residual C={Cc} {H}x{W} B={B}", "LASS_AFFINE", r, rr, br)


# ================================================================================================ LASS_UPCOL
def upcol_ref(y, s, t, no_guard=False):
    """y [B][h][w][C] -> (col [B][h][w + 1][4][C], bound, zero mask) for taps (dh, dw) in (0,0), (0,-1), (-1,0),
    (-1,-1): relu(y s + t) at (m + dh, n + dw), zero outside the map.  no_guard: the mutant that reads past the row end
    (the next row's first pixel) at n + dw = w."""
    B, h, w, Cc = y.shape
    v = y.double() * s.double() + t.double()
    a = v.clamp(min=0)
    if no_guard:      # column w of row m is pixel (m + 1, 0) in the flat map (zero past the last row)
        nxt = torch.cat([a[:, 1:, :1], torch.zeros_like(a[:, :1, :1])], dim=1)
        ap = F.pad(torch.cat([a, nxt], dim=2).permute(0, 3, 1, 2), (1, 0, 1, 0)).permute(0, 2, 3, 1)
        vp = F.pad(torch.cat([v, nxt], dim=2).permute(0, 3, 1, 2), (1, 0, 1, 0)).permute(0, 2, 3, 1)
    else:
        ap = F.pad(a.permute(0, 3, 1, 2), (1, 1, 1, 0)).permute(0, 2, 3, 1)      # [B][h + 1][w + 2][C]
        vp = F.pad(v.permute(0, 3, 1, 2), (1, 1, 1, 0)).permute(0, 2, 3, 1)
    mp = F.pad(torch.ones(B, 1, h, w, dtype=torch.float64, device=y.device), (1, 1, 1, 0)).permute(0, 2, 3, 1)
    cols, bnds, msk = [], [], []
    for k in range(4):
        dh, dw = k >> 1, k & 1
        sl = (slice(None), slice(1 - dh, 1 - dh + h), slice(1 - dw, 1 - dw + w + 1))
        cols.append(ap[sl])
        bnds.append(U * vp[sl].abs() + 2.0 ** -149)
        msk.append(mp[sl].expand(-1, -1, -1, Cc))
    st = lambda L: torch.stack(L, dim=3)   # noqa: E731
    return st(cols), st(bnds), st(msk) == 0


def upcol_shapes():
    """(C_in, h, w) of the six decoder levels of the shipped UNet at F = 513 and Tp = 64 (levels 5 .. 0)"""
    dec = specs.LASS_DEC
    Ws = [511]
    for _ in range(6):
        Ws.append(Ws[-1] // 2)
    return [(dec[j][0], 64 >> (6 - j), Ws[6 - j]) for j in range(6)]


@gpu
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("hmul", [1, 2, 10])
def test_lass_upcol(hmul, B):
    for Cc, h, w in upcol_shapes():
        h = h * hmul
        y = rnd((B, h, w, Cc), Cc + h + w, 1.2)
        s, t = rnd((Cc,), Cc + 1, 0.5, 1.0), rnd((Cc,), Cc + 2, 0.4)
        flat, col = out_f((B, h, w + 1, 4, Cc))
        yd = dev(y)
        probe("LASS_UPCOL", x=yd, s=dev(s), t=dev(t), y=col, B=B, hh=h, ww=w, C=Cc)
        written("LASS_UPCOL", flat)
        ref, bound, zero = upcol_ref(yd, dev(s), dev(t))
        exact(f"LASS_UPCOL zeros C={Cc} {h}x{w} B={B}", "LASS_UPCOL", col[zero], torch.zeros_like(col[zero]))
        check(f"LASS_UPCOL C={Cc} {h}x{w} B={B}", "LASS_UPCOL", col, ref, bound)


# ================================================================================================ LASS_SHUFFLE
def shuffle_ref(up, skip, swap=False):
    """up [B][h][w + 1][4][C], skip [B][2h][2w + 1][C] -> cat [B][2h][2w + 1][2C]; swap: phase bits exchanged"""
    B, h, w1, _, Cc = up.shape
    r = torch.arange(2 * h, device=up.device)
    c = torch.arange(2 * w1 - 1, device=up.device)
    R, Cl = torch.meshgrid(r, c, indexing="ij")
    ph = (Cl & 1) * 2 + (R & 1) if swap else (R & 1) * 2 + (Cl & 1)
    main = up[:, R >> 1, Cl >> 1, ph]                       # [B][2h][2w + 1][C]
    return torch.cat([main, skip], dim=-1)


@gpu
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("hmul", [1, 2, 10])
def test_lass_shuffle(hmul, B):
    for (cin, h, w), (_, cout) in zip(upcol_shapes(), specs.LASS_DEC):
        h = h * hmul
        up = rnd((B, h, w + 1, 4, cout), cout + h + w)
        skip = rnd((B, 2 * h, 2 * w + 1, cout), cout + h + w + 1)
        flat, cat = out_f((B, 2 * h, 2 * w + 1, 2 * cout))
        ud, sd = dev(up), dev(skip)
        probe("LASS_SHUFFLE", x=ud, x2=sd, y=cat, B=B, hh=h, ww=w, C=cout)
        written("LASS_SHUFFLE", flat)
        exact(f"LASS_SHUFFLE C={cout} {h}x{w} B={B}", "LASS_SHUFFLE", cat, shuffle_ref(ud, sd))


# ================================================================================================ LASS_FILM
def film_tables(nouts, nins, njobs, vec_len, seed, with_jb):
    """random FiLM tables: output o has nins[o] inputs at a random hid slice; job j writes dst[j] (a permutation slice
    of vec), ja / jb random outputs (jb -1 for about half the jobs when with_jb, else always -1)"""
    g = torch.Generator().manual_seed(seed)
    nin = torch.tensor(nins, dtype=torch.int32)
    woff = torch.cumsum(torch.cat([torch.zeros(1, dtype=torch.int64), nin[:-1].long()]), 0).int()
    hid_len = int(max(nins)) + 40
    hoff = torch.randint(0, 41, (nouts,), generator=g).int()
    dst = torch.randperm(vec_len, generator=g)[:njobs].int()
    ja = torch.randint(0, nouts, (njobs,), generator=g).int()
    jb = torch.randint(0, nouts, (njobs,), generator=g).int()
    if with_jb:
        jb[torch.rand(njobs, generator=g) < 0.5] = -1
    else:
        jb[:] = -1
    b2 = torch.randn(nouts, generator=g) * 0.1
    alpha = torch.randn(njobs, generator=g) * 0.8
    beta = torch.randn(njobs, generator=g) * 0.2
    w2 = torch.randn(int(nin.sum()), generator=g) / math.sqrt(max(nins))
    return dict(woff=woff, hoff=hoff, nin=nin, dst=dst, ja=ja, jb=jb, b2=b2, alpha=alpha, beta=beta, w2=w2,
                hid_len=hid_len)


def film_ref(hid, T, vec_len, ignore_jb=False):
    """vec [B][vec_len] (NaN where no job writes) and its bound from hid [B][hid_len] and the tables T (fp64)"""
    B = hid.shape[0]
    nouts = T["nin"].numel()
    h64, w64 = hid.double().cpu(), T["w2"].double()
    f = torch.zeros(B, nouts, dtype=torch.float64)
    Ef = torch.zeros(B, nouts, dtype=torch.float64)
    for o in range(nouts):
        n, wo, ho = int(T["nin"][o]), int(T["woff"][o]), int(T["hoff"][o])
        w, hs = w64[wo:wo + n], h64[:, ho:ho + n]
        acc = hs @ w + float(T["b2"][o])
        f[:, o] = acc.clamp(min=0)
        Ef[:, o] = gam(n + 6) * U * ((hs.abs() @ w.abs()) + abs(float(T["b2"][o])))
    ja, jb = T["ja"].long(), T["jb"].long()
    al, be = T["alpha"].double(), T["beta"].double()
    v = al * f[:, ja] + be
    E = al.abs() * Ef[:, ja] + U * v.abs()
    use = (jb >= 0) & (not ignore_jb)
    jbc = jb.clamp(min=0)
    v = torch.where(use, v + f[:, jbc], v)
    E = torch.where(use, E + Ef[:, jbc] + U * v.abs(), E)
    out = torch.full((B, vec_len), float("nan"), dtype=torch.float64)
    bnd = torch.full((B, vec_len), math.inf, dtype=torch.float64)
    out[:, T["dst"].long()] = v
    bnd[:, T["dst"].long()] = E + 2.0 ** -149
    return out, bnd


FILM_NINS = [1, 31, 32, 33, 768]


@gpu
@pytest.mark.parametrize("with_jb", [False, True])
@pytest.mark.parametrize("nin", FILM_NINS + ["mixed"])
@pytest.mark.parametrize("B", [1, 3])
def test_lass_film(nin, with_jb, B):
    """njobs * B not a multiple of the 8 warps of a block; vec entries no job writes keep their value"""
    nouts, njobs, vec_len = 13, 37, 44
    nins = [FILM_NINS[o % 5] for o in range(nouts)] if nin == "mixed" else [nin] * nouts
    T = film_tables(nouts, nins, njobs, vec_len, 50 + B + len(nins) + (nin if nin != "mixed" else 7), with_jb)
    hid = torch.relu(rnd((B, T["hid_len"]), 60 + B, 1.0))
    flat, vec = out_f((B, vec_len), fill=SENT)
    i32 = lambda k: T[k].to(DEV)   # noqa: E731
    probe("LASS_FILM", x=dev(hid), w2=dev(T["w2"]), woff=i32("woff"), hoff=i32("hoff"), nin=i32("nin"), b2=dev(T["b2"]),
          dst=i32("dst"), ja=i32("ja"), jb=i32("jb"), alpha=dev(T["alpha"]), beta=dev(T["beta"]), y=vec, nj=njobs, B=B,
          hid_len=T["hid_len"], vec_len=vec_len)
    n = B * vec_len
    assert torch.equal(flat[n:], torch.full_like(flat[n:], CANARY)), "LASS_FILM: written past the end of vec"
    ref, bound = film_ref(hid, T, vec_len)
    v = vec.cpu()
    hole = torch.isnan(ref)
    assert torch.all(v[hole] == SENT), "LASS_FILM: an entry no job writes changed"
    assert not torch.any(v[~hole] == SENT), "LASS_FILM: a job's entry was not written"
    check(f"LASS_FILM nin={nin} jb={with_jb} B={B}", "LASS_FILM", v[~hole], ref[~hole], bound[~hole])


# ================================================================================================ LASS handle ops
@pytest.fixture(scope="module")
def lass():
    """the small LASSNet (its UNet is the shipped one) with its handle built; (handle, fp64 state dict)"""
    from audiogpt_b200.sound_extraction.model.LASSNet import LASSNet
    m = LASSNet.from_config(specs.LASS_SMALL)
    m.load_state_dict(specs.synth_lass(specs.LASS_SMALL, 6060), strict=True)
    m = m.to(DEV).eval()
    m._ensure(torch.device(DEV))
    sd = {k: v.detach().double() for k, v in m.state_dict().items() if v.is_floating_point()}
    return m, sd


def lass_blocks(sd):
    """the ConvBlockResCond prefixes in forward order"""
    ps = []
    for i in range(len(specs.LASS_ENC)):
        ps += [f"UNet.encoder_block{i + 1}.conv_block1", f"UNet.encoder_block{i + 1}.conv_block2"]
    ps.append("UNet.conv_block7")
    for j in range(len(specs.LASS_DEC)):
        ps += [f"UNet.decoder_block{j + 1}.conv_block2", f"UNet.decoder_block{j + 1}.conv_block3"]
    ps.append("UNet.after_conv_block1")
    return ps


def film_vec_ref(sd, cond):
    """the FiLM vector [B][vec_len] in the documented layout and its bound (module docstring)"""
    import test_tapconv_gpu as tg
    c64 = cond.double().cpu()
    sd = {k: v.cpu() for k, v in sd.items()}
    vals, bnds = [], []

    def film(p):
        w1, b1 = sd[p + ".linear.0.weight"], sd[p + ".linear.0.bias"]
        w2, b2 = sd[p + ".linear.2.weight"], sd[p + ".linear.2.bias"]
        acc = c64 @ w1.T
        S = c64.abs() @ w1.abs().T
        n = tg.n_products({"kind": 0}, w1.shape[1], 1, True)
        E = tg.c_const(n, True) * tg.U * S + tg.FLOOR * w1.abs().sum(1) + \
            tg.FLOOR * tg.w_floor_scale(w1) * c64.abs().sum(1, keepdim=True)
        hb = acc + b1
        E = E + U * (acc.abs() + hb.abs())                      # the epilogue's bias add and the GEMM's fp32 store
        hid = hb.clamp(min=0)
        o = hid @ w2.T + b2
        Eo = gam(w2.shape[1] + 6) * U * (hid.abs() @ w2.abs().T + b2.abs()) + E @ w2.abs().T
        return o.clamp(min=0), Eo

    for p in lass_blocks(sd):
        f1, E1 = film(p + ".film1")
        g, be, rm, rv = (sd[p + ".bn2." + k] for k in ("weight", "bias", "running_mean", "running_var"))
        s2 = g / torch.sqrt(rv + 1e-5)
        t2 = be - rm * s2
        e1 = s2 * f1 + t2
        Ee = s2.abs() * E1 + 6 * U * (s2.abs() * f1.abs() + be.abs() + (rm * s2).abs()) + U * e1.abs()
        f2, E2 = film(p + ".film2")
        if p + ".shortcut.weight" in sd:
            fr, Er = film(p + ".film_res")
            r2 = f2 + fr
            Er2 = E2 + Er + U * r2.abs()
        else:
            r2, Er2 = f2, E2 + U * f2.abs()
        vals += [e1, r2]
        bnds += [Ee, Er2]
    return torch.cat(vals, 1), torch.cat(bnds, 1) * (1 + 1e-6) + 2.0 ** -140


@gpu
@pytest.mark.parametrize("B", [1, 3])
def test_lass_film_vec(lass, B):
    m, sd = lass
    h = m._engine.h.value
    info = np.full(2, -1, dtype=np.int32)
    probe("LASS_FILM_VEC", h=h, info=info, B=B)                     # y null: only vec_len
    vec_len = int(info[0])
    want_len = sum(2 * sd[p + ".conv1.weight"].shape[0] for p in lass_blocks(sd))
    assert vec_len == want_len, (vec_len, want_len)
    cond = torch.relu(rnd((B, 256), 80 + B, 1.0))
    flat, vec = out_f((B, vec_len))
    probe("LASS_FILM_VEC", h=h, x=dev(cond), y=vec, info=info, B=B)
    written("LASS_FILM_VEC", flat)
    ref, bound = film_vec_ref(sd, cond)
    check(f"LASS_FILM_VEC B={B}", "LASS_FILM_VEC", vec.cpu(), ref, bound)


def up_ref(sd, j, y, skip):
    """decoder_block{j + 1}: relu(bn1(y)) -> ConvTranspose2d(3, stride 2) -> [:, :, :-1, :] -> cat skip, on channels-
    last y [B][h][w][cin]; (ref [B][2h][2w + 1][2 cout], bound)"""
    import test_tapconv_gpu as tg
    p = f"UNet.decoder_block{j + 1}"
    W = sd[p + ".conv1.weight"]
    g, be, rm, rv = (sd[p + ".bn1." + k] for k in ("weight", "bias", "running_mean", "running_var"))
    s = g / torch.sqrt(rv + 1e-5)
    x = y.double().permute(0, 3, 1, 2)
    v = (x - rm[:, None, None]) * s[:, None, None] + be[:, None, None]
    a = v.clamp(min=0)
    Ea = U * v.abs() + 6 * U * ((x * s[:, None, None]).abs() + be.abs()[:, None, None] + (rm * s).abs()[:, None, None])
    ct = lambda inp, w: F.conv_transpose2d(inp, w, stride=2)[:, :, :-1, :]   # noqa: E731
    z = ct(a, W)
    n = tg.n_products({"kind": 0}, 4 * W.shape[0], 1, True)
    E = tg.c_const(n, True) * tg.U * ct(a.abs(), W.abs()) + tg.FLOOR * ct(torch.ones_like(a), W.abs()) + \
        tg.FLOOR * tg.w_floor_scale(W) * ct(a.abs(), torch.ones_like(W)) + ct(Ea, W.abs()) + U * z.abs()
    ref = torch.cat([z.permute(0, 2, 3, 1), skip.double()], dim=-1)
    bound = torch.cat([E.permute(0, 2, 3, 1), torch.zeros_like(skip, dtype=torch.float64)], dim=-1)
    return ref, bound * (1 + 1e-6) + 2.0 ** -140


@gpu
@pytest.mark.parametrize("B", [1, 2])
def test_lass_up(lass, B):
    """all six decoder levels of the shipped shape (F = 513, Tp = 64), the deepest the 7 -> 15 column one"""
    m, sd = lass
    h_ = m._engine.h.value
    for level in range(6):
        j = 5 - level
        cin, cout = specs.LASS_DEC[j]
        _, h, w = upcol_shapes()[j]
        y = rnd((B, h, w, cin), 90 + level, 1.0)
        skip = rnd((B, 2 * h, 2 * w + 1, cout), 91 + level)
        yd, sk = y.to(DEV).float(), skip.to(DEV).float()
        flat, cat = out_f((B, 2 * h, 2 * w + 1, 2 * cout))
        info = np.full(1, -1, dtype=np.int32)
        probe("LASS_UP", h=h_, level=level, x=yd, x2=sk, y=cat, info=info, B=B, hh=h, ww=w)
        written("LASS_UP", flat)
        ref, bound = up_ref({k: v.to(DEV) for k, v in sd.items() if k.startswith(f"UNet.decoder_block{j + 1}.")},
                            j, yd, sk)
        exact(f"LASS_UP skip half level={level}", "LASS_UP", cat[..., cout:], sk)
        check(f"LASS_UP level={level} {h}x{w} -> {2 * h}x{2 * w + 1} B={B}", "LASS_UP", cat, ref, bound)


@gpu
def test_lass_up_refuses_a_level_outside_the_decoder(lass):
    m, _ = lass
    for level in (-1, 6):
        with pytest.raises(RuntimeError, match=r"\[0, 6\)"):
            probe("LASS_UP", h=m._engine.h.value, level=level, B=1, hh=1, ww=7)


# ================================================================================================ TSD_PAD4
@gpu
@pytest.mark.parametrize("n", [1, 64, 64 * 333 + 5, 4096 * 256 + 37])
def test_tsd_pad4(n):
    x = rnd((n,), n)
    flat, y = out_f((n, 4))
    probe("TSD_PAD4", x=dev(x), y=y, rows=n)
    written("TSD_PAD4", flat)
    want = torch.zeros(n, 4)
    want[:, 0] = x
    exact(f"TSD_PAD4 n={n}", "TSD_PAD4", y, want)


# ================================================================================================ TSD_FUSE
def fuse_ref(f2, e1, n):
    """Fusion's AvgPool1d(n) of e1 * f2 (tsd_ref.fusion after the two ReLU'd convs): [B][Td][C n], [B][C n] -> [B][Td][C]"""
    B, Td, CN = f2.shape
    p = (f2.double() * e1.double()[:, None]).view(B, Td, CN // n, n)
    S = (f2.double() * e1.double()[:, None]).abs().view(B, Td, CN // n, n).sum(-1)
    out = p.mean(-1)
    return out, gam(n) * U * S + U * out.abs() + 2.0 ** -149


@gpu
@pytest.mark.parametrize("n", [1, 2, 4, 7])
@pytest.mark.parametrize("B,Td,Cc", [(1, 1, 512), (3, 62, 512), (3, 1000, 512), (2, 5, 3)])
def test_tsd_fuse(B, Td, Cc, n):
    f2 = torch.relu(rnd((B, Td, Cc * n), B + Td + n))
    e1 = torch.relu(rnd((B, Cc * n), B + Td + n + 1))
    flat, y = out_f((B, Td, Cc))
    probe("TSD_FUSE", x=dev(f2), x2=dev(e1), y=y, B=B, Td=Td, C=Cc, n=n)
    written("TSD_FUSE", flat)
    ref, bound = fuse_ref(f2, e1, n)
    check(f"TSD_FUSE B={B} Td={Td} C={Cc} n={n}", "TSD_FUSE", y.cpu(), ref, bound)


# ================================================================================================ TSD_REFEMB
def refemb_ref(E, att_pool, qw, qb, kw, kb, temp=TEMP):
    """RaDur_fusion's reference embedding on E [B][Trr][128] (the bn'd rows when att_pool): mean, or
    bmm(get_w(q, k, mean, E), E); (ref [B][128], bound).  temp: the mutant's temperature."""
    E64 = E.double()
    B, Trr, _ = E.shape
    m = E64.mean(1)
    Em = gam(Trr) * U * E64.abs().mean(1) + U * m.abs()
    if not att_pool:
        return m, Em + 2.0 ** -149
    # the attention starts from the kernel's own mean, reproduced exactly (a sequential fp32 sum, then / Trr); the
    # mean itself is gated against fp64 by the att_pool = 0 cases
    m32 = np.add.accumulate(E.float().cpu().numpy(), axis=1, dtype=np.float32)[:, -1] / np.float32(Trr)
    m = torch.from_numpy(m32.astype(np.float64)).to(E.device)
    qw, qb, kw, kb = (v.double().to(E.device) for v in (qw, qb, kw, kb))
    q = m @ qw.T + qb
    Eq = gam(129) * U * (m.abs() @ qw.abs().T + qb.abs())
    k = E64 @ kw.T + kb                                     # Linear k on every row
    sc = torch.einsum("bo,bto->bt", q, k) / temp
    u_ = q @ kw                                             # the kernel's folded kw^T q
    Eu = gam(128) * U * (q.abs() @ kw.abs()) + Eq @ kw.abs()
    qkb = q @ kb
    Eqb = gam(160) * U * (q.abs() @ kb.abs()) + Eq @ kb.abs()
    acc = torch.einsum("bc,btc->bt", u_, E64)
    Eacc = gam(129) * U * (torch.einsum("bc,btc->bt", u_.abs(), E64.abs()) + qkb.abs()[:, None]) + \
        torch.einsum("bc,btc->bt", Eu, E64.abs()) + Eqb[:, None]
    Es = Eacc / TEMP + U * sc.abs()
    p = torch.softmax(sc, dim=1)
    rel = softmax_rel(Es.max(1, keepdim=True).values, Trr)
    emb = torch.einsum("bt,btc->bc", p, E64)
    Ee = torch.einsum("bt,btc->bc", p * rel, E64.abs()) + gam(Trr) * U * torch.einsum("bt,btc->bc", p, E64.abs())
    return emb, Ee * (1 + 1e-6) + 2.0 ** -149


def refemb_inputs(B, Trr, seed):
    E = rnd((B, Trr, 128), seed, 1.0, 0.2)
    g = torch.Generator().manual_seed(seed + 1)
    qw, kw = (torch.randn(128, 128, generator=g) / math.sqrt(128) for _ in range(2))
    qb, kb = (torch.randn(128, generator=g) * 0.1 for _ in range(2))
    return E, qw, qb, kw, kb


@gpu
@pytest.mark.parametrize("att_pool", [0, 1])
@pytest.mark.parametrize("B,Trr", [(1, 1), (3, 2), (3, 62), (2, 11872), (2, 11873), (1, 131072)])
def test_tsd_refemb(B, Trr, att_pool):
    """Trr 11873 and 131072 kept their scores in more than the 48 KB of shared memory a launch allows by default"""
    E, qw, qb, kw, kb = refemb_inputs(B, Trr, Trr + B)
    Ed = dev(E)
    flat, y = out_f((B, 128))
    fs, scr = out_f((B, Trr))
    probe("TSD_REFEMB", x=Ed, w=dev(qw), b=dev(qb), w2=dev(kw), b2=dev(kb), scratch=scr if att_pool else None, y=y,
          B=B, T=Trr, att_pool=att_pool)
    written("TSD_REFEMB", flat)
    ref, bound = refemb_ref(Ed, att_pool, qw, qb, kw, kb)
    check(f"TSD_REFEMB att_pool={att_pool} B={B} Trr={Trr}", "TSD_REFEMB", y, ref, bound)


# ================================================================================================ TSD_HEAD
def head_ref(h, w, b, drop_last=False):
    """softmax(h w^T + b) over O (detect's fc -> outputlayer -> softmax, folded); drop_last: the mutant that
    normalises over O - 1 outputs"""
    z = h.double() @ w.double().T + b.double()
    Ez = gam(1030) * U * (h.double().abs() @ w.double().abs().T + b.double().abs())
    O = w.shape[0]
    if drop_last and O > 1:
        e = torch.exp(z - z.max(1, keepdim=True).values)
        p = e / e[:, :O - 1].sum(1, keepdim=True)
    else:
        p = torch.softmax(z, dim=1)
    rel = softmax_rel(Ez.max(1, keepdim=True).values, O)
    return p, p * rel * (1 + 1e-6) + 2.0 ** -149


@gpu
@pytest.mark.parametrize("O", [1, 2, 16])
@pytest.mark.parametrize("rows", [1, 7, 9, 1003])
def test_tsd_head(rows, O):
    h = torch.tanh(rnd((rows, 1024), rows + O))
    w = rnd((O, 1024), rows + O + 1, 0.08)
    b = rnd((O,), rows + O + 2, 0.3)
    flat, p = out_f((rows, O))
    probe("TSD_HEAD", x=dev(h), w=dev(w), b=dev(b), y=p, O=O, rows=rows)
    written("TSD_HEAD", flat)
    ref, bound = head_ref(h, w, b)
    check(f"TSD_HEAD rows={rows} O={O}", "TSD_HEAD", p.cpu(), ref, bound)


# ================================================================================================ TSD_MIX_INTERP
def mix_interp_ref(p1, p2, wmix, T, mutant=None):
    """fin = p1 (1 - w) + w p2 (RaDur_fusion.forward's two-pass mix), decision = fin[..., 0], up = tsd_ref.interpolate
    (fin, T) in fp64; (decision, bound, up, bound).  mutant: 'unclamped' (i1 = i0 + 1 even at the last frame, reading
    the next row of the flat array) or 'align' (the align_corners=True scale)."""
    B, Td, O = p1.shape
    p1d = p1.double()
    if p2 is None:
        fin, Ef = p1d, torch.zeros_like(p1d)
    else:
        w = wmix.double()[:, None, None]
        a, c = p1d * (1 - w), w * p2.double()
        fin = a + c
        Ef = U * (p1d.abs() * (1 - w).abs() + a.abs() + c.abs() + fin.abs())
    dec, Edec = fin[..., 0], Ef[..., 0]
    t = torch.arange(T, dtype=torch.float64)
    if mutant == "align":
        src = t * ((Td - 1) / (T - 1) if T > 1 else 0.0)
    else:
        src = ((Td / T) * (t + 0.5) - 0.5).clamp(min=0)
    i0 = src.floor().long().clamp(max=Td - 1)
    l1 = src - i0.double()
    if mutant == "unclamped":
        flat = torch.cat([fin.reshape(B * Td, O), torch.zeros(1, O, dtype=torch.float64)])
        i1 = i0 + 1
        rows = (torch.arange(B)[:, None] * Td + i1[None]).clamp(max=B * Td)
        f1 = flat[rows]
    else:
        i1 = (i0 + 1).clamp(max=Td - 1)
        f1 = fin[:, i1]
    f0 = fin[:, i0]
    up = (1 - l1)[None, :, None] * f0 + l1[None, :, None] * f1
    if mutant:
        return dec, None, up, None
    # the fp32 source index's rounding times the largest slope of the segments around it
    fp = torch.cat([fin[:, :1], fin, fin[:, -1:]], dim=1)          # fin[-1] = fin[0], fin[Td] = fin[Td - 1]
    slope = torch.maximum((fp[:, i0 + 1] - fp[:, i0]).abs(), (fp[:, i0 + 2] - fp[:, i0 + 1]).abs())
    slope = torch.maximum(slope, (fp[:, (i0 + 3).clamp(max=Td + 1)] - fp[:, i0 + 2]).abs())
    Esrc = 3 * U * ((Td / T) * (t + 0.5) + 1)
    l0 = (1 - l1)[None, :, None]
    Eup = l0 * Ef[:, i0] + l1[None, :, None] * Ef[:, i1] + slope * Esrc[None, :, None] + \
        U * (f0.abs() + (l0 * f0).abs() + (l1[None, :, None] * f1).abs() + up.abs())
    return dec, Edec * (1 + 1e-6) + 2.0 ** -149, up, Eup * (1 + 1e-6) + 2.0 ** -149


def probs(B, Td, O, seed):
    """per-frame class probabilities (uniform in [0, 1) when O = 1, where a softmax would be the constant 1)"""
    if O == 1:
        return torch.rand(B, Td, 1, generator=torch.Generator().manual_seed(seed))
    return torch.softmax(rnd((B, Td, O), seed, 2.0), dim=2)


MIX_CASES = [(1, 1, 7), (3, 1, 501), (3, 148, 149), (1, 62, 501), (3, 62, 1000), (3, 125, 1000), (3, 125, 4001),
             (3, 500, 501), (2, 500, 4001), (3, 500, 30000)]


@gpu
@pytest.mark.parametrize("two_pass", [False, True])
@pytest.mark.parametrize("O", [1, 2, 16])
@pytest.mark.parametrize("B,Td,T", MIX_CASES)
def test_tsd_mix_interp(B, Td, T, O, two_pass):
    """Td = 1; Td = T - 1 (time_resolution 'other', no time pooling: T = 149 gives Td = 148); Td 62 / 125 / 500 against
    T 501 / 1000 / 4001; and B T O past the grid-stride cap of 4096 blocks of 256"""
    p1 = probs(B, Td, O, Td + T + O)
    p2 = probs(B, Td, O, Td + T + O + 1) if two_pass else None
    wm = torch.tensor([0.0, 0.37, 0.5][:B] + [0.21] * max(0, B - 3))[:B]
    fd, dec = out_f((B, Td))
    fu, up = out_f((B, T, O))
    probe("TSD_MIX_INTERP", x=dev(p1), x2=dev(p2) if two_pass else None, vec=dev(wm), y=dec, y2=up, B=B, Td=Td, T=T,
          O=O)
    written("TSD_MIX_INTERP decision", fd)
    written("TSD_MIX_INTERP up", fu)
    rd, bd, ru, bu = mix_interp_ref(p1, p2, wm, T)
    tag = f"TSD_MIX_INTERP B={B} Td={Td} T={T} O={O} two_pass={two_pass}"
    check(tag + " decision", "TSD_MIX_INTERP", dec.cpu(), rd, bd)
    check(tag, "TSD_MIX_INTERP", up.cpu(), ru, bu)


def test_mix_interp_reference_is_atens():
    """the float64 reference interpolation agrees with tsd_ref.interpolate (F.interpolate linear, align_corners=False)"""
    from oracle import tsd_ref
    for Td, T in ((1, 7), (62, 501), (148, 149), (125, 4001)):
        p = probs(2, Td, 3, Td + T).double()
        _, _, up, _ = mix_interp_ref(p, None, None, T)
        assert torch.allclose(up, tsd_ref.interpolate(p, T), rtol=0, atol=1e-12), (Td, T)


# ================================================================================================ CLAP_EMBED(_TYPED)
def embed_inputs(N, L, H, vocab, ntypes, seed):
    g = torch.Generator().manual_seed(seed)
    word = torch.randn(vocab, H, generator=g)
    pos = torch.randn(L, H, generator=g)
    types = torch.randn(ntypes, H, generator=g)
    ids = torch.randint(0, vocab, (N, L), generator=g, dtype=torch.int32)
    edge = torch.tensor([-1, 0, vocab - 1, vocab, -(2 ** 31), 2 ** 31 - 1], dtype=torch.int32)
    k = min(edge.numel(), N * L)
    ids.view(-1)[:k] = edge[:k]
    tids = torch.randint(0, ntypes, (N, L), generator=g, dtype=torch.int32)
    tedge = torch.tensor([-1, ntypes, 5, 0], dtype=torch.int32)
    k = min(tedge.numel(), N * L)
    tids.view(-1)[-k:] = tedge[:k]
    mask = torch.ones(N, L, dtype=torch.int32)
    if L > 4:
        mask[:, L // 3:L // 2] = 0                           # padding in the middle
        mask[0, -2:] = 0
        mask[-1, 1] = 7                                     # nonzero but not 1: a real token
    return word, pos, types, ids, tids, mask


def embed_ref(word, pos, types, ids, tids, vocab, ntypes, assoc="left"):
    """BertEmbeddings in fp32 (torch's order): (word[id] + type[tid]) + pos[l]; assoc 'right': the mutant"""
    w = word[ids.long().clamp(0, vocab - 1)]
    t = types[tids.long().clamp(0, ntypes - 1)]
    p = pos[None, : ids.shape[1]]
    return (w + t) + p if assoc == "left" else w + (t + p)


EMB_CASES = [(2, 1, 256), (3, 77, 768), (2, 77, 100), (1, 512, 256), (2, 512, 100)]


@gpu
@pytest.mark.parametrize("N,L,H", EMB_CASES)
def test_clap_embed(N, L, H):
    vocab = 1000
    word, pos, types, ids, tids, _ = embed_inputs(N, L, H, vocab, 2, N + L + H)
    flat, x = out_f((N, L, H))
    probe("CLAP_EMBED", ids=ids.to(DEV), w=dev(word), x=dev(pos), x2=dev(types[0]), y=x, N=N, L=L, H=H, vocab=vocab)
    written("CLAP_EMBED", flat)
    exact(f"CLAP_EMBED N={N} L={L} H={H}", "CLAP_EMBED", x, embed_ref(word, pos, types, ids, torch.zeros_like(ids),
                                                                      vocab, 2))


@gpu
@pytest.mark.parametrize("N,L,H", EMB_CASES)
def test_clap_embed_typed(N, L, H):
    vocab, ntypes = 1000, 2
    word, pos, types, ids, tids, mask = embed_inputs(N, L, H, vocab, ntypes, N + L + H + 1)
    flat, x = out_f((N, L, H))
    kpm = torch.full((N * L + GUARD,), 0xA5, dtype=torch.uint8, device=DEV)
    probe("CLAP_EMBED_TYPED", ids=ids.to(DEV), type_ids=tids.to(DEV), mask=mask.to(DEV), w=dev(word), x=dev(pos),
          x2=dev(types), y=x, kpm=kpm, N=N, L=L, H=H, vocab=vocab, ntypes=ntypes)
    written("CLAP_EMBED_TYPED", flat)
    exact(f"CLAP_EMBED_TYPED N={N} L={L} H={H}", "CLAP_EMBED_TYPED", x,
          embed_ref(word, pos, types, ids, tids, vocab, ntypes))
    k = kpm.cpu()
    assert torch.all(k[N * L:] == 0xA5), "CLAP_EMBED_TYPED: kpm written past its end"
    assert torch.equal(k[:N * L].view(N, L), (mask == 0).to(torch.uint8)), "the key-padding mask must be mask == 0"


# ================================================================================================ CLAP_GELU
def gelu_ref(x):
    """fp64 erf-GELU and the bound of the kernel's 0.5 x (1 + erff(x fl(1 / sqrt 2)))"""
    x = x.double()
    z = x / math.sqrt(2)
    e = torch.erf(z)
    y = 0.5 * x * (1 + e)
    Ez = 2 * U * z.abs()
    Ee = (2 / math.sqrt(math.pi)) * torch.exp(-(z.abs() - Ez).clamp(min=0) ** 2) * Ez + 2 * 2.0 ** -23 * e.abs().clamp(
        min=2.0 ** -126)
    E = 0.5 * x.abs() * (Ee + U * (1 + e).abs()) + 2 * U * y.abs()
    return y, E * (1 + 1e-6) + 2.0 ** -149


@gpu
@pytest.mark.parametrize("max_blocks", [2368, 4096, 1])
@pytest.mark.parametrize("n", [1, 1000, 2368 * 256 + 1, 4096 * 256 + 77])
def test_clap_gelu(n, max_blocks):
    x = rnd((n,), n, 3.0)
    x[: min(n, 4)] = torch.tensor([-12.0, -9.5, 6.0, 1e-30][: min(n, 4)])
    flat, y = out_f((n,))
    probe("CLAP_GELU", x=dev(x), y=y, rows=n, max_blocks=max_blocks)
    written("CLAP_GELU", flat)
    ref, bound = gelu_ref(x)
    check(f"CLAP_GELU n={n} max_blocks={max_blocks}", "CLAP_GELU", y.cpu(), ref, bound)


@gpu
def test_clap_gelu_special_values_match_torch():
    x = torch.tensor([0.0, -0.0, math.inf, -math.inf, math.nan])
    flat, y = out_f((x.numel(),), fill=SENT)
    probe("CLAP_GELU", x=dev(x), y=y, rows=x.numel(), max_blocks=4096)
    written("CLAP_GELU special", flat, fill=SENT)
    want = F.gelu(x.to(DEV)).cpu()
    got = y.cpu()
    for i in range(x.numel()):
        g_, w_ = got[i].item(), want[i].item()
        same = (math.isnan(g_) and math.isnan(w_)) or (g_ == w_ and math.copysign(1, g_) == math.copysign(1, w_))
        assert same, f"CLAP_GELU({x[i].item()}): kernel {g_!r}, torch fp32 F.gelu {w_!r}"
    seen("CLAP_GELU")


# ================================================================================================ EMO_MEAN_NORM
def mean_norm_ref(h):
    """embed_utterance: raw = mean over the partials, raw / ||raw|| (inference.py:150-151); (ref [256], bound)"""
    h = h.double()
    N = h.shape[0]
    raw = h.mean(0)
    Er = gam(N) * U * h.abs().mean(0) + U * raw.abs()
    n2 = (raw * raw).sum()
    En2 = (2 * raw.abs() * Er + Er ** 2).sum() + (U + gam(264) * U) * n2
    nrm = n2.sqrt()
    En = En2 / (2 * nrm) + 2.0 ** -23 * nrm
    y = raw / nrm
    return y, (Er / nrm + raw.abs() * En / nrm ** 2 + U * y.abs()) * (1 + 1e-6) + 2.0 ** -149


def unit_rows(N, seed):
    h = torch.relu(rnd((N, 256), seed))
    return h / h.norm(dim=1, keepdim=True)


@gpu
@pytest.mark.parametrize("N", [1, 2, 10, 1000])
def test_emo_mean_norm(N):
    h = unit_rows(N, N)
    flat, y = out_f((256,))
    probe("EMO_MEAN_NORM", x=dev(h), y=y, N=N)
    written("EMO_MEAN_NORM", flat)
    ref, bound = mean_norm_ref(h.float())
    check(f"EMO_MEAN_NORM N={N}", "EMO_MEAN_NORM", y.cpu(), ref, bound)


# ================================================================================================ EMO_LINEAR_NORM
def linear_norm_ref(h, W, b, norm_first=False):
    """EmotionEncoder.forward's tail: relu(Linear(h)) / ||.|| (model.py:56-59); (ref [N][E], bound).  norm_first: the
    mutant that normalises before the ReLU"""
    h, W, b = h.double(), W.double(), b.double()
    acc = h @ W.T + b
    Ea = gam(257) * U * (h.abs() @ W.abs().T + b.abs())
    if norm_first:
        y = (acc / acc.norm(dim=1, keepdim=True)).clamp(min=0)
        return y, None
    r = acc.clamp(min=0)
    E = r.shape[1]
    n2 = (r * r).sum(1, keepdim=True)
    En2 = (2 * r.abs() * Ea + Ea ** 2).sum(1, keepdim=True) + (U + gam(E // 256 + 14) * U) * n2
    nrm = n2.sqrt()
    En = En2 / (2 * nrm) + 2.0 ** -23 * nrm
    y = r / nrm
    return y, (Ea / nrm + r.abs() * En / nrm ** 2 + U * y.abs()) * (1 + 1e-6) + 2.0 ** -149


def linear_norm_inputs(N, E, seed):
    h = torch.tanh(rnd((N, 256), seed))
    h[0] = 0.0                                              # with a non-positive bias: an all-zero ReLU row
    W = rnd((E, 256), seed + 1, 1 / 16)
    b = -rnd((E,), seed + 2, 0.1).abs()
    return h, W, b


@gpu
@pytest.mark.parametrize("N", [1, 74])
@pytest.mark.parametrize("E", [1, 255, 256, 257])
def test_emo_linear_norm(E, N):
    h, W, b = linear_norm_inputs(N, E, E + N)
    flat, y = out_f((N, E), fill=SENT)
    probe("EMO_LINEAR_NORM", x=dev(h), w=dev(W), b=dev(b), y=y, N=N, E=E)
    written("EMO_LINEAR_NORM", flat, fill=SENT)
    ref, bound = linear_norm_ref(h, W, b)
    assert torch.isnan(ref[0]).all(), "row 0 is the 0 / 0 case"
    check(f"EMO_LINEAR_NORM E={E} N={N}", "EMO_LINEAR_NORM", y.cpu(), ref, bound)


# ================================================================================================ preconditions (no device)
def _refused(op, match, **kw):
    with pytest.raises(RuntimeError, match=match):
        probe(op, stream=False, **kw)


FAKE = 256      # a non-null device address that is never dereferenced: the check throws first


def test_probe_refuses_lass_shapes_it_cannot_index():
    _refused("LASS_AFFINE", r"C % 4", rows=4, rows_per_sample=1, C=6)
    _refused("LASS_AFFINE", r"rows >= 1", rows=0, rows_per_sample=1, C=8)
    _refused("LASS_AFFINE", r"rows_per_sample >= 1", rows=4, rows_per_sample=0, C=8)
    _refused("LASS_AFFINE", r"must fit in vec_len", y2=FAKE, rows=4, rows_per_sample=1, C=8, vec_len=16, vec_off=12)
    _refused("LASS_AFFINE", r"must fit in vec_len", y2=FAKE, rows=4, rows_per_sample=1, C=8, vec_len=16, vec_off=-4)
    _refused("LASS_AFFINE", r"multiples of 4", y2=FAKE, rows=4, rows_per_sample=1, C=8, vec_len=18, vec_off=2)
    for op in ("LASS_UPCOL", "LASS_SHUFFLE"):
        _refused(op, r"C % 4", B=1, hh=2, ww=3, C=10)
        _refused(op, r"B, h, w >= 1", B=1, hh=0, ww=3, C=8)
        _refused(op, r"B, h, w >= 1", B=1, hh=2, ww=0, C=8)
    _refused("LASS_FILM", r"nj, B, hid_len, vec_len >= 1", nj=0, B=1, hid_len=4, vec_len=4)


def test_probe_refuses_a_lass_handle_op_without_a_lass_handle():
    _refused("LASS_UP", "invalid handle", level=0, B=1, hh=1, ww=7)
    _refused("LASS_FILM_VEC", "invalid handle", B=1)


def test_probe_refuses_tsd_shapes_it_cannot_index():
    _refused("TSD_PAD4", r"n >= 1", rows=0)
    _refused("TSD_FUSE", r"n >= 1", B=1, Td=4, C=8, n=0)
    _refused("TSD_FUSE", r"B, Td, C >= 1", B=1, Td=0, C=8, n=2)
    _refused("TSD_REFEMB", r"Trr >= 1", B=1, T=0, att_pool=0)
    _refused("TSD_REFEMB", r"score scratch", B=1, T=10, att_pool=1)
    for O in (0, 17):
        _refused("TSD_HEAD", r"1 <= O <= 16", O=O, rows=4)
        _refused("TSD_MIX_INTERP", r"1 <= O <= 16", B=1, Td=4, T=8, O=O)
    _refused("TSD_MIX_INTERP", r"B, Td, T >= 1", B=1, Td=0, T=8, O=1)
    _refused("TSD_MIX_INTERP", r"B, Td, T >= 1", B=1, Td=4, T=0, O=1)


def test_probe_refuses_empty_embedding_tables_and_rows():
    for k in ("vocab", "H", "L"):
        args = dict(N=1, L=4, H=8, vocab=10, ntypes=2)
        args[k] = 0
        _refused("CLAP_EMBED", r"vocab, H, L, N >= 1", **args)
        _refused("CLAP_EMBED_TYPED", r"vocab, ntypes, H, L, N >= 1", **args)
    _refused("CLAP_EMBED_TYPED", r"vocab, ntypes, H, L, N >= 1", N=1, L=4, H=8, vocab=10, ntypes=0)
    _refused("CLAP_GELU", r"n >= 1", rows=0, max_blocks=4096)
    _refused("CLAP_GELU", r"max_blocks >= 1", rows=10, max_blocks=0)


def test_probe_refuses_emotion_tails_it_cannot_launch():
    _refused("EMO_MEAN_NORM", r"N >= 1", N=0)
    _refused("EMO_LINEAR_NORM", r"E >= 1", N=1, E=0)
    _refused("EMO_LINEAR_NORM", r"48 KB", N=1, E=12001)


def test_probe_refuses_an_unknown_op():
    a = _lib.AnProbeArgs()
    a.op = len(_lib.AN_OPS)
    with pytest.raises(RuntimeError, match="unknown op"):
        _lib.check(_lib.lib().agpt_an_probe(C.byref(a), None))


# ================================================================================================ mutants (CPU)
def test_gate_catches_swapped_shuffle_phases():
    up, skip = rnd((2, 3, 8, 4, 8), 1), rnd((2, 6, 15, 8), 2)
    good = shuffle_ref(up, skip)
    assert not torch.equal(shuffle_ref(up, skip, swap=True), good)


def test_gate_catches_upcol_without_the_column_guard():
    y = rnd((2, 3, 7, 8), 3, 1.0, 0.5)
    s, t = rnd((8,), 4, 0.3, 1.0), rnd((8,), 5, 0.2, 0.3)
    ref, bound, zero = upcol_ref(y, s, t)
    assert passes(ref.float(), ref, bound)
    bad = upcol_ref(y, s, t, no_guard=True)[0]
    assert not (torch.equal(bad[zero], torch.zeros_like(bad[zero])) and passes(bad.float(), ref, bound))


def test_gate_catches_affine_sample_index_without_the_c4_division():
    rows, Cc, rps = 3 * 20, 16, 20
    x, s, t = affine_inputs(rows, Cc, 6)
    vec = rnd((3, 48), 7)
    _, _, r, br = affine_ref(x, s, t, vec, 16, rps)
    assert passes(r.float(), r, br)
    assert not passes(affine_ref(x, s, t, vec, 16, rps, mutant=True)[2].float(), r, br)


def test_gate_catches_embeddings_added_right_to_left():
    word, pos, types, ids, tids, _ = embed_inputs(2, 77, 256, 1000, 2, 8)
    good = embed_ref(word, pos, types, ids, tids, 1000, 2)
    assert not torch.equal(embed_ref(word, pos, types, ids, tids, 1000, 2, assoc="right"), good)


def test_gate_catches_a_mask_stored_as_mask_not_zero():
    mask = embed_inputs(2, 77, 8, 10, 2, 9)[5]
    assert not torch.equal((mask != 0).to(torch.uint8), (mask == 0).to(torch.uint8))


@pytest.mark.parametrize("mutant", ["unclamped", "align"])
def test_gate_catches_mix_interp_mutants(mutant):
    for B, Td, T in ((3, 62, 501), (2, 148, 149)):
        p1 = probs(B, Td, 2, 10)
        _, _, ru, bu = mix_interp_ref(p1, None, None, T)
        assert passes(ru.float(), ru, bu)
        assert not passes(mix_interp_ref(p1, None, None, T, mutant=mutant)[2].float(), ru, bu), (B, Td, T)


def test_gate_catches_refemb_without_the_temperature():
    E, qw, qb, kw, kb = refemb_inputs(2, 62, 11)
    ref, bound = refemb_ref(E, 1, qw, qb, kw, kb)
    assert passes(ref.float(), ref, bound)
    assert not passes(refemb_ref(E, 1, qw, qb, kw, kb, temp=1.0)[0].float(), ref, bound)


def test_gate_catches_the_head_normalising_over_one_output_less():
    h, w, b = torch.tanh(rnd((9, 1024), 12)), rnd((2, 1024), 13, 0.08), rnd((2,), 14, 0.3)
    ref, bound = head_ref(h, w, b)
    assert passes(ref.float(), ref, bound)
    assert not passes(head_ref(h, w, b, drop_last=True)[0].float(), ref, bound)


def test_gate_catches_linear_norm_normalising_before_the_relu():
    h, W, b = linear_norm_inputs(5, 256, 15)
    ref, bound = linear_norm_ref(h, W, b)
    assert passes(ref.float(), ref, bound)
    assert not passes(linear_norm_ref(h, W, b, norm_first=True)[0].float(), ref, bound)


def test_gate_catches_the_film_kernel_ignoring_jb():
    T = film_tables(13, [33] * 13, 37, 44, 16, True)
    hid = torch.relu(rnd((2, T["hid_len"]), 17))
    ref, bound = film_ref(hid, T, 44)
    w = ~torch.isnan(ref)
    assert passes(ref[w].float(), ref[w], bound[w])
    assert not passes(film_ref(hid, T, 44, ignore_jb=True)[0][w].float(), ref[w], bound[w])


@gpu
def test_every_op_exercised():
    """runs last in this module: every AGPT_AN_* selector has been through a gate"""
    missing = [op for op in _lib.AN_OPS if op not in EXERCISED]
    assert not missing, f"not exercised: {missing}"
