"""Conformance of the tap-GEMM primitive (tapconv_launch, the fused pair launch) against a float64 reference.

Every case runs ONE production launch through agpt_tapconv_probe_pipes -- the production weight packer, launch
parameters as given, caller-owned device tensors -- and compares it with torch.nn.functional in float64 on the device
(conv1d / conv2d / conv_transpose1d on the torch weight layouts, then the prologue and epilogue formulas of the
reference modules), written without any of the kernels' packing.  `ran`, what the probe reports as launched, is asserted for
every case, so a shape meant for one tile variant cannot quietly test another.

Tolerance, per output element, before the epilogue (U = 2^-22, S = |pro(x)| (*) |w|, the float64 conv of the
absolute values, n = the number of products summed into one output, u = the unit roundoff of the accumulator):

    |y - ref| <= c * U * S  +  2^-25 * (M (*) |w|)  +  2^-25 * s_w * (|pro(x)| (*) 1),   c = c_rep + LAMBDA sqrt(n) u / U

  * c_rep, the operands.  Tensor cores: each operand is split x = hi + lo into fp16 parts with
    |x - hi - lo| <= 2^-22 |x| (both parts carry 11 significand bits), likewise each weight, and the lo * lo product
    is dropped (<= 2^-22 |x w|): c_rep = 3.  fp32-FMA kernel: the operands are exact, but a SiLU prologue rounds
    (2 ulp): c_rep = 1.
  * LAMBDA sqrt(n) u, the accumulation: the probabilistic bound of Higham & Mary (SIAM J. Sci. Comput. 41(5), 2019)
    for a sum of n products with independent zero-mean rounding errors, |error| <= LAMBDA sqrt(n) u S except with
    probability 2 exp(-LAMBDA^2 / 2); LAMBDA = 6 (3e-8 per element).  Tensor cores: u = 2^-23 (the accumulation
    truncates), n = 3 products x taps x C_in rounded up to the 16-deep wgmma k-step.  fp32-FMA: u = 2^-24 (one
    rounding per fused multiply-add), n = taps x C_in rounded up to the 8-deep K chunk.  (The worst case n u S would
    not catch a single wrong tap of a long contraction; this bound still does, with room to spare.)
  * The fp16 limits (tensor cores only): the lo part of an activation below 2^-14 is subnormal, an absolute error of
    2^-25 per activation (M = 1 on the real input elements); weights are pre-scaled by a power of two so that
    max|w| lands in [2^13, 2^14), which gives each weight an absolute floor of 2^-25 * s_w, s_w = 2^(e - 14) for
    max|w| = m 2^e, m in [0.5, 1).  Activations are kept below the fp16 saturation at 65504.

The epilogue adds one fp32 rounding (2^-24 relative) per operation on the magnitudes it combines, and a
nonlinearity f maps the bound E of its argument to max |f(v +- E) - f(v)| plus 8 ulp of |f| + |v| for the device
transcendental functions.  Besides the per-element bound, the rms error must stay below half the rms bound.

The "pipelines" section reaches the persistent and two-CTA kernels HiFi-GAN runs (tcpair2_kernel, tcpair_pipe_kernel,
tcpair_narrow_kernel, tcconv_pipe_pl_kernel) through the probe's switches, checks each against the same bound, and
requires the same bits as the kernel the switches replace.  The mutants at the end (CPU only) show that plausible
pipeline bugs fail this gate.
"""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from audiogpt_b200 import _lib

gpu = pytest.mark.gpu

PRO_NONE, PRO_LRELU, PRO_ADDVEC, PRO_SILU = 0, 1, 2, 3
(EPI_BIAS, EPI_RES, EPI_ACC, EPI_RELU, EPI_ADDVEC, EPI_GATE, EPI_GEGLU, EPI_DIFFOUT, EPI_STORE_CF, EPI_TANH, EPI_MISH,
 EPI_SILU, EPI_GELU_SCALED) = range(13)
EPI_NAMES = ["BIAS", "RES", "ACC", "RELU", "ADDVEC", "GATE", "GEGLU", "DIFFOUT", "STORE_CF", "TANH", "MISH", "SILU",
             "GELU_SCALED"]

U = 2.0 ** -22
LAMBDA = 6.0
C_REP_TC, C_REP_FMA = 3.0, 1.0
U_ACC_TC, U_ACC_FMA = 2.0 ** -23, 2.0 ** -24
FLOOR = 2.0 ** -25
EPS32 = 2.0 ** -24
GUARD = 64              # canary floats after the last sample of every output buffer
DEV = "cuda"
NAN = float("nan")
TILE, DUAL, PAIR_PIPE, NARROW_PIPE, CONV_PIPE = range(len(_lib.TC_KERNS))   # ran[4], the kernel family
SWITCHES = ("tc_dual", "tc_pipe", "tc_narrow_pipe", "tc_conv_pipe")

EXERCISED = {}          # (kernel, BN, MT, plane-fed, family) -> worst error / bound over the cases that ran it


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    if EXERCISED:
        print("\ntap-GEMM variants exercised (kernel, BN, MT, plane-fed, family): worst error / bound")
        for k in sorted(EXERCISED):
            print(f"  {'wgmma' if k[0] == 1 else 'fma  '} BN {k[1]:3d} MT {k[2]:3d} plane {k[3]} "
                  f"{_lib.TC_KERNS[k[4]]:11s}: {EXERCISED[k]:.3f}")


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def cdiv(a, b):
    return -(-a // b)


def native_bn(cout):
    """tc_pick_bn: the weight image's own tile width"""
    if cout <= 32:
        return 32
    if cout <= 64:
        return 64
    return 128 if cdiv(cout, 128) * 128 <= cdiv(cout, 64) * 64 else 64


def pick_tile(cout, rows_v, G, tall):
    """The tile (BN, MT) pick_h_tile chooses for a 1-D launch of G samples x rows_v rows on this device (used only to
    choose shapes; every case asserts what actually ran)."""
    s = sms()
    cost = {128: 1.0, 96: 0.82, 64: 0.62, 32: 0.45}
    rt = cdiv(rows_v, 128) * G
    nat = native_bn(cout)
    best, bs = nat, cdiv(rt * cdiv(cout, nat), s) * cost[nat]
    cands = ([64] if nat == 128 else []) + ([96] if nat == 128 and cout > 128 else [])
    for bn in cands:
        sc = cdiv(rt * cdiv(cout, bn), s) * cost[bn]
        if sc < bs - 1e-9:
            best, bs = bn, sc
    mt = 256 if tall and best <= 64 and cdiv(rows_v, 256) * G * cdiv(cout, best) >= 4 * s else 128
    return best, mt


def rows_for(cout, G, bn, mt, tall):
    """The smallest L (a partial last row tile: L % 128 != 0) for which the picker lands on (bn, mt)."""
    for n in range(1, 2000):
        L = 128 * n - 37
        if pick_tile(cout, L, G, tall) == (bn, mt):
            return L
    raise AssertionError(f"no L lands on BN {bn} MT {mt} for Cout {cout} on {sms()} SMs")


# ------------------------------------------------------------------------------------------------ the fp64 reference
def pro_ref(x, pro, slope, pvec):
    if pro == PRO_LRELU:
        return F.leaky_relu(x, slope)
    if pro == PRO_SILU:
        return F.silu(x)
    if pro == PRO_ADDVEC:
        return x + pvec[:, None, :]     # on the real rows only: the conv's zero padding comes after the add
    return x


def conv_ref(sp, x, w):
    """x [G][rows][Cin] (float64) -> [G][rows][channels of the kernel's output], no bias."""
    G, rows = x.shape[0], x.shape[1]
    kind = sp["kind"]
    if kind == 1:
        H, W = rows // sp["Wreal"], sp["Wreal"]
        y = F.conv2d(x.permute(0, 2, 1).reshape(G, -1, H, W), w, padding=1)
        return y.reshape(G, y.shape[1], rows).permute(0, 2, 1)
    xt = x.permute(0, 2, 1)
    if kind == 2:
        u = sp["u"]
        y = F.conv_transpose1d(xt, w, stride=u, padding=sp["pad"])[:, :, :rows * u]   # the first L*u samples
        return y.permute(0, 2, 1).reshape(G, rows, u * w.shape[1])
    d = sp.get("dil", 1)
    return F.conv1d(xt, w, padding=d * (w.shape[2] - 1) // 2, dilation=d).permute(0, 2, 1)


def w_floor_scale(*ws):
    """s_w: the inverse power-of-two pre-scale of the fp16 weight image (pack_h_weights)"""
    mx = max(float(w.abs().max()) for w in ws)
    return 0.0 if mx == 0 else 2.0 ** (math.frexp(mx)[1] - 14)


def n_products(sp, cin, k, tc):
    """products summed into one output of the packed layer (an upper bound for the polyphase / grouped packings)"""
    kind = sp["kind"]
    taps = 9 if kind == 1 else (cdiv(k, sp["u"]) + 1 if kind == 2 else k)
    if kind == 3:
        g = sp["g"]
        cin, taps = g * cin, cdiv(k + g - 1, g) + 1
    return 3 * taps * cdiv(cin, 16) * 16 if tc else taps * cdiv(cin, 8) * 8


def c_const(n, tc):
    """c of the module docstring"""
    return (C_REP_TC + LAMBDA * math.sqrt(n) * U_ACC_TC / U) if tc else (C_REP_FMA + LAMBDA * math.sqrt(n) * U_ACC_FMA / U)


def conv_bound(sp, xp, w, tc, mask):
    """Per-element bound of the contraction (module docstring) for prologue output xp (float64)."""
    S = conv_ref(sp, xp.abs(), w.abs())
    cin = w.shape[0] if sp["kind"] == 2 else w.shape[1]
    c = c_const(n_products(sp, cin, w.shape[-1], tc), tc)
    if not tc:
        return c * U * S, S
    b = c * U * S + FLOOR * conv_ref(sp, mask, w.abs())
    sw = w_floor_scale(w)
    if sw:
        b = b + FLOOR * sw * conv_ref(sp, xp.abs(), torch.ones_like(w))
    return b, S


def f_bound(f, v, E):
    """bound of |f(v_hat) - f(v)| for |v_hat - v| <= E, plus the device function's own error"""
    fv = f(v)
    return torch.maximum((f(v + E) - fv).abs(), (f(v - E) - fv).abs()) + 8 * EPS32 * (fv.abs() + v.abs())


def gelu64(x):
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2.0)))


def mish64(x):
    return x * torch.tanh(torch.where(x > 20, x, torch.log1p(torch.exp(x))))


# ------------------------------------------------------------------------------------------------ buffers and the probe
def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def buffer(G, rows, pitch, gpad=0, fill=NAN):
    """flat fp32 device buffer of G samples of [rows][pitch] (+ gpad floats per sample) + a guard; returns (flat,
    sample stride)"""
    gs = rows * pitch + gpad
    return torch.full((G * gs + GUARD,), fill, dtype=torch.float32, device=DEV), gs


def view(flat, G, gs, rows, pitch, ch):
    return flat[:G * gs].view(G, gs)[:, :rows * pitch].view(G, rows, pitch)[:, :, :ch]


def region_mask(flat, G, gs, rows, pitch, ch):
    m = torch.zeros_like(flat, dtype=torch.bool)
    view(m, G, gs, rows, pitch, ch).fill_(True)
    return m


def bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def probe(**kw):
    """agpt_tapconv_probe_pipes with the arguments kw (the switches of SWITCHES among them); the 5 ints of ran"""
    a, sw = _lib.TapconvProbeArgs(), _lib.TapconvPipes()
    a.scale, a.slope, a.dil, a.dil2 = 1.0, 0.1, 1, 1
    for k, v in kw.items():
        if isinstance(v, torch.Tensor):
            v = v.data_ptr()
        setattr(sw if k in SWITCHES else a, k, v)
    ran = (C.c_int * 5)()
    _lib.check(_lib.lib().agpt_tapconv_probe_pipes(C.byref(a), C.byref(sw), ran, _lib.cur_stream()))
    return tuple(ran)


def verdict(y, ref, bound):
    """(failure or None, worst err / bound, rms err / rms bound) of the gate: every element written (no NaN canary
    left), |y - ref| <= bound element-wise and rms(err) <= rms(bound) / 2"""
    y = y.double()
    if not torch.isfinite(y).all():
        return "unwritten or non-finite output", math.inf, math.inf
    err = (y - ref).abs()
    bound = bound + 1e-300
    ratio = float((err / bound).max())
    rms_ratio = float(err.pow(2).mean().sqrt() / bound.pow(2).mean().sqrt())
    if ratio > 1.0:
        return f"error {ratio:.3g} x the bound", ratio, rms_ratio
    if rms_ratio > 0.5:
        return f"rms error {rms_ratio:.3g} x the rms bound", ratio, rms_ratio
    return None, ratio, rms_ratio


def check(name, y, ref, bound, path, ran):
    """assert the gate (verdict); returns the worst ratio"""
    fail, ratio, rms_ratio = verdict(y, ref, bound)
    print(f"{name} [{path} ran={ran}]: worst err/bound {ratio:.3f}, rms err/rms bound {rms_ratio:.3f}")
    assert fail is None, f"{name} [{path}]: {fail}"
    EXERCISED[tuple(ran)] = max(EXERCISED.get(tuple(ran), 0.0), ratio)
    return ratio


def pair_reference(sp, xp, w, b, w2, b2, slope, tc):
    """c2(lrelu(c1(xp))) + b2 of a ResBlock pair in float64 and its bound before the epilogue (module docstring).  c2
    runs over c1's view: plain rows with dilation sp["dil2"], or (kind 3) the time-grouped view, whose products the
    bound counts."""
    grouped = sp["kind"] == 3
    Eb1, _ = conv_bound(sp, xp, w, tc, torch.ones_like(xp))
    v = conv_ref(sp, xp, w) + b
    h = F.leaky_relu(v, slope)
    E_h = Eb1 + EPS32 * v.abs()
    sp2 = dict(kind=3 if grouped else 0, dil=sp.get("dil2", 1), u=1, g=sp["g"] if grouped else 1)
    vc2 = conv_ref(sp2, h, w2)
    Eb2, S2 = conv_bound(sp2, h, w2, tc, torch.ones_like(h))
    vv = vc2 + b2
    return vv, Eb2 + conv_ref(sp2, E_h, w2.abs()) + EPS32 * (S2 + vv.abs())


# ------------------------------------------------------------------------------------------------ one case
def run_case(name, kind=0, Cin=64, Cout=64, K=3, dil=1, G=2, L=200, Wreal=0, strip_w=0, u=1, pad=0, g=1,
             pro=PRO_LRELU, slope=0.1, epi=EPI_BIAS, bias=True, res=False, scale=1.0, accumulate=0, csplit=0,
             in_extra=0, out_extra=0, gpad=0, paths=("tc", "fma"), tall=0, plane_in=0, po=None, pl=None, pair=None,
             x_scale=1.0, w_spread=1.0, expect=None, seed=0, stats=None, switches=()):
    """Run one launch per path in `paths` and check it (see the module docstring).  expect: {path: (tc, BN, MT,
    plane, family)} asserted against `ran`; po / pl: None, "with" (and the fp32 tensor) or "only" (out = NULL).  stats:
    a dict that receives the worst {max |err| / rms(ref), rms(err) / rms(ref)} of the fp32 output over the paths.
    res: False, True (a tensor of its own), or "input" (the residual is the input tensor, Cin == Cout); a pair's
    residual is its input unless res == "own".  switches: pipeline switches of SWITCHES to set; such a launch must
    also be bit-identical to the same call with every switch off and tall = 0 (the kernels' own claim, DESIGN.md)."""
    sp = dict(kind=kind, dil=dil, Wreal=Wreal, u=u, pad=pad, g=g, dil2=(pair or {}).get("dil2", 1))
    gr = gen(seed)
    rows = L
    # --- weights (torch layouts, host arrays for the packers) and the per-sample vectors
    wshape = {0: (Cout, Cin, K), 1: (Cout, Cin, 3, 3), 2: (Cin, Cout, K), 3: (Cout, Cin, K), 4: (Cout, Cin, K)}[kind]
    fan = Cin * (9 if kind == 1 else K)
    w = torch.randn(wshape, generator=gr, device=DEV) / math.sqrt(fan)
    if w_spread > 1.0:   # weight-norm-like gain spread over the output channels (log-uniform over a factor w_spread)
        gain = w_spread ** (torch.rand(Cout, generator=gr, device=DEV) - 0.5)
        w = w * (gain[None, :, None] if kind == 2 else gain.view(-1, *([1] * (w.dim() - 1))))
    b = 0.05 * torch.randn(Cout, generator=gr, device=DEV) if bias else None
    w_h = w.cpu().contiguous()
    b_h = b.cpu().contiguous() if bias else None
    pvec = torch.randn(G, Cin, generator=gr, device=DEV) if pro == PRO_ADDVEC else None
    oc = u * Cout if kind == 2 else Cout             # channels of the kernel's output rows
    evec = torch.randn(G, oc, generator=gr, device=DEV) if epi == EPI_ADDVEC else None
    # --- pair: c2 weights
    if pair:
        K2 = pair.get("K2", K)
        w2 = torch.randn(Cout, Cout, K2, generator=gr, device=DEV) / math.sqrt(Cout * K2)
        b2 = 0.05 * torch.randn(Cout, generator=gr, device=DEV)
        w2_h, b2_h = w2.cpu().contiguous(), b2.cpu().contiguous()
    # --- input: [G][rows][in_pitch], NaN in the pitch padding past Cin and in the sample padding
    in_pitch = Cin + in_extra
    xin, in_gs = buffer(G, rows, in_pitch, gpad)
    x = view(xin, G, in_gs, rows, in_pitch, Cin)
    x.copy_(torch.randn(G, rows, Cin, generator=gr, device=DEV) * x_scale)
    # --- outputs
    gate = epi in (EPI_GATE, EPI_GEGLU)
    och = {EPI_GATE: oc // 2, EPI_GEGLU: oc // 2, EPI_DIFFOUT: csplit}.get(epi, oc)
    out_pitch = och + out_extra
    resv = None
    if (pair and res != "own") or res == "input":   # a ResBlock pair adds its own input: x + c2(lrelu(c1(lrelu(x))))
        rflat, res_gs, res_pitch, resv = xin, in_gs, in_pitch, x
    elif res:
        res_pitch = oc + out_extra
        rflat, res_gs = buffer(G, rows, res_pitch, gpad)
        resv = view(rflat, G, res_gs, rows, res_pitch, oc)
        resv.copy_(torch.randn(G, rows, oc, generator=gr, device=DEV))
    x64 = x.double()
    xp = pro_ref(x64, pro, slope, pvec.double() if pvec is not None else None)
    mask = torch.ones_like(x64)
    wref = w.double()
    v_conv = conv_ref(sp, xp, wref)
    if b is not None:
        bias_rows = b.double().repeat(u) if kind == 2 else b.double()
        v = v_conv + bias_rows
    else:
        bias_rows = torch.zeros(oc, dtype=torch.float64, device=DEV)
        v = v_conv
    old_out = torch.randn(G, rows, och, generator=gr, device=DEV) if (epi == EPI_ACC and accumulate) or epi == EPI_DIFFOUT else None
    old_out2 = torch.randn(G, rows, Cout - csplit, generator=gr, device=DEV) if epi == EPI_DIFFOUT and accumulate else None
    worst = 0.0
    for path in paths:
        tc = path != "fma"
        # c2 of a pair sees lrelu(c1 out) computed in fp32: its reference and bound come first
        if pair:
            vv, Ev = pair_reference(sp, xp, wref, b.double(), w2.double(), b2.double(), slope, tc)
        else:
            Eb, S = conv_bound(sp, xp, wref, tc, mask)
            vv = v
            Ev = Eb + EPS32 * (S + v.abs() + bias_rows.abs())
        # --- the epilogue reference and its bound
        r64 = resv.double() if resv is not None else 0.0
        if kind == 4 and resv is not None:   # the kernel reads res in the interleaved channel order of its weights
            r64 = torch.cat([r64[..., 0::2], r64[..., 1::2]], dim=-1)
        y2ref = None
        if epi == EPI_BIAS:
            ref, E = vv, Ev
        elif epi == EPI_RES:
            ref = vv + r64
            E = Ev + EPS32 * ref.abs()
        elif epi == EPI_ACC:
            t = vv + r64
            ref = scale * t + (old_out.double() if accumulate else 0.0)
            E = abs(scale) * (Ev + EPS32 * t.abs()) + EPS32 * (abs(scale) * t.abs() + ref.abs())
        elif epi == EPI_RELU:
            ref, E = F.relu(vv), Ev
        elif epi == EPI_ADDVEC:
            ref = vv + evec.double()[:, None, :]
            E = Ev + 2 * EPS32 * (evec.double().abs()[:, None, :] + ref.abs())
        elif epi == EPI_TANH:
            ref, E = torch.tanh(vv), f_bound(torch.tanh, vv, Ev)
        elif epi == EPI_MISH:
            ref, E = mish64(vv), f_bound(mish64, vv, Ev)
        elif epi == EPI_SILU:
            ref, E = F.silu(vv), f_bound(F.silu, vv, Ev)
        elif epi == EPI_GELU_SCALED:
            fs = lambda z: gelu64(scale * z)
            ref, E = fs(vv), f_bound(fs, vv, Ev)
        elif gate:
            pre = vv + r64
            Ep = Ev + EPS32 * pre.abs()
            a_, g_ = pre.chunk(2, dim=-1)
            Ea, Eg = Ep.chunk(2, dim=-1)
            if epi == EPI_GATE:   # DiffNet: gate, filter = chunk(y, 2); sigmoid(gate) * tanh(filter)
                fa, fg = torch.sigmoid, torch.tanh
            else:                 # GEGLU: x, gate = proj(x).chunk(2); x * gelu(gate)
                fa, fg = (lambda z: z), gelu64
            ref = fa(a_) * fg(g_)
            E = torch.zeros_like(ref)
            for sa in (-1, 1):
                for sg in (-1, 1):
                    E = torch.maximum(E, (fa(a_ + sa * Ea) * fg(g_ + sg * Eg) - ref).abs())
            E = E + 8 * EPS32 * (ref.abs() + a_.abs() + g_.abs())
        elif epi == EPI_DIFFOUT:  # DiffNet residual layer: x, skip = chunk(y); (x + residual) / sqrt(2), skip summed
            xo, sk = vv[..., :csplit], vv[..., csplit:]
            Ex, Es = Ev[..., :csplit], Ev[..., csplit:]
            ref = (old_out.double() + xo) / math.sqrt(2.0)
            E = (Ex + EPS32 * (old_out.double() + xo).abs()) / math.sqrt(2.0) + 2 * EPS32 * ref.abs()
            y2ref = sk + (old_out2.double() if accumulate else 0.0)
            E2 = Es + EPS32 * y2ref.abs()
        elif epi == EPI_STORE_CF:
            ref, E = vv, Ev
        cf = epi == EPI_STORE_CF
        only = (po == "only") or (pl == "only")
        o2p = Cout - csplit + out_extra

        def launch(sw, tall_):
            """fresh output buffers (NaN everywhere but where the kernel must read) and one probe call"""
            if cf:
                oflat, out_gs = buffer(G, oc, rows, gpad)
            else:
                oflat, out_gs = buffer(G, rows, out_pitch, gpad)
            if old_out is not None:
                view(oflat, G, out_gs, rows, out_pitch, och).copy_(old_out)
            o2flat, o2_gs = None, 0
            if epi == EPI_DIFFOUT:
                o2flat, o2_gs = buffer(G, rows, o2p, gpad)
                if accumulate:
                    view(o2flat, G, o2_gs, rows, o2p, Cout - csplit).copy_(old_out2)
            planes = {}
            for key, mode in (("po", po), ("pl", pl)):
                if mode:
                    planes[key] = [torch.full((G * out_gs + GUARD,), NAN, dtype=torch.float16, device=DEV) for _ in range(2)]
            kw = dict(kind=kind, Cin=Cin, Cout=Cout, K=K, dil=dil, Wreal=Wreal, strip_w=strip_w, u=u, pad=pad, g=g,
                      w=w_h.data_ptr(), b=b_h.data_ptr() if bias else None, G=G, L=L,
                      inp=x, in_gstride=in_gs, in_pitch=in_pitch,
                      out=None if only else oflat, out_gstride=out_gs, out_pitch=out_pitch,
                      pro=pro, slope=slope, epi=epi, scale=scale, accumulate=accumulate, csplit=csplit,
                      tc_tall=tall_, plane_in=plane_in if tc else 0, fma=0 if tc else 1)
            kw.update({k: 1 for k in sw})
            if resv is not None:
                kw.update(res=resv, res_gstride=res_gs, res_pitch=res_pitch)
            if pvec is not None:
                kw.update(pvec=pvec, pvec_gstride=Cin)
            if evec is not None:
                kw.update(evec=evec, evec_gstride=oc)
            if o2flat is not None:
                kw.update(out2=o2flat, out2_gstride=o2_gs, out2_pitch=o2p)
            if "po" in planes:
                kw.update(po_hi=planes["po"][0], po_lo=planes["po"][1], po_slope=0.2)
            if "pl" in planes:
                kw.update(pl_hi=planes["pl"][0], pl_lo=planes["pl"][1], pl_pitch=out_pitch)
            if pair:
                kw.update(pair=1, w2=w2_h.data_ptr(), b2=b2_h.data_ptr(), K2=pair.get("K2", K), dil2=pair.get("dil2", 1))
            return probe(**kw), oflat, out_gs, o2flat, o2_gs, planes

        saved_in = bits(xin).clone()
        saved_res = bits(rflat).clone() if resv is not None else None
        saved_pvec = pvec.clone() if pvec is not None else None
        ran, oflat, out_gs, o2flat, o2_gs, planes = launch(switches, tall)
        if expect and path in expect:
            assert ran == expect[path], f"{name} [{path}]: ran {ran}, meant to test {expect[path]}"
        elif not tc:
            assert ran == (0, native_bn(g * oc if kind == 3 else oc), 128, 0, TILE), f"{name} [fma]: ran {ran}"
        else:
            assert ran[0] == 1 and ran[3] == (1 if plane_in else 0) and ran[4] == TILE, f"{name} [{path}]: ran {ran}"
        if switches:   # the same sums in the same order as the kernel the switches replace: the same bits
            ran0, oflat0, _, o2flat0, _, planes0 = launch((), 0)
            assert ran0[4] == TILE, f"{name}: with the switches off, ran {ran0}"
            assert torch.equal(bits(oflat0), bits(oflat)), f"{name}: not bit-identical to {ran0} (ran {ran})"
            assert o2flat is None or torch.equal(bits(o2flat0), bits(o2flat)), f"{name}: out2 differs from {ran0}"
            for key in planes:
                for t, t0 in zip(planes[key], planes0[key]):
                    assert torch.equal(bits(t0), bits(t)), f"{name}: the {key} plane differs from {ran0}"
        tag = f"{name} {EPI_NAMES[epi]}"
        # --- inputs untouched
        assert torch.equal(bits(xin), saved_in), f"{tag}: the input was written"
        if resv is not None:
            assert torch.equal(bits(rflat), saved_res), f"{tag}: the residual was written"
        if pvec is not None:
            assert torch.equal(pvec, saved_pvec), f"{tag}: the prologue vector was written"
        # --- the fp32 outputs: every element written and within the bound, nothing else touched
        if not only:
            if cf:
                yv = view(oflat, G, out_gs, oc, rows, rows).permute(0, 2, 1)
                inside = region_mask(oflat, G, out_gs, oc, rows, rows)
            else:
                yv = view(oflat, G, out_gs, rows, out_pitch, och)
                inside = region_mask(oflat, G, out_gs, rows, out_pitch, och)
            assert torch.isnan(oflat[~inside]).all(), f"{tag} [{path}]: written outside [0, Cout) x rows x G"
            worst = max(worst, check(tag, yv, ref, E, path, ran))
            if stats is not None:
                err, rr = yv.double() - ref, ref.pow(2).mean().sqrt().clamp_min(1e-300)
                stats["max"] = max(stats.get("max", 0.0), float(err.abs().max() / rr))
                stats["rms"] = max(stats.get("rms", 0.0), float(err.pow(2).mean().sqrt() / rr))
        if o2flat is not None:
            inside2 = region_mask(o2flat, G, o2_gs, rows, o2p, Cout - csplit)
            assert torch.isnan(o2flat[~inside2]).all(), f"{tag} [{path}]: out2 written outside its region"
            worst = max(worst, check(tag + " out2", view(o2flat, G, o2_gs, rows, o2p, Cout - csplit), y2ref, E2, path, ran))
        # --- operand planes: hi + lo against float64, and bit for bit the split of the kernel's own fp32 value
        for key in planes:
            hi, lo = planes[key]
            hv, lv = (view(t, G, out_gs, rows, out_pitch, och) for t in (hi, lo))
            inside = region_mask(hi, G, out_gs, rows, out_pitch, och)
            assert torch.isnan(hi[~inside]).all() and torch.isnan(lo[~inside]).all(), f"{tag} {key}: written outside"
            if key == "po":   # hi + lo = lrelu(out, po_slope)
                pref, pE = F.leaky_relu(ref, 0.2), E
                val32 = F.leaky_relu(yv, 0.2) if not only else None
            else:
                pref, pE = ref, E
                val32 = yv if not only else None
            pE = pE + U * pref.abs() + FLOOR
            worst = max(worst, check(f"{tag} {key}-plane", hv.double() + lv.double(), pref, pE, path, ran))
            if val32 is not None:
                h_exp = val32.clamp(-65504, 65504).half()
                l_exp = (val32 - h_exp.float()).half()
                assert torch.equal(bits(hv.contiguous()), bits(h_exp.contiguous())), f"{tag} {key}: hi is not fp16(v)"
                assert torch.equal(bits(lv.contiguous()), bits(l_exp.contiguous())), f"{tag} {key}: lo is not fp16(v - hi)"
    return worst


# ================================================================================================ prologues
@pytest.mark.parametrize("pro,slope", [(PRO_NONE, 0.1), (PRO_LRELU, 0.1), (PRO_LRELU, 0.01), (PRO_SILU, 0.1),
                                       (PRO_ADDVEC, 0.1)])
@gpu
def test_prologues_1d(pro, slope):
    run_case(f"pro{pro}/{slope}", Cin=36, Cout=40, K=5, dil=3, G=3, L=257, pro=pro, slope=slope, epi=EPI_RES, res=True,
             in_extra=4, seed=pro)


@gpu
@pytest.mark.parametrize("pro", [PRO_ADDVEC, PRO_SILU])
def test_prologues_2d(pro):
    """3x3 conv: the virtual zero column and the rows above / below the image must stay zero after the prologue"""
    run_case(f"pro{pro} 2d", kind=1, Cin=64, Cout=32, G=2, L=10 * 13, Wreal=13, pro=pro, epi=EPI_BIAS, seed=10 + pro)


# ================================================================================================ epilogues
EPI_CASES = [
    dict(epi=EPI_BIAS), dict(epi=EPI_BIAS, bias=False), dict(epi=EPI_RES, res=True),
    dict(epi=EPI_ACC, res=True, accumulate=0, scale=1 / 3), dict(epi=EPI_ACC, res=True, accumulate=1, scale=1 / 3),
    dict(epi=EPI_ACC, accumulate=1, scale=0.75),
    dict(epi=EPI_RELU), dict(epi=EPI_ADDVEC), dict(epi=EPI_TANH), dict(epi=EPI_MISH), dict(epi=EPI_SILU),
    dict(epi=EPI_GELU_SCALED, scale=0.125),
    dict(epi=EPI_DIFFOUT, csplit=48, accumulate=0), dict(epi=EPI_DIFFOUT, csplit=48, accumulate=1),
    dict(epi=EPI_STORE_CF), dict(epi=EPI_STORE_CF, Cout=1, Cin=8), dict(epi=EPI_STORE_CF, Cout=2),
]


@gpu
@pytest.mark.parametrize("i", range(len(EPI_CASES)))
def test_epilogues(i):
    kw = dict(Cin=80, Cout=96, K=3, dil=1, G=2, L=300, pro=PRO_LRELU)
    kw.update(EPI_CASES[i])
    run_case(f"epi#{i}", seed=100 + i, **kw)


@gpu
def test_store_cf_2d():
    run_case("store_cf 2d", kind=1, Cin=32, Cout=4, G=2, L=12 * 9, Wreal=9, pro=PRO_SILU, epi=EPI_STORE_CF, seed=120)


@gpu
@pytest.mark.parametrize("epi", [EPI_GATE, EPI_GEGLU])
@pytest.mark.parametrize("res", [False, True])
def test_gate_epilogues(epi, res):
    run_case(f"pairs {'res' if res else ''}", kind=4, Cin=64, Cout=128, K=3, dil=2, G=2, L=250, pro=PRO_NONE, epi=epi,
             res=res, seed=130 + epi + 2 * res)


@gpu
@pytest.mark.parametrize("epi", [EPI_GATE, EPI_GEGLU])
@pytest.mark.parametrize("mode", ["with", "only"])
def test_gate_plane_output(epi, mode):
    """The GATE / GEGLU operand-plane output (G == 1: the UNet's GEGLU feeding a plane-fed ff2)"""
    run_case(f"pairs pl-{mode}", kind=4, Cin=320, Cout=640, K=1, G=1, L=333, pro=PRO_NONE, epi=epi, res=(epi == EPI_GATE),
             pl=mode, paths=("tc",), seed=140 + epi)


# ================================================================================================ shapes
@gpu
@pytest.mark.parametrize("Cin", [1, 2, 4, 8, 36, 64, 80, 100, 320, 1280])
def test_cin(Cin):
    """Cin in {1, 2} (and pitches not a multiple of 4) go to the FMA kernel by tcconv_supported"""
    exp = {"tc": (0, native_bn(40), 128, 0, TILE)} if Cin % 4 else None
    run_case(f"Cin {Cin}", Cin=Cin, Cout=40, K=3, G=2, L=131, epi=EPI_RES, res=True, expect=exp, seed=200 + Cin)


@gpu
@pytest.mark.parametrize("Cout", [4, 32, 40, 96, 100, 256, 320, 640])
def test_cout(Cout):
    run_case(f"Cout {Cout}", Cin=64, Cout=Cout, K=3, G=2, L=129, epi=EPI_BIAS, seed=300 + Cout)


@gpu
@pytest.mark.parametrize("L", [1, 127, 128, 129, 255, 256, 257, 3001])
@pytest.mark.parametrize("G", [1, 3])
def test_lengths(L, G):
    run_case(f"G {G} L {L}", Cin=32, Cout=32, K=7, dil=3, G=G, L=L, epi=EPI_RES, res=True, gpad=8, seed=400 + L + G)


@gpu
@pytest.mark.parametrize("K,dil", [(1, 1), (3, 1), (5, 3), (7, 5), (11, 1), (11, 5)])
def test_taps(K, dil):
    run_case(f"K {K} dil {dil}", Cin=64, Cout=64, K=K, dil=dil, G=2, L=300, epi=EPI_RES, res=True, seed=500 + K * dil)


@gpu
def test_input_pitch_view():
    """q / k / v style: the input is a Cin-channel view of a wider row (NaN in the rest of the row)"""
    run_case("pitch view", Cin=64, Cout=64, K=1, G=2, L=200, in_extra=128, out_extra=64, epi=EPI_BIAS, pro=PRO_NONE,
             seed=600)


# ================================================================================================ geometry
@gpu
@pytest.mark.parametrize("H,W", [(1, 13), (9, 1), (1, 1), (7, 24)])
def test_conv2d_edges(H, W):
    run_case(f"3x3 {H}x{W}", kind=1, Cin=64, Cout=64, G=2, L=H * W, Wreal=W, epi=EPI_RES, res=True, seed=700 + H * W)


@gpu
@pytest.mark.parametrize("W,strip", [(50, 16), (12, 16), (100, 32)])
def test_conv2d_strips(W, strip):
    """strip mode: Wreal % strip_w != 0 and Wreal < strip_w"""
    run_case(f"strips W {W} / {strip}", kind=1, Cin=32, Cout=64, G=2, L=6 * W, Wreal=W, strip_w=strip, epi=EPI_RES,
             res=True, seed=800 + W)


@gpu
@pytest.mark.parametrize("u,K", [(8, 16), (2, 4), (4, 8), (5, 11), (2, 5)])
def test_conv_transpose(u, K):
    """polyphase ConvTranspose1d(K, u, padding=(K-u)//2); with odd K - u the reference has L*u + 1 samples and the
    primitive computes the first L*u of them"""
    run_case(f"convT u {u} K {K}", kind=2, Cin=64, Cout=32, K=K, u=u, pad=(K - u) // 2, G=2, L=77, epi=EPI_BIAS,
             seed=900 + u * K)


@gpu
@pytest.mark.parametrize("g,K", [(2, 7), (2, 11), (4, 7), (4, 11)])
def test_grouped(g, K):
    """time-grouped conv (block-Toeplitz packing) against the plain conv1d"""
    run_case(f"grouped g {g} K {K}", kind=3, Cin=32, Cout=32, K=K, g=g, G=2, L=4 * 100, epi=EPI_RES, res=True,
             seed=1000 + g * K)


# ================================================================================================ tiles
TILES = [  # (BN, MT, Cout, G)
    (128, 128, 100, 2), (96, 128, 640, 2), (64, 128, 40, 2), (32, 128, 32, 2), (64, 256, 40, 3), (32, 256, 32, 3),
]


@gpu
@pytest.mark.parametrize("bn,mt,Cout,G", TILES)
@pytest.mark.parametrize("plane", [0, 1])
def test_tiles(bn, mt, Cout, G, plane):
    """every tile width and height of the wgmma kernel, fp32-fed and plane-fed (Cin % 64 != 0, pitch > Cin, G > 1
    except where one sample fills the SMs); rows chosen from this device's SM count; partial last row and column tiles"""
    tall = 1 if mt == 256 else 0
    L = rows_for(Cout, G, bn, mt, tall)
    Cin = 100 if Cout > 64 else 36
    run_case(f"tile {bn}x{mt} plane {plane}", Cin=Cin, Cout=Cout, K=3, dil=2, G=G, L=L, in_extra=4, epi=EPI_RES,
             res=True, tall=tall, plane_in=plane, paths=("tc",) if plane else ("tc", "fma"),
             expect={"tc": (1, bn, mt, plane, TILE)}, seed=1100 + bn + mt + plane)


@gpu
@pytest.mark.parametrize("mode", ["with", "only"])
def test_plane_output(mode):
    """po_*: the epilogue writes lrelu(out, po_slope) as an operand plane, with or without the fp32 tensor"""
    run_case(f"po-{mode}", Cin=128, Cout=256, K=3, G=2, L=300, epi=EPI_RES, res=True, plane_in=1, po=mode,
             paths=("tc",), seed=1200)


# ================================================================================================ fused pairs
PAIRS = [  # (C, K, dil, tall, plane)
    (128, 3, 1, 0, 0), (128, 11, 5, 0, 0), (64, 7, 3, 0, 0), (64, 3, 3, 1, 0), (32, 11, 5, 1, 0), (32, 7, 1, 0, 0),
]


@gpu
@pytest.mark.parametrize("C,K,dil,tall,plane", PAIRS)
@pytest.mark.parametrize("epi,acc", [(EPI_RES, 0), (EPI_ACC, 0), (EPI_ACC, 1)])
def test_pairs(C, K, dil, tall, plane, epi, acc):
    """fused ResBlock1 pair, x + c2(lrelu(c1(lrelu(x)))), at BN 128 / 64 / 32 and MT 128 / 256"""
    bn = native_bn(C)
    s = sms()
    if tall:   # enough 256-row tiles (MT - span(c2) outputs each) to fill every SM four times
        G = 4
        L = cdiv(4 * s, G) * (256 - (K - 1)) - 5
    else:
        G, L = 2, 300
    run_case(f"pair C {C} K {K} d {dil}", Cin=C, Cout=C, K=K, dil=dil, G=G, L=L, epi=epi, res=True, accumulate=acc,
             scale=1 / 3 if epi == EPI_ACC else 1.0, tall=tall, plane_in=plane, pair=dict(K2=K), paths=("tc",),
             expect={"tc": (1, bn, 256 if tall else 128, plane, TILE)}, seed=1300 + C + K + epi + acc)


@gpu
@pytest.mark.parametrize("L", [1, 2, 100, 118, 129, 300])
def test_pair_lengths(L):
    """pair tiles keep MT - span(c2) rows: lengths from 1 to past one tile"""
    run_case(f"pair L {L}", Cin=64, Cout=64, K=11, dil=1, G=2, L=L, epi=EPI_RES, res=True, pair=dict(K2=11),
             paths=("tc",), expect={"tc": (1, 64, 128, 0, TILE)}, seed=1400 + L)


@gpu
def test_probe_rejects_what_it_cannot_run():
    x = torch.zeros(2, 64, 32, device=DEV)
    y = torch.zeros(2, 64, 32, device=DEV)
    w = torch.zeros(32, 32, 3)
    base = dict(kind=0, Cin=32, Cout=32, K=3, w=w.data_ptr(), G=2, L=64, inp=x, in_gstride=64 * 32, in_pitch=32, out=y,
                out_gstride=64 * 32, out_pitch=32, epi=EPI_BIAS)
    with pytest.raises(RuntimeError, match="plane input"):
        probe(**dict(base, pro=PRO_SILU, plane_in=1))
    with pytest.raises(RuntimeError, match="pair"):
        probe(**dict(base, pro=PRO_LRELU, pair=1, w2=w.data_ptr(), K2=3, fma=1, res=x, res_gstride=64 * 32, res_pitch=32))
    pair = dict(base, pro=PRO_LRELU, pair=1, w2=w.data_ptr(), K2=3, res=x, res_gstride=64 * 32, res_pitch=32)
    with pytest.raises(RuntimeError, match="pair"):
        probe(**dict(pair, plane_in=1))
    with pytest.raises(RuntimeError, match="pair"):
        probe(**dict(pair, po_hi=y, po_lo=y))
    # agpt_tapconv_probe: the same launch without switches, reporting 4 ints
    ran4 = (C.c_int * 5)(*([-7] * 5))
    a = _lib.TapconvProbeArgs(**{k: (v.data_ptr() if isinstance(v, torch.Tensor) else v) for k, v in base.items()})
    a.scale, a.slope, a.dil, a.dil2 = 1.0, 0.1, 1, 1
    _lib.check(_lib.lib().agpt_tapconv_probe(C.byref(a), ran4, _lib.cur_stream()))
    assert tuple(ran4) == probe(**base)[:4] + (-7,)   # the fifth int is the caller's, untouched
    with pytest.raises(RuntimeError, match="pipeline switches"):
        probe(**dict(base, pro=PRO_LRELU, fma=1, tc_pipe=1))
    with pytest.raises(RuntimeError, match="grouped pair"):
        probe(**dict(pair, kind=3, g=2, dil2=2))


# ================================================================================================ pipelines
# The persistent and two-CTA kernels HiFi-GAN runs nearly every tap-GEMM launch on, selected through the probe's
# switches as Hifigan::forward sets them.  Each case is checked against float64, asserts the full `ran` (the kernel
# family included), and must be bit-identical to the same call with every switch off and tall = 0: tcpair_kernel<BN,
# 128> for the pairs, tcconv5_pl_kernel<128, 128> for the conv pipeline.  Tile counts come from this device's SM
# count s through the launchers' own formulas.
PAIR_SW = ("tc_dual", "tc_pipe", "tc_narrow_pipe")    # what the HiFi-GAN driver sets on every fused pair
K_MAX_DYN = 227 * 1024 - 256                         # kMaxDyn (tcconv5.cu)


def pair_span(K, dil=1, g=1):
    """span(c2) of tc5_rows: the tap span in rows of the view, (K - 1) dil, or the super-tap span of pack_conv_grouped"""
    if g == 1:
        return (K - 1) * dil
    c = (K - 1) // 2
    return (g - 1 + K - 1 - c) // g - (-c) // g


def pair_rows(tiles, K, g=1, G=1):
    """L with cdiv(L / g, 128 - span2) * G == tiles (tiles % G == 0), the last tile of each sample two-thirds full"""
    mto = 128 - pair_span(K, 1, g)
    n = tiles // G
    return (n * mto - mto // 3) * g


def tile_counts():
    s = sms()
    return [1, s - 1, s, s + 1, 2 * s + 1, 3 * s]


def narrow_plan(C, K, dil):
    """tcpair_narrow_try's shared-memory plan of a C-channel pair (c2: K taps, dilation 1): ("resident", sets) where
    every weight stage of c1 and c2 fits beside two sets, else ("ring", stages) beside two sets"""
    bn, iters = native_bn(C), 2 * K
    r1 = cdiv(128 + (K - 1) * dil, 8) * 8
    wbytes, set_ = 2 * bn * 128, 256 * r1 + 128 * cdiv(C, 32) * r1
    avail = K_MAX_DYN - 1024 - (2 * 22 + 4 * 4) * 8
    if avail - iters * wbytes >= 2 * set_:
        return "resident", min(4, (avail - iters * wbytes) // set_)
    return "ring", min(iters, (avail - 2 * set_) // wbytes)


def run_pair(name, C, K, dil, family, G=2, L=300, g=1, epi=EPI_RES, acc=0, res=True, in_extra=0, gpad=0, seed=0,
             switches=PAIR_SW):
    """one fused ResBlock pair (c2: K taps, dilation 1) on the kernel `family` (BN = the pair's native width)"""
    bn = native_bn(g * C)
    run_case(name, kind=3 if g > 1 else 0, Cin=C, Cout=C, K=K, dil=dil, g=g, G=G, L=L, epi=epi, res=res,
             accumulate=acc, scale=1 / 3 if epi == EPI_ACC else 1.0, in_extra=in_extra, gpad=gpad, pair=dict(K2=K),
             paths=("tc",), switches=switches, expect={"tc": (1, bn, 128, 0, family)}, seed=seed)


# ---- tcpair_pipe_kernel: C = 128 pairs and the time-grouped narrow pairs (128 -> 128 channels in the grouped view)
@gpu
@pytest.mark.parametrize("K,dil", [(k, d) for k in (3, 7, 11) for d in (1, 3, 5)])
def test_pair_pipe_taps(K, dil):
    """every C = 128 ResBlock pair of HiFi-GAN V1; k = 11 / d = 5 (c1 spans 50 rows) does not fit two operand sets and
    four weight half-stages, declines and runs tcpair_kernel<128, 128>"""
    run_pair(f"pipe k {K} d {dil}", 128, K, dil, TILE if (K, dil) == (11, 5) else PAIR_PIPE, seed=2000 + K * dil)


@gpu
@pytest.mark.parametrize("C,g,K", [(64, 2, 11), (32, 4, 7), (32, 4, 11)])
def test_pair_pipe_grouped(C, g, K):
    """a time-grouped pair (kind 3, dilation 1): both convs over the [L/g][g C] view, packed to 128 -> 128"""
    run_pair(f"pipe grouped C {C} g {g} k {K}", C, K, 1, PAIR_PIPE, g=g, L=pair_rows(2 * sms() + 2, K, g, 2),
             seed=2100 + C + K)


@gpu
@pytest.mark.parametrize("i", range(8))
def test_pair_pipe_tiles(i):
    """tiles = 1, s - 1, s, s + 1, 2 s + 1, 3 s over one sample (odd and even tiles per CTA), and 3 samples whose
    walk crosses sample boundaries; the last tile of every sample partial"""
    T, G = (tile_counts() + [3 * cdiv(sms() + 1, 3), 3 * cdiv(2 * sms() + 1, 3)])[i], 1 if i < 6 else 3
    run_pair(f"pipe tiles {T} G {G}", 128, 3, 3, PAIR_PIPE, G=G, L=pair_rows(T, 3, 1, G), gpad=8, seed=2200 + i)


@gpu
@pytest.mark.parametrize("L", [1, 2])
@pytest.mark.parametrize("G", [1, 3])
def test_pair_pipe_lengths(L, G):
    run_pair(f"pipe L {L} G {G}", 128, 7, 3, PAIR_PIPE, G=G, L=L, seed=2300 + L + G)


@gpu
@pytest.mark.parametrize("epi,acc", [(EPI_RES, 0), (EPI_ACC, 0), (EPI_ACC, 1)])
@pytest.mark.parametrize("res", [True, "own"])
def test_pair_pipe_epilogues(epi, acc, res):
    """EPI_RES, and EPI_ACC (the MRF sum at scale 1/3, accumulate 0 / 1); the residual the input or a tensor of its own"""
    run_pair(f"pipe epi {EPI_NAMES[epi]} acc {acc} res {res}", 128, 7, 1, PAIR_PIPE, G=3, L=pair_rows(sms() + 2, 7, 1, 1),
             epi=epi, acc=acc, res=res, seed=2400 + epi + 2 * acc + (res == "own"))


# ---- tcpair_narrow_kernel<64 / 32>: the residual read from the TMA-staged input rows
@gpu
@pytest.mark.parametrize("C,K,dil", [(64, k, d) for k in (3, 7) for d in (1, 3, 5)] +
                         [(32, k, d) for k in (3, 7, 11) for d in (1, 3, 5)])
def test_narrow_taps(C, K, dil):
    run_pair(f"narrow C {C} k {K} d {dil}", C, K, dil, NARROW_PIPE, seed=2500 + C + K * dil)


@gpu
@pytest.mark.parametrize("C", [16, 8])
def test_narrow_partial_box(C):
    """C < 32 at BN = 32: the 32-channel TMA box reaches past the tensor's channels (zero fill)"""
    run_pair(f"narrow C {C}", C, 7, 3, NARROW_PIPE, G=3, L=500, seed=2600 + C)


@gpu
@pytest.mark.parametrize("C", [64, 32])
def test_narrow_own_residual_runs_tcpair2(C):
    """a residual that is not the pair's input cannot be read from the staged rows: the narrow kernel declines and
    tcpair2_kernel runs"""
    run_pair(f"narrow own res C {C}", C, 3, 3, DUAL, res="own", seed=2700 + C)


@gpu
@pytest.mark.parametrize("C,K,dil,branch", [(32, 3, 1, "resident"), (32, 7, 1, "resident"), (64, 3, 5, "ring"),
                                            (32, 11, 5, "ring")])
def test_narrow_smem_plans(C, K, dil, branch):
    """both sides of the shared-memory plan (narrow_layout): C = 32, k = 3 keeps all 6 weight stages resident beside 3
    sets and k = 7, d = 1 all 14 beside 2; C = 64, k = 3, d = 5 streams a 5-stage ring with 2 sets, and C = 32,
    k = 11, d = 5 a 10-stage ring"""
    assert narrow_plan(C, K, dil)[0] == branch, narrow_plan(C, K, dil)
    run_pair(f"narrow {branch} {narrow_plan(C, K, dil)} C {C} k {K} d {dil}", C, K, dil, NARROW_PIPE, G=3,
             L=pair_rows(sms() + 3, K, 1, 3), seed=2800 + C + K + dil)


@gpu
def test_narrow_padded_pitch():
    """an input (and so residual) pitch of C + 4 floats: the TMA rows skip the padding, which holds NaN"""
    run_pair("narrow pitch 68", 64, 7, 3, NARROW_PIPE, G=3, L=400, in_extra=4, gpad=8, seed=2900)


@gpu
def test_narrow_pitch_tma_cannot_encode_is_refused():
    """a pitch that is not a multiple of 4 floats (16 bytes) is one TMA cannot encode; tcconv_supported refuses it
    first for every tensor-core pair, so no pair launch is taken (no narrow kernel, no tcpair2 fall-back)"""
    with pytest.raises(RuntimeError, match="pair launch was not taken"):
        run_pair("narrow pitch 66", 64, 3, 1, NARROW_PIPE, in_extra=2, seed=2901)


@gpu
@pytest.mark.parametrize("i", range(8))
def test_narrow_tiles(i):
    T, G = (tile_counts() + [3 * cdiv(sms() + 1, 3), 3 * cdiv(2 * sms() + 1, 3)])[i], 1 if i < 6 else 3
    run_pair(f"narrow tiles {T} G {G}", 32, 7, 3, NARROW_PIPE, G=G, L=pair_rows(T, 7, 1, G), gpad=8, seed=3000 + i)


@gpu
@pytest.mark.parametrize("C,K,dil", [(64, 3, 3), (32, 11, 5)])
@pytest.mark.parametrize("epi,acc", [(EPI_RES, 0), (EPI_ACC, 0), (EPI_ACC, 1)])
def test_narrow_epilogues(C, K, dil, epi, acc):
    run_pair(f"narrow epi {EPI_NAMES[epi]} acc {acc} C {C}", C, K, dil, NARROW_PIPE, G=3, L=333, epi=epi, acc=acc,
             seed=3100 + C + K + epi + 2 * acc)


@gpu
@pytest.mark.parametrize("L", [1, 2])
def test_narrow_lengths(L):
    run_pair(f"narrow L {L}", 32, 11, 5, NARROW_PIPE, G=3, L=L, seed=3200 + L)


# ---- tcpair2_kernel<64 / 32>: two 128-row CTAs per SM
@gpu
@pytest.mark.parametrize("dil", [1, 3, 5])
def test_dual_k11(dil):
    """C = 64, k = 11: 22 weight stages per tile, past the narrow kernel's 14"""
    run_pair(f"dual k 11 d {dil}", 64, 11, dil, DUAL, seed=3300 + dil)


@gpu
@pytest.mark.parametrize("C,K,dil", [(32, 7, 3), (64, 11, 3)])
@pytest.mark.parametrize("epi,acc", [(EPI_RES, 0), (EPI_ACC, 1)])
def test_dual_own_residual(C, K, dil, epi, acc):
    run_pair(f"dual own res C {C} k {K}", C, K, dil, DUAL, G=3, L=321, epi=epi, acc=acc, res="own",
             seed=3400 + C + K + epi)


@gpu
@pytest.mark.parametrize("i", range(8))
def test_dual_tiles(i):
    T, G = (tile_counts() + [3 * cdiv(sms() + 1, 3), 3 * cdiv(2 * sms() + 1, 3)])[i], 1 if i < 6 else 3
    run_pair(f"dual tiles {T} G {G}", 64, 11, 3, DUAL, G=G, L=pair_rows(T, 11, 1, G), gpad=8, seed=3500 + i)


# ---- tcconv_pipe_pl_kernel: plane-fed, BN = 128, 128-row tiles
def conv_units(cout, rows_v, G):
    return cdiv(rows_v, 128) * G * cdiv(cout, 128)


def conv_pipe_rows(cout, G, want):
    """the smallest L = 128 n - 37 (a partial last row tile) for which pick_h_tile lands on BN = 128, MT = 128 and the
    units satisfy want(units, s)"""
    s = sms()
    for n in range(1, 4000):
        L = 128 * n - 37
        if pick_tile(cout, L, G, 0) == (128, 128) and want(conv_units(cout, L, G), s):
            return L
    raise AssertionError(f"no L lands on the conv pipeline for Cout {cout}, G {G} on {s} SMs")


def run_conv_pipe(name, Cin, Cout, K, dil, G, L, epi, po, family=CONV_PIPE, bn=128, acc=0, kind=0, u=1, seed=0):
    res = epi in (EPI_RES, EPI_ACC)
    run_case(name, kind=kind, Cin=Cin, Cout=Cout, K=K, dil=dil, u=u, pad=(K - u) // 2 if kind == 2 else 0, G=G, L=L,
             epi=epi, res=res, accumulate=acc, scale=1 / 3 if epi == EPI_ACC else 1.0, plane_in=1, po=po,
             paths=("tc",), switches=("tc_conv_pipe",), expect={"tc": (1, bn, 128, 1, family)}, seed=seed)


@gpu
@pytest.mark.parametrize("K,dil", [(k, d) for k in (3, 7, 11) for d in (1, 3, 5)])
@pytest.mark.parametrize("conv", ["c1", "c2"])
def test_conv_pipe_resblock(K, dil, conv):
    """HiFi-GAN V1's C = 256 ResBlock convs: c1 (EPI_BIAS, only the operand plane of its output) and c2 (EPI_RES into
    the next residual, fp32 and plane); two 128-wide column units"""
    L = conv_pipe_rows(256, 2, lambda n, s: n >= 3 * s)
    if conv == "c1":
        run_conv_pipe(f"cpipe c1 k {K} d {dil}", 256, 256, K, dil, 2, L, EPI_BIAS, "only", seed=3600 + K * dil)
    else:
        run_conv_pipe(f"cpipe c2 k {K} d {dil}", 256, 256, K, dil, 2, L, EPI_RES, "with", seed=3700 + K * dil)


@gpu
@pytest.mark.parametrize("Cin,Cout", [(512, 256), (256, 128)])
def test_conv_pipe_upsamplers(Cin, Cout):
    """the plane-fed upsamplers as kind 2 (u = 8, K = 16): [L][8 Cout] rows, 16 / 8 column units"""
    L = conv_pipe_rows(8 * Cout, 1, lambda n, s: n >= 2 * s)
    run_conv_pipe(f"cpipe up {Cin}->{Cout}", Cin, Cout, 16, 1, 1, L, EPI_BIAS, "with" if Cout > 128 else None, kind=2,
                  u=8, seed=3800 + Cin)


@gpu
@pytest.mark.parametrize("Cin,K,dil", [(128, 3, 1), (256, 3, 1), (512, 3, 1), (256, 11, 5)])
def test_conv_pipe_buffers(Cin, K, dil):
    """Cin = 128 / 256 / 512: 2, 4 and (capped) 4 operand buffers; k = 11, d = 5: the 2-buffer, 4-stage plan"""
    L = conv_pipe_rows(256, 2, lambda n, s: n >= s)
    run_conv_pipe(f"cpipe Cin {Cin} k {K} d {dil}", Cin, 256, K, dil, 2, L, EPI_RES, "with", seed=3900 + Cin + K)


CPIPE_UNITS = {   # name -> (Cout, G, units predicate): pick_h_tile keeps BN = 128 only where narrower tiles do not
    "s/2 < units < s": (256, 1, lambda n, s: 2 * n > s and n < s),    # need fewer waves per tile cost
    "units = s": (128, 1, lambda n, s: n == s),
    "s < units < 2 s": (256, 3, lambda n, s: s < n < 2 * s),
    "units = 2 s": (256, 1, lambda n, s: n == 2 * s),
    "many units": (256, 3, lambda n, s: n >= 7 * s),
}


@gpu
@pytest.mark.parametrize("what", list(CPIPE_UNITS))
def test_conv_pipe_units(what):
    """unit counts against the SM count s: fewer than s (one unit per CTA), s, past one wave, many.  The half-unit grid
    of cpipe_grid (units <= s / 2) is not reachable through tcconv5_launch: pick_h_tile chooses 64-wide tiles there
    (test_conv_pipe_declines)."""
    Cout, G, want = CPIPE_UNITS[what]
    L = conv_pipe_rows(Cout, G, want)
    run_conv_pipe(f"cpipe {what} ({conv_units(Cout, L, G)} units)", 128, Cout, 7, 3, G, L, EPI_ACC, "with", acc=1,
                  seed=4000 + len(what))


@gpu
@pytest.mark.parametrize("acc", [0, 1])
def test_conv_pipe_accumulate(acc):
    L = conv_pipe_rows(256, 2, lambda n, s: n >= 2 * s)
    run_conv_pipe(f"cpipe acc {acc}", 256, 256, 11, 3, 2, L, EPI_ACC, None, acc=acc, seed=4100 + acc)


@gpu
@pytest.mark.parametrize("what", ["tanh", "bn64", "bn96"])
def test_conv_pipe_declines(what):
    """EPI_TANH is not a pipeline epilogue: tcconv5_pl_kernel<128, 128>.  Units <= s / 2 (Cout 128: 64-wide tiles fill
    the SMs in one wave) and a Cout 256 launch whose 96-wide tiles take one wave where 128-wide take two: tcconv5_pl at
    that BN"""
    s = sms()
    if what == "tanh":
        L = conv_pipe_rows(256, 2, lambda n, s_: n >= s_)
        run_conv_pipe("cpipe decline tanh", 256, 256, 3, 1, 2, L, EPI_TANH, None, family=TILE, seed=4200)
        return
    cout, bn = (128, 64) if what == "bn64" else (256, 96)
    L = next(128 * n - 37 for n in range(1, 4000) if pick_tile(cout, 128 * n - 37, 1, 0) == (bn, 128))
    assert what != "bn64" or 2 * conv_units(cout, L, 1) <= s
    run_conv_pipe(f"cpipe decline {what}", 256, cout, 3, 1, 1, L, EPI_RES, None, family=TILE, bn=bn, seed=4201 + bn)


# ================================================================================================ mutants (CPU)
# Each plausible pipeline bug, applied to the float64 reference of a pair (CPU), must fail the gate the kernels pass.
MUTANTS = ["res_row", "halo_zero", "straddle", "ring_slot", "acc_ignored", "lo_dropped", "phases", "unstored"]


def mutant_pair(mutant, seed=7):
    """(mutated fp32 output, float64 reference, bound) of a ResBlock pair, x + c2(lrelu(c1(lrelu(x)))) (EPI_ACC at
    scale 1/3 with accumulate = 1 for the MRF mutant), with tiles of 128 - span2 output rows"""
    g = 2 if mutant == "phases" else 1
    # C = 32 for the dropped lo plane: at C = 128 the bound of the other chunk's products and of the two 3-tap convs
    # hides it (error 0.12 x the bound); there only the bit-identity with the sibling kernel catches it
    C = 32 if mutant == "lo_dropped" else (64 if g > 1 else 128)
    G, K, dil = 2, 3, 3 if g == 1 else 1
    L = 300
    gr = torch.Generator().manual_seed(seed)
    x = torch.randn(G, L, C, generator=gr, dtype=torch.float64)
    w1 = torch.randn(C, C, K, generator=gr, dtype=torch.float64) / math.sqrt(C * K)
    w2 = torch.randn(C, C, K, generator=gr, dtype=torch.float64) / math.sqrt(C * K)
    b1, b2 = 0.05 * torch.randn(C, generator=gr, dtype=torch.float64), 0.05 * torch.randn(C, generator=gr, dtype=torch.float64)
    old = torch.randn(G, L, C, generator=gr, dtype=torch.float64)
    sp = dict(kind=3 if g > 1 else 0, dil=dil, g=g, u=1, dil2=1)
    acc = mutant == "acc_ignored"
    slope = 0.1

    def pair(xx, ww1=w1):
        return pair_reference(sp, F.leaky_relu(xx, slope), ww1, b1, w2, b2, slope, True)

    vv, Ev = pair(x)
    if acc:
        ref = (vv + x) / 3 + old
        E = (Ev + EPS32 * (vv + x).abs()) / 3 + EPS32 * ((vv + x).abs() / 3 + ref.abs())
    else:
        ref, E = vv + x, Ev + EPS32 * (vv + x).abs()
    mto = 128 - pair_span(K, 1, g)
    y = ref.clone()
    if mutant == "res_row":          # the staged residual read one row off
        y = vv + torch.cat([x[:, 1:], torch.zeros_like(x[:, :1])], dim=1)
    elif mutant == "halo_zero":      # each tile after the first computed as if it started the sequence
        for t0 in range(mto, L, mto):
            y[:, t0:t0 + mto] = pair(x[:, t0:])[0][:, :mto] + x[:, t0:t0 + mto]
    elif mutant == "straddle":       # the last tile of a sample takes its right halo from the next sample
        y[0] = pair(torch.cat([x[0], x[1]])[None])[0][0, :L] + x[0]
    elif mutant == "ring_slot":      # tap 1 of the second 64-channel chunk uses the weights of the previous ring slot
        wm = w1.clone()
        wm[:, 64:, 1] = w1[:, 64:, 0]
        y = pair(x, wm)[0] + x
    elif mutant == "acc_ignored":    # the old MRF sum not added
        y = (vv + x) / 3
    elif mutant == "lo_dropped":     # c1's (only) 64-channel chunk fed its fp16 hi part only
        xm = F.leaky_relu(x, slope).float().half().double()
        y = pair_reference(sp, xm, w1, b1, w2, b2, slope, True)[0] + x
    elif mutant == "phases":         # the g phases of the grouped view transposed
        y = ref.view(G, L // g, g, C).flip(2).reshape(G, L, C)
    elif mutant == "unstored":       # one tile of a CTA's walk not stored: the NaN canary stays
        y[1, mto:2 * mto] = NAN
    return y.float(), ref, E


def test_mutant_reference_passes_the_gate():
    for mutant in ("res_row", "phases", "acc_ignored", "lo_dropped"):   # the four reference configurations
        _, ref, E = mutant_pair(mutant)
        assert verdict(ref.float(), ref, E)[0] is None


@pytest.mark.parametrize("mutant", MUTANTS)
def test_gate_catches_pipeline_mutants(mutant):
    y, ref, E = mutant_pair(mutant)
    fail = verdict(y, ref, E)[0]
    assert fail is not None, f"{mutant}: passes the gate"
    if mutant == "unstored":
        assert fail.startswith("unwritten"), fail
