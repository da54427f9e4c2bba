"""Conformance of the tap-GEMM primitive (tapconv_launch, the fused pair launch) against a float64 reference.

Every case runs ONE production launch through agpt_tapconv_probe -- the production weight packer, launch parameters as
given, caller-owned device tensors -- and compares it with torch.nn.functional in float64 on the device (conv1d /
conv2d / conv_transpose1d on the torch weight layouts, then the prologue and epilogue formulas of the reference
modules), written without any of the kernels' packing.  `ran`, what the probe reports as launched, is asserted for
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
"""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from audiogpt_b200 import _lib

pytestmark = pytest.mark.gpu

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

EXERCISED = {}          # (kernel, BN, MT, plane-fed) -> worst error / bound over the cases that ran it


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    if EXERCISED:
        print("\ntap-GEMM variants exercised (kernel, BN, MT, plane-fed): worst error / bound")
        for k in sorted(EXERCISED):
            print(f"  {'wgmma' if k[0] == 1 else 'fma  '} BN {k[1]:3d} MT {k[2]:3d} plane {k[3]}: {EXERCISED[k]:.3f}")


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
    a = _lib.TapconvProbeArgs()
    a.scale, a.slope, a.dil, a.dil2 = 1.0, 0.1, 1, 1
    for k, v in kw.items():
        if isinstance(v, torch.Tensor):
            v = v.data_ptr()
        setattr(a, k, v)
    ran = (C.c_int * 4)()
    _lib.check(_lib.lib().agpt_tapconv_probe(C.byref(a), ran, _lib.cur_stream()))
    return tuple(ran)


def check(name, y, ref, bound, path, ran):
    """assert |y - ref| <= bound element-wise and rms(err) <= rms(bound) / 2; returns the worst ratio"""
    y = y.double()
    assert torch.isfinite(y).all(), f"{name} [{path}]: non-finite output"
    err = (y - ref).abs()
    bound = bound + 1e-300
    ratio = float((err / bound).max())
    rms_ratio = float(err.pow(2).mean().sqrt() / bound.pow(2).mean().sqrt())
    print(f"{name} [{path} ran={ran}]: worst err/bound {ratio:.3f}, rms err/rms bound {rms_ratio:.3f}")
    k = (ran[0], ran[1], ran[2], ran[3])
    EXERCISED[k] = max(EXERCISED.get(k, 0.0), ratio)
    assert ratio <= 1.0, f"{name} [{path}]: error {ratio:.3g} x the bound"
    assert rms_ratio <= 0.5, f"{name} [{path}]: rms error {rms_ratio:.3g} x the rms bound"
    return ratio


# ------------------------------------------------------------------------------------------------ one case
def run_case(name, kind=0, Cin=64, Cout=64, K=3, dil=1, G=2, L=200, Wreal=0, strip_w=0, u=1, pad=0, g=1,
             pro=PRO_LRELU, slope=0.1, epi=EPI_BIAS, bias=True, res=False, scale=1.0, accumulate=0, csplit=0,
             in_extra=0, out_extra=0, gpad=0, paths=("tc", "fma"), tall=0, plane_in=0, po=None, pl=None, pair=None,
             x_scale=1.0, w_spread=1.0, expect=None, seed=0, stats=None):
    """Run one launch per path in `paths` and check it (see the module docstring).  expect: {path: (tc, BN, MT,
    plane)} asserted against `ran`; po / pl: None, "with" (and the fp32 tensor) or "only" (out = NULL).  stats: a
    dict that receives the worst {max |err| / rms(ref), rms(err) / rms(ref)} of the fp32 output over the paths."""
    sp = dict(kind=kind, dil=dil, Wreal=Wreal, u=u, pad=pad, g=g)
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
    if pair:   # a ResBlock pair adds its own input: x + c2(lrelu(c1(lrelu(x))))
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
            Eb1, _ = conv_bound(sp, xp, wref, tc, mask)
            h = F.leaky_relu(v, slope)
            E_h = Eb1 + EPS32 * v.abs()
            sp2 = dict(kind=0, dil=pair.get("dil2", 1), u=1, g=1)
            vc2 = conv_ref(sp2, h, w2.double())
            Eb2, S2 = conv_bound(sp2, h, w2.double(), tc, torch.ones_like(h))
            vv = vc2 + b2.double()
            Ev = Eb2 + conv_ref(sp2, E_h, w2.double().abs()) + EPS32 * (S2 + vv.abs())
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
        # --- output buffers, NaN everywhere but where the kernel must read
        cf = epi == EPI_STORE_CF
        if cf:
            oflat, out_gs = buffer(G, oc, rows, gpad)
        else:
            oflat, out_gs = buffer(G, rows, out_pitch, gpad)
        if old_out is not None:
            view(oflat, G, out_gs, rows, out_pitch, och).copy_(old_out)
        o2flat = None
        if epi == EPI_DIFFOUT:
            o2p = Cout - csplit + out_extra
            o2flat, o2_gs = buffer(G, rows, o2p, gpad)
            if accumulate:
                view(o2flat, G, o2_gs, rows, o2p, Cout - csplit).copy_(old_out2)
        planes = {}
        for key, mode in (("po", po), ("pl", pl)):
            if mode:
                pp = out_pitch
                planes[key] = [torch.full((G * out_gs + GUARD,), NAN, dtype=torch.float16, device=DEV) for _ in range(2)]
        saved_in = bits(xin).clone()
        saved_res = bits(rflat).clone() if resv is not None else None
        saved_pvec = pvec.clone() if pvec is not None else None
        only = (po == "only") or (pl == "only")
        kw = dict(kind=kind, Cin=Cin, Cout=Cout, K=K, dil=dil, Wreal=Wreal, strip_w=strip_w, u=u, pad=pad, g=g,
                  w=w_h.data_ptr(), b=b_h.data_ptr() if bias else None, G=G, L=L,
                  inp=x, in_gstride=in_gs, in_pitch=in_pitch,
                  out=None if only else oflat, out_gstride=out_gs, out_pitch=out_pitch,
                  pro=pro, slope=slope, epi=epi, scale=scale, accumulate=accumulate, csplit=csplit,
                  tc_tall=tall, plane_in=plane_in if tc else 0, fma=0 if tc else 1)
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
        ran = probe(**kw)
        if expect and path in expect:
            assert ran == expect[path], f"{name} [{path}]: ran {ran}, meant to test {expect[path]}"
        elif not tc:
            assert ran == (0, native_bn(g * oc if kind == 3 else oc), 128, 0), f"{name} [fma]: ran {ran}"
        else:
            assert ran[0] == 1 and ran[3] == (1 if plane_in else 0), f"{name} [{path}]: ran {ran}"
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
def test_prologues_1d(pro, slope):
    run_case(f"pro{pro}/{slope}", Cin=36, Cout=40, K=5, dil=3, G=3, L=257, pro=pro, slope=slope, epi=EPI_RES, res=True,
             in_extra=4, seed=pro)


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


@pytest.mark.parametrize("i", range(len(EPI_CASES)))
def test_epilogues(i):
    kw = dict(Cin=80, Cout=96, K=3, dil=1, G=2, L=300, pro=PRO_LRELU)
    kw.update(EPI_CASES[i])
    run_case(f"epi#{i}", seed=100 + i, **kw)


def test_store_cf_2d():
    run_case("store_cf 2d", kind=1, Cin=32, Cout=4, G=2, L=12 * 9, Wreal=9, pro=PRO_SILU, epi=EPI_STORE_CF, seed=120)


@pytest.mark.parametrize("epi", [EPI_GATE, EPI_GEGLU])
@pytest.mark.parametrize("res", [False, True])
def test_gate_epilogues(epi, res):
    run_case(f"pairs {'res' if res else ''}", kind=4, Cin=64, Cout=128, K=3, dil=2, G=2, L=250, pro=PRO_NONE, epi=epi,
             res=res, seed=130 + epi + 2 * res)


@pytest.mark.parametrize("epi", [EPI_GATE, EPI_GEGLU])
@pytest.mark.parametrize("mode", ["with", "only"])
def test_gate_plane_output(epi, mode):
    """The GATE / GEGLU operand-plane output (G == 1: the UNet's GEGLU feeding a plane-fed ff2)"""
    run_case(f"pairs pl-{mode}", kind=4, Cin=320, Cout=640, K=1, G=1, L=333, pro=PRO_NONE, epi=epi, res=(epi == EPI_GATE),
             pl=mode, paths=("tc",), seed=140 + epi)


# ================================================================================================ shapes
@pytest.mark.parametrize("Cin", [1, 2, 4, 8, 36, 64, 80, 100, 320, 1280])
def test_cin(Cin):
    """Cin in {1, 2} (and pitches not a multiple of 4) go to the FMA kernel by tcconv_supported"""
    exp = {"tc": (0, native_bn(40), 128, 0)} if Cin % 4 else None
    run_case(f"Cin {Cin}", Cin=Cin, Cout=40, K=3, G=2, L=131, epi=EPI_RES, res=True, expect=exp, seed=200 + Cin)


@pytest.mark.parametrize("Cout", [4, 32, 40, 96, 100, 256, 320, 640])
def test_cout(Cout):
    run_case(f"Cout {Cout}", Cin=64, Cout=Cout, K=3, G=2, L=129, epi=EPI_BIAS, seed=300 + Cout)


@pytest.mark.parametrize("L", [1, 127, 128, 129, 255, 256, 257, 3001])
@pytest.mark.parametrize("G", [1, 3])
def test_lengths(L, G):
    run_case(f"G {G} L {L}", Cin=32, Cout=32, K=7, dil=3, G=G, L=L, epi=EPI_RES, res=True, gpad=8, seed=400 + L + G)


@pytest.mark.parametrize("K,dil", [(1, 1), (3, 1), (5, 3), (7, 5), (11, 1), (11, 5)])
def test_taps(K, dil):
    run_case(f"K {K} dil {dil}", Cin=64, Cout=64, K=K, dil=dil, G=2, L=300, epi=EPI_RES, res=True, seed=500 + K * dil)


def test_input_pitch_view():
    """q / k / v style: the input is a Cin-channel view of a wider row (NaN in the rest of the row)"""
    run_case("pitch view", Cin=64, Cout=64, K=1, G=2, L=200, in_extra=128, out_extra=64, epi=EPI_BIAS, pro=PRO_NONE,
             seed=600)


# ================================================================================================ geometry
@pytest.mark.parametrize("H,W", [(1, 13), (9, 1), (1, 1), (7, 24)])
def test_conv2d_edges(H, W):
    run_case(f"3x3 {H}x{W}", kind=1, Cin=64, Cout=64, G=2, L=H * W, Wreal=W, epi=EPI_RES, res=True, seed=700 + H * W)


@pytest.mark.parametrize("W,strip", [(50, 16), (12, 16), (100, 32)])
def test_conv2d_strips(W, strip):
    """strip mode: Wreal % strip_w != 0 and Wreal < strip_w"""
    run_case(f"strips W {W} / {strip}", kind=1, Cin=32, Cout=64, G=2, L=6 * W, Wreal=W, strip_w=strip, epi=EPI_RES,
             res=True, seed=800 + W)


@pytest.mark.parametrize("u,K", [(8, 16), (2, 4), (4, 8), (5, 11), (2, 5)])
def test_conv_transpose(u, K):
    """polyphase ConvTranspose1d(K, u, padding=(K-u)//2); with odd K - u the reference has L*u + 1 samples and the
    primitive computes the first L*u of them"""
    run_case(f"convT u {u} K {K}", kind=2, Cin=64, Cout=32, K=K, u=u, pad=(K - u) // 2, G=2, L=77, epi=EPI_BIAS,
             seed=900 + u * K)


@pytest.mark.parametrize("g,K", [(2, 7), (2, 11), (4, 7), (4, 11)])
def test_grouped(g, K):
    """time-grouped conv (block-Toeplitz packing) against the plain conv1d"""
    run_case(f"grouped g {g} K {K}", kind=3, Cin=32, Cout=32, K=K, g=g, G=2, L=4 * 100, epi=EPI_RES, res=True,
             seed=1000 + g * K)


# ================================================================================================ tiles
TILES = [  # (BN, MT, Cout, G)
    (128, 128, 100, 2), (96, 128, 640, 2), (64, 128, 40, 2), (32, 128, 32, 2), (64, 256, 40, 3), (32, 256, 32, 3),
]


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
             expect={"tc": (1, bn, mt, plane)}, seed=1100 + bn + mt + plane)


@pytest.mark.parametrize("mode", ["with", "only"])
def test_plane_output(mode):
    """po_*: the epilogue writes lrelu(out, po_slope) as an operand plane, with or without the fp32 tensor"""
    run_case(f"po-{mode}", Cin=128, Cout=256, K=3, G=2, L=300, epi=EPI_RES, res=True, plane_in=1, po=mode,
             paths=("tc",), seed=1200)


# ================================================================================================ fused pairs
PAIRS = [  # (C, K, dil, tall, plane)
    (128, 3, 1, 0, 0), (128, 11, 5, 0, 0), (64, 7, 3, 0, 0), (64, 3, 3, 1, 0), (32, 11, 5, 1, 0), (32, 7, 1, 0, 0),
]


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
             expect={"tc": (1, bn, 256 if tall else 128, plane)}, seed=1300 + C + K + epi + acc)


@pytest.mark.parametrize("L", [1, 2, 100, 118, 129, 300])
def test_pair_lengths(L):
    """pair tiles keep MT - span(c2) rows: lengths from 1 to past one tile"""
    run_case(f"pair L {L}", Cin=64, Cout=64, K=11, dil=1, G=2, L=L, epi=EPI_RES, res=True, pair=dict(K2=11),
             paths=("tc",), expect={"tc": (1, 64, 128, 0)}, seed=1400 + L)


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
