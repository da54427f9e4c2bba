"""CPU emulation of the tensor-core arithmetic of csrc/tcconv5.cu / attention_tc.cu ("3 x fp16 parts"):
documents the error bound the GPU parity tests rely on, without a GPU.

x = x_hi + x_lo (x_hi = fp16(x) with saturation, x_lo = fp16(x - x_hi)); weights the same after a per-layer
power-of-two scale that puts max|w| into [2^13, 2^14); y = sum x_hi w_hi + x_lo w_hi + x_hi w_lo in fp32."""
import numpy as np


def split_fp16(v):
    hi = np.clip(v, -65504.0, 65504.0).astype(np.float16)
    lo = np.clip(v - hi.astype(np.float32), -65504.0, 65504.0).astype(np.float16)   # cvt.rn.satfinite on both parts
    return hi.astype(np.float32), lo.astype(np.float32)


def weight_scale(w):
    mx = float(np.abs(w).max())
    if mx == 0.0:
        return 1.0
    _, e = np.frexp(np.float32(mx))          # mx = m * 2^e, m in [0.5, 1)
    return float(np.ldexp(1.0, int(np.clip(14 - e, -60, 60))))


def emulate(x, w):
    s = weight_scale(w)
    xh, xl = split_fp16(x.astype(np.float32))
    wh, wl = split_fp16((w * s).astype(np.float32))
    acc = (xh @ wh).astype(np.float32) + (xl @ wh).astype(np.float32) + (xh @ wl).astype(np.float32)
    return (acc / s).astype(np.float32)


def test_three_product_split_is_fp32_grade():
    rng = np.random.RandomState(0)
    for scale_x, scale_w, K in ((1.0, 0.05, 1408), (30.0, 0.01, 320), (1e-3, 2.0, 64), (5.0, 1e-4, 2880)):
        x = (rng.randn(64, K) * scale_x).astype(np.float32)
        w = (rng.randn(K, 48) * scale_w).astype(np.float32)
        ref = x.astype(np.float64) @ w.astype(np.float64)
        y = emulate(x, w)
        y32 = (x @ w).astype(np.float32)                           # plain fp32 GEMM for comparison
        den = np.sqrt((ref ** 2).mean())
        e3 = np.sqrt(((y - ref) ** 2).mean()) / den
        e32 = np.sqrt(((y32 - ref) ** 2).mean()) / den
        # single-pass fp16 (what kind::f16 alone would give) is ~3 orders of magnitude worse
        xh, _ = split_fp16(x)
        wh, _ = split_fp16((w * weight_scale(w)).astype(np.float32))
        e1 = np.sqrt((((xh @ wh) / weight_scale(w) - ref) ** 2).mean()) / den
        if scale_x >= 0.1:
            assert e3 < 2e-6, (scale_x, scale_w, K, e3)            # 2^-22 per term, averaged over K terms
            assert e3 < 20 * max(e32, 1e-8)                        # = what a plain fp32 GEMM gives
        else:
            # activations of order 1e-3: the lo part is an fp16 subnormal, absolute error floor 2^-25 per element
            # (DESIGN.md section 2) -- still well inside the 1e-4 bound, and no layer on this path is that small
            assert e3 < 5e-5, (scale_x, e3)
        assert e1 > 15 * e3


def test_weight_prescale_keeps_both_parts_normal_and_is_exact():
    rng = np.random.RandomState(1)
    for mag in (1e-6, 3e-3, 0.7, 40.0):
        w = (rng.randn(256, 16) * mag).astype(np.float32)
        s = weight_scale(w)
        assert np.log2(s) == np.round(np.log2(s))                  # power of two: scaling and un-scaling are exact
        mx = np.abs(w * s).max()
        assert 2.0 ** 13 <= mx < 2.0 ** 14
        wh, wl = split_fp16((w * s).astype(np.float32))
        big = np.abs(w * s) > 2.0 ** -3                            # everything down to max / 2^17 has a normal lo part
        rel = np.abs((wh + wl) - w * s)[big] / np.abs(w * s)[big]
        assert rel.max() < 2.0 ** -21


def test_activation_split_error_floor_and_saturation():
    x = np.array([1e-9, 3e-6, 1e-4, 0.11, 1.0, 777.7, 65504.0, 1e6, -1e6], dtype=np.float32)
    hi, lo = split_fp16(x)
    ok = np.abs(x) <= 65504
    err = np.abs((hi + lo) - x)[ok]
    tol = np.maximum(np.abs(x[ok]) * 2.0 ** -21, 2.0 ** -24)
    assert (err <= tol).all()
    assert np.isfinite(hi).all() and np.isfinite(lo).all()        # |x| > 65504 saturates instead of overflowing
