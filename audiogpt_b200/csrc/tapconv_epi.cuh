// Shared fused epilogue of the tapconv kernels (fp32 FMA version and tensor-core version):
// one call handles 4 consecutive output channels of one output row.  Split in two phases so
// that a kernel can issue the global READS of several items (residual, old accumulator) before
// consuming any of them (memory-level parallelism in the tensor-core epilogue).
#pragma once
#include "tapconv.cuh"
#include "tc_h16.cuh"

namespace agpt {

struct EpiPre {
  float4 a;   // residual / pre-activation additive term / old x (DIFFOUT, co < csplit) / old skip (co >= csplit)
  float4 b;   // old accumulator (EPI_ACC with accumulate)
};

__device__ __forceinline__ void epi_load(const TapConvParams& P, int g, int p, int co, EpiPre& pre) {
  pre.a = make_float4(0.f, 0.f, 0.f, 0.f);
  pre.b = pre.a;
  if (co >= P.Cout) return;
  switch (P.epi) {
    case EPI_RES:
    case EPI_ACC:
    case EPI_GATE:
    case EPI_GEGLU:
      if (P.res) pre.a = __ldg(reinterpret_cast<const float4*>(P.res + g * P.res_gstride + (long)p * P.res_pitch + co));
      if (P.epi == EPI_ACC && P.accumulate)
        pre.b = *reinterpret_cast<const float4*>(P.out + g * P.out_gstride + (long)p * P.out_pitch + co);
      break;
    case EPI_DIFFOUT:
      if (co < P.csplit) pre.a = *reinterpret_cast<const float4*>(P.out + g * P.out_gstride + (long)p * P.out_pitch + co);
      else if (P.accumulate)
        pre.a = *reinterpret_cast<const float4*>(P.out2 + g * P.out2_gstride + (long)p * P.out2_pitch + (co - P.csplit));
      break;
    default: break;
  }
}

// split form for register-tight callers: the additive term early, the old accumulator at use
__device__ __forceinline__ float4 epi_load_a(const TapConvParams& P, int g, int p, int co) {
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  if (co >= P.Cout) return a;
  switch (P.epi) {
    case EPI_RES:
    case EPI_ACC:
    case EPI_GATE:
    case EPI_GEGLU:
      if (P.res) a = __ldg(reinterpret_cast<const float4*>(P.res + g * P.res_gstride + (long)p * P.res_pitch + co));
      break;
    case EPI_DIFFOUT:
      if (co < P.csplit) a = *reinterpret_cast<const float4*>(P.out + g * P.out_gstride + (long)p * P.out_pitch + co);
      else if (P.accumulate)
        a = *reinterpret_cast<const float4*>(P.out2 + g * P.out2_gstride + (long)p * P.out2_pitch + (co - P.csplit));
      break;
    default: break;
  }
  return a;
}
__device__ __forceinline__ float4 epi_load_b(const TapConvParams& P, int g, int p, int co) {
  if (co < P.Cout && P.epi == EPI_ACC && P.accumulate)
    return *reinterpret_cast<const float4*>(P.out + g * P.out_gstride + (long)p * P.out_pitch + co);
  return make_float4(0.f, 0.f, 0.f, 0.f);
}

// per-(sample, output-channel) additive vector: bias (+ the EPI_ADDVEC vector).  Depends on (g, co) only, so
// a caller whose items share the channel group loads it once per block instead of once per item.
__device__ __forceinline__ float4 epi_colvec(const TapConvParams& P, int g, int co) {
  float4 c = make_float4(0.f, 0.f, 0.f, 0.f);
  if (co >= P.Cout) return c;
  if (P.bias) c = __ldg(reinterpret_cast<const float4*>(P.bias + co));
  if (P.epi == EPI_ADDVEC) {
    const float4 e = __ldg(reinterpret_cast<const float4*>(P.evec + (long)g * P.evec_gstride + co));
    c.x += e.x; c.y += e.y; c.z += e.z; c.w += e.w;
  }
  return c;
}

// operand plane of the 4 stored values (TapConvParams::po_hi): exactly pro_apply5 (leaky ReLU) + split2 of the
// transform a PRO_LRELU consumer would run on them
__device__ __forceinline__ void epi_store_plane(const TapConvParams& P, long off, float4 v) {
  v.x = lrelu(v.x, P.po_slope); v.y = lrelu(v.y, P.po_slope); v.z = lrelu(v.z, P.po_slope); v.w = lrelu(v.w, P.po_slope);
  uint2 h, l;
  h.x = split2(v.x, v.y, l.x);
  h.y = split2(v.z, v.w, l.y);
  *reinterpret_cast<uint2*>(P.po_hi + off) = h;
  *reinterpret_cast<uint2*>(P.po_lo + off) = l;
}

// PL: the plane-fed tensor-core kernels, which may write the output as an operand plane too (or only)
template <bool PL = false>
__device__ __forceinline__ void epi_store_cv(const TapConvParams& P, int g, int p, int co, float4 v, const EpiPre& pre,
                                             const float4 cv) {
  if (co >= P.Cout) return;
  v.x += cv.x; v.y += cv.y; v.z += cv.z; v.w += cv.w;
  switch (P.epi) {
    case EPI_BIAS: break;
    case EPI_RES:
    case EPI_ACC: {
      v.x += pre.a.x; v.y += pre.a.y; v.z += pre.a.z; v.w += pre.a.w;
      if (P.epi == EPI_ACC) {
        // explicit mul then add (no FMA contraction): bit-identical to the TMA epilogue, which stages
        // scale * (...) and lets the reduce-add store do the accumulation
        v.x = __fadd_rn(__fmul_rn(v.x, P.scale), pre.b.x); v.y = __fadd_rn(__fmul_rn(v.y, P.scale), pre.b.y);
        v.z = __fadd_rn(__fmul_rn(v.z, P.scale), pre.b.z); v.w = __fadd_rn(__fmul_rn(v.w, P.scale), pre.b.w);
      }
      break;
    }
    case EPI_RELU:
      v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
      break;
    case EPI_TANH:
      v.x = tanhf(v.x); v.y = tanhf(v.y); v.z = tanhf(v.z); v.w = tanhf(v.w);
      break;
    case EPI_MISH:
      v.x = mishf_(v.x); v.y = mishf_(v.y); v.z = mishf_(v.z); v.w = mishf_(v.w);
      break;
    case EPI_SILU:
      v.x = siluf_(v.x); v.y = siluf_(v.y); v.z = siluf_(v.z); v.w = siluf_(v.w);
      break;
    case EPI_GELU_SCALED:
      v.x = gelu_erf(v.x * P.scale); v.y = gelu_erf(v.y * P.scale); v.z = gelu_erf(v.z * P.scale); v.w = gelu_erf(v.w * P.scale);
      break;
    case EPI_ADDVEC: break;   // the vector is part of cv
    case EPI_GATE:
    case EPI_GEGLU: {
      v.x += pre.a.x; v.y += pre.a.y; v.z += pre.a.z; v.w += pre.a.w;   // pre-activation term (DiffNet conditioner)
      float2 o;
      if (P.epi == EPI_GATE) {
        o.x = sigmoidf_(v.x) * tanhf(v.y);
        o.y = sigmoidf_(v.z) * tanhf(v.w);
      } else {
        o.x = v.x * gelu_erf(v.y);
        o.y = v.z * gelu_erf(v.w);
      }
      if (P.out) *reinterpret_cast<float2*>(P.out + g * P.out_gstride + (long)p * P.out_pitch + (co >> 1)) = o;
      if (P.pl_hi) {
        const __half2 hh = __floats2half2_rn(fminf(fmaxf(o.x, -65504.f), 65504.f), fminf(fmaxf(o.y, -65504.f), 65504.f));
        const float2 hf = __half22float2(hh);
        const __half2 ll = __floats2half2_rn(o.x - hf.x, o.y - hf.y);
        const long off = (long)p * P.pl_pitch + (co >> 1);
        *reinterpret_cast<__half2*>(P.pl_hi + off) = hh;
        *reinterpret_cast<__half2*>(P.pl_lo + off) = ll;
      }
      return;
    }
    case EPI_DIFFOUT: {
      if (co < P.csplit) {
        const float r2 = 0.70710678118654752440f;
        const float4 x = make_float4((pre.a.x + v.x) * r2, (pre.a.y + v.y) * r2, (pre.a.z + v.z) * r2, (pre.a.w + v.w) * r2);
        *reinterpret_cast<float4*>(P.out + g * P.out_gstride + (long)p * P.out_pitch + co) = x;
      } else {
        v.x += pre.a.x; v.y += pre.a.y; v.z += pre.a.z; v.w += pre.a.w;   // zeros unless accumulate
        *reinterpret_cast<float4*>(P.out2 + g * P.out2_gstride + (long)p * P.out2_pitch + (co - P.csplit)) = v;
      }
      return;
    }
    case EPI_STORE_CF: {
      float* o = P.out + g * P.out_gstride + (long)co * P.L + p;
      o[0] = v.x;
      if (co + 1 < P.Cout) o[(long)P.L] = v.y;
      if (co + 2 < P.Cout) o[2 * (long)P.L] = v.z;
      if (co + 3 < P.Cout) o[3 * (long)P.L] = v.w;
      return;
    }
    default: break;
  }
  if constexpr (PL) {
    const long off = g * P.out_gstride + (long)p * P.out_pitch + co;
    if (P.out) *reinterpret_cast<float4*>(P.out + off) = v;
    if (P.po_hi) epi_store_plane(P, off, v);
  } else {
    *reinterpret_cast<float4*>(P.out + g * P.out_gstride + (long)p * P.out_pitch + co) = v;
  }
}

__device__ __forceinline__ void epi_store(const TapConvParams& P, int g, int p, int co, float4 v, const EpiPre& pre) {
  epi_store_cv(P, g, p, co, v, pre, epi_colvec(P, g, co));
}

__device__ __forceinline__ void tc_epilogue(const TapConvParams& P, int g, int p, int co, float4 v) {
  EpiPre pre;
  epi_load(P, g, p, co, pre);
  epi_store(P, g, p, co, v, pre);
}

}  // namespace agpt
