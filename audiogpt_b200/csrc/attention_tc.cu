// Multi-head attention on the Hopper tensor cores (wgmma): softmax_j(q_i . k_j * d^-0.5) v_j with heads outermost in
// the channel dimension ('b n (h d)'), as CrossAttention.forward computes it (ldm/modules/attention.py:170-193).
// Both contractions -- S = Q K^T and O = P V -- run as wgmma on error-compensated fp16 hi/lo parts (x = hi + lo;
// hi*hi + lo*hi + hi*lo with fp32 accumulation: the arithmetic of tcconv5.cu); the softmax is the exact online
// (running max / running sum) form in fp32 registers.
//
// One CTA = one warpgroup = 64 queries of one (sample, head).  Per block of 64 keys:
//   all threads   K block  [64 keys][d]  -> fp16 hi/lo, K-major SWIZZLE_128B tile (B operand of S)
//                 V block  [64 keys][d]  -> TRANSPOSED fp16 hi/lo tile [d rows][64 keys] (B operand of O, K = keys)
//   wgmma         S[64 x 64] = Q K^T in registers (Q tile converted once per CTA, pre-scaled by d^-0.5 * log2 e)
//   all threads   running max m, p = exp2(s - m), running sum l over the fragment rows (4 lanes share a row);
//                 P hi/lo -> K-major tile (A operand of O); O *= exp2(m_old - m_new)
//   wgmma         O[64 x DP] += P V in registers
#include <cuda_fp16.h>
#include "common.cuh"
#include "tc_common.cuh"
#include "tc_h16.cuh"
#include "models.h"
#include "nn_kernels.h"

namespace agpt {
namespace {

constexpr int AT_BK = 64;          // keys per block = one 128-byte swizzle span of fp16
constexpr int AT_ROWS = 64;        // queries per CTA (wgmma M)

// D = head dim (multiple of 8, <= 128; 128 is FastSpeech2's hidden 256 over 2 heads).  NCH = 64-channel chunks of the head dim; DP = D rounded up to 16 (the N of
// the P V wgmma and the K granularity of Q K^T)
template <int D>
struct AtCfg {
  static constexpr int NCH = (D + 63) / 64;
  static constexpr int DP = (D + 15) / 16 * 16;
  static constexpr uint32_t Q_BYTES = 2u * NCH * AT_ROWS * 128;          // hi + lo
  static constexpr uint32_t K_BYTES = 2u * NCH * AT_BK * 128;
  static constexpr uint32_t V_BYTES = 2u * DP * 128;                     // [DP rows][64 keys] hi + lo
  static constexpr uint32_t P_BYTES = 2u * AT_ROWS * 128;
  static constexpr uint32_t TOTAL = Q_BYTES + K_BYTES + V_BYTES + P_BYTES;
  static constexpr bool PF = D <= 64;      // software-prefetch the next K / V block into registers (register budget: d <= 64)
  static constexpr int KIT = (AT_BK * NCH * 8 + 127) / 128;   // K items (8 channels of one key) per thread
  static constexpr int VIT = (DP / 4 + 1) / 2;                // V channel quads per thread
};

template <int N>
__device__ __forceinline__ void wgmma_f16(float* d, uint64_t a, uint64_t b) {
  if constexpr (N == 16) wgmma_n16(d, a, b);
  else if constexpr (N == 32) wgmma_n32(d, a, b);
  else if constexpr (N == 48) wgmma_n48(d, a, b);
  else if constexpr (N == 64) wgmma_n64(d, a, b);
  else if constexpr (N == 80) wgmma_n80(d, a, b);
  else wgmma_n128(d, a, b);
}

// MASK: kpm [N][Lk] bytes, 1 = padding key (fairseq's key_padding_mask); a query whose keys are all padding gets zeros.
// The parameter is last and unread without MASK, so the unmasked instantiations are the kernels they were before it.
template <int D, bool MASK>
__global__ void __launch_bounds__(128) attention_tc_kernel(
    const float* __restrict__ q, int q_pitch, const float* __restrict__ k, int k_pitch,
    const float* __restrict__ v, int v_pitch, float* __restrict__ o, int o_pitch,
    int Lq, int Lk, float qscale /* d^-0.5 * log2(e) */, const uint8_t* __restrict__ kpm) {
  using Cf = AtCfg<D>;
  extern __shared__ uint8_t at_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(at_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* q_hi = smem;
  uint8_t* q_lo = q_hi + Cf::NCH * AT_ROWS * 128;
  uint8_t* k_hi = smem + Cf::Q_BYTES;
  uint8_t* k_lo = k_hi + Cf::NCH * AT_BK * 128;
  uint8_t* v_hi = smem + Cf::Q_BYTES + Cf::K_BYTES;
  uint8_t* v_lo = v_hi + Cf::DP * 128;
  uint8_t* p_hi = smem + Cf::Q_BYTES + Cf::K_BYTES + Cf::V_BYTES;
  uint8_t* p_lo = p_hi + AT_ROWS * 128;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * AT_ROWS;
  constexpr int CH8 = Cf::NCH * 8;                    // 16-byte chunks per row over all 64-channel chunks
  // ---- Q tile: [64 queries][D] fp32 -> pre-scaled fp16 hi/lo, 8-channel items like the conv transform
  {
    const float* qb = q + ((long)n * Lq) * q_pitch + h * D;
    for (int it = tid; it < AT_ROWS * CH8; it += 128) {
      const int row = it / CH8, c8 = it - row * CH8;
      const int ch = c8 * 8;
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
      if (q0 + row < Lq && ch < D) {
        const float* p = qb + (long)(q0 + row) * q_pitch + ch;
        a = *reinterpret_cast<const float4*>(p);
        b = *reinterpret_cast<const float4*>(p + 4);
      }
      uint4 hi, lo;
      hi.x = split2(a.x * qscale, a.y * qscale, lo.x);
      hi.y = split2(a.z * qscale, a.w * qscale, lo.y);
      hi.z = split2(b.x * qscale, b.y * qscale, lo.z);
      hi.w = split2(b.z * qscale, b.w * qscale, lo.w);
      const uint32_t off = (uint32_t)(c8 >> 3) * (AT_ROWS * 128) + sw128(row, c8 & 7);
      *reinterpret_cast<uint4*>(q_hi + off) = hi;
      *reinterpret_cast<uint4*>(q_lo + off) = lo;
    }
  }

  // fragment of this thread (wgmma accumulator layout): rows r and r + 8, columns 8i + 2 (lane % 4) + {0, 1}
  const int r = warp * 16 + (lane >> 2), cq = 2 * (lane & 3);
  float acc[Cf::DP / 2];
#pragma unroll
  for (int c = 0; c < Cf::DP / 2; ++c) acc[c] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};    // l_run: this thread's partial sums of its rows
  const float* kb = k + ((long)n * Lk) * k_pitch + h * D;
  const float* vb = v + ((long)n * Lk) * v_pitch + h * D;
  const int nblk = (Lk + AT_BK - 1) / AT_BK;

  // K items: (key row, 8-channel chunk) -> two float4; V items: (key, channel quad) -> one float4
  float4 kreg[Cf::KIT][2];
  float4 vreg[Cf::VIT];
  auto load_kv = [&](int j0) {
#pragma unroll
    for (int u = 0; u < Cf::KIT; ++u) {
      const int it = tid + 128 * u;
      const int row = it / CH8, c8 = it - row * CH8;
      const int ch = c8 * 8;
      kreg[u][0] = make_float4(0.f, 0.f, 0.f, 0.f); kreg[u][1] = kreg[u][0];
      if (it < AT_BK * CH8 && j0 + row < Lk && ch < D) {
        const float* p = kb + (long)(j0 + row) * k_pitch + ch;
        kreg[u][0] = *reinterpret_cast<const float4*>(p);
        kreg[u][1] = *reinterpret_cast<const float4*>(p + 4);
      }
    }
    const int key = tid & 63, half = tid >> 6;          // two groups of 64 threads split the channel quads
    const bool kok = j0 + key < Lk;
    const float* p = vb + (long)(j0 + key) * v_pitch;
#pragma unroll
    for (int u = 0; u < Cf::VIT; ++u) {
      const int ch = (half + 2 * u) * 4;
      vreg[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (kok && ch < D) vreg[u] = *reinterpret_cast<const float4*>(p + ch);
    }
  };
  auto store_kv = [&]() {
    // K -> K-major hi/lo tiles (rows = keys)
#pragma unroll
    for (int u = 0; u < Cf::KIT; ++u) {
      const int it = tid + 128 * u;
      if (it >= AT_BK * CH8) continue;
      const int row = it / CH8, c8 = it - row * CH8;
      const float4 a = kreg[u][0], b = kreg[u][1];
      uint4 hi, lo;
      hi.x = split2(a.x, a.y, lo.x); hi.y = split2(a.z, a.w, lo.y);
      hi.z = split2(b.x, b.y, lo.z); hi.w = split2(b.z, b.w, lo.w);
      const uint32_t off = (uint32_t)(c8 >> 3) * (AT_BK * 128) + sw128(row, c8 & 7);
      *reinterpret_cast<uint4*>(k_hi + off) = hi;
      *reinterpret_cast<uint4*>(k_lo + off) = lo;
    }
    // V -> transposed tiles [channel rows][64 keys]; lanes take consecutive keys (conflict-free columns)
    const int key = tid & 63, half = tid >> 6;
#pragma unroll
    for (int u = 0; u < Cf::VIT; ++u) {
      const int c4 = half + 2 * u;
      if (c4 >= Cf::DP / 4) continue;
      const int ch = c4 * 4;
      const float vals[4] = {vreg[u].x, vreg[u].y, vreg[u].z, vreg[u].w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const __half hh = __float2half_rn(vals[i]);
        const __half ll = __float2half_rn(vals[i] - __half2float(hh));
        const uint32_t off = sw128(ch + i, key >> 3) + (uint32_t)(key & 7) * 2u;
        *reinterpret_cast<__half*>(v_hi + off) = hh;
        *reinterpret_cast<__half*>(v_lo + off) = ll;
      }
    }
  };

  for (int blk = 0; blk < nblk; ++blk) {
    const int j0 = blk * AT_BK;
    // ---- K / V block of this iteration: from the prefetch registers (loaded one block ahead, so that the global
    //      latency hides behind the previous block's MMA / softmax phases) or straight from global memory
    if (!Cf::PF || blk == 0) load_kv(j0);
    store_kv();
    if (Cf::PF && blk + 1 < nblk) load_kv(j0 + AT_BK);
    fence_proxy_async();
    __syncthreads();
    // ---- S = Q K^T
    float s[AT_BK / 2];
#pragma unroll
    for (int i = 0; i < AT_BK / 2; ++i) s[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < Cf::NCH; ++c) {
      constexpr int kv_last = D - (Cf::NCH - 1) * 64;
      const int ksteps = ((c == Cf::NCH - 1 ? kv_last : 64) + 15) >> 4;
      const uint64_t dqh = make_desc(smem_u32(q_hi + c * AT_ROWS * 128)), dql = make_desc(smem_u32(q_lo + c * AT_ROWS * 128));
      const uint64_t dkh = make_desc(smem_u32(k_hi + c * AT_BK * 128)), dkl = make_desc(smem_u32(k_lo + c * AT_BK * 128));
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        if (ks < ksteps) {
          const uint64_t ko = (uint64_t)(2 * ks);
          wgmma_n64(s, dqh + ko, dkh + ko);
          wgmma_n64(s, dql + ko, dkh + ko);
          wgmma_n64(s, dqh + ko, dkl + ko);
        }
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    // ---- online softmax over the two rows of this thread (scores are already in log2 units)
    float mb[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < AT_BK / 8; ++i)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = j0 + 8 * i + cq + (e & 1);
        if (key >= Lk) s[4 * i + e] = -INFINITY;
        if constexpr (MASK) {
          if (key < Lk && kpm[(long)n * Lk + key]) s[4 * i + e] = -INFINITY;
        }
        mb[e >> 1] = fmaxf(mb[e >> 1], s[4 * i + e]);
      }
    float alpha[2], m_new[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      mb[rr] = fmaxf(mb[rr], __shfl_xor_sync(0xffffffffu, mb[rr], 1));
      mb[rr] = fmaxf(mb[rr], __shfl_xor_sync(0xffffffffu, mb[rr], 2));
      m_new[rr] = fmaxf(m_run[rr], mb[rr]);
      alpha[rr] = (m_run[rr] == -INFINITY) ? 0.f : exp2f(m_run[rr] - m_new[rr]);
      m_run[rr] = m_new[rr];
      if constexpr (MASK) {
        if (m_new[rr] == -INFINITY) m_new[rr] = 0.f;     // every key so far is padding: p = exp2(-inf) = 0, not NaN
      }
    }
    float lsum[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < AT_BK / 2; ++i) {
      s[i] = exp2f(s[i] - m_new[(i >> 1) & 1]);      // exp2(-inf) = 0 for masked keys
      lsum[(i >> 1) & 1] += s[i];
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) l_run[rr] = l_run[rr] * alpha[rr] + lsum[rr];
    // P hi/lo -> K-major [64 rows][64 keys] tiles
#pragma unroll
    for (int i = 0; i < AT_BK / 8; ++i)
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        uint32_t lo;
        const uint32_t hi = split2(s[4 * i + 2 * rr], s[4 * i + 2 * rr + 1], lo);
        const uint32_t off = sw128(r + 8 * rr, i) + (uint32_t)cq * 2u;
        *reinterpret_cast<uint32_t*>(p_hi + off) = hi;
        *reinterpret_cast<uint32_t*>(p_lo + off) = lo;
      }
#pragma unroll
    for (int c = 0; c < Cf::DP / 2; ++c) acc[c] *= alpha[(c >> 1) & 1];
    fence_proxy_async();
    __syncthreads();
    // ---- O += P V   (K = 64 keys: 4 k-steps)
    wgmma_fence();
    {
      const uint64_t dph = make_desc(smem_u32(p_hi)), dpl = make_desc(smem_u32(p_lo));
      const uint64_t dvh = make_desc(smem_u32(v_hi)), dvl = make_desc(smem_u32(v_lo));
#pragma unroll
      for (int ks = 0; ks < AT_BK / 16; ++ks) {
        const uint64_t ko = (uint64_t)(2 * ks);
        wgmma_f16<Cf::DP>(acc, dph + ko, dvh + ko);
        wgmma_f16<Cf::DP>(acc, dpl + ko, dvh + ko);
        wgmma_f16<Cf::DP>(acc, dph + ko, dvl + ko);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();      // every thread is done with the K, V, P tiles of this block
  }

#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    float l = l_run[rr];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int qi = q0 + r + 8 * rr;
    if (qi >= Lq) continue;
    float inv = 1.f / l;
    if constexpr (MASK) inv = l > 0.f ? inv : 0.f;      // all keys padding: zeros
    float* op = o + ((long)n * Lq + qi) * o_pitch + h * D;
#pragma unroll
    for (int i = 0; i < Cf::DP / 8; ++i) {
      const int c = 8 * i + cq;
      if (c < D) *reinterpret_cast<float2*>(op + c) = make_float2(acc[4 * i + 2 * rr] * inv, acc[4 * i + 2 * rr + 1] * inv);
    }
  }
}

template <int D, bool MASK>
void launch_at(const float* q, int q_pitch, const float* k, int k_pitch, const float* v, int v_pitch, float* o, int o_pitch,
               int N, int heads, int Lq, int Lk, const uint8_t* kpm, cudaStream_t st) {
  using Cf = AtCfg<D>;
  const size_t smem = Cf::TOTAL + 1024;
  static bool done[64] = {false};
  int dev = 0;
  AGPT_CUDA(cudaGetDevice(&dev));
  if (!done[dev & 63]) {
    AGPT_CUDA(cudaFuncSetAttribute(attention_tc_kernel<D, MASK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    done[dev & 63] = true;
  }
  const float qscale = (1.0f / sqrtf((float)D)) * 1.4426950408889634f;     // dim_head ** -0.5 (attention.py:158), in log2 units
  dim3 grid(cdiv(Lq, AT_ROWS), heads, N);
  attention_tc_kernel<D, MASK><<<grid, 128, smem, st>>>(q, q_pitch, k, k_pitch, v, v_pitch, o, o_pitch, Lq, Lk, qscale, kpm);
}

}  // namespace

// returns false when the head dim / alignment is not supported (caller uses the fp32 kernel)
bool attention_tc(const float* q, int q_pitch, const float* k, int k_pitch, const float* v, int v_pitch,
                  float* o, int o_pitch, int N, int heads, int d, int Lq, int Lk, cudaStream_t st, const uint8_t* kpm) {
  if ((q_pitch | k_pitch | v_pitch | o_pitch) % 4 != 0) return false;
  if (((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
        reinterpret_cast<uintptr_t>(o)) & 15) != 0) return false;
#define AGPT_ATC(D_)                                                                                   \
  (kpm ? launch_at<D_, true>(q, q_pitch, k, k_pitch, v, v_pitch, o, o_pitch, N, heads, Lq, Lk, kpm, st) \
       : launch_at<D_, false>(q, q_pitch, k, k_pitch, v, v_pitch, o, o_pitch, N, heads, Lq, Lk, nullptr, st))
  switch (d) {
    case 8: AGPT_ATC(8); break;
    case 16: AGPT_ATC(16); break;
    case 32: AGPT_ATC(32); break;
    case 40: AGPT_ATC(40); break;
    case 64: AGPT_ATC(64); break;
    case 80: AGPT_ATC(80); break;
    case 128: AGPT_ATC(128); break;
    default: return false;
  }
#undef AGPT_ATC
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
  return true;
}

}  // namespace agpt
