// Non-contraction kernels of the UNet path (channels-last rows [N][HW][C]):
// GroupNorm(+SiLU), LayerNorm, attention (fp32, online softmax), timestep embedding,
// concat / nearest-upsample / stride-2 im2col gathers, DDIM update.
// Reference semantics: ldm/modules/diffusionmodules/util.py:151-171,214-216;
// ldm/modules/attention.py:76-77,170-193,203-215; ldm/models/diffusion/ddim.py:198-225.
#include "common.cuh"
#include "models.h"
#include "nn_kernels.h"
#include "tapconv.cuh"
#include <cuda_fp16.h>

namespace agpt {

// fp16 hi/lo operand-plane split of one value (optional fp16 hi/lo output of the normalisation kernels)
__device__ __forceinline__ void plane_split(float v, __half& hi, __half& lo) {
  hi = __float2half_rn(fminf(fmaxf(v, -65504.f), 65504.f));
  lo = __float2half_rn(v - __half2float(hi));
}

// ------------------------------------------------------------------ GroupNorm
// One CTA per (sample, group): the group's slab -- HW rows x cpg contiguous channels -- is read ONCE into shared
// memory (when it fits: every UNet shape does; the VAE's 80x624 maps fall back to re-reading through L2), then
// mean, centred variance (exact two-pass, fp32 per thread / double across threads) and the normalised
// (+SiLU) output come from the cached copy.  Replaces round 1's gn_partial + gn_apply pair (fp64 shared
// atomics, a serial S x G fold per CTA: 57 us per call on the 8 MB UNet tensors).
// Reference: GroupNorm32 / Normalize, ldm/modules/diffusionmodules/util.py:199-216, attention.py:76-77.
constexpr int GN_THREADS = 512;
constexpr int GN_CACHE_FLOATS = 48 * 1024;   // 192 KB of dynamic shared memory

__device__ __forceinline__ double gn_block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  double t = 0.0;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
  return t;
}

template <int V>   // V = vector width in floats along the channel axis (cpg % V == 0)
__global__ void __launch_bounds__(GN_THREADS) gn_fused_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                               const float* __restrict__ gamma, const float* __restrict__ beta,
                                                               int HW, int C, int cpg, float eps, int silu /* 0 none, 1 SiLU, 2 ReLU */, int cached,
                                                               __half* __restrict__ phi, __half* __restrict__ plo,
                                                               const float* __restrict__ res /* added after the activation, or null */) {
  extern __shared__ __align__(16) float gn_cache[];
  __shared__ double red[GN_THREADS / 32];
  const int n = blockIdx.y, g = blockIdx.x;
  const long slab0 = (long)n * HW * C + g * cpg;   // this CTA's slab: element 0 of its rows in x, y, res and the planes
  const float* xb = x + slab0;
  float* yb = y + slab0;
  const float* rb = res ? res + slab0 : nullptr;
  const int vpr = cpg / V;                 // vectors per row
  const int nvec = HW * vpr;
  // pass 1: sum (and fill the cache)
  float s = 0.f;
  for (int i = threadIdx.x; i < nvec; i += GN_THREADS) {
    const int r = i / vpr, c = (i - r * vpr) * V;
    float v[V];
    if constexpr (V == 4) { const float4 t = __ldg(reinterpret_cast<const float4*>(xb + (long)r * C + c)); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; }
    else if constexpr (V == 2) { const float2 t = __ldg(reinterpret_cast<const float2*>(xb + (long)r * C + c)); v[0] = t.x; v[1] = t.y; }
    else v[0] = __ldg(xb + (long)r * C + c);
#pragma unroll
    for (int k = 0; k < V; ++k) { s += v[k]; if (cached) gn_cache[k * nvec + i] = v[k]; }
  }
  const double cnt = (double)HW * cpg;
  const float mean = (float)(gn_block_sum((double)s, red) / cnt);
  // pass 2: centred sum of squares
  float q = 0.f;
  for (int i = threadIdx.x; i < nvec; i += GN_THREADS) {
    const int r = i / vpr, c = (i - r * vpr) * V;
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const float d = (cached ? gn_cache[k * nvec + i] : __ldg(xb + (long)r * C + c + k)) - mean;
      q = fmaf(d, d, q);
    }
  }
  const float rstd = (float)(1.0 / sqrt(gn_block_sum((double)q, red) / cnt + (double)eps));
  // pass 3: normalise (+ SiLU)
  for (int i = threadIdx.x; i < nvec; i += GN_THREADS) {
    const int r = i / vpr, c = (i - r * vpr) * V;
    float o[V];
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const float xv = cached ? gn_cache[k * nvec + i] : __ldg(xb + (long)r * C + c + k);
      float t = (xv - mean) * rstd * __ldg(gamma + g * cpg + c + k) + __ldg(beta + g * cpg + c + k);
      if (silu == 1) t = siluf_(t);
      else if (silu == 2) t = fmaxf(t, 0.f);
      if (rb) t += __ldg(rb + (long)r * C + c + k);
      o[k] = t;
    }
    if (phi) {     // operand planes instead of the fp32 tensor (the consumer is a plane-fed GEMM)
      const long base = slab0 + (long)r * C + c;
#pragma unroll
      for (int k = 0; k < V; ++k) plane_split(o[k], phi[base + k], plo[base + k]);
      continue;
    }
    if constexpr (V == 4) *reinterpret_cast<float4*>(yb + (long)r * C + c) = make_float4(o[0], o[1], o[2], o[3]);
    else if constexpr (V == 2) *reinterpret_cast<float2*>(yb + (long)r * C + c) = make_float2(o[0], o[1]);
    else yb[(long)r * C + c] = o[0];
  }
}

void groupnorm(const float* x, float* y, const float* gamma, const float* beta, int N, int HW, int C, int G,
               float eps, bool silu, double* scratch, cudaStream_t st, __half* phi, __half* plo) {
  (void)scratch;
  groupnorm_ex(x, y, gamma, beta, N, HW, C, G, eps, silu ? 1 : 0, nullptr, st, phi, plo);
}

// act: 0 none, 1 SiLU, 2 ReLU; res (optional, same layout as y) is added after the activation (ConvStacks' x + f(x))
void groupnorm_ex(const float* x, float* y, const float* gamma, const float* beta, int N, int HW, int C, int G,
                  float eps, int act, const float* res, cudaStream_t st, __half* phi, __half* plo) {
  AGPT_CHECK(C % G == 0 && C % 4 == 0, "GroupNorm: channels must be divisible by the group count and by 4");
  const int cpg = C / G;
  const long slab = (long)HW * cpg;
  const int cached = slab <= GN_CACHE_FLOATS ? 1 : 0;
  const size_t smem = cached ? (size_t)slab * sizeof(float) : 0;
  int dev = 0;
  AGPT_CUDA(cudaGetDevice(&dev));
  static bool attr_done_dev[64] = {false};
  if (!attr_done_dev[dev & 63]) {
    AGPT_CUDA(cudaFuncSetAttribute(gn_fused_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, GN_CACHE_FLOATS * 4));
    AGPT_CUDA(cudaFuncSetAttribute(gn_fused_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, GN_CACHE_FLOATS * 4));
    AGPT_CUDA(cudaFuncSetAttribute(gn_fused_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, GN_CACHE_FLOATS * 4));
    attr_done_dev[dev & 63] = true;
  }
  const dim3 grid(G, N);
  const int si = act;
  if (cpg % 4 == 0) gn_fused_kernel<4><<<grid, dim3(GN_THREADS), smem, st>>>(x, y, gamma, beta, HW, C, cpg, eps, si, cached, phi, plo, res);
  else if (cpg % 2 == 0) gn_fused_kernel<2><<<grid, dim3(GN_THREADS), smem, st>>>(x, y, gamma, beta, HW, C, cpg, eps, si, cached, phi, plo, res);
  else gn_fused_kernel<1><<<grid, dim3(GN_THREADS), smem, st>>>(x, y, gamma, beta, HW, C, cpg, eps, si, cached, phi, plo, res);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}
size_t groupnorm_scratch_doubles(int N, int C) { (void)N; (void)C; return 16; }

// ------------------------------------------------------------------ LayerNorm (one warp per row)
__global__ void layernorm_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                 const float* __restrict__ beta, float* __restrict__ y, long rows, int C, float eps,
                                 __half* __restrict__ phi, __half* __restrict__ plo) {
  const long row = (long)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* xr = x + row * C;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += xr[c];
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)C;
  float v = 0.f;
  for (int c = lane; c < C; c += 32) { const float d = xr[c] - mean; v += d * d; }
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const float rstd = rsqrtf(v / (float)C + eps);
  if (phi) {       // operand planes instead of the fp32 tensor
    for (int c = lane; c < C; c += 32) plane_split((xr[c] - mean) * rstd * gamma[c] + beta[c], phi[row * C + c], plo[row * C + c]);
    return;
  }
  float* yr = y + row * C;
  for (int c = lane; c < C; c += 32) yr[c] = (xr[c] - mean) * rstd * gamma[c] + beta[c];
}

void layernorm(const float* x, float* y, const float* gamma, const float* beta, long rows, int C, float eps,
               cudaStream_t st, __half* phi, __half* plo) {
  const int wpb = 8;
  layernorm_kernel<<<dim3((unsigned)cdivl(rows, wpb)), dim3(wpb * 32), 0, st>>>(x, gamma, beta, y, rows, C, eps, phi, plo);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// ------------------------------------------------------------------ attention
// softmax_j(q_i . k_j * scale) v_j, heads outermost in the channel dim ('b n (h d)').
// Two lanes share one query row (each holds half of the head dim); K/V tiles of 32 keys
// are staged in shared memory and read as warp-wide broadcasts.
// MASK: kpm [N][Lk] bytes, 1 = padding key; a query whose keys are all padding gets zeros (last parameter, unread
// without MASK)
template <int DH, bool MASK>
__global__ void __launch_bounds__(128) attention_kernel(
    const float* __restrict__ q, int q_pitch, const float* __restrict__ k, int k_pitch,
    const float* __restrict__ v, int v_pitch, float* __restrict__ o, int o_pitch,
    int Lq, int Lk, float scale, const uint8_t* __restrict__ kpm) {
  constexpr int D = 2 * DH, KT = 32;
  __shared__ __align__(16) float Ks[KT][D];
  __shared__ __align__(16) float Vs[KT][D];
  const int n = blockIdx.z, h = blockIdx.y;
  const int half = threadIdx.x & 1;
  const int qi = blockIdx.x * 64 + (threadIdx.x >> 1);
  const bool valid = qi < Lq;
  float qr[DH], acc[DH];
  {
    const float* qp = q + ((long)n * Lq + (valid ? qi : 0)) * q_pitch + h * D + half * DH;
#pragma unroll
    for (int c = 0; c < DH; c += 4) {
      const float4 t = *reinterpret_cast<const float4*>(qp + c);
      qr[c] = t.x * scale; qr[c + 1] = t.y * scale; qr[c + 2] = t.z * scale; qr[c + 3] = t.w * scale;
    }
#pragma unroll
    for (int c = 0; c < DH; ++c) acc[c] = 0.f;
  }
  float m = -INFINITY, l = 0.f;
  const float* kb = k + (long)n * Lk * k_pitch + h * D;
  const float* vb = v + (long)n * Lk * v_pitch + h * D;
  for (int j0 = 0; j0 < Lk; j0 += KT) {
    __syncthreads();
    for (int i = threadIdx.x; i < KT * (D / 4); i += blockDim.x) {
      const int j = i / (D / 4), c = (i % (D / 4)) * 4;
      float4 kk = make_float4(0.f, 0.f, 0.f, 0.f), vv = kk;
      if (j0 + j < Lk) {
        kk = *reinterpret_cast<const float4*>(kb + (long)(j0 + j) * k_pitch + c);
        vv = *reinterpret_cast<const float4*>(vb + (long)(j0 + j) * v_pitch + c);
      }
      *reinterpret_cast<float4*>(&Ks[j][c]) = kk;
      *reinterpret_cast<float4*>(&Vs[j][c]) = vv;
    }
    __syncthreads();
    float s[KT];
    float tmax = -INFINITY;
#pragma unroll
    for (int j = 0; j < KT; ++j) {
      float d = 0.f;
#pragma unroll
      for (int c = 0; c < DH; c += 4) {
        const float4 kk = *reinterpret_cast<const float4*>(&Ks[j][half * DH + c]);
        d = fmaf(qr[c], kk.x, d); d = fmaf(qr[c + 1], kk.y, d); d = fmaf(qr[c + 2], kk.z, d); d = fmaf(qr[c + 3], kk.w, d);
      }
      d += __shfl_xor_sync(0xffffffffu, d, 1);
      if (j0 + j >= Lk) d = -INFINITY;
      if constexpr (MASK) {
        if (j0 + j < Lk && kpm[(long)n * Lk + j0 + j]) d = -INFINITY;
      }
      s[j] = d;
      tmax = fmaxf(tmax, d);
    }
    float mn = fmaxf(m, tmax);
    const float corr = (m == -INFINITY) ? 0.f : expf(m - mn);
    if constexpr (MASK) {
      if (mn == -INFINITY) { m = mn; continue; }     // every key so far is padding: nothing to accumulate
    }
    l *= corr;
#pragma unroll
    for (int c = 0; c < DH; ++c) acc[c] *= corr;
#pragma unroll
    for (int j = 0; j < KT; ++j) {
      const float p = expf(s[j] - mn);   // exp(-inf) = 0 for masked keys
      l += p;
#pragma unroll
      for (int c = 0; c < DH; c += 4) {
        const float4 vv = *reinterpret_cast<const float4*>(&Vs[j][half * DH + c]);
        acc[c] = fmaf(p, vv.x, acc[c]); acc[c + 1] = fmaf(p, vv.y, acc[c + 1]);
        acc[c + 2] = fmaf(p, vv.z, acc[c + 2]); acc[c + 3] = fmaf(p, vv.w, acc[c + 3]);
      }
    }
    m = mn;
  }
  if (valid) {
    float inv = 1.f / l;
    if constexpr (MASK) inv = l > 0.f ? inv : 0.f;     // all keys padding: zeros
    float* op = o + ((long)n * Lq + qi) * o_pitch + h * D + half * DH;
#pragma unroll
    for (int c = 0; c < DH; c += 4)
      *reinterpret_cast<float4*>(op + c) = make_float4(acc[c] * inv, acc[c + 1] * inv, acc[c + 2] * inv, acc[c + 3] * inv);
  }
}

static int g_attn_tc = -1;
void attention_set_tc(int on) { g_attn_tc = on; }
bool attention_tc_enabled() {
  if (g_attn_tc < 0) { const char* e = getenv("AGPT_ATTN_TC"); g_attn_tc = (e && e[0] == '0') ? 0 : 1; }
  return g_attn_tc >= 1;
}

void attention(const float* q, int q_pitch, const float* k, int k_pitch, const float* v, int v_pitch,
               float* o, int o_pitch, int N, int heads, int d, int Lq, int Lk, cudaStream_t st, const uint8_t* kpm) {
  // tensor-core path (QK^T and PV on wgmma, attention_tc.cu); the fp32 kernel below is the A/B reference
  if (attention_tc_enabled() && attention_tc(q, q_pitch, k, k_pitch, v, v_pitch, o, o_pitch, N, heads, d, Lq, Lk, st, kpm)) return;
  const float scale = 1.0f / sqrtf((float)d);   // dim_head ** -0.5  (attention.py:158)
  dim3 grid(cdiv(Lq, 64), heads, N);
#define AGPT_ATT(DH_)                                                                                                     \
  (kpm ? attention_kernel<DH_, true><<<grid, 128, 0, st>>>(q, q_pitch, k, k_pitch, v, v_pitch, o, o_pitch, Lq, Lk, scale, kpm) \
       : attention_kernel<DH_, false><<<grid, 128, 0, st>>>(q, q_pitch, k, k_pitch, v, v_pitch, o, o_pitch, Lq, Lk, scale, nullptr))
  switch (d) {
    case 8: AGPT_ATT(4); break;
    case 16: AGPT_ATT(8); break;
    case 32: AGPT_ATT(16); break;
    case 40: AGPT_ATT(20); break;
    case 64: AGPT_ATT(32); break;
    case 80: AGPT_ATT(40); break;
    case 128: AGPT_ATT(64); break;
    default: throw Error("attention: unsupported head dim " + std::to_string(d) + " (supported: 8,16,32,40,64,80,128)");
  }
#undef AGPT_ATT
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// ------------------------------------------------------------------ single-head attention with a wide head (VAE AttnBlock)
// softmax_j(q_i . k_j * C^-0.5) v_j with d = C = 256 / 512 and 780 / 3 120 tokens (ldm/modules/diffusionmodules/
// model.py:177-203) runs as two tap-GEMMs with an ACTIVATION as the weight operand (K^T, then V) and a row softmax
// in between; these helpers build the operand layouts the tap-GEMM expects ([cin_pad][cout_pad], zero padded).
__global__ void transpose_pad_kernel(const float* __restrict__ in, int in_pitch, int rows, int cols,
                                     float* __restrict__ out, int rows_pad) {
  __shared__ float tile[32][33];
  const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < rows && c < cols) ? in[(long)r * in_pitch + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (c < cols && r < rows_pad) out[(long)c * rows_pad + r] = tile[threadIdx.x][i];
  }
}
// out [cols][rows_pad] = in[rows][cols]^T, columns rows..rows_pad-1 zero
void transpose_pad(const float* in, int in_pitch, int rows, int cols, float* out, int rows_pad, cudaStream_t st) {
  dim3 grid(cdiv(rows_pad, 32), cdiv(cols, 32)), block(32, 8);
  transpose_pad_kernel<<<grid, block, 0, st>>>(in, in_pitch, rows, cols, out, rows_pad);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}
__global__ void copy_pad_rows_kernel(const float* __restrict__ in, int in_pitch, int rows, int cols,
                                     float* __restrict__ out, long total) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / cols;
    const int c = (int)(i - r * cols);
    out[i] = r < rows ? in[r * in_pitch + c] : 0.f;
  }
}
// out [rows_pad][cols] = in[rows][cols], rows beyond `rows` zero
void copy_pad_rows(const float* in, int in_pitch, int rows, int cols, float* out, int rows_pad, cudaStream_t st) {
  const long total = (long)rows_pad * cols;
  copy_pad_rows_kernel<<<(unsigned)std::min<long>(cdivl(total, 256), 4096), 256, 0, st>>>(in, in_pitch, rows, cols, out, total);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}
// in-place softmax over the first `cols` entries of every row of x [rows][pitch], after scaling by `scale`
// (torch: softmax(w_ * c^-0.5, dim=2)); entries cols..pitch-1 are set to zero.  One 256-thread block per row.
__global__ void __launch_bounds__(256) softmax_rows_kernel(float* __restrict__ x, int pitch, int cols, float scale) {
  __shared__ float red[8];
  float* xr = x + (long)blockIdx.x * pitch;
  float m = -INFINITY;
  for (int c = threadIdx.x; c < cols; c += 256) m = fmaxf(m, xr[c] * scale);
#pragma unroll
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
  __syncthreads();
  float s = 0.f;
  for (int c = threadIdx.x; c < cols; c += 256) { const float e = expf(xr[c] * scale - m); xr[c] = e; s += e; }
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += red[i];
  const float inv = 1.f / s;
  for (int c = threadIdx.x; c < pitch; c += 256) xr[c] = c < cols ? xr[c] * inv : 0.f;
}
void softmax_rows(float* x, int pitch, long rows, int cols, float scale, cudaStream_t st) {
  softmax_rows_kernel<<<(unsigned)rows, 256, 0, st>>>(x, pitch, cols, scale);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}


// ------------------------------------------------------------------ timestep embedding (cos || sin)
struct TParam { int t[256]; };
__global__ void timestep_embed_kernel(float* __restrict__ out, const __grid_constant__ TParam tp, int dim) {
  const int n = blockIdx.x, half = dim / 2;
  for (int j = threadIdx.x; j < dim; j += blockDim.x) {
    float v = 0.f;
    if (j < 2 * half) {
      const int i = j < half ? j : j - half;
      const float f = expf(-9.210340371976184f * (float)i / (float)half);   // -ln(10000) * i / half
      const float a = (float)tp.t[n] * f;
      v = j < half ? cosf(a) : sinf(a);
    }
    out[(long)n * dim + j] = v;
  }
}
void timestep_embedding(float* out, const int* t_host, int N, int dim, cudaStream_t st) {
  AGPT_CHECK(N <= 256, "at most 256 samples per UNet call");
  TParam tp;
  for (int i = 0; i < N; ++i) tp.t[i] = t_host[i];
  timestep_embed_kernel<<<N, 128, 0, st>>>(out, tp, dim);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// same, timesteps read from a device array (one row per DDIM step: the whole table is embedded once per sample() call)
__global__ void timestep_embed_dev_kernel(float* __restrict__ out, const int* __restrict__ t, int dim) {
  const int n = blockIdx.x, half = dim / 2;
  const float tv = (float)t[n];
  for (int j = threadIdx.x; j < dim; j += blockDim.x) {
    float v = 0.f;
    if (j < 2 * half) {
      const int i = j < half ? j : j - half;
      const float f = expf(-9.210340371976184f * (float)i / (float)half);
      const float a = tv * f;
      v = j < half ? cosf(a) : sinf(a);
    }
    out[(long)n * dim + j] = v;
  }
}
void timestep_embedding_dev(float* out, const int* t_dev, int rows, int dim, cudaStream_t st) {
  timestep_embed_dev_kernel<<<rows, 128, 0, st>>>(out, t_dev, dim);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// ------------------------------------------------------------------ device-side step counter (CUDA-graph replays)
// A denoising loop replays ONE captured step; everything that changes from step to step is read from device
// tables indexed by a device counter: out[c] = table[*step][c]; the counter is bumped by the last node of the step.
__global__ void select_row_kernel(const float* __restrict__ table, const int* __restrict__ step, float* __restrict__ out, int ncols) {
  const long k = *step;
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < ncols; c += gridDim.x * blockDim.x) out[c] = table[k * ncols + c];
}
void select_row(const float* table, const int* step_dev, float* out, int ncols, cudaStream_t st) {
  select_row_kernel<<<dim3(std::min(64, cdiv(ncols, 256))), dim3(256), 0, st>>>(table, step_dev, out, ncols);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}
__global__ void step_inc_kernel(int* step) { *step += 1; }
void step_inc(int* step_dev, cudaStream_t st) {
  step_inc_kernel<<<dim3(1), dim3(1), 0, st>>>(step_dev);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// ------------------------------------------------------------------ gathers
__global__ void concat_kernel(const float* __restrict__ a, int Ca, const float* __restrict__ b, int Cb,
                              float* __restrict__ out, long rows) {
  const int C = Ca + Cb;
  const long total = rows * (C / 4);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / (C / 4);
    const int c = (int)(i % (C / 4)) * 4;
    const float4 v = c < Ca ? *reinterpret_cast<const float4*>(a + r * Ca + c)
                            : *reinterpret_cast<const float4*>(b + r * Cb + (c - Ca));
    *reinterpret_cast<float4*>(out + r * C + c) = v;
  }
}
void concat_channels(const float* a, int Ca, const float* b, int Cb, float* out, long rows, cudaStream_t st) {
  AGPT_CHECK(Ca % 4 == 0 && Cb % 4 == 0, "concat channels must be multiples of 4");
  const long total = rows * ((Ca + Cb) / 4);
  concat_kernel<<<dim3((unsigned)std::min<long>(cdivl(total, 256), 4096)), dim3(256), 0, st>>>(a, Ca, b, Cb, out, rows);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// nearest x2: out[n][2H][2W][C] = in[n][h/2][w/2][C]   (F.interpolate(scale_factor=2, mode='nearest'))
__global__ void upsample2_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int H, int W, int C) {
  const long total = (long)N * 4 * H * W * (C / 4);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % (C / 4)) * 4;
    long r = i / (C / 4);
    const int wo = (int)(r % (2 * W)); r /= 2 * W;
    const int ho = (int)(r % (2 * H));
    const int n = (int)(r / (2 * H));
    const float4 v = *reinterpret_cast<const float4*>(in + (((long)n * H + ho / 2) * W + wo / 2) * C + c);
    *reinterpret_cast<float4*>(out + (((long)n * 2 * H + ho) * 2 * W + wo) * C + c) = v;
  }
}
void upsample_nearest2(const float* in, float* out, int N, int H, int W, int C, cudaStream_t st) {
  const long total = (long)N * 4 * H * W * (C / 4);
  upsample2_kernel<<<dim3((unsigned)std::min<long>(cdivl(total, 256), 4096)), dim3(256), 0, st>>>(in, out, N, H, W, C);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// 2x2 average pool with stride 2 and floor (the ResBlock down path's AvgPool2d(2, 2), openaimodel.py:134-160):
// out[n][ho][wo][C] = (x[2ho][2wo] + x[2ho][2wo+1] + x[2ho+1][2wo] + x[2ho+1][2wo+1]) / 4, summed in that order
__global__ void avgpool2_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int H, int W, int C) {
  const int Ho = H / 2, Wo = W / 2;
  const long total = (long)N * Ho * Wo * (C / 4);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % (C / 4)) * 4;
    long r = i / (C / 4);
    const int wo = (int)(r % Wo); r /= Wo;
    const int ho = (int)(r % Ho);
    const int n = (int)(r / Ho);
    const float* p = in + (((long)n * H + 2 * ho) * W + 2 * wo) * C + c;
    const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + C);
    const float4 d = *reinterpret_cast<const float4*>(p + (long)W * C), e = *reinterpret_cast<const float4*>(p + (long)W * C + C);
    *reinterpret_cast<float4*>(out + (((long)n * Ho + ho) * Wo + wo) * C + c) =
        make_float4((a.x + b.x + d.x + e.x) / 4.f, (a.y + b.y + d.y + e.y) / 4.f, (a.z + b.z + d.z + e.z) / 4.f,
                    (a.w + b.w + d.w + e.w) / 4.f);
  }
}
void avgpool2(const float* in, float* out, int N, int H, int W, int C, cudaStream_t st) {
  AGPT_CHECK(C % 4 == 0 && H >= 2 && W >= 2, "avgpool2: channels must be a multiple of 4 and the map at least 2x2");
  const long total = (long)N * (H / 2) * (W / 2) * (C / 4);
  avgpool2_kernel<<<dim3((unsigned)std::min<long>(cdivl(total, 256), 4096)), dim3(256), 0, st>>>(in, out, N, H, W, C);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// im2col for a 3x3 stride-2 Conv2d: col[n][ho][wo][tap*C + c] = x[n][2ho+kh-pad][2wo+kw-pad][c], zero outside x.
// pad 1: the UNet's Conv2d(k3, stride 2, padding 1); pad 0: the VAE encoder's Downsample, F.pad(x, (0,1,0,1)) then a
// conv without padding -- the one zero row / column past the end is the same out-of-range read
__global__ void im2col_s2_kernel(const float* __restrict__ in, float* __restrict__ col, int N, int H, int W, int C,
                                 int Ho, int Wo, int pad) {
  const long total = (long)N * Ho * Wo * 9 * (C / 4);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % (C / 4)) * 4;
    long r = i / (C / 4);
    const int tap = (int)(r % 9); r /= 9;
    const int wo = (int)(r % Wo); r /= Wo;
    const int ho = (int)(r % Ho);
    const int n = (int)(r / Ho);
    const int hi = 2 * ho + tap / 3 - pad, wi = 2 * wo + tap % 3 - pad;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (hi >= 0 && hi < H && wi >= 0 && wi < W) v = *reinterpret_cast<const float4*>(in + (((long)n * H + hi) * W + wi) * C + c);
    *reinterpret_cast<float4*>(col + ((((long)n * Ho + ho) * Wo + wo) * 9 + tap) * C + c) = v;
  }
}
void im2col_stride2(const float* in, float* col, int N, int H, int W, int C, int Ho, int Wo, int pad, cudaStream_t st) {
  const long total = (long)N * Ho * Wo * 9 * (C / 4);
  im2col_s2_kernel<<<dim3((unsigned)std::min<long>(cdivl(total, 256), 4096)), dim3(256), 0, st>>>(in, col, N, H, W, C, Ho, Wo, pad);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// [N][C][HW] -> [N][HW][Cpad] with zero fill for c >= C (tiny C, e.g. 4 latent channels)
// sample n reads source sample n % Nsrc: the doubled batch of classifier-free guidance (x_in = cat([x] * 2),
// ddim.py:178) is produced here instead of by two device-to-device copies
__global__ void cf_to_cl_pad_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int Cpad, int HW, long total, int Nsrc) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % Cpad);
    const long r = i / Cpad;
    const long n = (r / HW) % Nsrc, p = r % HW;
    out[i] = c < C ? in[(n * C + c) * HW + p] : 0.f;
  }
}
void cf_to_cl_pad(const float* in, float* out, int N, int C, int Cpad, int HW, cudaStream_t st, int Nsrc) {
  const long total = (long)N * HW * Cpad;
  cf_to_cl_pad_kernel<<<dim3((unsigned)std::min<long>(cdivl(total, 256), 4096)), dim3(256), 0, st>>>(in, out, C, Cpad, HW, total, Nsrc > 0 ? Nsrc : N);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// ------------------------------------------------------------------ DDIM update (ddim.py:198-225)
__global__ void ddim_update_kernel(const float* __restrict__ x, const float* __restrict__ eps2, int single, float s,
                                   float sqrt_at, float sqrt_aprev, float dir_coef, float sigma_t, float sqrt_om,
                                   const float* __restrict__ noise, float temperature, long total, long half_off,
                                   float* __restrict__ x_prev, float* __restrict__ pred_x0) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    float e;
    if (single) e = eps2[i];
    else { const float eu = eps2[i], ec = eps2[half_off + i]; e = eu + s * (ec - eu); }
    const float xv = x[i];
    const float p0 = (xv - sqrt_om * e) / sqrt_at;
    float o = sqrt_aprev * p0 + dir_coef * e;
    if (noise) o += sigma_t * noise[i] * temperature; else o += 0.f;
    x_prev[i] = o;
    if (pred_x0) pred_x0[i] = p0;
  }
}
// Table version for graph replays: coef[*step] = {sqrt_at, sqrt_aprev, dir_coef, sigma_t, sqrt_om, cfg_scale};
// x is updated in place (x_prev may alias x: every element is read before it is written by the same thread).
__global__ void ddim_update_tab_kernel(const float* __restrict__ x, const float* __restrict__ eps2, int single,
                                       const float* __restrict__ coef, const int* __restrict__ step, long total,
                                       float* __restrict__ x_prev, float* __restrict__ pred_x0) {
  const float* c = coef + 6 * (long)(*step);
  const float sqrt_at = c[0], sqrt_aprev = c[1], dir_coef = c[2], sqrt_om = c[4], s = c[5];
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    float e;
    if (single) e = eps2[i];
    else { const float eu = eps2[i], ec = eps2[total + i]; e = eu + s * (ec - eu); }
    const float xv = x[i];
    const float p0 = (xv - sqrt_om * e) / sqrt_at;
    x_prev[i] = sqrt_aprev * p0 + dir_coef * e + 0.f;
    if (pred_x0) pred_x0[i] = p0;
  }
}
void ddim_update_tab(const float* x, const float* eps2, int single, const float* coef_dev, const int* step_dev, int B, long n,
                     float* x_prev, float* pred_x0, cudaStream_t st) {
  const long total = (long)B * n;
  ddim_update_tab_kernel<<<(unsigned)std::min<long>(cdivl(total, 256), 2048), 256, 0, st>>>(x, eps2, single, coef_dev, step_dev,
                                                                                         total, x_prev, pred_x0);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// The UNet's `out` conv (GN -> SiLU -> conv3x3 C -> 4, openaimodel.py:686,742) FUSED with classifier-free guidance
// and the DDIM update (ddim.py:177-225): one warp per latent pixel computes the 4 output channels of BOTH guidance
// halves (samples b and b + B) from the normalised activation hn [N][H*W][C] (lanes stride the channels, 128-bit
// weight loads, warp-shuffle reduction), combines e = e_u + s (e_c - e_u) and writes x_prev / pred_x0 in place of
// eps -- the epsilon tensor never exists in memory.  coef[*step] as in ddim_update_tab_kernel.
__global__ void __launch_bounds__(256) conv_out_ddim_kernel(const float* __restrict__ hn, const float* __restrict__ w /*[9][C][4]*/,
                                                             const float* __restrict__ bias, float* __restrict__ x /*[B][4][HW] in place*/,
                                                             float* __restrict__ pred_x0, const float* __restrict__ coef,
                                                             const int* __restrict__ step, int B, int H, int W, int C, int single) {
  const int HW = H * W;
  const int lane = threadIdx.x & 31;
  const int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int b = blockIdx.y;
  if (p >= HW) return;
  const int ph = p / W, pw = p - ph * W;
  const float* hu = hn + (long)b * HW * C;                 // unconditional half (or the only one)
  const float* hc = hn + (long)(b + (single ? 0 : B)) * HW * C;
  float au[4] = {0.f, 0.f, 0.f, 0.f}, ac[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const int hh = ph + t / 3 - 1, ww = pw + t % 3 - 1;
    if (hh < 0 || hh >= H || ww < 0 || ww >= W) continue;
    const long row = (long)(hh * W + ww) * C;
    const float4* wt = reinterpret_cast<const float4*>(w) + (long)t * C;
    for (int c = lane; c < C; c += 32) {
      const float4 wv = __ldg(wt + c);
      const float xu = __ldg(hu + row + c);
      au[0] = fmaf(xu, wv.x, au[0]); au[1] = fmaf(xu, wv.y, au[1]); au[2] = fmaf(xu, wv.z, au[2]); au[3] = fmaf(xu, wv.w, au[3]);
      if (!single) {
        const float xc = __ldg(hc + row + c);
        ac[0] = fmaf(xc, wv.x, ac[0]); ac[1] = fmaf(xc, wv.y, ac[1]); ac[2] = fmaf(xc, wv.z, ac[2]); ac[3] = fmaf(xc, wv.w, ac[3]);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      au[k] += __shfl_xor_sync(0xffffffffu, au[k], o);
      ac[k] += __shfl_xor_sync(0xffffffffu, ac[k], o);
    }
  }
  if (lane < 4) {
    const int k = lane;
    const float* cf = coef + 6 * (long)(*step);
    const float sqrt_at = cf[0], sqrt_aprev = cf[1], dir_coef = cf[2], sqrt_om = cf[4], s = cf[5];
    const float sel_u = k == 0 ? au[0] : (k == 1 ? au[1] : (k == 2 ? au[2] : au[3]));
    const float sel_c = k == 0 ? ac[0] : (k == 1 ? ac[1] : (k == 2 ? ac[2] : ac[3]));
    const float eu = sel_u + bias[k];
    float e = eu;
    if (!single) { const float ec = sel_c + bias[k]; e = eu + s * (ec - eu); }
    const long xi = ((long)b * 4 + k) * HW + p;
    const float xv = x[xi];
    const float p0 = (xv - sqrt_om * e) / sqrt_at;
    x[xi] = sqrt_aprev * p0 + dir_coef * e + 0.f;
    if (pred_x0) pred_x0[xi] = p0;
  }
}
void conv_out_ddim(const float* hn, const float* w9c4, const float* bias4, float* x_io, float* pred_x0, const float* coef_dev,
                   const int* step_dev, int B, int H, int W, int C, int single, cudaStream_t st) {
  dim3 grid(cdiv(H * W, 8), B);
  conv_out_ddim_kernel<<<grid, dim3(256), 0, st>>>(hn, w9c4, bias4, x_io, pred_x0, coef_dev, step_dev, B, H, W, C, single);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

void ddim_update(const float* x, const float* eps2, int single, float cfg_scale, float a_t, float a_prev,
                 float sigma_t, float sqrt_om, const float* noise, float temperature, int B, long n,
                 float* x_prev, float* pred_x0, cudaStream_t st) {
  const long total = (long)B * n;
  // fp32 scalar algebra exactly as torch.full(...).sqrt() etc. would do it
  const float sqrt_at = sqrtf(a_t), sqrt_aprev = sqrtf(a_prev);
  const float dir_coef = sqrtf(1.0f - a_prev - sigma_t * sigma_t);
  ddim_update_kernel<<<(unsigned)std::min<long>(cdivl(total, 256), 2048), 256, 0, st>>>(
      x, eps2, single, cfg_scale, sqrt_at, sqrt_aprev, dir_coef, sigma_t, sqrt_om, noise, temperature, total, total,
      x_prev, pred_x0);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

}  // namespace agpt
