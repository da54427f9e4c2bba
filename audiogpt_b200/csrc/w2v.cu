// wav2vec2 CTC (transformers' Wav2Vec2ForCTC, post-LN base layout) on sm_90a: the reference-audio ASR of the TTS_OOD
// tool (NeuralSeq/inference/tts/base_tts_infer.py:83-101: asr_model(input_values).logits, eval mode, no mask).
//
//   conv stem      conv0 (1 -> C, k0, stride s0, no bias) + GroupNorm(C groups, C) + GELU, two launches over the
//                  waveform: statistics (per-CTA centred partials, merged in chunk order by the last CTA of a sample),
//                  then conv0 again (k0 MACs per output) with the affine norm and GELU, written once
//   conv 1..n-1    stride-s convs as stride-1 tap-GEMMs over super-rows: [T][C] read as [ceil(T/s)][s C], ceil(k/s)
//                  taps of s C channels (specs.w2v_superrow_weight packs them), exact-GELU epilogue
//   projection     LayerNorm(C) + Linear(C -> H)
//   positional     Conv1d(H -> H, K, padding K/2, groups G, bias), SamePad, GELU, added to the projection:
//                  one wgmma launch (pos_conv_tc_kernel), fused epilogue y = x + gelu(conv + bias)
//   trunk          LayerNorm + post-LN BERT layers (ClapNet::trunk), then lm_head
#include <algorithm>
#include <cmath>
#include <cuda_fp16.h>
#include "common.cuh"
#include "tapconv.cuh"
#include "tc_common.cuh"
#include "tc_h16.cuh"
#include "nn_kernels.h"
#include "models.h"
#include "clap.cuh"
#include "audio_front.cuh"

namespace agpt {

namespace {

constexpr int kStemRows = 128;        // conv0 output rows per CTA of both stem launches
constexpr int kStemMaxK = 16;
constexpr int kPosCG = 48;            // channels per positional-conv group (768 / 16)
constexpr int kPosMaxK = 128;         // positional-conv taps
constexpr int PC_ROWS = 64;           // output rows per CTA of the wgmma positional conv (one warpgroup, wgmma M)
constexpr int PC_TAPS = 2;            // taps per weight stage
constexpr int PC_TAP_BYTES = 2 * kPosCG * 128;                       // hi + lo [48 rows][128 B] per tap
constexpr int PC_WIN = (PC_ROWS + kPosMaxK - 1 + 7) / 8 * 8;         // operand window rows
constexpr int PC_SMEM = 2 * PC_WIN * 128 + 2 * PC_TAPS * PC_TAP_BYTES + 1024;
constexpr int PF_ROWS = 32;           // output rows per CTA of the fp32 positional conv

// conv0 of row t, channel c: sum_k w[k] x[s t + k] over the staged segment xs (row t0 at xs[0])
__device__ __forceinline__ float stem_conv(const float* xs, const float* w, int k0, int s0, int r) {
  float v = 0.f;
#pragma unroll
  for (int k = 0; k < kStemMaxK; ++k)
    if (k < k0) v = fmaf(w[k], xs[r * s0 + k], v);
  return v;
}

__device__ __forceinline__ void stem_stage(const float* __restrict__ x, float* xs, long S, int b, int t0, int nrows, int k0,
                                           int s0) {
  const long base = (long)b * S + (long)t0 * s0;
  const int n = (nrows - 1) * s0 + k0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) xs[i] = x[base + i];
}

// Launch 1: per (sample, chunk of kStemRows rows, channel) the chunk mean and centred sum of squares (fp64), merged by
// the sample's last CTA in chunk order (Chan et al.) into mean / rstd.  cnt[b] is back at 0 when the launch ends.
__global__ void w2v_stem_stats_kernel(const float* __restrict__ x, long S, int T0, int C, const float* __restrict__ w0, int k0,
                                      int s0, double2* __restrict__ part, float2* __restrict__ stat, int* __restrict__ cnt,
                                      float eps) {
  extern __shared__ float xs[];
  const int b = blockIdx.y, ch = blockIdx.x, c = threadIdx.x;
  const int t0 = ch * kStemRows, nrows = min(kStemRows, T0 - t0);
  stem_stage(x, xs, S, b, t0, nrows, k0, s0);
  float w[kStemMaxK];
#pragma unroll
  for (int k = 0; k < kStemMaxK; ++k) w[k] = k < k0 ? w0[c * k0 + k] : 0.f;
  __syncthreads();
  double sum = 0.0;
  for (int r = 0; r < nrows; ++r) sum += (double)stem_conv(xs, w, k0, s0, r);
  const double mean = sum / nrows;
  double m2 = 0.0;
  for (int r = 0; r < nrows; ++r) {
    const double d = (double)stem_conv(xs, w, k0, s0, r) - mean;
    m2 += d * d;
  }
  part[((long)b * gridDim.x + ch) * C + c] = make_double2(mean, m2);
  __threadfence();
  __syncthreads();
  __shared__ bool last;
  if (threadIdx.x == 0) last = atomicAdd(&cnt[b], 1) == (int)gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  double n = 0.0, mu = 0.0, M2 = 0.0;
  for (int j = 0; j < (int)gridDim.x; ++j) {
    const double2 p = __ldcg(&part[((long)b * gridDim.x + j) * C + c]);
    const double nb = (double)min(kStemRows, T0 - j * kStemRows), nn = n + nb;
    const double d = p.x - mu;
    mu += d * (nb / nn);
    M2 += p.y + d * d * (n * nb / nn);
    n = nn;
  }
  stat[(long)b * C + c] = make_float2((float)mu, (float)(1.0 / sqrt(M2 / n + (double)eps)));
  if (threadIdx.x == 0) cnt[b] = 0;
}

// Launch 2: conv0 again, GroupNorm affine, GELU -> out [B][R][C] (sample stride R rows); rows T0 .. T0 + zpad - 1 get
// zeros (the first super-row view's padding)
__global__ void w2v_stem_apply_kernel(const float* __restrict__ x, long S, int T0, int zpad, int C, const float* __restrict__ w0,
                                      int k0, int s0, const float2* __restrict__ stat, const float* __restrict__ gamma,
                                      const float* __restrict__ beta, float* __restrict__ out, long R) {
  extern __shared__ float xs[];
  const int b = blockIdx.y, c = threadIdx.x;
  const int t0 = blockIdx.x * kStemRows, nrows = max(0, min(kStemRows, T0 - t0));
  if (nrows > 0) stem_stage(x, xs, S, b, t0, nrows, k0, s0);
  float w[kStemMaxK];
#pragma unroll
  for (int k = 0; k < kStemMaxK; ++k) w[k] = k < k0 ? w0[c * k0 + k] : 0.f;
  const float2 st = stat[(long)b * C + c];
  const float g = gamma[c] * st.y, bb = beta[c];
  __syncthreads();
  float* o = out + ((long)b * R + t0) * C + c;
  for (int r = 0; r < nrows; ++r) o[(long)r * C] = gelu_erf((stem_conv(xs, w, k0, s0, r) - st.x) * g + bb);
  const int zend = min(kStemRows, T0 + zpad - t0);
  for (int r = max(nrows, T0 - t0); r < zend; ++r) o[(long)r * C] = 0.f;
}

__device__ __forceinline__ void fence_acc24(float* a) {
#pragma unroll
  for (int i = 0; i < kPosCG / 2; ++i) asm volatile("" : "+f"(a[i])::"memory");
}

// Grouped positional conv on the tensor cores.  CTA = 64 output rows x one 48-channel group x one sample, one warpgroup.
// The input window (rows t0 - K/2 .. t0 + 63 + K - 1 - K/2, zero outside the sample) is converted once into K-major
// SWIZZLE_128B fp16 hi / lo tiles (48 of each row's 64 fp16 slots used); tap k is the window shifted by k rows.  The
// weight image wimg [G][K][hi | lo][48 co rows][128 B] (pre-split, pre-swizzled, pre-scaled by 1 / descale) streams
// through two stages of PC_TAPS taps by cp.async.  y[t][g 48 + co] = x[t][..] + gelu(conv * descale + bias).
// Each stage's wgmmas start from a zero accumulator, which is then added into the fp32 total: the tensor cores' own
// accumulation truncates at every k-step: over all 1152 of a 128-tap conv that put x + conv 1.1e-5 off fp64; with
// per-stage totals the conv alone is 5e-7 off, below the fp32 reference's own rounding.
__global__ void __launch_bounds__(128) pos_conv_tc_kernel(const float* __restrict__ x, float* __restrict__ y, int T, int H, int K,
                                                          const uint8_t* __restrict__ wimg, const float* __restrict__ bias,
                                                          float descale) {
  extern __shared__ uint8_t pc_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(pc_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* a_hi = smem;
  uint8_t* a_lo = smem + PC_WIN * 128;
  uint8_t* wst = smem + 2 * PC_WIN * 128;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int t0 = blockIdx.x * PC_ROWS, g = blockIdx.y, b = blockIdx.z;
  const int pad = K / 2, nwin = PC_ROWS + K - 1;
  const float* xb = x + (long)b * T * H + g * kPosCG;
  const uint8_t* wg = wimg + (size_t)g * K * PC_TAP_BYTES;
  const int nst = (K + PC_TAPS - 1) / PC_TAPS;

  auto issue_stage = [&](int s) {
    const int k0 = s * PC_TAPS, nt = min(PC_TAPS, K - k0);
    const uint8_t* src = wg + (size_t)k0 * PC_TAP_BYTES;
    uint8_t* dst = wst + (s & 1) * PC_TAPS * PC_TAP_BYTES;
    for (int i = tid; i < nt * PC_TAP_BYTES / 16; i += 128) cp_async16_zfill(dst + 16 * i, src + 16 * i, 16u);
    cp_async_commit_();
  };
  issue_stage(0);
  // the operand window: 6 items of 8 channels per row
  for (int it = tid; it < nwin * 6; it += 128) {
    const int row = it / 6, j = it - row * 6;
    const int t = t0 - pad + row;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), c = a;
    if (t >= 0 && t < T) {
      const float* p = xb + (long)t * H + 8 * j;
      a = *reinterpret_cast<const float4*>(p);
      c = *reinterpret_cast<const float4*>(p + 4);
    }
    uint4 hi, lo;
    hi.x = split2(a.x, a.y, lo.x); hi.y = split2(a.z, a.w, lo.y);
    hi.z = split2(c.x, c.y, lo.z); hi.w = split2(c.z, c.w, lo.w);
    *reinterpret_cast<uint4*>(a_hi + sw128(row, j)) = hi;
    *reinterpret_cast<uint4*>(a_lo + sw128(row, j)) = lo;
  }

  float acc[kPosCG / 2], tot[kPosCG / 2];
#pragma unroll
  for (int i = 0; i < kPosCG / 2; ++i) tot[i] = 0.f;
  const uint32_t ah = smem_u32(a_hi), al = smem_u32(a_lo);
  for (int s = 0; s < nst; ++s) {
    cp_async_wait_all_();
    fence_proxy_async();
    __syncthreads();                  // stage s (and, at s = 0, the window) visible to the async proxy of every thread
    if (s + 1 < nst) issue_stage(s + 1);   // its buffer's wgmmas (stage s - 1) completed before the barrier
    const uint32_t ws = smem_u32(wst + (s & 1) * PC_TAPS * PC_TAP_BYTES);
    const int nt = min(PC_TAPS, K - s * PC_TAPS);
#pragma unroll
    for (int i = 0; i < kPosCG / 2; ++i) acc[i] = 0.f;
    fence_acc24(acc);
    wgmma_fence();
    for (int kk = 0; kk < nt; ++kk) {
      const int k = s * PC_TAPS + kk;
      const uint64_t dah = make_desc(ah + k * 128), dal = make_desc(al + k * 128);
      const uint64_t dwh = make_desc(ws + kk * PC_TAP_BYTES), dwl = make_desc(ws + kk * PC_TAP_BYTES + kPosCG * 128);
#pragma unroll
      for (int ks = 0; ks < kPosCG / 16; ++ks) {
        const uint64_t ko = (uint64_t)(2 * ks);
        wgmma_n48(acc, dah + ko, dwh + ko);
        wgmma_n48(acc, dal + ko, dwh + ko);
        wgmma_n48(acc, dah + ko, dwl + ko);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc24(acc);
#pragma unroll
    for (int i = 0; i < kPosCG / 2; ++i) tot[i] += acc[i];
  }

  const int r = warp * 16 + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int t = t0 + r + 8 * rr;
    if (t >= T) continue;
    const long off = ((long)b * T + t) * H + g * kPosCG;
#pragma unroll
    for (int i = 0; i < kPosCG / 8; ++i) {
      const int co = 8 * i + cq;
      const float2 xv = *reinterpret_cast<const float2*>(x + off + co);
      const float v0 = fmaf(tot[4 * i + 2 * rr], descale, bias[g * kPosCG + co]);
      const float v1 = fmaf(tot[4 * i + 2 * rr + 1], descale, bias[g * kPosCG + co + 1]);
      *reinterpret_cast<float2*>(y + off + co) = make_float2(xv.x + gelu_erf(v0), xv.y + gelu_erf(v1));
    }
  }
}

// The same conv on the fp32 FMA units (AGPT_TENSOR_CORES=0): CTA = 32 rows x one group x one sample, w [G][K][ci][co].
__global__ void __launch_bounds__(192) pos_conv_fma_kernel(const float* __restrict__ x, float* __restrict__ y, int T, int H,
                                                           int K, const float* __restrict__ w, const float* __restrict__ bias) {
  extern __shared__ float win[];                // [PF_ROWS + K - 1][48]
  const int t0 = blockIdx.x * PF_ROWS, g = blockIdx.y, b = blockIdx.z;
  const int pad = K / 2, nwin = PF_ROWS + K - 1;
  const float* xb = x + (long)b * T * H + g * kPosCG;
  for (int i = threadIdx.x; i < nwin * kPosCG; i += blockDim.x) {
    const int row = i / kPosCG, ci = i - row * kPosCG, t = t0 - pad + row;
    win[i] = (t >= 0 && t < T) ? xb[(long)t * H + ci] : 0.f;
  }
  __syncthreads();
  const int co = threadIdx.x % kPosCG, r0 = (threadIdx.x / kPosCG) * (PF_ROWS / 4);
  float acc[PF_ROWS / 4];
#pragma unroll
  for (int j = 0; j < PF_ROWS / 4; ++j) acc[j] = 0.f;
  const float* wg = w + (size_t)g * K * kPosCG * kPosCG + co;
  for (int k = 0; k < K; ++k)
    for (int ci = 0; ci < kPosCG; ++ci) {
      const float wv = __ldg(wg + ((size_t)k * kPosCG + ci) * kPosCG);
#pragma unroll
      for (int j = 0; j < PF_ROWS / 4; ++j) acc[j] = fmaf(win[(r0 + j + k) * kPosCG + ci], wv, acc[j]);
    }
#pragma unroll
  for (int j = 0; j < PF_ROWS / 4; ++j) {
    const int t = t0 + r0 + j;
    if (t >= T) continue;
    const long o = ((long)b * T + t) * H + g * kPosCG + co;
    y[o] = x[o] + gelu_erf(acc[j] + bias[g * kPosCG + co]);
  }
}

}  // namespace

void w2v_stem(const float* x, long S, int B, int T0, int zpad, int C, const float* w0, int k0, int s0, const float* gamma,
              const float* beta, float eps, void* part, void* stat, int* cnt, float* out, long R, cudaStream_t st) {
  AGPT_CHECK(k0 >= 1 && k0 <= kStemMaxK && s0 >= 1 && s0 <= 64, "conv0: k0 must be 1..16 and s0 1..64");
  AGPT_CHECK(C >= 1 && C <= 1024, "conv0: at most 1024 channels (one thread each)");
  AGPT_CHECK(B >= 1 && T0 >= 1 && zpad >= 0 && R >= (long)T0 + zpad && (long)(T0 - 1) * s0 + k0 <= S, "conv0: bad sizes");
  const int nch = cdiv(T0, kStemRows);
  const size_t xs_bytes = sizeof(float) * ((kStemRows - 1) * s0 + k0);
  w2v_stem_stats_kernel<<<dim3(nch, B), C, xs_bytes, st>>>(x, S, T0, C, w0, k0, s0, static_cast<double2*>(part),
                                                         static_cast<float2*>(stat), cnt, eps);
  w2v_stem_apply_kernel<<<dim3(cdiv(T0 + zpad, kStemRows), B), C, xs_bytes, st>>>(
      x, S, T0, zpad, C, w0, k0, s0, static_cast<const float2*>(stat), gamma, beta, out, R);
  count_launch(2);
}

// conv output lengths T_0 .. T_{n-1} of an S-sample input (0 from the first layer without a frame on)
static void w2v_conv_lengths(const agpt_w2v_cfg& c, long S, std::vector<int>& T) {
  T.assign(c.conv_layers, 0);
  long t = S;
  for (int i = 0; i < c.conv_layers; ++i) {
    t = t >= c.conv_kernel[i] ? (t - c.conv_kernel[i]) / c.conv_stride[i] + 1 : 0;
    T[i] = (int)std::min<long>(t, 1L << 30);
  }
}

// The engine: every buffer is grown to the largest call seen.
struct W2vNet : Handle {
  agpt_w2v_cfg cfg;
  DevBuf w0, gng, gnb;                  // conv0 [C][k0], GroupNorm scale / shift
  std::vector<PackedConv> convs;        // conv 1 .. n-1 on super-rows
  DevBuf fplng, fplnb;
  PackedConv proj, head;
  DevBuf pos_w, pos_b;                  // fp32 [G][K][ci][co] (FMA kernel), bias [H]
  DevBuf pos_img;                       // fp16 hi / lo weight image of pos_conv_tc_kernel (bytes)
  float pos_descale = 1.f;
  ClapNet bert;                         // encoder.layer_norm and the encoder layers
  DevBuf fa, fb, part, stat, cnt;       // conv-stack ping-pong, stem partials / statistics / CTA counters

  void features(const float* x, int B, long S, cudaStream_t st);    // -> out_feat (rows T_last at stride feat_stride)
  void pos_conv(const float* xin, float* yout, int B, int T, cudaStream_t st);
  void logits(const float* x, int B, long S, float* out, cudaStream_t st);
  const float* out_feat = nullptr;
  long feat_stride = 0;                 // rows per sample of out_feat
};

void W2vNet::features(const float* x, int B, long S, cudaStream_t st) {
  std::vector<int> T;
  w2v_conv_lengths(cfg, S, T);
  const int n = cfg.conv_layers, C = cfg.conv_dim;
  AGPT_CHECK(B >= 1 && T[n - 1] >= 1, "input too short: the conv feature encoder yields no frame");
  AGPT_CHECK(T[0] <= (1 << 24), "input too long");
  const int k0 = cfg.conv_kernel[0], s0 = cfg.conv_stride[0];
  const long R = T[0] + 8;                                    // rows per sample of the conv stack's buffers
  fa.ensure((size_t)B * R * C);
  fb.ensure((size_t)B * R * C);
  const int nch = cdiv(T[0], kStemRows);
  part.ensure((size_t)B * nch * C * 2 * 2);                   // double2 per (sample, chunk, channel)
  stat.ensure((size_t)B * C * 2);
  if (cnt.n < (size_t)B) {
    cnt.ensure(B);
    AGPT_CUDA(cudaMemsetAsync(cnt.p, 0, sizeof(int) * B, st));
  }
  const float gn_eps = 1e-5f;                                 // nn.GroupNorm's default (Wav2Vec2GroupNormConvLayer)
  const int zpad = n > 1 ? round_up(T[0], cfg.conv_stride[1]) - T[0] : 0;
  w2v_stem(x, S, B, T[0], zpad, C, w0.p, k0, s0, gng.p, gnb.p, gn_eps, part.p, stat.p, reinterpret_cast<int*>(cnt.p), fa.p, R, st);
  AGPT_CUDA(cudaGetLastError());
  float* cur = fa.p;
  float* nxt = fb.p;
  for (int i = 1; i < n; ++i) {
    const int s = cfg.conv_stride[i];
    const int Lin = cdiv(T[i - 1], s);                        // super-rows of the input (the last one zero-padded)
    const bool last = i == n - 1;
    const long Rout = last ? Lin : R;                         // the last stage's rows are packed for the projection
    TapConvParams P = tapconv_params(convs[i - 1], B, Lin, 0, 1);
    P.in = cur; P.in_gstride = R * C; P.in_pitch = s * C;
    P.out = nxt; P.out_gstride = Rout * C; P.out_pitch = C;
    P.epi = EPI_GELU_SCALED; P.scale = 1.f;
    tapconv_launch(P, st);
    // rows T_i .. of the output hold partial sums of the zero padding: the next super-row view needs them zero
    if (!last) {
      const int z = round_up(T[i], cfg.conv_stride[i + 1]) - T[i];
      if (z > 0)
        AGPT_CUDA(cudaMemset2DAsync(nxt + (long)T[i] * C, sizeof(float) * R * C, 0, sizeof(float) * z * C, B, st));
    }
    std::swap(cur, nxt);
    feat_stride = Rout;
  }
  if (n == 1) feat_stride = R;
  out_feat = cur;
}

void W2vNet::pos_conv(const float* xin, float* yout, int B, int T, cudaStream_t st) {
  const int H = cfg.hidden_size, G = cfg.num_conv_pos_embedding_groups, K = cfg.num_conv_pos_embeddings;
  if (tc_enabled()) {
    pos_conv_tc_kernel<<<dim3(cdiv(T, PC_ROWS), G, B), 128, PC_SMEM, st>>>(
        xin, yout, T, H, K, reinterpret_cast<const uint8_t*>(pos_img.p), pos_b.p, pos_descale);
  } else {
    const size_t sm = sizeof(float) * (PF_ROWS + K - 1) * kPosCG;
    pos_conv_fma_kernel<<<dim3(cdiv(T, PF_ROWS), G, B), 192, sm, st>>>(xin, yout, T, H, K, pos_w.p, pos_b.p);
  }
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

void W2vNet::logits(const float* x, int B, long S, float* out, cudaStream_t st) {
  features(x, B, S, st);
  std::vector<int> T;
  w2v_conv_lengths(cfg, S, T);
  const int Tf = T[cfg.conv_layers - 1], C = cfg.conv_dim, H = cfg.hidden_size;
  const long rows = (long)B * Tf;
  bert.ensure_work(rows);
  // feature projection: LayerNorm over the packed rows (feat_stride >= Tf per sample), then the Linear compacts them
  float* ln = fa.p == out_feat ? fb.p : fa.p;
  layernorm(out_feat, ln, fplng.p, fplnb.p, (long)B * feat_stride, C, cfg.layer_norm_eps, st);
  TapConvParams P = tapconv_params(proj, B, Tf, 0, 1);
  P.in = ln; P.in_gstride = feat_stride * C; P.in_pitch = C;
  P.out = bert.x.p; P.out_gstride = (long)Tf * H; P.out_pitch = H;
  P.epi = EPI_BIAS;
  tapconv_launch(P, st);
  pos_conv(bert.x.p, bert.y.p, B, Tf, st);                   // y = x + pos(x): what the trunk's first LayerNorm reads
  bert.trunk(B, Tf, nullptr, st);
  TapConvParams Q = tapconv_params(head, 1, (int)rows, 0, 1);
  Q.in = bert.x.p; Q.in_gstride = rows * H; Q.in_pitch = H;
  Q.out = out; Q.out_gstride = rows * cfg.vocab_size; Q.out_pitch = cfg.vocab_size;
  Q.epi = EPI_BIAS;
  tapconv_launch(Q, st);
  AGPT_CUDA(cudaGetLastError());
}

void w2v_lengths(const agpt_w2v_cfg* cfg, long S, int* frames) {
  std::vector<int> T;
  w2v_conv_lengths(*cfg, S, T);
  *frames = T[cfg->conv_layers - 1];
}

static void w2v_check_cfg(const agpt_w2v_cfg* c) {
  AGPT_CHECK(c->conv_layers >= 1 && c->conv_layers <= AGPT_W2V_MAX_CONV, "conv_layers must be 1..8");
  AGPT_CHECK(c->conv_dim >= 32 && c->conv_dim <= 1024 && c->conv_dim % 32 == 0, "conv_dim must be a multiple of 32 in [32, 1024]");
  AGPT_CHECK(c->conv_kernel[0] >= 1 && c->conv_kernel[0] <= kStemMaxK && c->conv_stride[0] >= 1 && c->conv_stride[0] <= 64,
             "conv_kernel[0] must be 1..16 (and conv_stride[0] 1..64)");
  for (int i = 1; i < c->conv_layers; ++i)
    AGPT_CHECK(c->conv_kernel[i] >= 1 && c->conv_stride[i] >= 1 && c->conv_stride[i] <= 8 &&
                   cdiv(c->conv_kernel[i], c->conv_stride[i]) <= kMaxTaps,
               "conv_kernel / conv_stride of layers 1.. must give at most 12 super-row taps (stride <= 8)");
  AGPT_CHECK(c->hidden_size > 0 && c->num_heads >= 1 && c->hidden_size % c->num_heads == 0, "hidden_size % num_heads != 0");
  const int d = c->hidden_size / c->num_heads;
  AGPT_CHECK(d == 8 || d == 16 || d == 32 || d == 40 || d == 64 || d == 80 || d == 128,
             "head dim must be one of 8, 16, 32, 40, 64, 80, 128 (the attention kernel's)");
  AGPT_CHECK(c->num_conv_pos_embedding_groups >= 1 && c->hidden_size == kPosCG * c->num_conv_pos_embedding_groups,
             "the positional conv needs 48 channels per group (hidden_size = 48 * num_conv_pos_embedding_groups)");
  AGPT_CHECK(c->num_conv_pos_embeddings >= 1 && c->num_conv_pos_embeddings <= kPosMaxK, "num_conv_pos_embeddings must be 1..128");
  AGPT_CHECK(c->num_layers >= 0 && c->intermediate_size > 0 && c->intermediate_size % 4 == 0 && c->vocab_size >= 1 &&
                 c->layer_norm_eps > 0.f,
             "bad wav2vec2 config");
}

Handle* w2v_create(const agpt_w2v_cfg* cfg, const float* const* W, int nW, int device) {
  DeviceGuard dg_(device);
  w2v_check_cfg(cfg);
  std::unique_ptr<W2vNet> h(new W2vNet());
  h->magic = kMagicW2v; h->device = device; h->cfg = *cfg;
  const int C = cfg->conv_dim, H = cfg->hidden_size, G = cfg->num_conv_pos_embedding_groups, K = cfg->num_conv_pos_embeddings;
  WeightCursor wc{W, nW};
  h->w0.upload(wc.next(), (size_t)C * cfg->conv_kernel[0]);
  h->gng.upload(wc.next(), C);
  h->gnb.upload(wc.next(), C);
  h->convs.resize(cfg->conv_layers - 1);
  for (int i = 1; i < cfg->conv_layers; ++i) {
    const int s = cfg->conv_stride[i], nt = cdiv(cfg->conv_kernel[i], s);
    PackedConv& pc = h->convs[i - 1];
    pack_conv(pc, wc.next(), nullptr, C, s * C, nt, false);   // [C][s C][nt]: specs.w2v_superrow_weight
    for (int t = 0; t < nt; ++t) pc.tap_off_1d[t] = t;
    pc.useful = (float)cfg->conv_kernel[i] / (float)(nt * s);
  }
  h->fplng.upload(wc.next(), C);
  h->fplnb.upload(wc.next(), C);
  { auto w = wc.next(); auto b = wc.next(); pack_conv(h->proj, w, b, H, C, 1, false); }
  // positional conv: the folded weight [H][48][K] (g v / |v| per tap) -> [G][K][ci][co] fp32 and the fp16 hi / lo image
  {
    const float* w = wc.next();
    h->pos_b.upload(wc.next(), H);
    std::vector<float> wf((size_t)G * K * kPosCG * kPosCG);
    float mx = 0.f;
    for (int g = 0; g < G; ++g)
      for (int co = 0; co < kPosCG; ++co)
        for (int ci = 0; ci < kPosCG; ++ci)
          for (int k = 0; k < K; ++k) {
            const float v = w[((size_t)(g * kPosCG + co) * kPosCG + ci) * K + k];
            wf[(((size_t)g * K + k) * kPosCG + ci) * kPosCG + co] = v;
            mx = std::max(mx, std::fabs(v));
          }
    h->pos_w.upload(wf);
    int e = 0;
    float wscale = 1.f;
    if (mx > 0.f && std::isfinite(mx)) {                      // max |w| into [2^13, 2^14), as pack_h_weights does
      std::frexp(mx, &e);
      wscale = std::ldexp(1.f, std::max(-60, std::min(60, 14 - e)));
    }
    h->pos_descale = 1.f / wscale;
    const size_t bytes = (size_t)G * K * PC_TAP_BYTES;
    std::vector<__half> img(bytes / 2, __float2half(0.f));
    for (int g = 0; g < G; ++g)
      for (int k = 0; k < K; ++k) {
        __half* hi = img.data() + ((size_t)g * K + k) * (PC_TAP_BYTES / 2);
        __half* lo = hi + kPosCG * 64;
        for (int co = 0; co < kPosCG; ++co)
          for (int ci = 0; ci < kPosCG; ++ci) {
            const float v = wf[(((size_t)g * K + k) * kPosCG + ci) * kPosCG + co] * wscale;
            const __half vh = __float2half_rn(v);
            const __half vl = __float2half_rn(v - __half2float(vh));
            const int j = ci >> 3, slot = (co * 128 + (((j ^ (co & 7)) << 4)) + (ci & 7) * 2) / 2;   // sw128(co, j)
            hi[slot] = vh;
            lo[slot] = vl;
          }
      }
    h->pos_img.ensure(cdiv((long)bytes, 4));
    AGPT_CUDA(cudaMemcpy(h->pos_img.p, img.data(), bytes, cudaMemcpyHostToDevice));
    // the attribute belongs to the kernel on this device, shared by every handle, and PC_SMEM is the same for all of
    // them: setting it at each create (under this create's DeviceGuard) needs no host-side flag
    AGPT_CUDA(cudaFuncSetAttribute(pos_conv_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PC_SMEM));
  }
  agpt_clap_cfg& b = h->bert.cfg;
  memset(&b, 0, sizeof(b));
  b.hidden_size = H; b.num_layers = cfg->num_layers; b.num_heads = cfg->num_heads;
  b.intermediate_size = cfg->intermediate_size; b.layer_norm_eps = cfg->layer_norm_eps;
  h->bert.load_trunk(wc);
  { auto w = wc.next(); auto bb = wc.next(); pack_conv(h->head, w, bb, cfg->vocab_size, H, 1, false); }
  wc.done();
  return h.release();
}

void w2v_logits(Handle* hh, const float* x, int B, long S, float* logits, cudaStream_t st) {
  auto* h = static_cast<W2vNet*>(hh);
  DeviceGuard dg_(h->device);
  h->logits(x, B, S, logits, st);
}

void w2v_features(Handle* hh, const float* x, int B, long S, float* feats, cudaStream_t st) {
  auto* h = static_cast<W2vNet*>(hh);
  DeviceGuard dg_(h->device);
  h->features(x, B, S, st);
  std::vector<int> T;
  w2v_conv_lengths(h->cfg, S, T);
  const int Tf = T[h->cfg.conv_layers - 1];
  const size_t row = sizeof(float) * h->cfg.conv_dim;
  AGPT_CUDA(cudaMemcpy2DAsync(feats, row * Tf, h->out_feat, row * h->feat_stride, row * Tf, B, cudaMemcpyDeviceToDevice, st));
}

void w2v_pos_conv(Handle* hh, const float* x, int B, int T, float* y, cudaStream_t st) {
  auto* h = static_cast<W2vNet*>(hh);
  DeviceGuard dg_(h->device);
  AGPT_CHECK(B >= 1 && T >= 1, "empty input");
  AGPT_CHECK(x != y, "x and y must not alias");
  // the tensor-core kernel reads hidden rows as float4 and writes float2 pairs (hidden_size is a multiple of 48)
  AGPT_CHECK(reinterpret_cast<uintptr_t>(x) % 16 == 0 && reinterpret_cast<uintptr_t>(y) % 8 == 0,
             "hidden must be 16-byte and out 8-byte aligned");
  h->pos_conv(x, y, B, T, st);
}

}  // namespace agpt
