// HiFi-GAN generator on sm_90a: host driver + the small non-contraction kernels.
// Arithmetic follows NeuralSeq/modules/hifigan/hifigan.py:144-169 (reference) and is
// parity-checked against oracle/hifigan_ref.py in tests/test_hifigan_gpu.py.
#include "common.cuh"
#include "tapconv.cuh"
#include "models.h"
#include "voc_kernels.cuh"

namespace agpt {

// [B][C][T] (channels-first, as the reference passes mel) -> [B][T][C] rows
__global__ void cf_to_cl_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int T) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const float* ib = in + (long)b * C * T;
  float* ob = out + (long)b * C * T;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, t = t0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && t < T) ? ib[(long)c * T + t] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i, c = c0 + threadIdx.x;
    if (t < T && c < C) ob[(long)t * C + c] = tile[threadIdx.x][i];
  }
}

void launch_cf_to_cl(const float* in, float* out, int B, int C, int T, cudaStream_t st) {
  dim3 grid(cdiv(T, 32), cdiv(C, 32), B), block(32, 8);
  cf_to_cl_kernel<<<grid, block, 0, st>>>(in, out, C, T);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// conv_post: leaky_relu(0.01) -> Conv1d(C -> c_out, k7, pad 3) -> tanh   (hifigan.py:165-167)
// in [B][L][C] rows, out [B][c_out][L].  Memory-bound (C*4 bytes in per sample out).
__global__ void conv_post_kernel(const float* __restrict__ in, const float* __restrict__ w /*[c_out][7][C]*/,
                                 const float* __restrict__ bias, float* __restrict__ out,
                                 int L, int C, int c_out, float slope) {
  extern __shared__ float ws[];
  for (int i = threadIdx.x; i < c_out * 7 * C; i += blockDim.x) ws[i] = w[i];
  __syncthreads();
  const int b = blockIdx.y;
  const long p = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= L) return;
  const float* ib = in + (long)b * L * C;
  for (int oc = 0; oc < c_out; ++oc) {
    float acc = bias[oc];
    const float* wo = ws + oc * 7 * C;
#pragma unroll
    for (int k = 0; k < 7; ++k) {
      const long q = p + k - 3;
      if (q < 0 || q >= L) continue;
      const float4* row = reinterpret_cast<const float4*>(ib + q * C);
      const float* wk = wo + k * C;
      for (int c4 = 0; c4 < C / 4; ++c4) {
        const float4 x = __ldg(row + c4);
        acc = fmaf(lrelu(x.x, slope), wk[4 * c4 + 0], acc);
        acc = fmaf(lrelu(x.y, slope), wk[4 * c4 + 1], acc);
        acc = fmaf(lrelu(x.z, slope), wk[4 * c4 + 2], acc);
        acc = fmaf(lrelu(x.w, slope), wk[4 * c4 + 3], acc);
      }
    }
    out[((long)b * c_out + oc) * L + p] = tanhf(acc);
  }
}

// conv_post for the common C == 32 case: the block stages its (256 + 6) activated input rows ONCE in shared
// memory with coalesced 128-bit loads (16-byte chunk c of row r at slot c ^ (r & 7): the row-per-thread reads
// below are then bank-conflict free); same accumulation order as the generic kernel (bit-identical results).
constexpr int CP_ROWS = 256;
__global__ void __launch_bounds__(CP_ROWS) conv_post32_kernel(const float* __restrict__ in, const float* __restrict__ w,
                                                               const float* __restrict__ bias, float* __restrict__ out,
                                                               int L, int c_out, float slope) {
  __shared__ float4 xs[(CP_ROWS + 6) * 8];
  extern __shared__ float ws[];
  for (int i = threadIdx.x; i < c_out * 7 * 32; i += CP_ROWS) ws[i] = w[i];
  const int b = blockIdx.y;
  const long p0 = (long)blockIdx.x * CP_ROWS;
  const float4* ib = reinterpret_cast<const float4*>(in + (long)b * L * 32);
  for (int i = threadIdx.x; i < (CP_ROWS + 6) * 8; i += CP_ROWS) {
    const int r = i >> 3, c = i & 7;
    const long q = p0 + r - 3;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q >= 0 && q < L) {
      v = __ldg(ib + q * 8 + c);
      v.x = lrelu(v.x, slope); v.y = lrelu(v.y, slope); v.z = lrelu(v.z, slope); v.w = lrelu(v.w, slope);
    }
    xs[r * 8 + (c ^ (r & 7))] = v;
  }
  __syncthreads();
  const long p = p0 + threadIdx.x;
  if (p >= L) return;
  for (int oc = 0; oc < c_out; ++oc) {
    float acc = bias[oc];
    const float* wo = ws + oc * 7 * 32;
#pragma unroll
    for (int k = 0; k < 7; ++k) {
      const long q = p + k - 3;
      if (q < 0 || q >= L) continue;          // (zero rows contribute nothing; skipping keeps the generic kernel's order)
      const int r = threadIdx.x + k;
      const float* wk = wo + k * 32;
#pragma unroll
      for (int c4 = 0; c4 < 8; ++c4) {
        const float4 x = xs[r * 8 + (c4 ^ (r & 7))];
        acc = fmaf(x.x, wk[4 * c4 + 0], acc);
        acc = fmaf(x.y, wk[4 * c4 + 1], acc);
        acc = fmaf(x.z, wk[4 * c4 + 2], acc);
        acc = fmaf(x.w, wk[4 * c4 + 3], acc);
      }
    }
    out[((long)b * c_out + oc) * L + p] = tanhf(acc);
  }
}

bool launch_conv_post(const float* in, const float* w, const float* b, float* out, int B, int L, int C, int c_out,
                      float slope, cudaStream_t st) {
  AGPT_CHECK(B >= 1 && L >= 1 && c_out >= 1 && C >= 4 && C % 4 == 0, "conv_post: needs C % 4 == 0 (float4 rows)");
  const size_t smem = (size_t)c_out * 7 * C * sizeof(float);
  AGPT_CHECK(smem <= 48 * 1024, "conv_post: c_out * 7 * C weights exceed 48 KB of shared memory");
  const int threads = 256;
  dim3 grid(cdiv(L, threads), B);
  const bool c32 = C == 32 && smem <= 8 * 1024;
  if (c32)
    conv_post32_kernel<<<grid, CP_ROWS, smem, st>>>(in, w, b, out, L, c_out, slope);
  else
    conv_post_kernel<<<grid, threads, smem, st>>>(in, w, b, out, L, C, c_out, slope);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
  return c32;
}

// Anti-aliased periodic activation of BigVGAN (Activation1d(Snake | SnakeBeta),
// vocoder/bigvgan/alias_free_torch/act.py:22-27, resample.py:22-31, filter.py:80-90, activations.py:46-57,104-117):
//   u = 2 * upfir2(replicate_pad(x, 5))[15:-15]          (12-tap Kaiser sinc, zero-stuffing stride 2: 6 taps per sample)
//   s = u + inv_b[c] * sin^2(a[c] * u)
//   y[t] = sum_k f[k] * replicate_pad(s, 5, 6)[2 t + k]   (stride-2 low-pass)
// on channels-last rows [B][L][C].  One block: AA_TT output rows x 32 channels; the x tile, then the
// activated 2x-rate samples are staged in shared memory so every sin() is evaluated once.
struct AaFilter { float f[12]; };
constexpr int AA_TT = 64;
__global__ void __launch_bounds__(256) aa_snake_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                        const float* __restrict__ a, const float* __restrict__ inv_b,
                                                        int L, int C, AaFilter F) {
  __shared__ float xs[AA_TT + 12][32];
  __shared__ float ss[2 * AA_TT + 10][32];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int c = blockIdx.y * 32 + tx;
  const int b = blockIdx.z;
  const int t0 = blockIdx.x * AA_TT;
  const bool cok = c < C;
  const float* xb = x + (long)b * L * C;
  for (int r = ty; r < AA_TT + 12; r += 8) {
    const int t = min(max(t0 - 6 + r, 0), L - 1);
    xs[r][tx] = cok ? __ldg(xb + (long)t * C + c) : 0.f;
  }
  __syncthreads();
  const float av = cok ? a[c] : 0.f, ib = cok ? inv_b[c] : 0.f;
  // up-FIR: sample m = 2 i + r of the zero-stuffed convolution touches the 6 taps k = (n & 1) + 2 q, n = m + 15,
  // applied to x[(n >> 1) - 5 - q] (replicate-clamped); taps are visited in ascending k like a direct convolution
  for (int j = ty; j < 2 * AA_TT + 10; j += 8) {
    const int m = min(max(2 * t0 - 5 + j, 0), 2 * L - 1);
    const int n = m + 15;
    const bool odd = (n & 1) != 0;
    const int base = (n >> 1) - 5;
    float u = 0.f;
#pragma unroll
    for (int q = 0; q < 6; ++q) {
      const int xi = min(max(base - q, 0), L - 1) - (t0 - 6);
      u = fmaf(odd ? F.f[2 * q + 1] : F.f[2 * q], xs[xi][tx], u);
    }
    u *= 2.f;
    const float sn = sinf(u * av);
    ss[j][tx] = u + ib * (sn * sn);
  }
  __syncthreads();
  float* yb = y + (long)b * L * C;
  for (int r = ty; r < AA_TT; r += 8) {
    const int t = t0 + r;
    if (t >= L || !cok) continue;
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 12; ++k) acc = fmaf(F.f[k], ss[2 * r + k][tx], acc);
    yb[(long)t * C + c] = acc;
  }
}

void aa_snake(const float* x, float* y, const float* a, const float* inv_b, const float* taps, int B, int L, int C,
              cudaStream_t st) {
  AGPT_CHECK(B >= 1 && L >= 1 && C >= 1 && taps, "aa_snake: needs L >= 1 and the 12 filter taps");
  AaFilter F;
  for (int k = 0; k < 12; ++k) F.f[k] = taps[k];
  dim3 block(32, 8), grid(cdiv(L, AA_TT), cdiv(C, 32), B);
  aa_snake_kernel<<<grid, block, 0, st>>>(x, y, a, inv_b, L, C, F);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// NSF excitation add: x[b][p][c] += bias[c] + sum_k w[c][k] * har[b][p*st - pad + k]   (hifigan.py:155-157)
__global__ void nsf_add_kernel(float* __restrict__ x, const float* __restrict__ har, const float* __restrict__ w,
                               const float* __restrict__ bias, int L, int C, int Lh, int K, int st, int pad) {
  const int b = blockIdx.z;
  const int p = blockIdx.x * blockDim.y + threadIdx.y;
  const int c = blockIdx.y * blockDim.x + threadIdx.x;
  if (p >= L || c >= C) return;
  const float* hb = har + (long)b * Lh;
  float acc = bias[c];
  const int base = p * st - pad;
  for (int k = 0; k < K; ++k) {
    const int q = base + k;
    if (q >= 0 && q < Lh) acc = fmaf(w[c * K + k], hb[q], acc);
  }
  x[((long)b * L + p) * C + c] += acc;
}

void nsf_add(float* x, const float* har, const float* w, const float* bias, int B, int L, int C, int Lh, int K, int stride,
             int pad, cudaStream_t st) {
  AGPT_CHECK(B >= 1 && L >= 1 && C >= 1 && K >= 1 && stride >= 1, "nsf_add: needs K >= 1 and stride >= 1");
  dim3 block(32, 8), grid(cdiv(L, 8), cdiv(C, 32), B);
  nsf_add_kernel<<<grid, block, 0, st>>>(x, har, w, bias, L, C, Lh, K, stride, pad);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// ------------------------------------------------------------------ NSF harmonic source (SourceModuleHnNSF)
// NeuralSeq/modules/parallel_wavegan/models/source.py:311-441 (SineGen), :484-532 (SourceModuleHnNSF):
//   rad[t,h]  = (f0[t] * (h+1) / sr) mod 1          (+ rand_ini[h] at t = 0, rand_ini[0] = 0)
//   sines     = sin(2 pi * cumsum_t(rad)) * sine_amp   -- the reference subtracts 1 whenever the running sum wraps
//                                                         (source.py:369-377); sin is 1-periodic in that sum, so the
//                                                         phase is the FRACTIONAL part of the prefix sum
//   x[t,h]    = sines * uv[t] + (uv * noise_std + (1 - uv) * sine_amp / 3) * noise[t,h],   uv = f0 > threshold
//   har[t]    = tanh(b + sum_h w[h] * x[t,h])
// The prefix sum over the 10^5 samples of an utterance is a three-level scan in double precision (chunk sums ->
// one sequential pass over the chunk sums per (utterance, harmonic) -> in-chunk block scan), so the phase is exact to
// fp64 rounding where the reference's sequential fp32 cumsum drifts by ~1e-5 cycles; the random draws (initial
// phases, noise) stay with the caller in the reference's torch call order.
constexpr int NSF_CHUNK = 1024, NSF_MAXH = 16;
struct NsfLin { float w[NSF_MAXH]; float b; };

__device__ __forceinline__ float nsf_rad(float f0, int h, float sr) {
  const float v = (f0 * (float)(h + 1)) / sr;      // f0_buf[:, :, h] = f0 * (h + 1); (f0_values / sampling_rate) % 1
  return v - floorf(v);                             // torch's % on floats: result in [0, 1)
}

// chunk sums: grid (nchunks, dim, B)
__global__ void nsf_chunk_sum_kernel(const float* __restrict__ f0, double* __restrict__ csum, int L, int dim, float sr) {
  __shared__ double red[8];
  const int c = blockIdx.x, h = blockIdx.y, b = blockIdx.z, nch = gridDim.x;
  const float* fb = f0 + (long)b * L;
  double s = 0.0;
  for (int i = threadIdx.x; i < NSF_CHUNK; i += blockDim.x) {
    const int t = c * NSF_CHUNK + i;
    if (t < L) s += (double)nsf_rad(fb[t], h, sr);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
    csum[((long)b * dim + h) * nch + c] = t;
  }
}
// exclusive scan of the chunk sums (fractional part), seeded with the initial phase: one thread per (b, h)
__global__ void nsf_chunk_scan_kernel(double* __restrict__ csum, const float* __restrict__ rand_ini, int nch, int dim, int B) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * dim) return;
  const int h = i % dim;
  double acc = (h == 0 || !rand_ini) ? 0.0 : (double)rand_ini[i];
  double* cs = csum + (long)i * nch;
  for (int c = 0; c < nch; ++c) {
    const double v = cs[c];
    cs[c] = acc;
    acc += v;
    acc -= floor(acc);
  }
}
// in-chunk inclusive scan + sines + merge: grid (nchunks, B), 256 threads x 4 samples
__global__ void __launch_bounds__(256) nsf_source_kernel(const float* __restrict__ f0, const double* __restrict__ cbase,
                                                          const float* __restrict__ noise, float* __restrict__ har,
                                                          int L, int dim, float sr, float sine_amp, float noise_std, float thr,
                                                          NsfLin lin) {
  __shared__ double wsum[8];
  const int c = blockIdx.x, b = blockIdx.y, nch = gridDim.x;
  const int t0 = c * NSF_CHUNK + threadIdx.x * 4;
  const float* fb = f0 + (long)b * L;
  float fv[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) fv[k] = (t0 + k < L) ? fb[t0 + k] : 0.f;
  float acc[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) acc[k] = lin.b;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int h = 0; h < dim; ++h) {
    double r[4], run = 0.0;
#pragma unroll
    for (int k = 0; k < 4; ++k) { run += (double)nsf_rad(fv[k], h, sr); r[k] = run; }     // thread-local inclusive sums
    double inc = run;                                                                       // warp inclusive scan of the thread totals
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const double v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
    __syncthreads();
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    double base = cbase[((long)b * dim + h) * nch + c];
    for (int w = 0; w < warp; ++w) base += wsum[w];
    base += inc - run;                                                                      // exclusive prefix of this thread
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int t = t0 + k;
      if (t >= L) continue;
      double ph = base + r[k];
      ph -= floor(ph);
      const float sn = sinf((float)ph * 6.283185307179586f) * sine_amp;
      const float uv = fv[k] > thr ? 1.f : 0.f;
      const float na = uv * noise_std + (1.f - uv) * sine_amp / 3.f;
      const float nz = noise ? noise[((long)b * L + t) * dim + h] : 0.f;
      acc[k] = fmaf(lin.w[h], sn * uv + na * nz, acc[k]);
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (t0 + k < L) har[(long)b * L + t0 + k] = tanhf(acc[k]);
}

static DevBuf g_nsf_scratch[16];

// f0 [B][L] (already at the sample rate), rand_ini [B][dim] or null, noise [B][L][dim] or null -> har [B][L]
void nsf_source(const float* f0, int B, int L, int dim, float sr, const float* lin_w_host, float lin_b,
                const float* rand_ini, const float* noise, float sine_amp, float noise_std, float thr, float* har,
                cudaStream_t st) {
  AGPT_CHECK(B >= 1 && L >= 1 && dim >= 1 && dim <= NSF_MAXH, "nsf_source: bad shape (at most 16 harmonics)");
  int dev = 0;
  AGPT_CUDA(cudaGetDevice(&dev));
  const int nch = cdiv(L, NSF_CHUNK);
  double* cs = reinterpret_cast<double*>(g_nsf_scratch[dev & 15].ensure((size_t)B * dim * nch * 2 + 2));
  NsfLin lin;
  for (int h = 0; h < NSF_MAXH; ++h) lin.w[h] = h < dim ? lin_w_host[h] : 0.f;
  lin.b = lin_b;
  nsf_chunk_sum_kernel<<<dim3(nch, dim, B), 256, 0, st>>>(f0, cs, L, dim, sr);
  nsf_chunk_scan_kernel<<<cdiv(B * dim, 64), 64, 0, st>>>(cs, rand_ini, nch, dim, B);
  nsf_source_kernel<<<dim3(nch, B), 256, 0, st>>>(f0, cs, noise, har, L, dim, sr, sine_amp, noise_std, thr, lin);
  count_launch(3);
  AGPT_CUDA(cudaGetLastError());
}

struct SnakeW { DevBuf a, inv_b; };   // per-channel exp(alpha) (or alpha) and 1 / (beta + 1e-9)

struct ResBlockW {
  int ks = 0;
  std::vector<int> dil;
  std::vector<PackedConv> c1, c2;  // c2 empty for ResBlock2
  std::vector<PackedConv> c1g, c2g;  // time-grouped images of the dilation-1 convs of narrow stages (pack_conv_grouped)
  std::vector<int> g1, g2;           // their group factor (0: not grouped)
  std::vector<SnakeW> act;          // BigVGAN: one anti-aliased snake per conv (AMPBlock1: 2 per pair)
};

struct NoiseConvW {
  DevBuf w, b;
  int K = 0, st = 1, pad = 0, C = 0;
};

struct Hifigan : Handle {
  agpt_hifigan_cfg cfg;
  PackedConv conv_pre;
  std::vector<PackedConv> ups;
  std::vector<ResBlockW> rbs;
  std::vector<NoiseConvW> noise;
  DevBuf post_w, post_b;
  SnakeW act_post;                  // BigVGAN activation_post
  AaFilter aaf;                     // the 12 Kaiser-sinc taps (state-dict buffer)
  int c_last = 0, hop = 1;
  DevBuf melT, buf[6], sbuf;        // sbuf: activated conv input (BigVGAN only)
  DevBuf plane[6];                  // plane[k]: operand plane of buf[k] (fp16 hi, then lo), HiFi-GAN plane feed only
  DevBuf io_mel, io_wav, io_har;  // staging for the host-buffer entry point
  float* pin_mel = nullptr; float* pin_wav = nullptr; size_t pin_mel_n = 0, pin_wav_n = 0;
  cudaStream_t own_stream = nullptr;
  bool fuse_resblock = true;        // AGPT_FUSE_RESBLOCK=0: every ResBlock1 conv as its own launch
  bool tall_tiles = true;           // AGPT_TALL_TILES=0: 128-row tiles only (TapConvParams::tc_tall)
  bool plane_feed = true;           // AGPT_PLANE_FEED=0: every tap-GEMM converts its fp32 input itself
  bool pair_dual = true;            // AGPT_PAIR_DUAL=0: no fused pair runs two CTAs per SM (TapConvParams::tc_dual)
  bool pair_pipe = true;            // AGPT_PAIR_PIPE=0: no C = 128 pair runs two tiles per CTA (TapConvParams::tc_pipe)
  bool pair_pipe_stage = true;      // AGPT_PAIR_PIPE_STAGE=0: those pairs load their input and residual per thread
  bool narrow_pipe = true;          // AGPT_NARROW_PIPE=0: narrow pairs keep two CTAs per SM (TapConvParams::tc_narrow_pipe)
  bool conv_pipe = true;            // AGPT_CONV_PIPE=0: plane-fed convs keep one tile per CTA (TapConvParams::tc_conv_pipe)

  ~Hifigan() override {
    if (pin_mel) cudaFreeHost(pin_mel);
    if (pin_wav) cudaFreeHost(pin_wav);
    if (own_stream) cudaStreamDestroy(own_stream);
  }

  void forward(const float* mel, const float* har, int B, int T, float* wav, cudaStream_t st) {
    AGPT_CHECK(B >= 1 && T >= 1, "empty batch");
    const int C0 = cfg.upsample_initial_channel;
    // buffer sizing: max over stages of L_i * C_i
    size_t mx = (size_t)T * C0;
    {
      long L = T; int C = C0;
      for (int i = 0; i < cfg.num_upsamples; ++i) { L *= cfg.upsample_rates[i]; C /= 2; mx = std::max(mx, (size_t)L * C); }
    }
    mx *= (size_t)B;
    for (auto& b : buf) b.ensure(mx);
    melT.ensure((size_t)B * T * cfg.n_mels);
    float *cur = buf[0].p, *acc = buf[1].p, *X = buf[2].p, *A = buf[3].p, *R0 = buf[4].p, *R1 = buf[5].p;
    const bool big = cfg.activation != 0;          // BigVGAN: anti-aliased snake instead of leaky-relu
    if (big) sbuf.ensure(mx);
    float* S = sbuf.p;
    // Operand planes (TapConvParams::pi_hi / po_hi): a leaky-ReLU(0.1) tap-GEMM reads its input as a pre-split fp16
    // hi / lo plane, written once by the epilogue that produced the tensor (or by plane_split where no tap-GEMM did),
    // instead of converting the fp32 tensor in every tile.  Only tensors of more than 128 channels get a plane: their
    // consumers (the unfused convs of the first stage, the upsamplers) run several 128-wide co-tiles, each of which
    // would convert the same rows again, so the plane saves more than the 4 bytes per element its write costs.  The
    // consumers of narrower tensors (the fused pairs, ups of C <= 128) run one co-tile; there, writing the plane in
    // the producer's epilogue costs more than the conversion it saves (measured on H100, DESIGN.md section 4).
    const bool planes = plane_feed && !big && tc_enabled();
    auto has_plane = [&](int ch) { return planes && ch > 128 && ch % 8 == 0; };
    size_t mxp = 0;   // elements of the largest tensor with a plane
    {
      long Lp = T; int Cp = C0;
      for (int i = 0; i <= cfg.num_upsamples; ++i) {
        if (has_plane(Cp)) mxp = std::max(mxp, (size_t)B * Lp * Cp);
        if (i < cfg.num_upsamples) { Lp *= cfg.upsample_rates[i]; Cp /= 2; }
      }
    }
    if (mxp) for (auto& p : plane) p.ensure(mxp);   // mxp floats = 2 mxp halves: hi [mxp], lo [mxp]
    auto plane_hi = [&](const float* t) -> __half* {
      for (int k = 0; k < 6; ++k)
        if (buf[k].p == t) return reinterpret_cast<__half*>(plane[k].p);
      throw Error("hifigan: no operand plane for this tensor");
    };
    // ch: channels of the tensor (the plane view of a time-grouped launch has the same plane)
    auto feed = [&](TapConvParams& P, int ch) {                // P reads its input's plane
      if (!has_plane(ch)) return;
      P.pi_hi = plane_hi(P.in); P.pi_lo = P.pi_hi + mxp;
      P.tc_conv_pipe = conv_pipe;
    };
    auto emit = [&](TapConvParams& P, int ch, bool keep_fp32) {   // P's epilogue writes its output's plane too (or only)
      if (!has_plane(ch)) return;
      P.po_hi = plane_hi(P.out); P.po_lo = P.po_hi + mxp; P.po_slope = 0.1f;
      if (!keep_fp32) P.out = nullptr;
    };
    auto split = [&](const float* t, long rows, int ch) {
      if (has_plane(ch)) plane_split(t, plane_hi(t), plane_hi(t) + mxp, rows * ch, 0.1f, st);
    };
    auto snake = [&](const float* src, float* dst, long Lr, int Cr, const SnakeW& w) {
      aa_snake(src, dst, w.a.p, w.inv_b.p, aaf.f, B, (int)Lr, Cr, st);
    };
    launch_cf_to_cl(mel, melT.p, B, cfg.n_mels, T, st);
    {
      TapConvParams P = tapconv_params(conv_pre, B, T, 0, 1);
      P.in = melT.p; P.in_gstride = (long)T * cfg.n_mels; P.in_pitch = cfg.n_mels;
      P.out = cur; P.out_gstride = (long)T * C0; P.out_pitch = C0;
      P.pro = PRO_NONE; P.epi = EPI_BIAS;
      P.tc_tall = tall_tiles;
      tapconv_launch(P, st);
    }
    split(cur, (long)B * T, C0);   // conv_pre reads the mel, not a plane: its output's plane comes from a split pass
    long L = T; int C = C0;
    const float inv_nk = 1.f / (float)cfg.num_kernels;
    for (int i = 0; i < cfg.num_upsamples; ++i) {
      const int u = cfg.upsample_rates[i];
      const int Co = C / 2;
      {  // leaky_relu(0.1) -> ConvTranspose1d   (hifigan.py:153-154)
        TapConvParams P = tapconv_params(ups[i], B, (int)L, 0, 1);
        P.in = cur; P.in_gstride = L * C; P.in_pitch = C;
        P.out = X; P.out_gstride = L * u * Co; P.out_pitch = u * Co;
        P.pro = big ? PRO_NONE : PRO_LRELU; P.slope = 0.1f; P.epi = EPI_BIAS;   // BigVGAN upsamples x directly (models.py:184-186)
        P.tc_tall = tall_tiles;
        feed(P, C);
        if (!har) emit(P, Co, true);   // X is also every first pair's residual
        tapconv_launch(P, st);
      }
      L *= u; C = Co;
      if (har) {
        AGPT_CHECK(cfg.use_nsf, "har_source given but the generator has no noise_convs");
        const NoiseConvW& nc = noise[i];
        nsf_add(X, har, nc.w.p, nc.b.p, B, (int)L, C, T * hop, nc.K, nc.st, nc.pad, st);
        split(X, (long)B * L, C);   // the plane of X after the excitation add
      }
      const long gs = L * C;
      auto gview = [&](int g) { return (g && L % g == 0) ? g : 1; };   // time-grouped view [L/g][g*C] of the same memory
      // one conv of a ResBlock over the view gq (1: plain rows [L][C]); the caller sets the epilogue
      auto conv = [&](const PackedConv& plain, const PackedConv& grouped, int gq, int dil, const float* in, float* out) {
        TapConvParams P = gq > 1 ? tapconv_params(grouped, B, (int)(L / gq), 0, 1) : tapconv_params(plain, B, (int)L, 0, dil);
        P.in = in; P.in_gstride = gs; P.in_pitch = gq * C;
        P.out = out; P.out_gstride = gs; P.out_pitch = gq * C;
        P.pro = big ? PRO_NONE : PRO_LRELU; P.slope = 0.1f;
        P.tc_tall = tall_tiles;
        return P;
      };
      for (int j = 0; j < cfg.num_kernels; ++j) {
        const ResBlockW& rb = rbs[i * cfg.num_kernels + j];
        const float* x = X;
        const int nd = (int)rb.dil.size();
        for (int n = 0; n < nd; ++n) {
          const bool last = (n == nd - 1);
          float* dst = last ? acc : ((n & 1) ? R1 : R0);
          // dst feeds the next pair, or (the completed MRF sum) the next upsampler; conv_post reads the fp32 sum
          const bool dst_plane = !last || (j == cfg.num_kernels - 1 && i + 1 < cfg.num_upsamples);
          auto residual_epi = [&](TapConvParams& P) {   // x + conv(...), on the last pair into the MRF accumulator
            P.res = x; P.res_gstride = gs; P.res_pitch = P.in_pitch;
            if (last) { P.epi = EPI_ACC; P.scale = inv_nk; P.accumulate = (j > 0); }
            else P.epi = EPI_RES;
          };
          const bool t1 = cfg.resblock_type == 1;
          if (t1 && !big && fuse_resblock) {
            // both convs in one launch (tcpair_launch; not taken for C > 128 or without tensor cores).  c2 takes c1's
            // view, so a grouped c2 after a dilated c1 runs ungrouped: on H100 that pair is still faster fused.
            const int gq = gview(rb.g1[n]) == gview(rb.g2[n]) ? gview(rb.g1[n]) : 1;
            TapConvParams P1 = conv(rb.c1[n], rb.c1g[n], gq, rb.dil[n], x, A);
            P1.epi = EPI_BIAS;
            P1.tc_dual = pair_dual;
            P1.tc_pipe = pair_pipe ? (pair_pipe_stage ? 1 : 2) : 0;
            P1.tc_narrow_pipe = narrow_pipe;
            feed(P1, C);
            TapConvParams P2 = conv(rb.c2[n], rb.c2g[n], gq, 1, A, dst);
            residual_epi(P2);
            if (dst_plane) emit(P2, C, true);
            if (tcpair_launch(P1, P2, st)) { x = dst; continue; }
          }
          const float* conv_in = x;
          if (t1) {
            if (big) snake(x, S, L, C, rb.act[2 * n]);      // xt = a1(x)   (AMPBlock1.forward, models.py:75-76)
            TapConvParams P = conv(rb.c1[n], rb.c1g[n], gview(rb.g1[n]), rb.dil[n], big ? S : x, A);
            P.epi = EPI_BIAS;
            feed(P, C);
            emit(P, C, false);   // A is read only by c2, as a plane
            tapconv_launch(P, st);
            conv_in = A;
          }
          if (big) {                                        // a2(xt) resp. AMPBlock2's a(x)
            snake(conv_in, S, L, C, rb.act[t1 ? 2 * n + 1 : n]);
            conv_in = S;
          }
          TapConvParams P = t1 ? conv(rb.c2[n], rb.c2g[n], gview(rb.g2[n]), 1, conv_in, dst)
                               : conv(rb.c1[n], rb.c1g[n], gview(rb.g1[n]), rb.dil[n], conv_in, dst);
          residual_epi(P);
          feed(P, C);
          if (dst_plane) emit(P, C, true);
          tapconv_launch(P, st);
          x = dst;
        }
      }
      std::swap(cur, acc);
    }
    {
      const float* pin = cur;
      float slope = 0.01f;                      // HiFi-GAN: F.leaky_relu default slope (hifigan.py:165)
      if (big) { snake(cur, S, L, C, act_post); pin = S; slope = 1.f; }   // BigVGAN: activation_post, no leaky-relu
      launch_conv_post(pin, post_w.p, post_b.p, wav, B, (int)L, C, cfg.c_out, slope, st);
    }
  }
};

Handle* hifigan_create(const agpt_hifigan_cfg* cfg, const float* const* W, int nW, int device) {
  DeviceGuard dg_(device);
  const int nu = cfg->num_upsamples, nk = cfg->num_kernels;
  AGPT_CHECK(nu >= 1 && nu <= AGPT_MAX_UPS && nk >= 1 && nk <= AGPT_MAX_RBK, "bad config");
  const int C0 = cfg->upsample_initial_channel;
  for (int i = 0, C = C0; i < nu; ++i, C /= 2)
    AGPT_CHECK(C % 2 == 0 && (C / 2) % 4 == 0, "channel counts must stay multiples of 4");
  for (int j = 0; j < nk; ++j)
    AGPT_CHECK(cfg->resblock_kernel_sizes[j] % 2 == 1 && cfg->resblock_kernel_sizes[j] <= kMaxTaps,
               "resblock kernel size must be odd and <= 11");
  // ConvTranspose1d(k, u, padding=(k-u)//2) yields L*u + (k-u) % 2 samples: the engine's polyphase upsampler and its
  // T * hop output are exactly L*u, so an odd k - u would silently drop the reference's last sample of every stage
  for (int i = 0; i < nu; ++i)
    AGPT_CHECK(cfg->upsample_rates[i] >= 1 && cfg->upsample_kernel_sizes[i] >= cfg->upsample_rates[i] &&
                   (cfg->upsample_kernel_sizes[i] - cfg->upsample_rates[i]) % 2 == 0,
               "upsample kernel size k and rate u need k >= u and an even k - u (else the stage does not output L*u samples)");
  std::unique_ptr<Hifigan> h(new Hifigan());
  h->magic = kMagicHifigan; h->device = device; h->cfg = *cfg;
  { const char* e = getenv("AGPT_FUSE_RESBLOCK"); h->fuse_resblock = !(e && e[0] == '0'); }
  { const char* e = getenv("AGPT_TALL_TILES"); h->tall_tiles = !(e && e[0] == '0'); }
  { const char* e = getenv("AGPT_PLANE_FEED"); h->plane_feed = !(e && e[0] == '0'); }
  { const char* e = getenv("AGPT_PAIR_DUAL"); h->pair_dual = !(e && e[0] == '0'); }
  { const char* e = getenv("AGPT_PAIR_PIPE"); h->pair_pipe = !(e && e[0] == '0'); }
  { const char* e = getenv("AGPT_PAIR_PIPE_STAGE"); h->pair_pipe_stage = !(e && e[0] == '0'); }
  { const char* e = getenv("AGPT_NARROW_PIPE"); h->narrow_pipe = !(e && e[0] == '0'); }
  { const char* e = getenv("AGPT_CONV_PIPE"); h->conv_pipe = !(e && e[0] == '0'); }
  WeightCursor wc{W, nW};
  { const float* w = wc.next(); const float* b = wc.next(); pack_conv(h->conv_pre, w, b, C0, cfg->n_mels, 7, false); }
  h->ups.resize(nu);
  int C = C0; h->hop = 1;
  for (int i = 0; i < nu; ++i) {
    const float* w = wc.next(); const float* b = wc.next();
    const int u = cfg->upsample_rates[i], k = cfg->upsample_kernel_sizes[i];
    pack_convtranspose(h->ups[i], w, b, C, C / 2, k, u, (k - u) / 2);
    C /= 2; h->hop *= u;
  }
  h->c_last = C;
  // BigVGAN (cfg.activation 1 = Snake, 2 = SnakeBeta): alpha [, beta] vectors follow each block's convs
  auto load_snake = [&](SnakeW& sw, int ch) {
    const float* al = wc.next();
    const float* be = (cfg->activation == 2) ? wc.next() : al;
    std::vector<float> a(ch), ib(ch);
    for (int c = 0; c < ch; ++c) {
      const float av = cfg->snake_logscale ? std::exp(al[c]) : al[c];
      const float bv = cfg->snake_logscale ? std::exp(be[c]) : be[c];
      a[c] = av;
      ib[c] = 1.0f / (bv + 0.000000001f);
    }
    sw.a.upload(a); sw.inv_b.upload(ib);
  };
  h->rbs.resize((size_t)nu * nk);
  C = C0;
  for (int i = 0; i < nu; ++i) {
    C /= 2;
    for (int j = 0; j < nk; ++j) {
      ResBlockW& rb = h->rbs[i * nk + j];
      rb.ks = cfg->resblock_kernel_sizes[j];
      const int nd = cfg->resblock_num_dilations[j];
      rb.dil.assign(cfg->resblock_dilations[j], cfg->resblock_dilations[j] + nd);
      // narrow stages: dilation-1 convs with k >= 7 also get a time-grouped image (N = 128 per MMA instead of C)
      auto group_of = [&](int dil) {
        if (cfg->activation != 0 || dil != 1 || rb.ks < 7) return 0;
        if (C == 32) return 4;
        if (C == 64 && rb.ks >= 11) return 2;
        return 0;
      };
      rb.c1.resize(nd); rb.c1g.resize(nd); rb.g1.assign(nd, 0);
      for (int n = 0; n < nd; ++n) {
        const float* w = wc.next(); const float* b = wc.next();
        pack_conv(rb.c1[n], w, b, C, C, rb.ks, false);
        rb.g1[n] = group_of(rb.dil[n]);
        if (rb.g1[n]) pack_conv_grouped(rb.c1g[n], w, b, C, rb.ks, rb.g1[n]);
      }
      if (cfg->resblock_type == 1) {
        rb.c2.resize(nd); rb.c2g.resize(nd); rb.g2.assign(nd, 0);
        for (int n = 0; n < nd; ++n) {
          const float* w = wc.next(); const float* b = wc.next();
          pack_conv(rb.c2[n], w, b, C, C, rb.ks, false);
          rb.g2[n] = group_of(1);
          if (rb.g2[n]) pack_conv_grouped(rb.c2g[n], w, b, C, rb.ks, rb.g2[n]);
        }
      }
      if (cfg->activation != 0) {
        rb.act.resize(cfg->resblock_type == 1 ? 2 * nd : nd);
        for (auto& a : rb.act) load_snake(a, C);
      }
    }
  }
  if (cfg->activation != 0) load_snake(h->act_post, C);
  {  // conv_post [c_out][C][7] -> [c_out][7][C]
    const float* w = wc.next(); const float* b = wc.next();
    std::vector<float> pw((size_t)cfg->c_out * 7 * C);
    for (int oc = 0; oc < cfg->c_out; ++oc)
      for (int c = 0; c < C; ++c)
        for (int k = 0; k < 7; ++k) pw[((size_t)oc * 7 + k) * C + c] = w[((size_t)oc * C + c) * 7 + k];
    h->post_w.upload(pw);
    h->post_b.upload(b, cfg->c_out);
  }
  if (cfg->activation != 0) {   // the Kaiser-sinc taps (identical upsample / downsample buffers of every Activation1d)
    const float* f = wc.next();
    for (int k = 0; k < 12; ++k) h->aaf.f[k] = f[k];
  }
  if (cfg->use_nsf) {
    wc.next(); wc.next();  // m_source.l_linear.{weight,bias}: the source module stays on the host side (RNG)
    h->noise.resize(nu);
    int Cc = C0;
    for (int i = 0; i < nu; ++i) {
      Cc /= 2;
      NoiseConvW& nc = h->noise[i];
      nc.C = Cc;
      if (i + 1 < nu) {
        int stv = 1; for (int q = i + 1; q < nu; ++q) stv *= cfg->upsample_rates[q];
        nc.st = stv; nc.K = 2 * stv; nc.pad = stv / 2;
      } else { nc.st = 1; nc.K = 1; nc.pad = 0; }
      const float* w = wc.next(); const float* b = wc.next();
      nc.w.upload(w, (size_t)Cc * nc.K);
      nc.b.upload(b, Cc);
    }
  }
  wc.done();
  return h.release();
}

void hifigan_forward(Handle* hh, const float* mel, const float* har, int B, int T, float* wav, cudaStream_t st) {
  auto* h = static_cast<Hifigan*>(hh);
  DeviceGuard dg_(h->device);
  h->forward(mel, har, B, T, wav, st);
}

void hifigan_vocode_host(Handle* hh, const float* mel_host, const float* har_host, int B, int T, float* wav_host) {
  auto* h = static_cast<Hifigan*>(hh);
  DeviceGuard dg_(h->device);
  if (!h->own_stream) AGPT_CUDA(cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking));
  const size_t nmel = (size_t)B * h->cfg.n_mels * T, nwav = (size_t)B * h->cfg.c_out * T * h->hop;
  const size_t nhar = (size_t)B * T * h->hop;
  if (h->pin_mel_n < nmel) { if (h->pin_mel) cudaFreeHost(h->pin_mel); AGPT_CUDA(cudaMallocHost(&h->pin_mel, nmel * 4)); h->pin_mel_n = nmel; }
  if (h->pin_wav_n < nwav) { if (h->pin_wav) cudaFreeHost(h->pin_wav); AGPT_CUDA(cudaMallocHost(&h->pin_wav, nwav * 4)); h->pin_wav_n = nwav; }
  h->io_mel.ensure(nmel); h->io_wav.ensure(nwav);
  memcpy(h->pin_mel, mel_host, nmel * 4);
  cudaStream_t st = h->own_stream;
  AGPT_CUDA(cudaMemcpyAsync(h->io_mel.p, h->pin_mel, nmel * 4, cudaMemcpyHostToDevice, st));
  const float* har_dev = nullptr;
  if (har_host) {
    h->io_har.ensure(nhar);
    AGPT_CUDA(cudaMemcpyAsync(h->io_har.p, har_host, nhar * 4, cudaMemcpyHostToDevice, st));
    har_dev = h->io_har.p;
  }
  h->forward(h->io_mel.p, har_dev, B, T, h->io_wav.p, st);
  AGPT_CUDA(cudaMemcpyAsync(h->pin_wav, h->io_wav.p, nwav * 4, cudaMemcpyDeviceToHost, st));
  AGPT_CUDA(cudaStreamSynchronize(st));
  memcpy(wav_host, h->pin_wav, nwav * 4);
}

}  // namespace agpt
