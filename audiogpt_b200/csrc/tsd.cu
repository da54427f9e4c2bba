// The target-sound-detection tool's RaDur_fusion on sm_90a: a log-mel clip and the log-mel of a reference example of
// the target event -> framewise probabilities that the event is present.
// Reference: audio_detection/target_sound_detection/src/models.py:175-218 (ConvBlock), :220-256 (ConvBlock_GLU),
// :304-377 (Cnn14, which here takes the mel directly), :422-479 (Cnn10_mul_scale), :698-718 (conv1d = 1-wide Conv1d +
// ReLU), :770-788 (Fusion), :1058-1106 (CDur_CNN_mul_scale_fusion), :1109-1291 (RaDur_fusion, eval mode).
// Activations are channels-last [B][H = time][W = mel][C], as Cnn14Net's; the reference's transpose(1, 2).flatten(-2)
// after each CNN is then the identity, since both CNNs end at width 1.  Eval BatchNorm is folded into the preceding
// convs, RaDur_fusion.bn into a second copy of encoder.fc1, and detection.fc -> outputlayer (no activation between
// them) into one [outputdim][1024] matrix.
// On the tap-GEMM: every 3 x 3 conv (convblock.cuh), encoder.fc1, both Fusion layers that vary over time, and the GRU's
// input projections of both directions (one 512 -> 3072 GEMM).  New kernels: the fused multi-scale GLU stem, a general
// average pool, the bidirectional GRU recurrence (one 16-CTA cluster per direction, W_hh resident in shared memory, h
// exchanged over DSMEM), the attention pooling of the reference embeddings, the enhancement tail, the Fusion product,
// the fc / outputlayer / softmax head and the two-pass mix + linear interpolation.
#include <cooperative_groups.h>
#include "common.cuh"
#include "tapconv.cuh"
#include "models.h"
#include "convblock.cuh"
#include "an_kernels.cuh"

namespace cg = cooperative_groups;

namespace agpt {

namespace {

constexpr float kBnEps = 1e-5f;
constexpr int kMel = 64;
constexpr int kEmb = 128;                       // Cnn14.fc1 width = the embedding width
constexpr int kEnc = 6;
constexpr int kEncCh[kEnc] = {64, 128, 256, 512, 1024, 2048};
constexpr int kDetCh[3] = {128, 256, 512};      // Cnn10_mul_scale.conv_block2..4
constexpr int kStemC = 96;                      // three GLU branches of 32 channels
constexpr int kStemRowsMax = 500;               // x1[:, :, :500, :32]
constexpr int kFeat = 512;                      // GRU input and hidden size
constexpr int kFuse = 1024;                     // detection.fusion: 2 x 512
constexpr float kTemperature = 11.3f;           // RaDur_fusion.temperature, as written
constexpr int kMaxFramesDet = 500;              // T' <= the stem's 500-row crop

// ---- the GRU cluster: 16 CTAs per direction, each owning 32 hidden units (96 rows of W_hh in fp32 = 192 KB)
constexpr int kGruH = 512, kGruCta = 16, kGruU = kGruH / kGruCta, kGruRows = 3 * kGruU, kGruThreads = 512, kGruMaxB = 4;
constexpr size_t kGruSmem = sizeof(float) * ((size_t)kGruRows * kGruH + 2 * kGruMaxB * kGruH + kGruMaxB * kGruRows + kGruMaxB * kGruU);

// Cnn10_mul_scale's pool sizes (models.py:436-455) from time_resolution (CDur_CNN_mul_scale_fusion.__init__: 125 -> 8,
// 250 -> 4, 500 -> 2, anything else -> 0)
void det_pools(int time_resolution, int p[4][2]) {
  static const int tab[4][4][2] = {{{2, 2}, {2, 2}, {2, 4}, {1, 4}},    // scale 8
                                   {{2, 2}, {2, 2}, {1, 4}, {1, 4}},    // scale 4
                                   {{2, 2}, {1, 2}, {1, 4}, {1, 4}},    // scale 2
                                   {{1, 2}, {1, 2}, {1, 4}, {1, 4}}};   // scale 0
  const int s = time_resolution == 125 ? 0 : time_resolution == 250 ? 1 : time_resolution == 500 ? 2 : 3;
  memcpy(p, tab[s], sizeof(tab[s]));
}

// ---- Cnn14's first conv reads a 4-channel input: img[b][t][m] = (mel[b][t][m], 0, 0, 0)
__global__ void tsd_pad4_kernel(const float* __restrict__ mel, float4* __restrict__ img, long n) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    img[i] = make_float4(mel[i], 0.f, 0.f, 0.f);
}

// ---- F.avg_pool2d(kernel = stride = (ph, pw)), floor: out [B][H / ph][W / pw][C]; the window is summed row by row,
// then divided by ph * pw, as ATen's CPU kernel does
__global__ void tsd_avgpool_kernel(const float4* __restrict__ in, float4* __restrict__ out, int H, int W, int C4, int ph, int pw,
                                   int Ho, int Wo, long total) {
  const float d = (float)(ph * pw);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    long r = i / C4;
    const int wo = (int)(r % Wo); r /= Wo;
    const int ho = (int)(r % Ho);
    const long b = r / Ho;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int dy = 0; dy < ph; ++dy)
      for (int dx = 0; dx < pw; ++dx) {
        const float4 v = in[((b * H + ho * ph + dy) * W + wo * pw + dx) * C4 + c];
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      }
    out[i] = make_float4(s.x / d, s.y / d, s.z / d, s.w / d);
  }
}

// ---- the multi-scale GLU stem of Cnn10_mul_scale (models.py:457-468), fused: mel [B][T][64] -> out [B][m][32][96].
// Branch k in {1, 3, 5} (channels 32 * branch ...): Conv2d(1, 64, k, padding 1) with BatchNorm folded (w [3][64][25],
// the k * k taps first; b [3][64]), sigmoid(first 32) * last 32, avg_pool (ph, 2).  The 1 x 1 branch is (T + 2) x 66
// (its border is GLU of the bias alone) and keeps pooled columns < 32; the 5 x 5 branch is (T - 2) x 62, pooled to
// H3 x 31 and replication-padded by one row and one column; every branch keeps the first m rows.
constexpr int kStemThreads = 256;
__global__ void __launch_bounds__(kStemThreads) tsd_stem_kernel(const float* __restrict__ mel, const float* __restrict__ w,
                                                                 const float* __restrict__ bias, int T, int ph, int H3, int m,
                                                                 float* __restrict__ out, long total) {
  __shared__ float ws[3 * 64 * 25], bs[3 * 64];
  for (int i = threadIdx.x; i < 3 * 64 * 25; i += blockDim.x) ws[i] = w[i];
  for (int i = threadIdx.x; i < 3 * 64; i += blockDim.x) bs[i] = bias[i];
  __syncthreads();
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int o = (int)(i % kStemC);
    long r = i / kStemC;
    int c = (int)(r % 32); r /= 32;
    int row = (int)(r % m);
    const long b = r / m;
    const int br = o / 32, g = o % 32, k = 2 * br + 1;
    if (br == 2) { row = min(row, H3 - 1); c = min(c, 30); }     // ReplicationPad2d((0, 1, 0, 1))
    const float* wa = ws + (br * 64 + g) * 25;
    const float* wb = ws + (br * 64 + g + 32) * 25;
    const float ba = bs[br * 64 + g], bb = bs[br * 64 + g + 32];
    const float* mb = mel + b * T * kMel;
    float s = 0.f;
    for (int dy = 0; dy < ph; ++dy)
      for (int dx = 0; dx < 2; ++dx) {
        const int y = row * ph + dy, x = c * 2 + dx;     // conv output position; input rows y - 1 .. y + k - 2
        float va = 0.f, vb = 0.f;
        for (int ky = 0; ky < k; ++ky) {
          const int yi = y + ky - 1;
          if (yi < 0 || yi >= T) continue;
          for (int kx = 0; kx < k; ++kx) {
            const int xi = x + kx - 1;
            if (xi < 0 || xi >= kMel) continue;
            const float v = __ldg(mb + (long)yi * kMel + xi);
            va = fmaf(wa[ky * k + kx], v, va);
            vb = fmaf(wb[ky * k + kx], v, vb);
          }
        }
        s += sigmoidf_(va + ba) * (vb + bb);
      }
    out[i] = s / (float)(ph * 2);
  }
}

// ---- Fusion's product and pool: out[r][j] = mean_q e1[r / rows_per_b][j n + q] * f2[r][j n + q], q < n
__global__ void tsd_fuse_kernel(const float* __restrict__ f2, const float* __restrict__ e1, int rows_per_b, int C, int n,
                                float* __restrict__ out, long total) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int j = (int)(i % C);
    const long r = i / C, b = r / rows_per_b;
    const float* a = e1 + b * (long)C * n + (long)j * n;
    const float* f = f2 + r * (long)C * n + (long)j * n;
    float s = 0.f;
    for (int q = 0; q < n; ++q) s += a[q] * f[q];
    out[i] = s / (float)n;
  }
}

__device__ float block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[w] = v;
  __syncthreads();
  float s = 0.f;
  for (int k = 0; k < nw; ++k) s += red[k];
  return s;
}
__device__ float block_max(float v, float* red) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[w] = v;
  __syncthreads();
  float s = -INFINITY;
  for (int k = 0; k < nw; ++k) s = fmaxf(s, red[k]);
  return s;
}

// y[o] = W[o] . x + b[o] for o < n_out (W [n_out][128] row-major, x in shared memory), relu optional
__device__ void linear128(const float* __restrict__ W, const float* __restrict__ b, const float* x, float* y, int n_out, bool relu) {
  for (int o = threadIdx.x; o < n_out; o += blockDim.x) {
    const float4* w4 = reinterpret_cast<const float4*>(W + (long)o * kEmb);
    float acc = 0.f;
#pragma unroll 8
    for (int c = 0; c < kEmb / 4; ++c) {
      const float4 v = __ldg(w4 + c);
      acc = fmaf(v.x, x[4 * c], acc); acc = fmaf(v.y, x[4 * c + 1], acc);
      acc = fmaf(v.z, x[4 * c + 2], acc); acc = fmaf(v.w, x[4 * c + 3], acc);
    }
    acc += b[o];
    y[o] = relu ? fmaxf(acc, 0.f) : acc;
  }
}

// attention weights of `rows` embeddings E[row_of(i)] against q (get_w / get_w_ee): score_i = (W_k E_i + b_k) . q / 11.3
// = (W_k^T q) . E_i / 11.3 + q . b_k / 11.3, softmax over i.  u, sc: shared scratch [128], [rows].
template <typename RowOf>
__device__ void attend(const float* __restrict__ Wk, const float* __restrict__ bk, const float* q, const float* __restrict__ E,
                       int rows, RowOf row_of, float* u, float* sc, float* red) {
  for (int c = threadIdx.x; c < kEmb; c += blockDim.x) {
    float acc = 0.f;
    for (int o = 0; o < kEmb; ++o) acc = fmaf(__ldg(Wk + (long)o * kEmb + c), q[o], acc);
    u[c] = acc;
  }
  float part = 0.f;
  for (int o = threadIdx.x; o < kEmb; o += blockDim.x) part = fmaf(q[o], bk[o], part);
  const float qb = block_sum(part, red);   // (syncs: u is complete)
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < rows; i += blockDim.x) {
    const float* e = E + (long)row_of(i) * kEmb;
    float acc = 0.f;
    for (int c = 0; c < kEmb; ++c) acc = fmaf(u[c], e[c], acc);
    sc[i] = (acc + qb) / kTemperature;
    mx = fmaxf(mx, sc[i]);
  }
  mx = block_max(mx, red);
  float sum = 0.f;
  for (int i = threadIdx.x; i < rows; i += blockDim.x) { sc[i] = expf(sc[i] - mx); sum += sc[i]; }
  sum = block_sum(sum, red);
  for (int i = threadIdx.x; i < rows; i += blockDim.x) sc[i] /= sum;
  __syncthreads();
}

// ---- the reference embedding (RaDur_fusion.forward before the detection): E [B][Tr][128] -> emb [B][128].
// att_pool: E holds bn(fc1(.)) rows; emb = sum_t softmax_t(get_w(mean_t E, E)) E_t.  Otherwise emb = mean_t E.
// The scores live in global scratch [B][Tr] (a long reference clip's Tr floats would not fit in shared memory).
constexpr int kTailThreads = 256;
__global__ void __launch_bounds__(kTailThreads) tsd_refemb_kernel(const float* __restrict__ E, int Tr, int att_pool,
                                                                  const float* __restrict__ qw, const float* __restrict__ qb,
                                                                  const float* __restrict__ kw, const float* __restrict__ kb,
                                                                  float* __restrict__ scores, float* __restrict__ emb) {
  __shared__ float m[kEmb], q[kEmb], u[kEmb], red[32];
  const long b = blockIdx.x;
  const float* Eb = E + b * Tr * kEmb;
  for (int c = threadIdx.x; c < kEmb; c += blockDim.x) {
    float s = 0.f;
    for (int t = 0; t < Tr; ++t) s += Eb[(long)t * kEmb + c];
    m[c] = s / (float)Tr;
  }
  __syncthreads();
  if (!att_pool) {
    for (int c = threadIdx.x; c < kEmb; c += blockDim.x) emb[b * kEmb + c] = m[c];
    return;
  }
  float* sc = scores + b * Tr;
  linear128(qw, qb, m, q, kEmb, false);
  __syncthreads();
  attend(kw, kb, q, Eb, Tr, [](int i) { return i; }, u, sc, red);
  for (int c = threadIdx.x; c < kEmb; c += blockDim.x) {
    float s = 0.f;
    for (int t = 0; t < Tr; ++t) s = fmaf(sc[t], Eb[(long)t * kEmb + c], s);
    emb[b * kEmb + c] = s;
  }
}

// ---- the enhancement tail of orcal_EE (models.py:1209-1232) for one sample per block:
// top-k (k = min(top, T')) of the first decision p1[:, :, 0], descending, ties to the lower frame; the mixture's
// embeddings at those frames, weighted by softmax(get_w_ee(emb, .)) * (v > tao ? v : 0) and averaged; EE_fusion with
// emb -> me [128].  wmix = mean(v) > tao ? mean(v) / 2 : 0 (the raw top-k mean).  Frames at or past Te (possible when
// T' > Te) are clamped for the read; the launcher rejects them.
__global__ void __launch_bounds__(kTailThreads) tsd_enhance_kernel(const float* __restrict__ p1, int Td, int O,
                                                                   const float* __restrict__ Emix, int Te, const float* __restrict__ emb,
                                                                   int k, float tao, const float* __restrict__ qw, const float* __restrict__ qb,
                                                                   const float* __restrict__ kw, const float* __restrict__ kb,
                                                                   const float* __restrict__ f1w, const float* __restrict__ f1b,
                                                                   const float* __restrict__ f2w, const float* __restrict__ f2b,
                                                                   float* __restrict__ me, float* __restrict__ wmix, int* __restrict__ idx_out,
                                                                   float* __restrict__ val_out) {
  __shared__ float s[kMaxFramesDet], sc[kMaxFramesDet], e[kEmb], q[kEmb], u[kEmb], mix[kEmb], red[32];
  __shared__ float g1[4 * kEmb], g2[4 * kEmb];
  __shared__ int sidx[kMaxFramesDet];
  const long b = blockIdx.x;
  for (int t = threadIdx.x; t < Td; t += blockDim.x) s[t] = p1[(b * Td + t) * O];
  for (int c = threadIdx.x; c < kEmb; c += blockDim.x) e[c] = emb[b * kEmb + c];
  __syncthreads();
  for (int t = threadIdx.x; t < Td; t += blockDim.x) {
    const float v = s[t];
    int rank = 0;
    for (int j = 0; j < Td; ++j) rank += (s[j] > v) || (s[j] == v && j < t);
    if (rank < k) sidx[rank] = t;
  }
  linear128(qw, qb, e, q, kEmb, false);
  __syncthreads();
  float vs = 0.f;
  for (int i = threadIdx.x; i < k; i += blockDim.x) {
    vs += s[sidx[i]];
    idx_out[b * k + i] = sidx[i];
    if (val_out) val_out[b * k + i] = s[sidx[i]];
  }
  const float vmean = block_sum(vs, red) / (float)k;
  const float* Eb = Emix + b * Te * kEmb;
  attend(kw, kb, q, Eb, k, [&](int i) { return min(sidx[i], Te - 1); }, u, sc, red);
  for (int c = threadIdx.x; c < kEmb; c += blockDim.x) {
    float acc = 0.f;
    for (int i = 0; i < k; ++i) {
      const float v = s[sidx[i]];
      const float a = sc[i] * (v > tao ? v : 0.f);
      acc += Eb[(long)min(sidx[i], Te - 1) * kEmb + c] * a;
    }
    mix[c] = acc / (float)k;
  }
  __syncthreads();
  linear128(f1w, f1b, mix, g1, 4 * kEmb, true);    // EE_fusion.fuse_layer1(mix_embedding)
  linear128(f2w, f2b, e, g2, 4 * kEmb, true);      // EE_fusion.fuse_layer2(embedding)
  __syncthreads();
  for (int c = threadIdx.x; c < kEmb; c += blockDim.x) {
    float a = 0.f;
    for (int qq = 0; qq < 4; ++qq) a += g1[4 * c + qq] * g2[4 * c + qq];
    me[b * kEmb + c] = a / 4.f;
  }
  if (threadIdx.x == 0) wmix[b] = vmean > tao ? vmean / 2.f : 0.f;
}

// ---- detection.fc -> outputlayer (folded: w [O][1024], bias [O]) and the softmax over O: one warp per row
constexpr int kHeadWarps = 8, kMaxOut = 16;
__global__ void __launch_bounds__(kHeadWarps * 32) tsd_head_kernel(const float* __restrict__ h, const float* __restrict__ w,
                                                                   const float* __restrict__ bias, int O, long rows, float* __restrict__ p) {
  const int lane = threadIdx.x & 31;
  const long r = (long)blockIdx.x * kHeadWarps + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* x = h + r * (2 * kFeat);
  float z[kMaxOut];
  float mx = -INFINITY;
  for (int o = 0; o < O; ++o) {
    float acc = 0.f;
    for (int c = lane; c < 2 * kFeat; c += 32) acc = fmaf(w[(long)o * 2 * kFeat + c], x[c], acc);
#pragma unroll
    for (int s = 16; s; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
    z[o] = acc + bias[o];
    mx = fmaxf(mx, z[o]);
  }
  float sum = 0.f;
  for (int o = 0; o < O; ++o) { z[o] = expf(z[o] - mx); sum += z[o]; }
  if (lane == 0)
    for (int o = 0; o < O; ++o) p[r * O + o] = z[o] / sum;
}

// ---- the two-pass mix and interpolate(size = T, mode = 'linear', align_corners = False):
// fin = p1 (1 - w) + w p2 (p2 / w absent: fin = p1); decision[b][i] = fin[b][i][0]; up[b][t][o] from ATen's source
// index src = max(T' / T * (t + 0.5) - 0.5, 0), i0 = floor(src), i1 = i0 + (i0 < T' - 1), l1 = src - i0
__device__ __forceinline__ float mixed(const float* p1, const float* p2, float w, long i) {
  return p2 ? p1[i] * (1.f - w) + w * p2[i] : p1[i];
}
__global__ void tsd_mix_interp_kernel(const float* __restrict__ p1, const float* __restrict__ p2, const float* __restrict__ wmix, int B,
                                      int Td, int T, int O, float* __restrict__ decision, float* __restrict__ up) {
  const long nup = (long)B * T * O, ndec = (long)B * Td;
  const float scale = (float)Td / (float)T;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < nup + ndec; i += (long)gridDim.x * blockDim.x) {
    if (i < nup) {
      const int o = (int)(i % O);
      const long r = i / O;
      const int t = (int)(r % T);
      const long b = r / T;
      const float w = p2 ? wmix[b] : 0.f;
      float src = scale * ((float)t + 0.5f) - 0.5f;
      src = src < 0.f ? 0.f : src;
      const int i0 = (int)src, i1 = i0 + (i0 < Td - 1 ? 1 : 0);
      const float l1 = src - (float)i0, l0 = 1.f - l1;
      up[i] = l0 * mixed(p1, p2, w, (b * Td + i0) * O + o) + l1 * mixed(p1, p2, w, (b * Td + i1) * O + o);
    } else {
      const long j = i - nup, b = j / Td;
      decision[j] = mixed(p1, p2, p2 ? wmix[b] : 0.f, j * O);
    }
  }
}

// ---- the bidirectional GRU recurrence (PyTorch gate order r, z, n; h0 = 0):
//   r = sig(xr + W_hr h + b_hr), z = sig(xz + W_hz h + b_hz), n = tanh(xn + r (W_hn h + b_hn)), h' = (h - n) z + n
// x* = the input projections W_i* x + b_i* (xp [B][T][3072]: forward r, z, n | backward r, z, n).  One cluster of 16
// CTAs per (direction, group of up to 4 samples); CTA `rank` owns hidden units 32 rank .. 32 rank + 31 and keeps their
// 96 W_hh rows in shared memory for the whole sequence.  Every step each CTA forms its rows' W_hh h, updates its units,
// writes them into the next h buffer of all 16 CTAs over DSMEM and meets the others at a cluster barrier.  fp32 FMA.
__global__ void __launch_bounds__(kGruThreads, 1) tsd_gru_kernel(const float* __restrict__ whh, const float* __restrict__ bhh,
                                                                 const float* __restrict__ xp, int B, int T, float* __restrict__ out) {
  cg::cluster_group cluster = cg::this_cluster();
  extern __shared__ float4 gru_sm4[];
  float* w = reinterpret_cast<float*>(gru_sm4);      // [96][512]
  float* hbuf = w + kGruRows * kGruH;               // [2][kGruMaxB][512]
  float* g = hbuf + 2 * kGruMaxB * kGruH;           // [kGruMaxB][96]
  float* hn = g + kGruMaxB * kGruRows;              // [kGruMaxB][32]
  const int rank = (int)cluster.block_rank();
  const int dir = blockIdx.y;
  const int b0 = blockIdx.z * kGruMaxB, nb = min(kGruMaxB, B - b0);
  const int u0 = rank * kGruU;
  const float* wd = whh + (size_t)dir * 3 * kGruH * kGruH;
  for (int i = threadIdx.x; i < kGruRows * kGruH / 4; i += blockDim.x) {
    const int lr = i / (kGruH / 4), c4 = i % (kGruH / 4);
    const int gr = (lr / kGruU) * kGruH + u0 + lr % kGruU;
    gru_sm4[i] = reinterpret_cast<const float4*>(wd + (size_t)gr * kGruH)[c4];
  }
  for (int i = threadIdx.x; i < 2 * kGruMaxB * kGruH; i += blockDim.x) hbuf[i] = 0.f;
  const float* bd = bhh + dir * 3 * kGruH;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int kWarps = kGruThreads / 32, kPer = kGruH / 32;
  cluster.sync();    // every CTA runs and has zeroed its buffers before any remote write
  for (int s = 0; s < T; ++s) {
    const int t = dir ? T - 1 - s : s;
    const float* hc = hbuf + (s & 1) * kGruMaxB * kGruH;
    float* hnext = hbuf + ((s + 1) & 1) * kGruMaxB * kGruH;
    for (int b = 0; b < nb; ++b) {
      float hr[kPer];
#pragma unroll
      for (int k = 0; k < kPer; ++k) hr[k] = hc[b * kGruH + lane + 32 * k];
      for (int row = warp; row < kGruRows; row += kWarps) {
        const float* wr = w + row * kGruH + lane;
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < kPer; ++k) acc = fmaf(wr[32 * k], hr[k], acc);
#pragma unroll
        for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) g[b * kGruRows + row] = acc;
      }
    }
    __syncthreads();
    if (threadIdx.x < nb * kGruU) {
      const int b = threadIdx.x / kGruU, j = threadIdx.x % kGruU, u = u0 + j;
      const float* x = xp + ((size_t)(b0 + b) * T + t) * (6 * kGruH) + dir * 3 * kGruH;
      const float* gb = g + b * kGruRows;
      const float r = sigmoidf_(x[u] + (gb[j] + bd[u]));
      const float z = sigmoidf_(x[kGruH + u] + (gb[kGruU + j] + bd[kGruH + u]));
      const float n = tanhf(x[2 * kGruH + u] + r * (gb[2 * kGruU + j] + bd[2 * kGruH + u]));
      const float h = (hc[b * kGruH + u] - n) * z + n;
      hn[b * kGruU + j] = h;
      out[((size_t)(b0 + b) * T + t) * (2 * kGruH) + dir * kGruH + u] = h;
    }
    __syncthreads();
    if (s + 1 < T)
      for (int i = threadIdx.x; i < kGruCta * nb * kGruU; i += blockDim.x) {
        const int q = i / (nb * kGruU), bj = i % (nb * kGruU), b = bj / kGruU, j = bj % kGruU;
        float* dst = cluster.map_shared_rank(hnext, q);
        dst[b * kGruH + u0 + j] = hn[bj];
      }
    cluster.sync();
  }
}

unsigned ew_blocks(long n) { return (unsigned)std::max<long>(1, std::min<long>(cdivl(n, 256), 4096)); }

}  // namespace

// ---------------------------------------------------------------- launchers (also the unit tests' entry points)
void tsd_pad4(const float* mel, float* img, long n, cudaStream_t st) {
  AGPT_CHECK(n >= 1, "pad4: n >= 1");
  tsd_pad4_kernel<<<ew_blocks(n), 256, 0, st>>>(mel, reinterpret_cast<float4*>(img), n);
  count_launch(1);
}

void tsd_fuse(const float* f2, const float* e1, int B, int Td, int C, int n, float* out, cudaStream_t st) {
  AGPT_CHECK(n >= 1, "fuse: n >= 1");
  AGPT_CHECK(B >= 1 && Td >= 1 && C >= 1, "fuse: B, Td, C >= 1");
  const long total = (long)B * Td * C;
  tsd_fuse_kernel<<<ew_blocks(total), 256, 0, st>>>(f2, e1, Td, C, n, out, total);
  count_launch(1);
}

void tsd_refemb(const float* E, int B, int Trr, int att_pool, const float* qw, const float* qb, const float* kw, const float* kb,
                float* scratch, float* emb, cudaStream_t st) {
  AGPT_CHECK(Trr >= 1, "refemb: Trr >= 1");
  AGPT_CHECK(B >= 1, "refemb: B >= 1");
  AGPT_CHECK(!att_pool || scratch, "refemb: attention pooling needs a [B][Trr] score scratch");
  tsd_refemb_kernel<<<B, kTailThreads, 0, st>>>(E, Trr, att_pool, qw, qb, kw, kb, scratch, emb);
  count_launch(1);
}

void tsd_head(const float* h, const float* w, const float* bias, int O, long rows, float* p, cudaStream_t st) {
  AGPT_CHECK(O >= 1 && O <= kMaxOut, "head: 1 <= O <= 16");
  AGPT_CHECK(rows >= 1, "head: rows >= 1");
  tsd_head_kernel<<<(unsigned)cdivl(rows, kHeadWarps), kHeadWarps * 32, 0, st>>>(h, w, bias, O, rows, p);
  count_launch(1);
}

void tsd_mix_interp(const float* p1, const float* p2, const float* wmix, int B, int Td, int T, int O, float* decision, float* up,
                    cudaStream_t st) {
  AGPT_CHECK(O >= 1 && O <= kMaxOut, "mix_interp: 1 <= O <= 16");
  AGPT_CHECK(B >= 1 && Td >= 1 && T >= 1, "mix_interp: B, Td, T >= 1");
  const long n = (long)B * T * O + (long)B * Td;
  tsd_mix_interp_kernel<<<ew_blocks(n), 256, 0, st>>>(p1, p2, wmix, B, Td, T, O, decision, up);
  count_launch(1);
}

void tsd_avgpool(const float* in, int B, int H, int W, int C, int ph, int pw, float* out, cudaStream_t st) {
  AGPT_CHECK(B >= 1 && ph >= 1 && pw >= 1 && C >= 4 && C % 4 == 0, "avgpool: C must be a multiple of 4");
  AGPT_CHECK(H >= ph && W >= pw, "avgpool: the map is smaller than the pool window");
  const int Ho = H / ph, Wo = W / pw;
  const long total = (long)B * Ho * Wo * (C / 4);
  tsd_avgpool_kernel<<<ew_blocks(total), 256, 0, st>>>(reinterpret_cast<const float4*>(in), reinterpret_cast<float4*>(out), H, W, C / 4,
                                                       ph, pw, Ho, Wo, total);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// the stem's pooled row counts for a T-frame mel and row pool ph: {H1 (1 x 1), H2 (3 x 3), H3 (5 x 5, before the pad), m}
static void stem_rows(int T, int ph, int r[4]) {
  AGPT_CHECK(T >= 3 && T - 2 >= ph, "clip too short: the 5 x 5 stem branch has no pooled row");
  r[0] = (T + 2) / ph; r[1] = T / ph; r[2] = (T - 2) / ph;
  r[3] = std::min(std::min(r[0], kStemRowsMax), std::min(r[1], r[2] + 1));
}

void tsd_stem(const float* mel, const float* w, const float* b, int B, int T, int ph, float* out, cudaStream_t st) {
  AGPT_CHECK(B >= 1 && (ph == 1 || ph == 2), "stem: ph must be 1 or 2");
  int r[4];
  stem_rows(T, ph, r);
  const long total = (long)B * r[3] * 32 * kStemC;
  tsd_stem_kernel<<<(unsigned)std::min<long>(cdivl(total, kStemThreads), 8192), kStemThreads, 0, st>>>(mel, w, b, T, ph, r[2], r[3],
                                                                                                      out, total);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

void tsd_gru(const float* whh, const float* bhh, const float* xp, int B, int T, float* out, cudaStream_t st) {
  AGPT_CHECK(B >= 1 && T >= 1, "gru: empty input");
  static bool configured[64] = {};
  int dev = 0;
  AGPT_CUDA(cudaGetDevice(&dev));
  if (dev >= 64 || !configured[dev]) {
    AGPT_CUDA(cudaFuncSetAttribute(tsd_gru_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kGruSmem));
    AGPT_CUDA(cudaFuncSetAttribute(tsd_gru_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    if (dev < 64) configured[dev] = true;
  }
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(kGruCta, 2, cdiv(B, kGruMaxB));
  cfg.blockDim = dim3(kGruThreads);
  cfg.dynamicSmemBytes = kGruSmem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = kGruCta; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, tsd_gru_kernel, whh, bhh, xp, B, T, out);
  if (e != cudaSuccess)
    throw Error(std::string("gru: the 16-CTA cluster launch was refused: ") + cudaGetErrorString(e));
  count_launch(1);
}

void tsd_enhance(const float* p1, int B, int Td, int O, const float* Emix, int Te, const float* emb, int top, float tao,
                 const float* const wts[8], float* me, float* wmix, int* idx, float* val, cudaStream_t st) {
  AGPT_CHECK(B >= 1 && Td >= 1 && Td <= kMaxFramesDet && O >= 1 && Te >= 1 && top >= 1, "enhance: bad sizes (1 <= T' <= 500)");
  const int k = std::min(top, Td);
  tsd_enhance_kernel<<<B, kTailThreads, 0, st>>>(p1, Td, O, Emix, Te, emb, k, tao, wts[0], wts[1], wts[2], wts[3], wts[4], wts[5],
                                                 wts[6], wts[7], me, wmix, idx, val);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
  if (Td > Te) {   // the reference's gather raises for a selected frame the mixture encoder does not have
    std::vector<int> h((size_t)B * k);
    AGPT_CUDA(cudaMemcpyAsync(h.data(), idx, sizeof(int) * h.size(), cudaMemcpyDeviceToHost, st));
    AGPT_CUDA(cudaStreamSynchronize(st));
    for (int v : h)
      AGPT_CHECK(v < Te, "enhancement: a top-k frame of the detection lies past the mixture encoder's frames "
                         "(the reference's torch.gather fails here too)");
  }
}

// frames[0] = T' (detection frames), frames[1] = the reference encoder's frames, frames[2] = the mixture encoder's
// frames (0 without enhancement)
void tsd_frames(const agpt_tsd_cfg* cfg, int T, int Tr, int frames[3]) {
  AGPT_CHECK(cfg->mel_bins == kMel, "RaDur_fusion: mel_bins must be 64");
  AGPT_CHECK(T >= 1 && Tr >= 1 && T <= (1 << 20) && Tr <= (1 << 20), "bad clip lengths");
  int p[4][2];
  det_pools(cfg->time_resolution, p);
  AGPT_CHECK(T - 2 >= p[0][0], "clip too short: the stem has no output row");
  int r[4];
  stem_rows(T, p[0][0], r);
  int H = r[3];
  for (int i = 1; i < 4; ++i) {
    AGPT_CHECK(H >= p[i][0], "clip too short: a detection pool has no output row");
    H /= p[i][0];
  }
  frames[0] = H;
  AGPT_CHECK(Tr >= 8, "reference clip too short: Cnn14 needs 8 frames for one output frame");
  frames[1] = Tr / 8;
  frames[2] = 0;
  if (cfg->enhancement) {
    AGPT_CHECK(T >= 8, "clip too short: the enhancement's Cnn14 needs 8 frames for one output frame");
    frames[2] = T / 8;
  }
}

namespace {

struct TsdNet : Handle {
  agpt_tsd_cfg cfg;
  int pools[4][2];
  PackedConv enc[kEnc][2], fc1, fc1_bn;
  DevBuf stem_w, stem_b;
  PackedConv det[3][2];
  PackedConv wih, fuse1, fuse2;
  DevBuf whh, bhh, headw, headb;
  DevBuf qw, qb, kw, kb, qew, qeb, kew, keb, ee1w, ee1b, ee2w, ee2b;
  DevBuf img, bA, bB, bC, eref, emix, emb, me, e1, stem, f2, fused, xp, hs, p1, p2, wmix, idx, scores;
  cudaEvent_t ev[kTsdStages + 1] = {};
  bool timed = false;

  void mark(int i, cudaStream_t st) { if (timed) AGPT_CUDA(cudaEventRecord(ev[i], st)); }

  void linear(const PackedConv& pc, const float* in, float* out, long rows, int epi, cudaStream_t st) {
    TapConvParams P = tapconv_params(pc, 1, (int)rows, 0, 1);
    P.in = in; P.in_pitch = pc.Cin;
    P.out = out; P.out_pitch = pc.Cout;
    P.epi = epi;
    tapconv_launch(P, st);
  }

  // Cnn14.forward on mel [B][T][64] -> [B][T / 8][128] through fc (fc1, or fc1 with bn folded)
  void encode(const float* mel, int B, int T, const PackedConv& fc, float* out, cudaStream_t st) {
    tsd_pad4(mel, img.p, (long)B * T * kMel, st);
    const float* in = img.p;
    int H = T, W = kMel;
    for (int i = 0; i < kEnc; ++i) {
      conv3x3_relu(enc[i][0], in, bB.p, B, H, W, st);
      conv3x3_relu(enc[i][1], bB.p, bC.p, B, H, W, st);
      const int ph = i < 3 ? 2 : 1;
      tsd_avgpool(bC.p, B, H, W, kEncCh[i], ph, 2, bA.p, st);
      H /= ph; W /= 2;
      in = bA.p;
    }
    linear(fc, bA.p, out, (long)B * H, EPI_BIAS, st);
  }

  // one detection pass from the fused-in embedding's fuse_layer1 output e1 [B][1024]: Fusion product, GRU, head -> p
  void pass(int B, int Td, const float* e1v, float* p, cudaStream_t st) {
    const long rows = (long)B * Td;
    tsd_fuse(f2.p, e1v, B, Td, kFeat, 2, fused.p, st);
    linear(wih, fused.p, xp.p, rows, EPI_BIAS, st);
    tsd_gru(whh.p, bhh.p, xp.p, B, Td, hs.p, st);
    tsd_head(hs.p, headw.p, headb.p, cfg.outputdim, rows, p, st);
    AGPT_CUDA(cudaGetLastError());
  }

  void forward(const float* x, const float* ref, int B, int T, int Tr, float* decision, float* decision_up, cudaStream_t st) {
    AGPT_CHECK(B >= 1, "empty batch");
    int fr[3];
    tsd_frames(&cfg, T, Tr, fr);
    const int Td = fr[0], Trr = fr[1], Te = fr[2];
    int sr[4];
    stem_rows(T, pools[0][0], sr);
    const size_t big = (size_t)B * std::max(T, Tr) * kMel * kEncCh[0];
    img.ensure((size_t)B * std::max(T, Tr) * kMel * 4);
    bA.ensure(big); bB.ensure(big); bC.ensure(big);
    eref.ensure((size_t)B * Trr * kEmb); emix.ensure((size_t)B * std::max(Te, 1) * kEmb);
    emb.ensure((size_t)B * kEmb); me.ensure((size_t)B * kEmb); e1.ensure((size_t)B * kFuse);
    stem.ensure((size_t)B * sr[3] * 32 * kStemC);
    const size_t rows = (size_t)B * Td;
    f2.ensure(rows * kFuse); fused.ensure(rows * kFeat); xp.ensure(rows * 6 * kGruH); hs.ensure(rows * 2 * kGruH);
    p1.ensure(rows * cfg.outputdim); p2.ensure(rows * cfg.outputdim); wmix.ensure(B); idx.ensure((size_t)B * cfg.top);
    mark(0, st);
    // the reference embedding
    encode(ref, B, Tr, cfg.att_pool ? fc1_bn : fc1, eref.p, st);
    if (cfg.att_pool) scores.ensure((size_t)B * Trr);
    tsd_refemb(eref.p, B, Trr, cfg.att_pool, qw.p, qb.p, kw.p, kb.p, scores.p, emb.p, st);
    AGPT_CUDA(cudaGetLastError());
    mark(1, st);
    if (cfg.enhancement) encode(x, B, T, fc1_bn, emix.p, st);   // the mixture's embeddings, bn applied
    mark(2, st);
    // detection features: stem, conv blocks 2-4, and fusion.fuse_layer2 (the same in both passes)
    tsd_stem(x, stem_w.p, stem_b.p, B, T, pools[0][0], stem.p, st);
    const float* in = stem.p;
    int H = sr[3], W = 32, cin = kStemC;
    for (int i = 0; i < 3; ++i) {
      conv3x3_relu(det[i][0], in, bB.p, B, H, W, st);
      conv3x3_relu(det[i][1], bB.p, bC.p, B, H, W, st);
      tsd_avgpool(bC.p, B, H, W, kDetCh[i], pools[i + 1][0], pools[i + 1][1], bA.p, st);
      H /= pools[i + 1][0]; W /= pools[i + 1][1];
      in = bA.p;
      cin = kDetCh[i];
    }
    AGPT_CHECK(H == Td && W == 1 && cin == kFeat, "detection feature shape");
    linear(fuse2, bA.p, f2.p, (long)rows, EPI_RELU, st);
    mark(3, st);
    linear(fuse1, emb.p, e1.p, B, EPI_RELU, st);
    pass(B, Td, e1.p, p1.p, st);
    mark(4, st);
    if (cfg.enhancement) {
      const float* wts[8] = {qew.p, qeb.p, kew.p, keb.p, ee1w.p, ee1b.p, ee2w.p, ee2b.p};
      tsd_enhance(p1.p, B, Td, cfg.outputdim, emix.p, Te, emb.p, cfg.top, cfg.tao, wts, me.p, wmix.p, reinterpret_cast<int*>(idx.p),
                  nullptr, st);
      linear(fuse1, me.p, e1.p, B, EPI_RELU, st);
      pass(B, Td, e1.p, p2.p, st);
    }
    mark(5, st);
    tsd_mix_interp(p1.p, cfg.enhancement ? p2.p : nullptr, wmix.p, B, Td, T, cfg.outputdim, decision, decision_up, st);
    AGPT_CUDA(cudaGetLastError());
    mark(6, st);
  }
};

}  // namespace

Handle* tsd_create(const agpt_tsd_cfg* cfg, const float* const* Wt, int nW, int device) {
  DeviceGuard dg_(device);
  AGPT_CHECK(cfg->mel_bins == kMel, "RaDur_fusion: mel_bins must be 64 (both CNNs pool the mel axis down to one column)");
  AGPT_CHECK(cfg->outputdim >= 1 && cfg->outputdim <= kMaxOut, "RaDur_fusion: outputdim must be in [1, 16]");
  AGPT_CHECK(cfg->top >= 1, "RaDur_fusion: top must be >= 1");
  AGPT_CHECK(cfg->att_pool == 0 || cfg->att_pool == 1, "att_pool is 0 or 1");
  AGPT_CHECK(cfg->enhancement == 0 || cfg->enhancement == 1, "enhancement is 0 or 1");
  std::unique_ptr<TsdNet> h(new TsdNet());
  h->magic = kMagicTsd; h->device = device; h->cfg = *cfg;
  det_pools(cfg->time_resolution, h->pools);
  WeightCursor wc{Wt, nW};
  int cin = 1;
  for (int i = 0; i < kEnc; ++i) {   // encoder.conv_block1..6
    const int c = kEncCh[i];
    const float* w1 = wc.next(); const float* w2 = wc.next();
    load_conv_bn(h->enc[i][0], w1, wc, c, cin, round_up(cin, 4), kBnEps);
    load_conv_bn(h->enc[i][1], w2, wc, c, c, c, kBnEps);
    cin = c;
  }
  const float* fc1w = wc.next(); const float* fc1b = wc.next();
  pack_conv(h->fc1, fc1w, fc1b, kEmb, cin, 1, false);
  {  // detection.features.conv_block1_1 / 1_2 / 1_3: folded into [3][64][25] (k * k taps first) and [3][64]
    std::vector<float> w(3 * 64 * 25, 0.f), b(3 * 64);
    for (int br = 0; br < 3; ++br) {
      const int k = 2 * br + 1;
      const float* cw = wc.next();
      const float* g = wc.next(); const float* be = wc.next(); const float* rm = wc.next(); const float* rv = wc.next();
      for (int co = 0; co < 64; ++co) {
        const float s = g[co] / sqrtf(rv[co] + kBnEps);
        b[br * 64 + co] = be[co] - rm[co] * s;
        for (int t = 0; t < k * k; ++t) w[(br * 64 + co) * 25 + t] = cw[co * k * k + t] * s;
      }
    }
    h->stem_w.upload(w); h->stem_b.upload(b);
  }
  cin = kStemC;
  for (int i = 0; i < 3; ++i) {      // detection.features.conv_block2..4
    const int c = kDetCh[i];
    const float* w1 = wc.next(); const float* w2 = wc.next();
    load_conv_bn(h->det[i][0], w1, wc, c, cin, cin, kBnEps);
    load_conv_bn(h->det[i][1], w2, wc, c, c, c, kBnEps);
    cin = c;
  }
  {  // detection.gru: weight_ih, weight_hh, bias_ih, bias_hh, then the same _reverse
    const float* p[2][4];
    for (int d = 0; d < 2; ++d)
      for (int j = 0; j < 4; ++j) p[d][j] = wc.next();
    const size_t G = 3 * kGruH;
    std::vector<float> wi(2 * G * kFeat), bi(2 * G), wh(2 * G * kGruH), bh(2 * G);
    for (int d = 0; d < 2; ++d) {
      memcpy(&wi[d * G * kFeat], p[d][0], sizeof(float) * G * kFeat);
      memcpy(&wh[d * G * kGruH], p[d][1], sizeof(float) * G * kGruH);
      memcpy(&bi[d * G], p[d][2], sizeof(float) * G);
      memcpy(&bh[d * G], p[d][3], sizeof(float) * G);
    }
    pack_conv(h->wih, wi.data(), bi.data(), (int)(2 * G), kFeat, 1, false);
    h->whh.upload(wh); h->bhh.upload(bh);
  }
  const float* fcw = wc.next(); const float* fcb = wc.next();          // detection.fc [256][1024]
  { const float* w = wc.next(); const float* b = wc.next(); pack_conv(h->fuse1, w, b, kFuse, kEmb, 1, false); }
  { const float* w = wc.next(); const float* b = wc.next(); pack_conv(h->fuse2, w, b, kFuse, kFeat, 1, false); }
  {  // detection.outputlayer [O][256] after fc: one [O][1024] matrix, summed in fp64
    const float* ow = wc.next(); const float* ob = wc.next();
    const int O = cfg->outputdim, F = 256, D = 2 * kFeat;
    std::vector<double> acc((size_t)O * D, 0.0);
    std::vector<float> w((size_t)O * D), b(O);
    for (int o = 0; o < O; ++o) {
      double bb = ob[o];
      for (int j = 0; j < F; ++j) {
        const double a = ow[o * F + j];
        bb += a * fcb[j];
        for (int i = 0; i < D; ++i) acc[(size_t)o * D + i] += a * fcw[(size_t)j * D + i];
      }
      b[o] = (float)bb;
      for (int i = 0; i < D; ++i) w[(size_t)o * D + i] = (float)acc[(size_t)o * D + i];
    }
    h->headw.upload(w); h->headb.upload(b);
  }
  h->qw.upload(wc.next(), kEmb * kEmb); h->qb.upload(wc.next(), kEmb);
  h->kw.upload(wc.next(), kEmb * kEmb); h->kb.upload(wc.next(), kEmb);
  h->qew.upload(wc.next(), kEmb * kEmb); h->qeb.upload(wc.next(), kEmb);
  h->kew.upload(wc.next(), kEmb * kEmb); h->keb.upload(wc.next(), kEmb);
  {  // RaDur_fusion.bn folded into a second copy of encoder.fc1: W' = s W, b' = s (b - mean) + beta
    const float* g = wc.next(); const float* be = wc.next(); const float* rm = wc.next(); const float* rv = wc.next();
    std::vector<float> w((size_t)kEmb * 2048), b(kEmb);
    for (int o = 0; o < kEmb; ++o) {
      const float s = g[o] / sqrtf(rv[o] + kBnEps);
      b[o] = (fc1b[o] - rm[o]) * s + be[o];
      for (int i = 0; i < 2048; ++i) w[(size_t)o * 2048 + i] = fc1w[(size_t)o * 2048 + i] * s;
    }
    pack_conv(h->fc1_bn, w.data(), b.data(), kEmb, 2048, 1, false);
  }
  h->ee1w.upload(wc.next(), 4 * kEmb * kEmb); h->ee1b.upload(wc.next(), 4 * kEmb);
  h->ee2w.upload(wc.next(), 4 * kEmb * kEmb); h->ee2b.upload(wc.next(), 4 * kEmb);
  wc.done();
  return h.release();
}

void tsd_forward(Handle* hh, const float* x, const float* ref, int B, int T, int Tr, float* decision, float* decision_up, cudaStream_t st) {
  auto* h = static_cast<TsdNet*>(hh);
  DeviceGuard dg_(h->device);
  h->forward(x, ref, B, T, Tr, decision, decision_up, st);
}

void tsd_stage_events(Handle* hh, void* const* events, int n) {
  auto* h = static_cast<TsdNet*>(hh);
  AGPT_CHECK(n == 0 || n == kTsdStages + 1, "stage events: pass none or kTsdStages + 1");
  h->timed = n > 0;
  for (int i = 0; i < n; ++i) h->ev[i] = static_cast<cudaEvent_t>(events[i]);
}

}  // namespace agpt
