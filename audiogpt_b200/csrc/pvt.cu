// The sound-event-detection tool's PVT on sm_90a: a 32 kHz clip -> framewise / clipwise class probabilities.
// Reference: audio_detection/audio_infer/pytorch/models.py:141-237 (PVT.forward, eval mode), :619-658 (Mlp), :661-733
// (Attention with spatial reduction), :749-786 (Block), :789-829 (OverlapPatchEmbed), :832-927
// (PyramidVisionTransformerV2), :929-940 (DWConv), pytorch_utils.py:103-117 (interpolate).
// Activations are token-major [B][H * W][C] (H = time, W = mel), which is the channels-last image every stage reads, so
// the reference's [B, C, H, W] <-> [B, N, C] permutes disappear.  The log-mel front end is Cnn14's (logmel.cuh); every
// Linear, the stage 2-4 patch embeddings (over im2col rows) and the sr convs (over gathered patches) are 1-tap
// tap-GEMMs; attention is the d = 64 attention kernel with K and V read from the kv buffer at pitch 2C.  New here: the
// 7 x 7 patch embedding, the sr patch gather, the Mlp's depthwise conv + GELU and the head.
#include "common.cuh"
#include "tapconv.cuh"
#include "tc_h16.cuh"
#include "nn_kernels.h"
#include "models.h"
#include "fs_layers.cuh"
#include "logmel.cuh"

namespace agpt {

namespace {

constexpr float kBnEps = 1e-5f;
constexpr int kStages = 4;
constexpr int kHeadDim = 64;

// ---- stage 1 patch embedding: Conv2d(1, C, 7, stride 4, padding 2) on img [B][H][W], then LayerNorm over the C
// outputs -> tokens [B][Ho * Wo][C].  One warp per token: the 49 taps of its patch go through shared memory, lane l
// owns channels l, l + 32, ...; the [49][C] weights are staged once per block of kPatchTokens tokens.
constexpr int kPatchTaps = 49, kPatchWarps = 8, kPatchTokens = 64, kPatchMaxCpl = 4;
__global__ void __launch_bounds__(kPatchWarps * 32) pvt_patch7_kernel(const float* __restrict__ img, const float* __restrict__ w,
                                                                      const float* __restrict__ bias, const float* __restrict__ gamma,
                                                                      const float* __restrict__ beta, float eps, int H, int W, int C,
                                                                      int Ho, int Wo, long tokens, float* __restrict__ out) {
  extern __shared__ float sm[];
  float* ws = sm;                          // [49][C]
  float* patch = sm + kPatchTaps * C;      // [warps][52]
  for (int i = threadIdx.x; i < kPatchTaps * C; i += blockDim.x) {
    const int c = i / kPatchTaps, k = i - c * kPatchTaps;
    ws[k * C + c] = w[i];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, cpl = C >> 5;
  float* pp = patch + warp * 52;
  const long t0 = (long)blockIdx.x * kPatchTokens;
  for (long t = t0 + warp; t < min(t0 + kPatchTokens, tokens); t += kPatchWarps) {
    const int wo = (int)(t % Wo);
    const long r = t / Wo;
    const int ho = (int)(r % Ho);
    const long b = r / Ho;
    __syncwarp();
    for (int k = lane; k < kPatchTaps; k += 32) {
      const int hi = 4 * ho - 2 + k / 7, wi = 4 * wo - 2 + k % 7;
      pp[k] = (hi >= 0 && hi < H && wi >= 0 && wi < W) ? img[(b * H + hi) * W + wi] : 0.f;
    }
    __syncwarp();
    float acc[kPatchMaxCpl];
#pragma unroll
    for (int j = 0; j < kPatchMaxCpl; ++j) acc[j] = j < cpl ? bias[lane + 32 * j] : 0.f;
    for (int k = 0; k < kPatchTaps; ++k) {
      const float v = pp[k];
#pragma unroll
      for (int j = 0; j < kPatchMaxCpl; ++j)
        if (j < cpl) acc[j] = fmaf(v, ws[k * C + lane + 32 * j], acc[j]);
    }
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < kPatchMaxCpl; ++j) s += acc[j];
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float)C;
    float v2 = 0.f;
#pragma unroll
    for (int j = 0; j < kPatchMaxCpl; ++j)
      if (j < cpl) { const float d = acc[j] - mean; v2 += d * d; }
#pragma unroll
    for (int o = 16; o; o >>= 1) v2 += __shfl_xor_sync(0xffffffffu, v2, o);
    const float rstd = rsqrtf(v2 / (float)C + eps);
#pragma unroll
    for (int j = 0; j < kPatchMaxCpl; ++j)
      if (j < cpl) {
        const int c = lane + 32 * j;
        out[t * C + c] = (acc[j] - mean) * rstd * gamma[c] + beta[c];
      }
  }
}

// ---- Attention.sr's input: the non-overlapping sr x sr patches of x [B][H * W][C] as rows
// out[b][hr * Wr + wr][(ky * sr + kx) * C + c] = x[b][(hr * sr + ky) * W + wr * sr + kx][c], Hr = H / sr, Wr = W / sr
// (rows and columns that do not fill a patch are dropped, as the unpadded strided conv drops them)
__global__ void pvt_sr_gather_kernel(const float4* __restrict__ x, float4* __restrict__ out, int H, int W, int C4, int sr, int Hr,
                                     int Wr, long total) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    long r = i / C4;
    const int kx = (int)(r % sr); r /= sr;
    const int ky = (int)(r % sr); r /= sr;
    const int wr = (int)(r % Wr); r /= Wr;
    const int hr = (int)(r % Hr);
    const long b = r / Hr;
    out[i] = x[((b * H + hr * sr + ky) * W + wr * sr + kx) * C4 + c];
  }
}

// ---- Mlp's DWConv + GELU: depthwise 3 x 3, padding 1, bias, exact GELU on x [B][H][W][C].  One block per (64-channel
// slice, strip of image rows, sample): the strip and its two halo rows sit in shared memory as float4s, each thread
// produces 4 channels of one pixel per step and stores them as fp32 or as the fp16 hi / lo operand plane fc2 reads.
constexpr int kDwCC = 64, kDwThreads = 256;
__global__ void __launch_bounds__(kDwThreads) pvt_dwconv_gelu_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                                     const float* __restrict__ bias, int H, int W, int C, int RS,
                                                                     float* __restrict__ out, __half* __restrict__ phi,
                                                                     __half* __restrict__ plo) {
  extern __shared__ float4 tile[];                    // [(RS + 2) * W][16]
  __shared__ float4 ws[9][kDwCC / 4], bs[kDwCC / 4];
  constexpr int L4 = kDwCC / 4;
  const int c0 = blockIdx.x * kDwCC, h0 = blockIdx.y * RS;
  const long b = blockIdx.z;
  const int rows = min(RS, H - h0);
  for (int i = threadIdx.x; i < 10 * kDwCC; i += blockDim.x) {
    const int k = i / kDwCC, c = i - k * kDwCC;
    const float v = c0 + c < C ? (k < 9 ? w[(long)(c0 + c) * 9 + k] : bias[c0 + c]) : 0.f;
    (k < 9 ? reinterpret_cast<float*>(ws[k]) : reinterpret_cast<float*>(bs))[c] = v;
  }
  const float* xb = x + b * H * W * C;
  for (int i = threadIdx.x; i < (rows + 2) * W * L4; i += blockDim.x) {
    const int l = i % L4, px = i / L4;
    const int h = h0 - 1 + px / W, c = c0 + 4 * l;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (h >= 0 && h < H && c < C) v = *reinterpret_cast<const float4*>(xb + ((long)h * W + px % W) * C + c);
    tile[i] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < rows * W * L4; i += blockDim.x) {
    const int l = i % L4, px = i / L4;
    const int hh = px / W, ww = px - hh * W, c = c0 + 4 * l;
    if (c >= C) continue;
    float4 a = bs[l];
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int wi = ww + kx - 1;
        if (wi < 0 || wi >= W) continue;
        const float4 v = tile[((hh + ky) * W + wi) * L4 + l], k4 = ws[ky * 3 + kx][l];
        a.x = fmaf(v.x, k4.x, a.x); a.y = fmaf(v.y, k4.y, a.y); a.z = fmaf(v.z, k4.z, a.z); a.w = fmaf(v.w, k4.w, a.w);
      }
    a.x = gelu_erf(a.x); a.y = gelu_erf(a.y); a.z = gelu_erf(a.z); a.w = gelu_erf(a.w);
    const long off = ((b * H + h0 + hh) * W + ww) * C + c;
    if (phi) {
      uint2 hv, lv;
      hv.x = split2(a.x, a.y, lv.x);
      hv.y = split2(a.z, a.w, lv.y);
      *reinterpret_cast<uint2*>(phi + off) = hv;
      *reinterpret_cast<uint2*>(plo + off) = lv;
    } else {
      *reinterpret_cast<float4*>(out + off) = a;
    }
  }
}

// ---- head: mean over the mel axis of x [B][H][W][C], fc_audioset, sigmoid, the row repeat of interpolate() and the
// clipwise mean over H.  One block per (8 classes, sample): its warps hold one class row each in shared memory and
// walk the H rows in order, so the clipwise sum is a fixed-order fp32 sum.
constexpr int kHeadWarps = 8;
__global__ void __launch_bounds__(kHeadWarps * 32) pvt_head_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                                   const float* __restrict__ bias, int H, int W, int C, int classes,
                                                                   int ratio, float* __restrict__ framewise, float* __restrict__ clipwise,
                                                                   float* __restrict__ logits) {
  extern __shared__ float sm[];
  float* mean = sm;            // [C]
  float* wrow = sm + C;        // [warps][C]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int cls = blockIdx.x * kHeadWarps + warp;
  const long b = blockIdx.y;
  if (cls < classes)
    for (int c = lane; c < C; c += 32) wrow[warp * C + c] = w[(long)cls * C + c];
  const float bv = cls < classes ? bias[cls] : 0.f;
  float clip = 0.f;
  for (int h = 0; h < H; ++h) {
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      float s = 0.f;
      for (int j = 0; j < W; ++j) s += x[((b * H + h) * W + j) * C + c];
      mean[c] = s / (float)W;
    }
    __syncthreads();
    if (cls >= classes) continue;
    float d = 0.f;
    for (int c = lane; c < C; c += 32) d = fmaf(mean[c], wrow[warp * C + c], d);
#pragma unroll
    for (int o = 16; o; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    const float z = d + bv, p = sigmoidf_(z);
    clip += p;
    if (logits && lane == 0) logits[(b * H + h) * classes + cls] = z;
    for (int r = lane; r < ratio; r += 32) framewise[((b * H + h) * ratio + r) * classes + cls] = p;
  }
  if (cls < classes && lane == 0) clipwise[b * classes + cls] = clip / (float)H;
}

}  // namespace

// ---------------------------------------------------------------- launchers (also the unit tests' entry points)
void pvt_patch7(const float* img, const float* w, const float* bias, const float* gamma, const float* beta, float eps, int B, int H,
                int W, int C, float* out, cudaStream_t st) {
  AGPT_CHECK(B >= 1 && H >= 3 && W >= 3, "patch7: the image must be at least 3 x 3");
  AGPT_CHECK(C >= 32 && C % 32 == 0 && C <= 32 * kPatchMaxCpl, "patch7: C must be 32, 64, 96 or 128");
  const int Ho = (H - 3) / 4 + 1, Wo = (W - 3) / 4 + 1;
  const long tokens = (long)B * Ho * Wo;
  const size_t smem = sizeof(float) * (kPatchTaps * C + kPatchWarps * 52);
  pvt_patch7_kernel<<<(unsigned)cdivl(tokens, kPatchTokens), kPatchWarps * 32, smem, st>>>(img, w, bias, gamma, beta, eps, H, W, C, Ho,
                                                                                           Wo, tokens, out);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

void pvt_sr_gather(const float* x, int B, int H, int W, int C, int sr, float* out, cudaStream_t st) {
  AGPT_CHECK(B >= 1 && sr >= 1 && H >= sr && W >= sr && C % 4 == 0, "sr_gather: the grid must hold one sr x sr patch, C % 4 == 0");
  const int Hr = H / sr, Wr = W / sr;
  const long total = (long)B * Hr * Wr * sr * sr * (C / 4);
  pvt_sr_gather_kernel<<<(unsigned)std::min<long>(cdivl(total, 256), 4096), 256, 0, st>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(out), H, W, C / 4, sr, Hr, Wr, total);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

void pvt_dwconv_gelu(const float* x, const float* w, const float* bias, int B, int H, int W, int C, float* out, __half* phi,
                     __half* plo, cudaStream_t st) {
  AGPT_CHECK(B >= 1 && H >= 1 && W >= 1 && C >= 4 && C % 4 == 0, "dwconv_gelu: C must be a multiple of 4");
  AGPT_CHECK((out != nullptr) != (phi != nullptr) && (phi != nullptr) == (plo != nullptr),
             "dwconv_gelu: either the fp32 output or both operand planes");
  const long row_bytes = (long)W * kDwCC * sizeof(float);
  AGPT_CHECK(3 * row_bytes <= 40 * 1024, "dwconv_gelu: image too wide for the shared-memory strip");
  const int RS = (int)std::max<long>(1, std::min<long>(std::min(8, H), 40 * 1024 / row_bytes - 2));
  dim3 grid(cdiv(C, kDwCC), cdiv(H, RS), B);
  pvt_dwconv_gelu_kernel<<<grid, kDwThreads, (size_t)(RS + 2) * row_bytes, st>>>(x, w, bias, H, W, C, RS, out, phi, plo);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

void pvt_head(const float* x, const float* w, const float* bias, int B, int H, int W, int C, int classes, int ratio, float* framewise,
              float* clipwise, float* logits, cudaStream_t st) {
  AGPT_CHECK(B >= 1 && H >= 1 && W >= 1 && C >= 1 && classes >= 1 && ratio >= 1, "head: empty input");
  const size_t smem = sizeof(float) * (size_t)C * (1 + kHeadWarps);
  AGPT_CHECK(smem <= 48 * 1024, "head: too many channels");
  pvt_head_kernel<<<dim3(cdiv(classes, kHeadWarps), B), kHeadWarps * 32, smem, st>>>(x, w, bias, H, W, C, classes, ratio, framewise,
                                                                                     clipwise, logits);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// The stage grids of a clip (agpt_pvt_frames)
void pvt_frames(const agpt_pvt_cfg* cfg, long n, int grid[4][2]) {
  AGPT_CHECK(cfg->hop_size >= 1 && cfg->window_size >= 8, "bad PVT config");
  AGPT_CHECK(n > cfg->window_size / 2, "clip too short: reflect padding needs more than window_size / 2 samples");
  AGPT_CHECK(n <= (1L << 30), "clip too long");
  int H = (int)(n / cfg->hop_size) + 1, W = cfg->mel_bins;
  for (int i = 0; i < kStages; ++i) {
    AGPT_CHECK(H >= (i ? 1 : 3) && W >= (i ? 1 : 3), "clip too short: a stage's token grid is empty");
    if (i == 0) { H = (H - 3) / 4 + 1; W = (W - 3) / 4 + 1; }
    else { H = (H - 1) / 2 + 1; W = (W - 1) / 2 + 1; }
    AGPT_CHECK(H >= cfg->sr_ratios[i] && W >= cfg->sr_ratios[i],
               "clip too short: a stage's token grid is smaller than its sr_ratio, so attention would have no keys");
    grid[i][0] = H; grid[i][1] = W;
  }
}

namespace {

struct PvtBlock {
  DevBuf n1g, n1b, n2g, n2b, srg, srb, dww, dwb;
  PackedConv q, kv, proj, sr, fc1, fc2;
};
struct PvtStage {
  DevBuf pw, pb;             // stage 1: the 7 x 7 conv's [C][49] weight and bias (fp32 kernel)
  PackedConv patch;          // stages 2-4: [C][(ky, kx, ci)] over im2col rows
  DevBuf eg, eb, ng, nb;     // patch_embed.norm, norm{i}
  std::vector<PvtBlock> blocks;
};

// Conv2d weight [Cout][Cin][k][k] -> [Cout][(ky, kx, ci)], the row order of im2col_stride2 and pvt_sr_gather
std::vector<float> repack_kkc(const float* w, int cout, int cin, int k) {
  std::vector<float> r((size_t)cout * cin * k * k);
  for (int co = 0; co < cout; ++co)
    for (int ci = 0; ci < cin; ++ci)
      for (int t = 0; t < k * k; ++t) r[((size_t)co * k * k + t) * cin + ci] = w[((size_t)co * cin + ci) * k * k + t];
  return r;
}

struct PvtNet : Handle {
  agpt_pvt_cfg cfg;
  LogmelFront front;
  PvtStage stage[kStages];
  DevBuf fcw, fcb;
  DevBuf img, x, y, n, q, kv, ctx, gat, s, sn, hid, act, col;

  void linear(const PackedConv& pc, const float* in, float* out, long rows, int epi, cudaStream_t st, const float* res = nullptr) {
    fs_conv(pc, in, pc.Cin, out, pc.Cout, 1, (int)rows, epi, st, res);
  }

  void forward(const float* wav, int B, long nsamp, float* framewise, float* clipwise, float* logits, cudaStream_t st) {
    AGPT_CHECK(B >= 1, "empty batch");
    int grid[4][2];
    pvt_frames(&cfg, nsamp, grid);
    AGPT_CHECK((long)B * grid[0][0] * grid[0][1] <= (1L << 30) / 64, "batch x clip length too large");
    const int T = LogmelFront::frames_of(nsamp, cfg.hop_size), nm = cfg.mel_bins;
    img.ensure((size_t)B * T * nm);
    front.run<1>(wav, (int)nsamp, B, img.p, st);
    size_t mx = 0, mh = 0, mg = 0, mc = 0;
    for (int i = 0; i < kStages; ++i) {
      const size_t rows = (size_t)B * grid[i][0] * grid[i][1], C = cfg.embed_dims[i];
      mx = std::max(mx, rows * C);
      mh = std::max(mh, rows * C * cfg.mlp_ratios[i]);
      if (cfg.sr_ratios[i] > 1) mg = std::max(mg, rows * C);     // the gather keeps (almost) every element
      if (i) mc = std::max(mc, rows * 9 * cfg.embed_dims[i - 1]);
    }
    x.ensure(mx); y.ensure(mx); n.ensure(mx); q.ensure(mx); ctx.ensure(mx); kv.ensure(2 * mx);
    s.ensure(mx); sn.ensure(mx); hid.ensure(mh); act.ensure(mh); gat.ensure(std::max<size_t>(mg, 4)); col.ensure(std::max<size_t>(mc, 4));
    const bool planes = tc_enabled();   // fc2 reads the GELU output as fp16 hi / lo operand planes (tensor-core arm only)
    int H = T, W = nm;
    for (int i = 0; i < kStages; ++i) {
      PvtStage& S = stage[i];
      const int C = cfg.embed_dims[i], heads = cfg.num_heads[i], sr = cfg.sr_ratios[i], hdim = C * cfg.mlp_ratios[i];
      const int Ho = grid[i][0], Wo = grid[i][1];
      const long rows = (long)B * Ho * Wo;
      if (i == 0) {
        pvt_patch7(img.p, S.pw.p, S.pb.p, S.eg.p, S.eb.p, cfg.embed_norm_eps, B, H, W, C, x.p, st);
      } else {
        const int Cp = cfg.embed_dims[i - 1];
        im2col_stride2(n.p, col.p, B, H, W, Cp, Ho, Wo, 1, st);      // n holds the previous stage's normed output
        linear(S.patch, col.p, y.p, rows, EPI_BIAS, st);
        layernorm(y.p, x.p, S.eg.p, S.eb.p, rows, C, cfg.embed_norm_eps, st);
      }
      H = Ho; W = Wo;
      const int Hr = H / sr, Wr = W / sr;
      const long krows = (long)B * Hr * Wr;
      for (PvtBlock& K : S.blocks) {
        layernorm(x.p, n.p, K.n1g.p, K.n1b.p, rows, C, cfg.layer_norm_eps, st);
        linear(K.q, n.p, q.p, rows, EPI_BIAS, st);
        if (sr > 1) {
          pvt_sr_gather(n.p, B, H, W, C, sr, gat.p, st);
          linear(K.sr, gat.p, s.p, krows, EPI_BIAS, st);
          layernorm(s.p, sn.p, K.srg.p, K.srb.p, krows, C, cfg.embed_norm_eps, st);
          linear(K.kv, sn.p, kv.p, krows, EPI_BIAS, st);
        } else {
          linear(K.kv, n.p, kv.p, rows, EPI_BIAS, st);
        }
        attention(q.p, C, kv.p, 2 * C, kv.p + C, 2 * C, ctx.p, C, B, heads, kHeadDim, H * W, Hr * Wr, st);
        linear(K.proj, ctx.p, y.p, rows, EPI_RES, st, x.p);
        layernorm(y.p, n.p, K.n2g.p, K.n2b.p, rows, C, cfg.layer_norm_eps, st);
        linear(K.fc1, n.p, hid.p, rows, EPI_BIAS, st);
        if (planes && hdim % 8 == 0) {
          __half* hi = reinterpret_cast<__half*>(act.p);
          __half* lo = hi + (size_t)rows * hdim;
          pvt_dwconv_gelu(hid.p, K.dww.p, K.dwb.p, B, H, W, hdim, nullptr, hi, lo, st);
          TapConvParams P = tapconv_params(K.fc2, 1, (int)rows, 0, 1);
          P.in = hid.p; P.in_pitch = hdim; P.in_gstride = rows * hdim;   // the planes below are read, not the fp32 tensor
          P.pi_hi = hi; P.pi_lo = lo;
          P.pro = PRO_LRELU; P.slope = 1.f;            // the planes hold lrelu(x, 1) = x
          P.out = x.p; P.out_pitch = C;
          P.epi = EPI_RES; P.res = y.p; P.res_pitch = C;
          tapconv_launch(P, st);
        } else {
          pvt_dwconv_gelu(hid.p, K.dww.p, K.dwb.p, B, H, W, hdim, act.p, nullptr, nullptr, st);
          linear(K.fc2, act.p, x.p, rows, EPI_RES, st, y.p);
        }
      }
      layernorm(x.p, n.p, S.ng.p, S.nb.p, rows, C, cfg.layer_norm_eps, st);
    }
    pvt_head(n.p, fcw.p, fcb.p, B, H, W, cfg.embed_dims[kStages - 1], cfg.classes_num, cfg.interpolate_ratio, framewise, clipwise,
             logits, st);
  }
};

}  // namespace

Handle* pvt_create(const agpt_pvt_cfg* cfg, const float* const* Wt, int nW, int device) {
  DeviceGuard dg_(device);
  AGPT_CHECK(cfg->window_size >= 8 && cfg->window_size % 4 == 0 && cfg->hop_size >= 1 && cfg->classes_num >= 1 &&
                 cfg->interpolate_ratio >= 1 && cfg->layer_norm_eps > 0.f && cfg->embed_norm_eps > 0.f,
             "bad PVT config");
  AGPT_CHECK(cfg->mel_bins == 64, "PVT: mel_bins must be 64 (bn0 is BatchNorm2d(64))");
  for (int i = 0; i < kStages; ++i) {
    AGPT_CHECK(cfg->num_heads[i] >= 1 && cfg->embed_dims[i] == kHeadDim * cfg->num_heads[i], "PVT: every head must be 64 wide");
    AGPT_CHECK(cfg->depths[i] >= 1 && cfg->mlp_ratios[i] >= 1 && cfg->sr_ratios[i] >= 1, "bad PVT stage config");
  }
  AGPT_CHECK(cfg->embed_dims[0] <= 32 * kPatchMaxCpl, "PVT: the first stage is at most 128 wide");
  AGPT_CHECK((size_t)cfg->embed_dims[kStages - 1] * (1 + kHeadWarps) * sizeof(float) <= 48 * 1024, "PVT: the last stage is too wide");
  std::unique_ptr<PvtNet> h(new PvtNet());
  h->magic = kMagicPvt; h->device = device; h->cfg = *cfg;
  WeightCursor wc{Wt, nW};
  h->front.load(wc, cfg->window_size, cfg->hop_size, cfg->mel_bins, kBnEps);
  auto up2 = [&](DevBuf& a, DevBuf& b, size_t na, size_t nb) { const float* p = wc.next(); const float* r = wc.next(); a.upload(p, na); b.upload(r, nb); };
  auto lin = [&](PackedConv& pc, int cout, int cin) { const float* w = wc.next(); const float* b = wc.next(); pack_conv(pc, w, b, cout, cin, 1, false); };
  for (int i = 0; i < kStages; ++i) {
    PvtStage& S = h->stage[i];
    const int C = cfg->embed_dims[i], sr = cfg->sr_ratios[i], hd = C * cfg->mlp_ratios[i];
    if (i == 0) {
      up2(S.pw, S.pb, (size_t)C * kPatchTaps, C);
    } else {
      const int Cp = cfg->embed_dims[i - 1];
      const float* w = wc.next(); const float* b = wc.next();
      pack_conv(S.patch, repack_kkc(w, C, Cp, 3).data(), b, C, 9 * Cp, 1, false);
    }
    up2(S.eg, S.eb, C, C);
    S.blocks.resize(cfg->depths[i]);
    for (PvtBlock& K : S.blocks) {
      up2(K.n1g, K.n1b, C, C);
      lin(K.q, C, C); lin(K.kv, 2 * C, C); lin(K.proj, C, C);
      if (sr > 1) {
        const float* w = wc.next(); const float* b = wc.next();
        pack_conv(K.sr, repack_kkc(w, C, C, sr).data(), b, C, sr * sr * C, 1, false);
        up2(K.srg, K.srb, C, C);
      }
      up2(K.n2g, K.n2b, C, C);
      lin(K.fc1, hd, C);
      up2(K.dww, K.dwb, (size_t)hd * 9, hd);
      lin(K.fc2, C, hd);
    }
    up2(S.ng, S.nb, C, C);
  }
  up2(h->fcw, h->fcb, (size_t)cfg->classes_num * cfg->embed_dims[kStages - 1], cfg->classes_num);
  wc.done();
  return h.release();
}

void pvt_forward(Handle* hh, const float* wav, int B, long n_samples, float* framewise, float* clipwise, float* logits,
                 cudaStream_t st) {
  auto* h = static_cast<PvtNet*>(hh);
  DeviceGuard dg_(h->device);
  h->forward(wav, B, n_samples, framewise, clipwise, logits, st);
}

}  // namespace agpt
