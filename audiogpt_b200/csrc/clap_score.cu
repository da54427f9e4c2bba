// Audio tower of the CLAP candidate scorer on sm_90a: a 16 kHz clip -> the L2-normalised [B][d_proj] audio embedding
// that T2A.select_best_audio compares with its prompt.
// Reference: text_to_audio/Make_An_Audio/wav_evaluation/models/CLAPWrapper.py:119-143 (resample_and_duration),
// :184-206 (get_audio_embeddings), models/audio.py:107-179 (Cnn14 with torchlibrosa's Spectrogram / LogmelFilterBank),
// models/clap.py:8-40 (Projection, AudioEncoder), torchaudio.transforms.Resample (sinc_interp_hann polyphase filter).
// The DFT, the 12 convs (eval BatchNorm folded), fc1 and the projection's Linears are tap-GEMMs (tcconv5 on the tensor
// cores); the resampler, framing, power / mel / log / bn0, pooling head, L2 norms and the score dots are fp32 kernels.
#include "common.cuh"
#include "tapconv.cuh"
#include "nn_kernels.h"
#include "models.h"
#include "fs_layers.cuh"
#include "clap.cuh"

namespace agpt {

namespace {

constexpr int kCnn14Blocks = 6;
constexpr int kCnn14Ch[kCnn14Blocks] = {64, 128, 256, 512, 1024, 2048};
constexpr float kBnEps = 1e-5f;

// out[b][i] = y_b[(start_b + i) mod R] for i < clip, y_b the resampled clip b: one rule for the crop (start_b >= 0,
// start_b + clip <= R) and the tiling (start_b = 0, R <= clip) of resample_and_duration.
// y[k * nw + p] = sum_j ker[p][j] * x[k * orig + j - width]  (torchaudio's conv1d over the zero-padded clip)
__global__ void cnn14_resample_kernel(const float* __restrict__ x, long L, const float* __restrict__ ker, int taps, int orig,
                                      int nw, int width, long R, const int* __restrict__ starts, int clip,
                                      float* __restrict__ out, long total) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long b = i / clip, o = i - b * clip;
    const long n = ((long)max(starts[b], 0) + o) % R;
    const long k = n / nw;
    const int p = (int)(n - k * nw);
    const long base = k * orig - width;
    const float* xb = x + b * L;
    const float* kp = ker + (long)p * taps;
    float acc = 0.f;
    for (int j = 0; j < taps; ++j) {
      const long xi = base + j;
      if (xi >= 0 && xi < L) acc = fmaf(kp[j], xb[xi], acc);
    }
    out[i] = acc;
  }
}

// frames[b][t][j] = x_b[reflect(t * hop + j - n / 2)]  (center=True, pad_mode='reflect')
__global__ void cnn14_frames_kernel(const float* __restrict__ x, int clip, int T, int hop, int n, float* __restrict__ fr, long total) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long bt = i / n;
    const int j = (int)(i - bt * n);
    const long b = bt / T;
    const int t = (int)(bt - b * T);
    int s = t * hop + j - n / 2;
    s = s < 0 ? -s : (s >= clip ? 2 * (clip - 1) - s : s);
    fr[i] = x[b * clip + s];
  }
}

// one block per frame: re^2 + im^2 -> melW projection -> 10 log10(max(., 1e-10)) -> bn0 (folded scale / shift per mel
// bin) -> img[b][t][m][0..3] (the first conv's 4-channel padded input)
__global__ void cnn14_logmel_kernel(const float* __restrict__ spec, int pitch, int nb, const float* __restrict__ melW,
                                    int nm, const float* __restrict__ bn_s, const float* __restrict__ bn_t, float* __restrict__ img) {
  extern __shared__ float pw[];
  const long f = blockIdx.x;
  const float* re = spec + f * pitch;
  const float* im = re + nb;
  for (int k = threadIdx.x; k < nb; k += blockDim.x) pw[k] = re[k] * re[k] + im[k] * im[k];
  __syncthreads();
  for (int m = threadIdx.x; m < nm; m += blockDim.x) {
    float acc = 0.f;
    for (int k = 0; k < nb; ++k) acc = fmaf(pw[k], melW[(long)k * nm + m], acc);
    const float db = 10.f * log10f(fmaxf(acc, 1e-10f));
    *reinterpret_cast<float4*>(img + (f * nm + m) * 4) = make_float4(db * bn_s[m] + bn_t[m], 0.f, 0.f, 0.f);
  }
}

// x [B][T][F][C] -> out[b][c] = max_t mean_f x + mean_t mean_f x  (Cnn14.forward after conv_block6)
__global__ void cnn14_head_kernel(const float* __restrict__ x, int T, int F, int C, float* __restrict__ out, int B) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * C) return;
  const long b = i / C;
  const int c = (int)(i - b * C);
  const float* xb = x + b * T * F * C + c;
  float mx = -INFINITY, sum = 0.f;
  for (int t = 0; t < T; ++t) {
    float s = 0.f;
    for (int f = 0; f < F; ++f) s += xb[((long)t * F + f) * C];
    s /= (float)F;
    mx = fmaxf(mx, s);
    sum += s;
  }
  out[i] = mx + sum / (float)T;
}

__device__ float block_sum(float v, float* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[w] = v;
  __syncthreads();
  float s = 0.f;
  for (int k = 0; k < nw; ++k) s += red[k];
  return s;
}

// out[r] = in[r] / |in[r]|, twice (the scorer divides by the norm in _get_*_embeddings and again in get_*_embeddings)
__global__ void clap_l2norm2_kernel(const float* __restrict__ in, float* __restrict__ out, int D) {
  __shared__ float red[32];
  const float* x = in + (long)blockIdx.x * D;
  float* y = out + (long)blockIdx.x * D;
  float s = 0.f;
  for (int c = threadIdx.x; c < D; c += blockDim.x) s = fmaf(x[c], x[c], s);
  const float n1 = sqrtf(block_sum(s, red));
  s = 0.f;
  for (int c = threadIdx.x; c < D; c += blockDim.x) { const float v = x[c] / n1; s = fmaf(v, v, s); }
  const float n2 = sqrtf(block_sum(s, red));
  for (int c = threadIdx.x; c < D; c += blockDim.x) y[c] = (x[c] / n1) / n2;
}

// out[i][j] = scale * <a_i, t_j>  (compute_similarity: (t @ a.T).T), one block per (i, j), fp32 FMA
__global__ void clap_similarity_kernel(const float* __restrict__ a, const float* __restrict__ t, int Nt, int D, float scale,
                                       float* __restrict__ out) {
  __shared__ float red[32];
  const int i = blockIdx.x / Nt, j = blockIdx.x % Nt;
  float s = 0.f;
  for (int c = threadIdx.x; c < D; c += blockDim.x) s = fmaf(a[(long)i * D + c], t[(long)j * D + c], s);
  s = block_sum(s, red);
  if (threadIdx.x == 0) out[blockIdx.x] = scale * s;
}

__global__ void clap_gelu2_kernel(const float* __restrict__ in, float* __restrict__ out, long n) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) out[i] = gelu_erf(in[i]);
}

unsigned ew_blocks(long n) { return (unsigned)std::min<long>(cdivl(n, 256), 4096); }

}  // namespace

void clap_l2norm2(const float* in, float* out, int rows, int D, cudaStream_t st) {
  clap_l2norm2_kernel<<<rows, 256, 0, st>>>(in, out, D);
  count_launch(1);
}

void clap_similarity(const float* a, int Na, const float* t, int Nt, int D, float scale, float* out, cudaStream_t st) {
  AGPT_CHECK(Na >= 1 && Nt >= 1 && D >= 1, "empty similarity");
  clap_similarity_kernel<<<(unsigned)(Na * Nt), 256, 0, st>>>(a, t, Nt, D, scale, out);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// CLAP's Projection (clap.py:8-20, dropout off) on [rows][d_in] rows of pitch in_pitch, then the two L2 norms:
// out = l2(l2(LayerNorm(e1 + linear2(gelu(e1))))), e1 = linear1(x)
void ClapProjection::run(const float* x, int in_pitch, int rows, float* out, cudaStream_t st) {
  const int D = lin1.Cout;
  e1.ensure((size_t)rows * D); g1.ensure((size_t)rows * D); e12.ensure((size_t)rows * D); z.ensure((size_t)rows * D);
  TapConvParams P = tapconv_params(lin1, 1, rows, 0, 1);
  P.in = x; P.in_pitch = in_pitch;
  P.out = e1.p; P.out_pitch = D;
  P.epi = EPI_BIAS;
  tapconv_launch(P, st);
  clap_gelu2_kernel<<<ew_blocks((long)rows * D), 256, 0, st>>>(e1.p, g1.p, (long)rows * D);
  count_launch(1);
  fs_conv(lin2, g1.p, D, e12.p, D, 1, rows, EPI_RES, st, e1.p);
  layernorm(e12.p, z.p, lng.p, lnb.p, rows, D, eps, st);
  clap_l2norm2(z.p, out, rows, D, st);
}

void ClapProjection::load(WeightCursor& wc, int d_in, int d_out, float eps_) {
  pack_conv(lin1, wc.next(), nullptr, d_out, d_in, 1, false);
  pack_conv(lin2, wc.next(), nullptr, d_out, d_out, 1, false);
  { auto g = wc.next(); auto b = wc.next(); lng.upload(g, d_out); lnb.upload(b, d_out); }
  eps = eps_;
}

struct Cnn14Net : Handle {
  agpt_cnn14_cfg cfg;
  PackedConv dft;
  DevBuf melW, bn0_s, bn0_t;
  PackedConv conv[kCnn14Blocks][2];
  PackedConv fc1;
  ClapProjection proj;
  // resampler (agpt_cnn14_set_resample)
  DevBuf ker;
  int orig = 0, nw = 0, width = 0, taps = 0, clip = 0;
  DevBuf starts, wav, frames, spec, img, bufA, bufB, bufC, pooled, emb;

  void embed(const float* x, long L, int B, const int* start_host, float* out, cudaStream_t st) {
    AGPT_CHECK(clip > 0, "agpt_cnn14_set_resample was not called");
    AGPT_CHECK(B >= 1 && L >= 1, "empty batch");
    const long R = cdivl((long)nw * L, orig);   // ceil(new * L / orig): the resampled length
    for (int b = 0; b < B; ++b) {
      const int s = start_host[b];
      if (R > clip) AGPT_CHECK(s >= 0 && (long)s < R - clip, "crop start outside [0, resampled length - clip)");
      else AGPT_CHECK(s == -1, "a clip no longer than the target is tiled: its start must be -1");
    }
    const int n = cfg.window_size, hop = cfg.hop_size, nb = n / 2 + 1, nm = cfg.mel_bins;
    AGPT_CHECK(clip > n / 2, "the fitted clip must be longer than half a window (reflect padding)");
    const int T = clip / hop + 1;
    int* sd = reinterpret_cast<int*>(starts.ensure(B));
    AGPT_CUDA(cudaMemcpyAsync(sd, start_host, sizeof(int) * B, cudaMemcpyHostToDevice, st));
    wav.ensure((size_t)B * clip);
    const long tot = (long)B * clip;
    cnn14_resample_kernel<<<ew_blocks(tot), 256, 0, st>>>(x, L, ker.p, taps, orig, nw, width, R, sd, clip, wav.p, tot);
    frames.ensure((size_t)B * T * n);
    cnn14_frames_kernel<<<ew_blocks((long)B * T * n), 256, 0, st>>>(wav.p, clip, T, hop, n, frames.p, (long)B * T * n);
    count_launch(2);
    spec.ensure((size_t)B * T * dft.cout_pad);
    {
      TapConvParams P = tapconv_params(dft, 1, B * T, 0, 1);
      P.in = frames.p; P.in_pitch = n;
      P.out = spec.p; P.out_pitch = dft.cout_pad;
      P.epi = EPI_BIAS;
      tapconv_launch(P, st);
    }
    img.ensure((size_t)B * T * nm * 4);
    cnn14_logmel_kernel<<<(unsigned)(B * T), 64, sizeof(float) * nb, st>>>(spec.p, dft.cout_pad, nb, melW.p, nm, bn0_s.p, bn0_t.p, img.p);
    count_launch(1);
    // conv blocks: (3x3 conv -> folded BN -> ReLU) x 2, then AvgPool2d(2) (blocks 1-5) on [B][H=T][W=F][C]
    const size_t big = (size_t)B * T * nm * kCnn14Ch[0];
    bufA.ensure(big); bufB.ensure(big); bufC.ensure(big);
    const float* in = img.p;
    int H = T, W = nm;
    for (int i = 0; i < kCnn14Blocks; ++i) {
      conv3x3(conv[i][0], in, bufB.p, B, H, W, st);
      conv3x3(conv[i][1], bufB.p, bufC.p, B, H, W, st);
      if (i < kCnn14Blocks - 1) {
        avgpool2(bufC.p, bufA.p, B, H, W, kCnn14Ch[i], st);
        H /= 2; W /= 2;
        in = bufA.p;
      } else {
        in = bufC.p;
      }
    }
    const int C = kCnn14Ch[kCnn14Blocks - 1];
    pooled.ensure((size_t)B * C); emb.ensure((size_t)B * cfg.out_emb);
    cnn14_head_kernel<<<(unsigned)cdivl((long)B * C, 256), 256, 0, st>>>(in, H, W, C, pooled.p, B);
    count_launch(1);
    fs_conv(fc1, pooled.p, C, emb.p, cfg.out_emb, 1, B, EPI_RELU, st);
    proj.run(emb.p, cfg.out_emb, B, out, st);
    AGPT_CUDA(cudaGetLastError());
  }

  void conv3x3(const PackedConv& pc, const float* in, float* out, int B, int H, int W, cudaStream_t st) {
    TapConvParams P = tapconv_params(pc, B, H * W, W, 1);
    P.in = in; P.in_gstride = (long)H * W * pc.Cin; P.in_pitch = pc.Cin;
    P.out = out; P.out_gstride = (long)H * W * pc.Cout; P.out_pitch = pc.Cout;
    P.epi = EPI_RELU;
    tapconv_launch(P, st);
  }
};

// BatchNorm2d (eval) folded into the preceding bias-free conv: w' = w * s, b' = beta - mean * s, s = gamma / sqrt(var + eps)
static void load_conv_bn(PackedConv& pc, const float* w, WeightCursor& wc, int cout, int cin, int cin_pad) {
  const float* g = wc.next(); const float* be = wc.next(); const float* rm = wc.next(); const float* rv = wc.next();
  std::vector<float> wf((size_t)cout * cin_pad * 9, 0.f), bf(cout);
  for (int co = 0; co < cout; ++co) {
    const float s = g[co] / sqrtf(rv[co] + kBnEps);
    bf[co] = be[co] - rm[co] * s;
    for (int ci = 0; ci < cin; ++ci)
      for (int k = 0; k < 9; ++k) wf[((size_t)co * cin_pad + ci) * 9 + k] = w[((size_t)co * cin + ci) * 9 + k] * s;
  }
  pack_conv(pc, wf.data(), bf.data(), cout, cin_pad, 9, true);
}

Handle* cnn14_create(const agpt_cnn14_cfg* cfg, const float* const* W, int nW, int device) {
  DeviceGuard dg_(device);
  AGPT_CHECK(cfg->window_size >= 8 && cfg->window_size % 4 == 0 && cfg->hop_size >= 1 && cfg->mel_bins == 64 &&
                 cfg->out_emb >= 4 && cfg->out_emb % 4 == 0 && cfg->d_proj >= 4 && cfg->d_proj % 4 == 0,
             "bad Cnn14 config (mel_bins must be 64: Cnn14's bn0 is BatchNorm2d(64))");
  std::unique_ptr<Cnn14Net> h(new Cnn14Net());
  h->magic = kMagicCnn14; h->device = device; h->cfg = *cfg;
  const int n = cfg->window_size, nb = n / 2 + 1, nm = cfg->mel_bins;
  WeightCursor wc{W, nW};
  {  // conv_real / conv_imag [nb][1][n] -> one [n] -> [re | im] 1-tap GEMM
    const float* re = wc.next(); const float* im = wc.next();
    std::vector<float> w((size_t)2 * nb * n);
    memcpy(w.data(), re, sizeof(float) * nb * n);
    memcpy(w.data() + (size_t)nb * n, im, sizeof(float) * nb * n);
    pack_conv(h->dft, w.data(), nullptr, 2 * nb, n, 1, false);
  }
  h->melW.upload(wc.next(), (size_t)nb * nm);
  {
    const float* g = wc.next(); const float* be = wc.next(); const float* rm = wc.next(); const float* rv = wc.next();
    std::vector<float> s(nm), t(nm);
    for (int m = 0; m < nm; ++m) { s[m] = g[m] / sqrtf(rv[m] + kBnEps); t[m] = be[m] - rm[m] * s[m]; }
    h->bn0_s.upload(s); h->bn0_t.upload(t);
  }
  int cin = 1;
  for (int i = 0; i < kCnn14Blocks; ++i) {
    const int c = kCnn14Ch[i];
    const float* w1 = wc.next(); const float* w2 = wc.next();
    load_conv_bn(h->conv[i][0], w1, wc, c, cin, round_up(cin, 4));
    load_conv_bn(h->conv[i][1], w2, wc, c, c, c);
    cin = c;
  }
  { auto w = wc.next(); auto b = wc.next(); pack_conv(h->fc1, w, b, cfg->out_emb, cin, 1, false); }
  h->proj.load(wc, cfg->out_emb, cfg->d_proj, kBnEps);
  wc.done();
  return h.release();
}

void cnn14_set_resample(Handle* hh, int orig, int nw, int width, const float* table, int clip) {
  auto* h = static_cast<Cnn14Net*>(hh);
  DeviceGuard dg_(h->device);
  AGPT_CHECK(orig >= 1 && nw >= 1 && width >= 0 && clip >= 1 && table, "bad resampler");
  h->orig = orig; h->nw = nw; h->width = width; h->taps = 2 * width + orig; h->clip = clip;
  h->ker.upload(table, (size_t)nw * h->taps);
}

void cnn14_embed(Handle* hh, const float* wav, long n_samples, int B, const int* start_host, float* out, cudaStream_t st) {
  auto* h = static_cast<Cnn14Net*>(hh);
  DeviceGuard dg_(h->device);
  h->embed(wav, n_samples, B, start_host, out, st);
}

}  // namespace agpt
