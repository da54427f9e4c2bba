// The out-of-domain TTS tool's emotion encoder on sm_90a: a preprocessed 16 kHz wav -> the L2-normalised mean of the
// last LSTM layer's final h over 1.6 s partial utterances (emo_embed, an input of GenerSpeech).
// Reference: NeuralSeq/data_gen/tts/emotion/inference.py:59-164 (compute_partial_slices, embed_utterance),
// audio.py:43-55 (wav_to_mel_spectrogram: librosa's power mel, n_fft 400, hop 160, 40 Slaney bands, no log) and
// model.py:41-77 (EmotionEncoder: nn.LSTM(40, 256, 3, batch_first) from h0 = c0 = 0; forward adds Linear, ReLU and an
// L2 norm).
// Front end: reflect-padded framing (cnn14_frames), one 1-tap tap-GEMM against the periodic-Hann DFT rows, then
// emo_powmel_kernel (re^2 + im^2 projected on the mel matrix).  Each layer's input projection W_ih x + b_ih + b_hh is
// one tap-GEMM; layer 0 runs it once over the mel frames the partials cover, and partial p reads rows step p ..
// step p + T - 1 of it (the partials overlap by half, so this halves layer 0's projection).  The recurrence is
// emo_lstm_kernel: an 8-CTA cluster per group of sequences, W_hh resident in shared memory, h exchanged over DSMEM.
#include <cmath>
#include <cooperative_groups.h>
#include "common.cuh"
#include "tapconv.cuh"
#include "models.h"
#include "audio_front.cuh"
#include "an_kernels.cuh"

namespace cg = cooperative_groups;

namespace agpt {

namespace {

constexpr int kNfft = 400, kHop = 160, kBins = kNfft / 2 + 1, kMels = 40;
constexpr int kEmoH = 256;                   // model_hidden_size
constexpr int kGates = 4 * kEmoH;            // i, f, g, o (PyTorch's order)

// ---- the LSTM cluster: 8 CTAs, each owning 32 hidden units (their 4 x 32 rows of W_hh in fp32 = 128 KB)
constexpr int kLstmCta = 8, kLstmU = kEmoH / kLstmCta, kLstmRows = 4 * kLstmU, kLstmThreads = 512, kLstmMaxB = 16;
constexpr size_t kLstmSmem = sizeof(float) * ((size_t)kLstmRows * kEmoH + 2 * kLstmMaxB * kEmoH + kLstmMaxB * kLstmRows + kLstmMaxB * kLstmU);

// one block per frame: mel[f][m] = sum_k (re_k^2 + im_k^2) melW[k][m] (no log, no normalisation)
constexpr int kMelThreads = 64;
__global__ void __launch_bounds__(kMelThreads) emo_powmel_kernel(const float* __restrict__ spec, int pitch, const float* __restrict__ melW,
                                                                 float* __restrict__ mel) {
  __shared__ float pw[kBins];
  const long f = blockIdx.x;
  const float* re = spec + f * pitch;
  const float* im = re + kBins;
  for (int k = threadIdx.x; k < kBins; k += blockDim.x) pw[k] = re[k] * re[k] + im[k] * im[k];
  __syncthreads();
  for (int m = threadIdx.x; m < kMels; m += blockDim.x) {
    float acc = 0.f;
    for (int k = 0; k < kBins; ++k) acc = fmaf(pw[k], melW[k * kMels + m], acc);
    mel[f * kMels + m] = acc;
  }
}

// ---- one LSTM layer's recurrence (PyTorch gate order i, f, g, o; h0 = c0 = 0):
//   z = xp + W_hh h,  c' = sig(z_f) c + sig(z_i) tanh(z_g),  h' = sig(z_o) tanh(c')
// xp holds the input projections W_ih x + b_ih + b_hh: sequence n's step t is row n * seq_stride + t of [rows][1024].
// One cluster of 8 CTAs per group of up to 16 sequences; CTA `rank` owns hidden units 32 rank .. 32 rank + 31 and keeps
// their 128 W_hh rows in shared memory for the whole sequence.  Every step each CTA forms its rows' W_hh h, updates its
// units (c stays in the updating thread's register), writes them into the next h buffer of all 8 CTAs over DSMEM and
// meets the others at a cluster barrier.  h_seq [N][T][256] (optional) gets every step, h_last [N][256] (optional) the
// final h.  fp32 FMA.
__global__ void __launch_bounds__(kLstmThreads, 1) emo_lstm_kernel(const float* __restrict__ whh, const float* __restrict__ xp, int N,
                                                                   int T, long seq_stride, int nb_max, float* __restrict__ h_seq,
                                                                   float* __restrict__ h_last) {
  cg::cluster_group cluster = cg::this_cluster();
  extern __shared__ float4 lstm_sm4[];
  float* w = reinterpret_cast<float*>(lstm_sm4);      // [128][256]
  float* hbuf = w + kLstmRows * kEmoH;               // [2][kLstmMaxB][256]
  float* g = hbuf + 2 * kLstmMaxB * kEmoH;           // [kLstmMaxB][128]
  float* hn = g + kLstmMaxB * kLstmRows;             // [kLstmMaxB][32]
  const int rank = (int)cluster.block_rank();
  const int n0 = blockIdx.z * nb_max, nb = min(nb_max, N - n0);
  const int u0 = rank * kLstmU;
  for (int i = threadIdx.x; i < kLstmRows * kEmoH / 4; i += blockDim.x) {
    const int lr = i / (kEmoH / 4), c4 = i % (kEmoH / 4);
    const int gr = (lr / kLstmU) * kEmoH + u0 + lr % kLstmU;
    lstm_sm4[i] = reinterpret_cast<const float4*>(whh + (size_t)gr * kEmoH)[c4];
  }
  for (int i = threadIdx.x; i < 2 * kLstmMaxB * kEmoH; i += blockDim.x) hbuf[i] = 0.f;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int kWarps = kLstmThreads / 32, kPer = kEmoH / 32;
  // the unit this thread updates (threads past nb * 32 only help with W_hh h); its c lives in a register
  const int ub = threadIdx.x / kLstmU, uj = threadIdx.x % kLstmU, u = u0 + uj;
  float c = 0.f;
  cluster.sync();    // every CTA runs and has zeroed its buffers before any remote write
  for (int t = 0; t < T; ++t) {
    const float* hc = hbuf + (t & 1) * kLstmMaxB * kEmoH;
    float* hnext = hbuf + ((t + 1) & 1) * kLstmMaxB * kEmoH;
    for (int row = warp; row < kLstmRows; row += kWarps) {
      float wr[kPer];
#pragma unroll
      for (int k = 0; k < kPer; ++k) wr[k] = w[row * kEmoH + lane + 32 * k];
      for (int b = 0; b < nb; ++b) {
        const float* hb = hc + b * kEmoH + lane;
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < kPer; ++k) acc = fmaf(wr[k], hb[32 * k], acc);
#pragma unroll
        for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) g[b * kLstmRows + row] = acc;
      }
    }
    __syncthreads();
    if (ub < nb) {
      const float* x = xp + ((size_t)(n0 + ub) * seq_stride + t) * kGates;
      const float* gb = g + ub * kLstmRows;
      const float ig = sigmoidf_(x[u] + gb[uj]);
      const float fg = sigmoidf_(x[kEmoH + u] + gb[kLstmU + uj]);
      const float gg = tanhf(x[2 * kEmoH + u] + gb[2 * kLstmU + uj]);
      const float og = sigmoidf_(x[3 * kEmoH + u] + gb[3 * kLstmU + uj]);
      c = fg * c + ig * gg;
      const float h = og * tanhf(c);
      hn[ub * kLstmU + uj] = h;
      if (h_seq) h_seq[((size_t)(n0 + ub) * T + t) * kEmoH + u] = h;
      if (h_last && t == T - 1) h_last[(size_t)(n0 + ub) * kEmoH + u] = h;
    }
    __syncthreads();
    if (t + 1 < T) {
      for (int i = threadIdx.x; i < kLstmCta * nb * kLstmU; i += blockDim.x) {
        const int q = i / (nb * kLstmU), bj = i % (nb * kLstmU), b = bj / kLstmU, j = bj % kLstmU;
        float* dst = cluster.map_shared_rank(hnext, q);
        dst[b * kEmoH + u0 + j] = hn[bj];
      }
      cluster.sync();
    }
  }
}

constexpr int kTailThreads = 256;
__device__ float emo_block_sum(float v, float* red) {
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

// embed_utterance's tail: raw = mean over the N partials of h [N][256], embed = raw / ||raw||_2.  One block.
__global__ void __launch_bounds__(kTailThreads) emo_mean_norm_kernel(const float* __restrict__ h, int N, float* __restrict__ embed) {
  __shared__ float red[32];
  const int u = threadIdx.x;
  float s = 0.f;
  for (int n = 0; n < N; ++n) s += h[(size_t)n * kEmoH + u];
  const float raw = s / (float)N;
  const float nrm = sqrtf(emo_block_sum(raw * raw, red));
  embed[u] = raw / nrm;
}

// EmotionEncoder.forward's tail: e = relu(W h + b) [E], e / ||e||_2.  One block per row; W [E][256] row-major.
__global__ void __launch_bounds__(kTailThreads) emo_linear_norm_kernel(const float* __restrict__ h, const float* __restrict__ W,
                                                                       const float* __restrict__ bias, int E, float* __restrict__ out) {
  extern __shared__ float e[];                   // [E]
  __shared__ float x[kEmoH], red[32];
  const long n = blockIdx.x;
  for (int k = threadIdx.x; k < kEmoH; k += blockDim.x) x[k] = h[n * kEmoH + k];
  __syncthreads();
  float ss = 0.f;
  for (int o = threadIdx.x; o < E; o += blockDim.x) {
    const float4* w4 = reinterpret_cast<const float4*>(W + (size_t)o * kEmoH);
    float acc = 0.f;
#pragma unroll 8
    for (int k = 0; k < kEmoH / 4; ++k) {
      const float4 v = __ldg(w4 + k);
      acc = fmaf(v.x, x[4 * k], acc); acc = fmaf(v.y, x[4 * k + 1], acc);
      acc = fmaf(v.z, x[4 * k + 2], acc); acc = fmaf(v.w, x[4 * k + 3], acc);
    }
    const float r = fmaxf(acc + bias[o], 0.f);
    e[o] = r;
    ss += r * r;
  }
  const float nrm = sqrtf(emo_block_sum(ss, red));
  for (int o = threadIdx.x; o < E; o += blockDim.x) out[n * E + o] = e[o] / nrm;
}

// sequences per cluster: spread N over the clusters the device can hold at once, at most kLstmMaxB each
int lstm_group(int N) {
  static int max_clusters[64] = {};
  int dev = 0;
  AGPT_CUDA(cudaGetDevice(&dev));
  int& mc = max_clusters[dev < 64 ? dev : 0];
  if (dev >= 64 || mc == 0) {
    AGPT_CUDA(cudaFuncSetAttribute(emo_lstm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kLstmSmem));
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(kLstmCta, 1, 1);
    cfg.blockDim = dim3(kLstmThreads);
    cfg.dynamicSmemBytes = kLstmSmem;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = kLstmCta; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    int n = 0;
    AGPT_CUDA(cudaOccupancyMaxActiveClusters(&n, emo_lstm_kernel, &cfg));
    AGPT_CHECK(n >= 1, "lstm: the device cannot hold one 8-CTA cluster of 128 KB CTAs");
    mc = n;
  }
  return std::min(kLstmMaxB, cdiv(N, mc));
}

}  // namespace

// ---------------------------------------------------------------- launchers (also the unit tests' entry points)
void emo_mean_norm(const float* h, int N, float* embed, cudaStream_t st) {
  AGPT_CHECK(N >= 1, "mean_norm: N >= 1");
  emo_mean_norm_kernel<<<1, kEmoH, 0, st>>>(h, N, embed);
  count_launch(1);
}

void emo_linear_norm(const float* h, const float* W, const float* bias, int N, int E, float* out, cudaStream_t st) {
  AGPT_CHECK(E >= 1 && N >= 1, "linear_norm: E >= 1 and N >= 1");
  AGPT_CHECK(sizeof(float) * ((size_t)E + kEmoH + 32) <= 48 * 1024,
             "linear_norm: E floats of dynamic shared memory exceed the 48 KB a launch allows");
  emo_linear_norm_kernel<<<(unsigned)N, kTailThreads, sizeof(float) * E, st>>>(h, W, bias, E, out);
  count_launch(1);
}

void emo_powmel(const float* spec, int pitch, const float* melW, float* mel, long frames, cudaStream_t st) {
  AGPT_CHECK(frames >= 1 && pitch >= 2 * kBins, "power mel: bad sizes");
  emo_powmel_kernel<<<(unsigned)frames, kMelThreads, 0, st>>>(spec, pitch, melW, mel);
  count_launch(1);
}

void emo_lstm(const float* whh, const float* xp, int N, int T, long seq_stride, float* h_seq, float* h_last, cudaStream_t st) {
  AGPT_CHECK(N >= 1 && T >= 1, "lstm: empty input");
  AGPT_CHECK(seq_stride >= 0, "lstm: negative sequence stride");
  AGPT_CHECK(h_seq || h_last, "lstm: no output");
  const int nb = lstm_group(N);
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(kLstmCta, 1, cdiv(N, nb));
  cfg.blockDim = dim3(kLstmThreads);
  cfg.dynamicSmemBytes = kLstmSmem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = kLstmCta; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, emo_lstm_kernel, whh, xp, N, T, seq_stride, nb, h_seq, h_last);
  if (e != cudaSuccess) throw Error(std::string("lstm: the 8-CTA cluster launch was refused: ") + cudaGetErrorString(e));
  count_launch(1);
}

// compute_partial_slices(n_samples, partial_frames, min_pad_coverage, overlap) (inference.py:59-108) in frames of 160
// samples: the partial count, the frame step and the length the wav is zero-padded to (wav_slices[-1].stop when that
// is at least n_samples, else n_samples itself).  np.round rounds half to even, as nearbyint does by default.
void emo_partials(long n_samples, int partial_frames, double min_pad_coverage, double overlap, int* n_partials, int* frame_step,
                  long* padded) {
  AGPT_CHECK(n_samples >= 0 && partial_frames >= 1, "partials: bad sizes");
  AGPT_CHECK(overlap >= 0.0 && overlap < 1.0, "partials: overlap must be in [0, 1)");
  AGPT_CHECK(min_pad_coverage > 0.0 && min_pad_coverage <= 1.0, "partials: min_pad_coverage must be in (0, 1]");
  const long n_frames = (n_samples + 1 + kHop - 1) / kHop;
  const long step = std::max(1L, (long)std::nearbyint(partial_frames * (1.0 - overlap)));
  const long steps = std::max(1L, n_frames - partial_frames + step + 1);
  long n = (steps + step - 1) / step;
  const long last = (n - 1) * step * kHop;
  const double coverage = (double)(n_samples - last) / (double)((long)partial_frames * kHop);
  if (coverage < min_pad_coverage && n > 1) --n;
  AGPT_CHECK(n <= (1 << 20), "partials: too many");
  *n_partials = (int)n;
  *frame_step = (int)step;
  *padded = std::max(n_samples, ((n - 1) * step + partial_frames) * kHop);
}

namespace {

struct EmoNet : Handle {
  agpt_emo_cfg cfg;
  PackedConv dft;
  std::vector<PackedConv> wih;
  std::vector<DevBuf> whh;
  DevBuf melW, linw, linb;
  DevBuf wav, frames, spec, mel, xp, hsa, hsb, last;

  void linear(const PackedConv& pc, const float* in, float* out, long rows, cudaStream_t st) {
    TapConvParams P = tapconv_params(pc, 1, (int)rows, 0, 1);
    P.in = in; P.in_pitch = pc.Cin;
    P.out = out; P.out_pitch = pc.Cout;
    P.epi = EPI_BIAS;
    tapconv_launch(P, st);
  }

  // x [clip] (device, at least 201 samples) -> mel [clip / 160 + 1][40]
  void mel_of(const float* x, long clip, float* out, cudaStream_t st) {
    AGPT_CHECK(clip > kNfft / 2, "the wav must have at least n_fft / 2 + 1 = 201 samples (reflect padding)");
    AGPT_CHECK(clip < (1L << 31), "the wav is too long");
    const int F = (int)(clip / kHop) + 1;
    frames.ensure((size_t)F * kNfft);
    cnn14_frames(x, (int)clip, 1, kHop, kNfft, frames.p, st);
    AGPT_CUDA(cudaGetLastError());
    spec.ensure((size_t)F * dft.cout_pad);
    TapConvParams P = tapconv_params(dft, 1, F, 0, 1);
    P.in = frames.p; P.in_pitch = kNfft;
    P.out = spec.p; P.out_pitch = dft.cout_pad;
    P.epi = EPI_BIAS;
    tapconv_launch(P, st);
    emo_powmel(spec.p, dft.cout_pad, melW.p, out, F, st);
    AGPT_CUDA(cudaGetLastError());
  }

  // the LSTM stack over N sequences of T steps whose layer-0 inputs are rows n * in_stride + t of x [.][40]; the last
  // layer's final h -> out [N][256]
  void stack(const float* x, long in_rows, long in_stride, int N, int T, float* out, cudaStream_t st) {
    const size_t rows = (size_t)N * T;
    xp.ensure(std::max<size_t>(rows, (size_t)in_rows) * kGates);
    const int L = cfg.num_layers;
    if (L > 1) { hsa.ensure(rows * kEmoH); if (L > 2) hsb.ensure(rows * kEmoH); }
    linear(wih[0], x, xp.p, in_rows, st);
    const float* in = nullptr;
    for (int l = 0; l < L; ++l) {
      if (l > 0) linear(wih[l], in, xp.p, (long)rows, st);
      float* seq = l + 1 < L ? (l % 2 == 0 ? hsa.p : hsb.p) : nullptr;
      emo_lstm(whh[l].p, xp.p, N, T, l == 0 ? in_stride : T, seq, l + 1 < L ? nullptr : out, st);
      in = seq;
    }
  }

  void hidden(const float* x, int N, int T, float* out, cudaStream_t st) {
    AGPT_CHECK(N >= 1 && T >= 1, "empty batch");
    AGPT_CHECK((long)N * T < (1L << 31), "too many frames");
    stack(x, (long)N * T, T, N, T, out, st);
  }

  void forward(const float* x, int N, int T, float* out, cudaStream_t st) {
    last.ensure((size_t)N * kEmoH);
    hidden(x, N, T, last.p, st);
    const int E = cfg.embedding_size;
    emo_linear_norm(last.p, linw.p, linb.p, N, E, out, st);
    AGPT_CUDA(cudaGetLastError());
  }

  void embed(const float* x, long n, int partial_frames, double cover, double overlap, float* out, float* partials, cudaStream_t st) {
    AGPT_CHECK(n >= 1, "empty wav");
    if (partial_frames == 0) {   // using_partials=False: the whole mel as one sequence
      const int F = (int)(n / kHop) + 1;
      mel.ensure((size_t)F * kMels);
      mel_of(x, n, mel.p, st);
      last.ensure(kEmoH);
      hidden(mel.p, 1, F, last.p, st);
      AGPT_CUDA(cudaMemcpyAsync(out, last.p, sizeof(float) * kEmoH, cudaMemcpyDeviceToDevice, st));
      return;
    }
    int N = 0, step = 0;
    long padded = 0;
    emo_partials(n, partial_frames, cover, overlap, &N, &step, &padded);
    wav.ensure((size_t)padded);
    AGPT_CUDA(cudaMemcpyAsync(wav.p, x, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
    if (padded > n) AGPT_CUDA(cudaMemsetAsync(wav.p + n, 0, sizeof(float) * (padded - n), st));
    const int F = (int)(padded / kHop) + 1;
    const long used = (long)(N - 1) * step + partial_frames;   // the mel frames the partials cover
    AGPT_CHECK(used <= F, "partials: a slice runs past the mel");
    mel.ensure((size_t)F * kMels);
    mel_of(wav.p, padded, mel.p, st);
    float* h = partials;
    if (!h) { last.ensure((size_t)N * kEmoH); h = last.p; }
    stack(mel.p, used, step, N, partial_frames, h, st);
    emo_mean_norm(h, N, out, st);
    AGPT_CUDA(cudaGetLastError());
  }
};

}  // namespace

Handle* emo_create(const agpt_emo_cfg* cfg, const float* const* Wt, int nW, int device) {
  DeviceGuard dg_(device);
  AGPT_CHECK(cfg->input_size == kMels, "EmotionEncoder: input_size must be 40 (mel_n_channels)");
  AGPT_CHECK(cfg->hidden_size == kEmoH, "EmotionEncoder: hidden_size must be 256");
  AGPT_CHECK(cfg->num_layers >= 1 && cfg->num_layers <= 16, "EmotionEncoder: num_layers must be in [1, 16]");
  AGPT_CHECK(cfg->embedding_size >= 1 && cfg->embedding_size <= 4096, "EmotionEncoder: embedding_size must be in [1, 4096]");
  std::unique_ptr<EmoNet> h(new EmoNet());
  h->magic = kMagicEmo; h->device = device; h->cfg = *cfg;
  WeightCursor wc{Wt, nW};
  h->wih.resize(cfg->num_layers);
  h->whh.resize(cfg->num_layers);
  for (int l = 0; l < cfg->num_layers; ++l) {
    const float* wi = wc.next(); const float* wh = wc.next(); const float* b = wc.next();
    // K = 40 already meets the tap-GEMM's channel granularity (a multiple of 8, 16-byte rows), so no zero columns
    pack_conv(h->wih[l], wi, b, kGates, l == 0 ? kMels : kEmoH, 1, false);
    h->whh[l].upload(wh, (size_t)kGates * kEmoH);
  }
  h->linw.upload(wc.next(), (size_t)cfg->embedding_size * kEmoH);
  h->linb.upload(wc.next(), cfg->embedding_size);
  {  // the DFT rows (real | imaginary) as one [400] -> [402] 1-tap GEMM
    const float* re = wc.next(); const float* im = wc.next();
    std::vector<float> w((size_t)2 * kBins * kNfft);
    memcpy(w.data(), re, sizeof(float) * kBins * kNfft);
    memcpy(w.data() + (size_t)kBins * kNfft, im, sizeof(float) * kBins * kNfft);
    pack_conv(h->dft, w.data(), nullptr, 2 * kBins, kNfft, 1, false);
  }
  h->melW.upload(wc.next(), (size_t)kBins * kMels);
  wc.done();
  return h.release();
}

void emo_mel(Handle* hh, const float* wav, long n, float* mel, cudaStream_t st) {
  auto* h = static_cast<EmoNet*>(hh);
  DeviceGuard dg_(h->device);
  h->mel_of(wav, n, mel, st);
}

void emo_hidden(Handle* hh, const float* frames, int N, int T, float* hidden, cudaStream_t st) {
  auto* h = static_cast<EmoNet*>(hh);
  DeviceGuard dg_(h->device);
  h->hidden(frames, N, T, hidden, st);
}

void emo_forward(Handle* hh, const float* frames, int N, int T, float* embeds, cudaStream_t st) {
  auto* h = static_cast<EmoNet*>(hh);
  DeviceGuard dg_(h->device);
  h->forward(frames, N, T, embeds, st);
}

void emo_embed(Handle* hh, const float* wav, long n, int partial_frames, double min_pad_coverage, double overlap, float* embed,
               float* partials, cudaStream_t st) {
  auto* h = static_cast<EmoNet*>(hh);
  DeviceGuard dg_(h->device);
  AGPT_CHECK(partial_frames >= 0, "partial_frames must be >= 0 (0: the whole utterance as one sequence)");
  h->embed(wav, n, partial_frames, min_pad_coverage, overlap, embed, partials, st);
}

}  // namespace agpt
