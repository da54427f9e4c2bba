// The torchlibrosa log-mel front end shared by Cnn14 (clap_score.cu) and the sound-event-detection PVT (pvt.cu):
// Spectrogram(n_fft = win = n, hop, periodic Hann, center + reflect, power 2) -> LogmelFilterBank(ref 1, amin 1e-10, no
// top_db) -> bn0 (eval BatchNorm over the mel axis).  Reflect-padded framing, one 1-tap tap-GEMM against the
// checkpoint's DFT rows, then one fused fp32 kernel per frame.
#pragma once
#include "common.cuh"
#include "tapconv.cuh"
#include "models.h"

namespace agpt {

// frames[b][t][j] = x_b[reflect(t * hop + j - n / 2)]  (center=True, pad_mode='reflect')
static __global__ void cnn14_frames_kernel(const float* __restrict__ x, int clip, int T, int hop, int n, float* __restrict__ fr, long total) {
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
// bin) -> CH == 4: img[b][t][m][0..3] (Cnn14's first conv reads a 4-channel padded input); CH == 1: img[b][t][m]
template <int CH>
static __global__ void cnn14_logmel_kernel(const float* __restrict__ spec, int pitch, int nb, const float* __restrict__ melW,
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
    const float v = db * bn_s[m] + bn_t[m];
    if constexpr (CH == 4) *reinterpret_cast<float4*>(img + (f * nm + m) * 4) = make_float4(v, 0.f, 0.f, 0.f);
    else img[f * nm + m] = v;
  }
}

struct LogmelFront {
  PackedConv dft;
  DevBuf melW, bn0_s, bn0_t, frames, spec;
  int n = 0, hop = 0, nm = 0;

  // consumes conv_real.weight, conv_imag.weight [n / 2 + 1][1][n], melW [n / 2 + 1][nm], bn0 weight / bias / running_mean
  // / running_var [nm]
  void load(WeightCursor& wc, int n_, int hop_, int nm_, float bn_eps) {
    n = n_; hop = hop_; nm = nm_;
    const int nb = n / 2 + 1;
    {  // conv_real / conv_imag -> one [n] -> [re | im] 1-tap GEMM
      const float* re = wc.next(); const float* im = wc.next();
      std::vector<float> w((size_t)2 * nb * n);
      memcpy(w.data(), re, sizeof(float) * nb * n);
      memcpy(w.data() + (size_t)nb * n, im, sizeof(float) * nb * n);
      pack_conv(dft, w.data(), nullptr, 2 * nb, n, 1, false);
    }
    melW.upload(wc.next(), (size_t)nb * nm);
    const float* g = wc.next(); const float* be = wc.next(); const float* rm = wc.next(); const float* rv = wc.next();
    std::vector<float> s(nm), t(nm);
    for (int m = 0; m < nm; ++m) { s[m] = g[m] / sqrtf(rv[m] + bn_eps); t[m] = be[m] - rm[m] * s[m]; }
    bn0_s.upload(s); bn0_t.upload(t);
  }

  static int frames_of(long clip, int hop) { return (int)(clip / hop) + 1; }

  // wav [B][clip] (device) -> img [B][T][nm][CH], T = clip / hop + 1; clip > n / 2 (reflect padding)
  template <int CH>
  void run(const float* wav, int clip, int B, float* img, cudaStream_t st) {
    const int nb = n / 2 + 1, T = frames_of(clip, hop);
    const long tot = (long)B * T * n;
    frames.ensure((size_t)tot);
    cnn14_frames_kernel<<<(unsigned)std::min<long>(cdivl(tot, 256), 4096), 256, 0, st>>>(wav, clip, T, hop, n, frames.p, tot);
    count_launch(1);
    spec.ensure((size_t)B * T * dft.cout_pad);
    TapConvParams P = tapconv_params(dft, 1, B * T, 0, 1);
    P.in = frames.p; P.in_pitch = n;
    P.out = spec.p; P.out_pitch = dft.cout_pad;
    P.epi = EPI_BIAS;
    tapconv_launch(P, st);
    cnn14_logmel_kernel<CH><<<(unsigned)(B * T), 64, sizeof(float) * nb, st>>>(spec.p, dft.cout_pad, nb, melW.p, nm, bn0_s.p, bn0_t.p, img);
    count_launch(1);
  }
};

}  // namespace agpt
