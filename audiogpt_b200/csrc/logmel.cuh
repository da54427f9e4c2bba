// The torchlibrosa log-mel front end shared by Cnn14 (clap_score.cu) and the sound-event-detection PVT (pvt.cu):
// Spectrogram(n_fft = win = n, hop, periodic Hann, center + reflect, power 2) -> LogmelFilterBank(ref 1, amin 1e-10, no
// top_db) -> bn0 (eval BatchNorm over the mel axis).  Reflect-padded framing, one 1-tap tap-GEMM against the
// checkpoint's DFT rows, then one fused fp32 kernel per frame (cnn14_frames / cnn14_logmel, clap_score.cu).
#pragma once
#include "common.cuh"
#include "tapconv.cuh"
#include "models.h"
#include "audio_front.cuh"

namespace agpt {

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
    frames.ensure((size_t)B * T * n);
    cnn14_frames(wav, clip, B, hop, n, frames.p, st);
    spec.ensure((size_t)B * T * dft.cout_pad);
    TapConvParams P = tapconv_params(dft, 1, B * T, 0, 1);
    P.in = frames.p; P.in_pitch = n;
    P.out = spec.p; P.out_pitch = dft.cout_pad;
    P.epi = EPI_BIAS;
    tapconv_launch(P, st);
    cnn14_logmel(spec.p, dft.cout_pad, nb, melW.p, nm, bn0_s.p, bn0_t.p, img, (long)B * T, CH, st);
  }
};

}  // namespace agpt
