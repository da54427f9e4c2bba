// The PANNs ConvBlock on the tap-GEMM, shared by the CLAP scorer's Cnn14 (clap_score.cu) and the target-sound-detection
// RaDur_fusion (tsd.cu): 3x3 conv (padding 1, no bias) -> eval BatchNorm2d folded into the weights -> ReLU, on
// channels-last images [B][H][W][C].
#pragma once
#include <vector>
#include "common.cuh"
#include "tapconv.cuh"

namespace agpt {

// out = relu(conv3x3(in) + b'): one 9-tap launch over the [H][W] grid of every sample
inline void conv3x3_relu(const PackedConv& pc, const float* in, float* out, int B, int H, int W, cudaStream_t st) {
  TapConvParams P = tapconv_params(pc, B, H * W, W, 1);
  P.in = in; P.in_gstride = (long)H * W * pc.Cin; P.in_pitch = pc.Cin;
  P.out = out; P.out_gstride = (long)H * W * pc.Cout; P.out_pitch = pc.Cout;
  P.epi = EPI_RELU;
  tapconv_launch(P, st);
}

// BatchNorm2d (eval) folded into the preceding bias-free conv: w' = w * s, b' = beta - mean * s, s = gamma / sqrt(var + eps).
// Consumes the BatchNorm's weight, bias, running_mean, running_var from the cursor; cin_pad >= cin input channels are
// packed (the extra ones zero).
inline void load_conv_bn(PackedConv& pc, const float* w, WeightCursor& wc, int cout, int cin, int cin_pad, float eps) {
  const float* g = wc.next(); const float* be = wc.next(); const float* rm = wc.next(); const float* rv = wc.next();
  std::vector<float> wf((size_t)cout * cin_pad * 9, 0.f), bf(cout);
  for (int co = 0; co < cout; ++co) {
    const float s = g[co] / sqrtf(rv[co] + eps);
    bf[co] = be[co] - rm[co] * s;
    for (int ci = 0; ci < cin; ++ci)
      for (int k = 0; k < 9; ++k) wf[((size_t)co * cin_pad + ci) * 9 + k] = w[((size_t)co * cin + ci) * 9 + k] * s;
  }
  pack_conv(pc, wf.data(), bf.data(), cout, cin_pad, 9, true);
}

}  // namespace agpt
