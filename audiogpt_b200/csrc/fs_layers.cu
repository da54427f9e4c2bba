// Layers shared by the FastSpeech-family drivers (fs_layers.cuh).
// Reference: NeuralSeq/modules/fastspeech/tts_modules.py:217-264 (PitchPredictor / EnergyPredictor),
// modules/commons/common_layers.py:87-142 (SinusoidalPositionalEmbedding), utils/__init__.py:145-157 (make_positions).
#include "fs_layers.cuh"
#include "models.h"
#include "nn_kernels.h"

namespace agpt {

__global__ void fs_affine_mask_kernel(float* __restrict__ x, const float* __restrict__ a, const float* __restrict__ b,
                                      const float* __restrict__ mask, long total, int C) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / C;
    const int c = (int)(i - r * C);
    float v = x[i];
    if (a) v = v * a[c] + b[c];
    x[i] = v * mask[r];
  }
}
__global__ void fs_positions_kernel(const float* __restrict__ x, int* __restrict__ pos, int T, int C) {
  if (threadIdx.x != 0) return;                       // one sequential scan per utterance (T <= a few thousand frames)
  const int b = blockIdx.x;
  int run = 0;
  for (int t = 0; t < T; ++t) {
    const bool nz = x[((long)b * T + t) * C] != 0.f;
    run += nz ? 1 : 0;
    pos[(long)b * T + t] = nz ? run : 0;
  }
}
__global__ void fs_posemb_add_kernel(const float* __restrict__ in, float* __restrict__ out, const int* __restrict__ pos, float alpha,
                                     long total, int C, float neg_emb) {
  const int half = C / 2;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / C;
    const int c = (int)(i - r * C);
    const int p = pos[r];
    float v = in[i];
    if (p != 0 && c < 2 * half) {                       // the padding row of the table is zero; odd dims pad with a zero column
      const int k = c < half ? c : c - half;
      const float a = (float)p * expf((float)k * neg_emb);
      v += alpha * (c < half ? sinf(a) : cosf(a));
    }
    out[i] = v;
  }
}

static unsigned ew_grid(long total) { return (unsigned)std::min<long>(cdivl(total, 256), 2368); }

void fs_conv(const PackedConv& pc, const float* in, int cin, float* out, int cout_pitch, int B, int T, int epi, cudaStream_t st,
             const float* res, float scale) {
  TapConvParams P = tapconv_params(pc, B, T, 0, 1);
  P.in = in; P.in_gstride = (long)T * cin; P.in_pitch = cin;
  P.out = out; P.out_gstride = (long)T * cout_pitch; P.out_pitch = cout_pitch;
  P.epi = epi;
  P.scale = scale;
  if (res) { P.res = res; P.res_gstride = (long)T * cout_pitch; P.res_pitch = cout_pitch; }
  tapconv_launch(P, st);
}

void fs_affine_mask(float* x, const float* a, const float* b, const float* mask, long rows, int C, cudaStream_t st) {
  fs_affine_mask_kernel<<<ew_grid(rows * C), 256, 0, st>>>(x, a, b, mask, rows * C, C);
  count_launch(1);
}

void fs_positions(const float* x, int* pos, int B, int T, int C, cudaStream_t st) {
  fs_positions_kernel<<<B, 32, 0, st>>>(x, pos, T, C);
  count_launch(1);
}

void fs_posemb_add(const float* in, float* out, const int* pos, float alpha, long rows, int C, cudaStream_t st) {
  const float neg_emb = (float)(-(std::log(10000.0) / (double)(C / 2 - 1)));
  fs_posemb_add_kernel<<<ew_grid(rows * C), 256, 0, st>>>(in, out, pos, alpha, rows * C, C, neg_emb);
  count_launch(1);
}

void PitchPredictorNet::load(WeightCursor& wc, int H, int P_, int k, int layers, int odim) {
  AGPT_CHECK(odim >= 1 && odim <= 4 && k % 2 == 1 && k <= kMaxTaps, "bad pitch predictor config");
  P = P_;
  alpha = wc.next()[0];
  conv.resize(layers); g.resize(layers); b.resize(layers);
  int cin = H;
  for (int l = 0; l < layers; ++l) {
    { auto w = wc.next(); auto bb = wc.next(); pack_conv(conv[l], w, bb, P, cin, k, false); }
    { auto gg = wc.next(); auto bb = wc.next(); g[l].upload(gg, P); b[l].upload(bb, P); }
    cin = P;
  }
  {  // Linear(P -> odim), padded to 4 output channels so that rows stay float4-addressable
    auto w = wc.next(); auto bb = wc.next();
    std::vector<float> wp((size_t)4 * P, 0.f), bp(4, 0.f);
    memcpy(wp.data(), w, sizeof(float) * odim * P);
    for (int i = 0; i < odim; ++i) bp[i] = bb[i];
    pack_conv(lin, wp.data(), bp.data(), 4, P, 1, false);
  }
  wc.next();                           // embed_positions._float_tensor (a device marker buffer)
}

void PitchPredictorNet::forward(const float* x, int H, int B, int T, float* s0, float* s1, float* s2, float* pred4, cudaStream_t st) {
  const long rows = (long)B * T;
  pos.ensure(rows);
  int* ipos = reinterpret_cast<int*>(pos.p);
  fs_positions(x, ipos, B, T, H, st);
  fs_posemb_add(x, s0, ipos, alpha, rows, H, st);
  float *cur = s0, *a = s1, *c = s2;
  int cin = H;
  for (size_t l = 0; l < conv.size(); ++l) {
    fs_conv(conv[l], cur, cin, a, P, B, T, EPI_RELU, st);
    layernorm(a, c, g[l].p, b[l].p, rows, P, 1e-5f, st);
    std::swap(cur, c);
    cin = P;
  }
  fs_conv(lin, cur, P, pred4, 4, 1, (int)rows, EPI_BIAS, st);
  AGPT_CUDA(cudaGetLastError());
}

}  // namespace agpt
