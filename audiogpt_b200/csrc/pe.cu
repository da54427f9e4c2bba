// PitchExtractor on sm_90a: mel [B][T][80] -> (pitch_pred [B][T][2], f0_denorm_pred [B][T]) -- the network that
// recovers F0 from a generated mel-spectrogram for the NSF vocoder on the text-to-singing path.
// Reference: NeuralSeq/modules/fastspeech/pe.py:119-148 (PitchExtractor), :7-42 (Prenet), :44-116 (ConvBlock /
// ConvStacks), modules/fastspeech/tts_modules.py:217-260 (PitchPredictor), modules/commons/common_layers.py:87-142
// (SinusoidalPositionalEmbedding), utils/__init__.py:145-157 (make_positions), utils/pitch_utils.py:63-76 (denorm_f0).
// The mel is already channels-last; every Conv1d / Linear is a tap-GEMM on the tensor-core kernel, BatchNorm1d (eval) is
// a per-channel affine fused with the non-padding mask, GroupNorm + ReLU + residual is one gn_fused launch.
// Parity: tests/test_pe_gpu.py against tests/golden/pe_{small,base}.npz (made by the reference module) and oracle/pe_ref.py.
#include "common.cuh"
#include "tapconv.cuh"
#include "nn_kernels.h"
#include "models.h"
#include "fs_layers.cuh"

namespace agpt {

// mask[b*T + t] = 1 if the frame has any non-zero bin  (pe.py:29: x.abs().sum(-1).eq(0) is the PADDING mask)
__global__ void pe_mask_kernel(const float* __restrict__ mel, float* __restrict__ mask, long rows, int M) {
  const long r = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  float s = 0.f;
  for (int c = lane; c < M; c += 32) s += fabsf(mel[r * M + c]);
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) mask[r] = s == 0.f ? 0.f : 1.f;
}
// pred4 [rows][4] (channels 0, 1 used) -> pitch_pred [rows][2], f0 [rows] = denorm_f0(pred[..., 0], pred[..., 1] > 0, padding)
__global__ void pe_denorm_kernel(const float* __restrict__ pred4, const float* __restrict__ mask, float* __restrict__ pitch_pred,
                                 float* __restrict__ f0, long rows, int use_uv, int norm_mode, float f0_mean, float f0_std) {
  for (long r = (long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long)gridDim.x * blockDim.x) {
    const float p0 = pred4[r * 4], p1 = pred4[r * 4 + 1];
    pitch_pred[r * 2] = p0; pitch_pred[r * 2 + 1] = p1;
    float v = p0;
    v = denorm(v, norm_mode, f0_mean, f0_std);
    if (use_uv && p1 > 0.f) v = 0.f;
    if (mask[r] == 0.f) v = 0.f;
    f0[r] = v;
  }
}

void pe_mask(const float* mel, float* mask, long rows, int M, cudaStream_t st) {
  pe_mask_kernel<<<(unsigned)cdivl(rows, 8), 256, 0, st>>>(mel, mask, rows, M);
  count_launch(1);
}

void pe_denorm(const float* pred4, const float* mask, float* pitch_pred, float* f0, long rows, int use_uv, int norm, float mean,
               float std_, cudaStream_t st) {
  pe_denorm_kernel<<<(unsigned)std::min<long>(cdivl(rows, 256), 1184), 256, 0, st>>>(pred4, mask, pitch_pred, f0, rows, use_uv, norm, mean,
                                                                                  std_);
  count_launch(1);
}

struct PeNet : Handle {
  agpt_pe_cfg cfg;
  PackedConv pre_conv[3], pre_out, enc_in, enc_out;
  DevBuf bn_a[3], bn_b[3];
  std::vector<PackedConv> enc_conv;
  std::vector<DevBuf> enc_g, enc_b;
  PitchPredictorNet pp;
  DevBuf mask, buf[4], pred4;

  void forward(const float* mel, int B, int T, float* pitch_pred, float* f0, int use_uv, int norm_mode, float f0_mean, float f0_std,
               cudaStream_t st) {
    AGPT_CHECK(B >= 1 && T >= 1, "empty batch");
    const int H = cfg.hidden_size, P_ = cfg.predictor_hidden, M = cfg.n_mel_bins;
    const long rows = (long)B * T;
    const int Cmax = std::max(H, P_);
    mask.ensure(rows); pred4.ensure(rows * 4);
    for (auto& b : buf) b.ensure((size_t)rows * Cmax);
    float *x = buf[0].p, *y = buf[1].p, *z = buf[2].p;
    pe_mask(mel, mask.p, rows, M, st);
    // ---- Prenet (pe.py:23-42): 3 x [Conv1d k5 -> ReLU -> BatchNorm1d(eval) -> x mask], out_proj, x mask
    const float* in = mel;
    int cin = M;
    for (int l = 0; l < 3; ++l) {
      fs_conv(pre_conv[l], in, cin, x, H, B, T, EPI_RELU, st);
      fs_affine_mask(x, bn_a[l].p, bn_b[l].p, mask.p, rows, H, st);
      std::swap(x, y);
      in = y; cin = H;
    }
    fs_conv(pre_out, in, H, x, H, 1, (int)rows, EPI_BIAS, st);
    fs_affine_mask(x, nullptr, nullptr, mask.p, rows, H, st);
    // ---- ConvStacks (pe.py:98-116): in_proj, n x [x + ReLU(GroupNorm(C/16 groups)(ConvNorm k5 (x)))], out_proj
    if (!enc_conv.empty()) {
      fs_conv(enc_in, x, H, y, H, 1, (int)rows, EPI_BIAS, st);
      std::swap(x, y);
      for (size_t l = 0; l < enc_conv.size(); ++l) {
        fs_conv(enc_conv[l], x, H, y, H, B, T, EPI_BIAS, st);
        groupnorm_ex(y, z, enc_g[l].p, enc_b[l].p, B, T, H, H / 16, 1e-5f, 2, x, st);
        std::swap(x, z);
      }
      fs_conv(enc_out, x, H, y, H, 1, (int)rows, EPI_BIAS, st);
      std::swap(x, y);
    }
    // ---- PitchPredictor (tts_modules.py:247-260)
    pp.forward(x, H, B, T, y, z, buf[3].p, pred4.p, st);
    pe_denorm(pred4.p, mask.p, pitch_pred, f0, rows, use_uv, norm_mode, f0_mean, f0_std, st);
    AGPT_CUDA(cudaGetLastError());
  }
};

Handle* pe_create(const agpt_pe_cfg* cfg, const float* const* W, int nW, int device) {
  DeviceGuard dg_(device);
  const int H = cfg->hidden_size, M = cfg->n_mel_bins, P = cfg->predictor_hidden, k = cfg->predictor_kernel;
  AGPT_CHECK(H % 16 == 0 && P % 4 == 0 && M % 4 == 0 && k % 2 == 1 && k <= kMaxTaps, "bad PitchExtractor config");
  std::unique_ptr<PeNet> h(new PeNet());
  h->magic = kMagicPe; h->device = device; h->cfg = *cfg;
  WeightCursor wc{W, nW};
  int cin = M;
  for (int l = 0; l < 3; ++l) {
    auto w = wc.next(); auto b = wc.next();
    pack_conv(h->pre_conv[l], w, b, H, cin, 5, false);
    auto g = wc.next(); auto be = wc.next(); auto mu = wc.next(); auto var = wc.next();
    wc.next();                            // num_batches_tracked
    std::vector<float> a(H), bb(H);
    for (int c = 0; c < H; ++c) {      // BatchNorm1d eval: (x - mean) / sqrt(var + eps) * gamma + beta, eps = 1e-5
      a[c] = g[c] / std::sqrt(var[c] + 1e-5f);
      bb[c] = be[c] - mu[c] * a[c];
    }
    h->bn_a[l].upload(a); h->bn_b[l].upload(bb);
    cin = H;
  }
  { auto w = wc.next(); auto b = wc.next(); pack_conv(h->pre_out, w, b, H, H, 1, false); }
  h->enc_conv.resize(cfg->conv_layers); h->enc_g.resize(cfg->conv_layers); h->enc_b.resize(cfg->conv_layers);
  for (int l = 0; l < cfg->conv_layers; ++l) {
    { auto w = wc.next(); auto b = wc.next(); pack_conv(h->enc_conv[l], w, b, H, H, 5, false); }
    { auto g = wc.next(); auto b = wc.next(); h->enc_g[l].upload(g, H); h->enc_b[l].upload(b, H); }
  }
  if (cfg->conv_layers > 0) {
    { auto w = wc.next(); auto b = wc.next(); pack_conv(h->enc_in, w, b, H, H, 1, false); }
    { auto w = wc.next(); auto b = wc.next(); pack_conv(h->enc_out, w, b, H, H, 1, false); }
  }
  h->pp.load(wc, H, P, k, cfg->predictor_layers, 2);
  wc.done();
  return h.release();
}

void pe_forward(Handle* hh, const float* mel, int B, int T, float* pitch_pred, float* f0, int use_uv, int norm_mode,
                float f0_mean, float f0_std, cudaStream_t st) {
  auto* h = static_cast<PeNet*>(hh);
  DeviceGuard dg_(h->device);
  h->forward(mel, B, T, pitch_pred, f0, use_uv, norm_mode, f0_mean, f0_std, st);
}

}  // namespace agpt
