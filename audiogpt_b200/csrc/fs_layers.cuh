// Layers shared by the FastSpeech-family drivers (pe.cu: PitchExtractor, fs2.cu: FastSpeech2 / FastSpeech2MIDI).
// Activations are channels-last rows [B][T][C].
#pragma once
#include <vector>
#include "common.cuh"
#include "tapconv.cuh"

namespace agpt {

// One Conv1d ("same" zero padding per utterance) or Linear (1 tap) of a [B][T][cin] tensor on the tap-GEMM.
void fs_conv(const PackedConv& pc, const float* in, int cin, float* out, int cout_pitch, int B, int T, int epi,
             cudaStream_t st, const float* res = nullptr, float scale = 1.f);
// x[r][c] = (x[r][c] * a[c] + b[c]) * mask[r]; a / b may be null (then x *= mask)
void fs_affine_mask(float* x, const float* a, const float* b, const float* mask, long rows, int C, cudaStream_t st);
// fairseq make_positions on x[..., 0] with padding_idx 0: pos = cumsum(x[..., 0] != 0) * (x[..., 0] != 0)
// (x is [B][T][C]; one sequential scan per utterance)
void fs_positions(const float* x, int* pos, int B, int T, int C, cudaStream_t st);
// out = in + alpha * SinusoidalPositionalEmbedding(pos) (sin || cos halves, (C/2 - 1) divisor, row 0 = 0); out may be in
void fs_posemb_add(const float* in, float* out, const int* pos, float alpha, long rows, int C, cudaStream_t st);

// PitchPredictor / EnergyPredictor (NeuralSeq/modules/fastspeech/tts_modules.py:217-264): + alpha * positions of
// x[..., 0], n x [Conv1d k SAME -> ReLU -> LayerNorm over channels], Linear -> odim (padded to 4 output channels).
struct PitchPredictorNet {
  std::vector<PackedConv> conv;
  std::vector<DevBuf> g, b;
  PackedConv lin;
  float alpha = 1.f;
  int P = 0;
  DevBuf pos;
  // consumes, in state-dict order: pos_embed_alpha, conv.{l}.1.weight / .bias, conv.{l}.3.weight / .bias, linear.weight /
  // .bias, embed_positions._float_tensor
  void load(WeightCursor& wc, int H, int P_, int k, int layers, int odim);
  // x [B][T][H] (read only) -> pred4 [B][T][4] (channels >= odim are zero); s0 / s1 / s2: scratch of B*T*max(H, P) floats
  void forward(const float* x, int H, int B, int T, float* s0, float* s1, float* s2, float* pred4, cudaStream_t st);
};

}  // namespace agpt
