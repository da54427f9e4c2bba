// Layers shared by the FastSpeech-family drivers (pe.cu: PitchExtractor, fs2.cu: FastSpeech2 / FastSpeech2MIDI,
// generspeech.cu: GenerSpeech).
// Activations are channels-last rows [B][T][C].
#pragma once
#include <vector>
#include "common.cuh"
#include "tapconv.cuh"

namespace agpt {

// utils/pitch_utils.py:22-32 f0_to_coarse, in the fp32 operation order torch applies (numpy constants rounded to fp32)
__device__ __forceinline__ int f0_coarse(float f0, float mel_min, float mel_range) {
  float m = __fmul_rn(1127.f, logf(__fadd_rn(1.f, __fdiv_rn(f0, 700.f))));
  if (m > 0.f) m = __fadd_rn(__fdiv_rn(__fmul_rn(__fsub_rn(m, mel_min), 254.f), mel_range), 1.f);
  if (m <= 1.f) m = 1.f;
  if (m > 255.f) m = 255.f;
  return (int)(m + 0.5f);
}
__device__ __forceinline__ float denorm(float f, int norm, float mean, float std_) {
  if (norm == 1) f = f * std_ + mean;      // 'standard'
  if (norm == 2) f = exp2f(f);             // 'log': 2 ** f0
  return f;
}

constexpr int kRelMaxLen = 5000;    // RelPositionalEncoding's table length (positions run backwards from max_len - 1)

// Token embedding + encoder positions + source masks (see fs_embed_tokens_kernel in fs_layers.cu); the MIDI inputs may be null
void fs_embed_tokens(const int* tok, const int* pmidi, const float* mdur, const int* slur, const float* E, const float* midiE,
                     const float* mdw, const float* mdb, const float* slurE, int ntok, float escale, int pos_mode, const float* rel_div,
                     float neg_emb, float xscale, float* x, float* nonpad, uint8_t* kpm, int B, int T, int H, cudaStream_t st);
// FFTBlocks' padding mask from the rows themselves: nonpad[r] = any(x[r] != 0), kpm[r] = !nonpad[r]
void fs_rowmask(const float* x, float* nonpad, uint8_t* kpm, long rows, int C, cudaStream_t st);
// DurationPredictor.inference: dur[r] = pred4[r][0] * nonpad[r]; dch (may be null) = clamp(round(exp(dur) - 1), 0)
void fs_dur(const float* pred4, const float* nonpad, float* dur, int* dch, long rows, cudaStream_t st);
// LengthRegulator: per-utterance cumsum of dch -> cum, mel_len[b]; then mel2ph [B][Tm] from them
void fs_lr_scan(const int* dch, int* cum, int* mel_len, int B, int T, cudaStream_t st);
void fs_lr_fill(const int* cum, const int* mel_len, int* mel2ph, int B, int Tt, int Tm, cudaStream_t st);
// expand_states: out = gather(pad(enc, 1 leading zero row), mel2ph) [B][Tm][H]; tgt = mel2ph > 0
void fs_gather(const float* enc, const int* mel2ph, float* out, float* tgt, int B, int Tt, int Tm, int H, cudaStream_t st);

// EncSALayer (common_layers.py:541-587), norm 'ln', act 'gelu', padding 'SAME'
struct FftLayer {
  DevBuf ln1g, ln1b, ln2g, ln2b;
  PackedConv qkv, out, ffn1, ffn2;
  int k = 9;
};
struct FftStack {
  std::vector<FftLayer> layers;
  DevBuf lng, lnb;
  // consumes L x (layer_norm1, in_proj_weight, out_proj.weight, layer_norm2, ffn_1, ffn_2), then the last layer_norm
  void load(WeightCursor& wc, int H, int L, int k);
  // FFTBlocks.forward after the input positions (tts_modules.py:307-332): x * nonpad, layers, last LayerNorm * nonpad.
  // xs [B*T][H] is overwritten; the result goes to out (which may be y).  Scratch: y, z [B*T][H], qkv [B*T][3H],
  // ffn [B*T][4H].
  void forward(float* xs, float* out, int B, int T, int H, int heads, const float* nonpad, const uint8_t* kpm, float* y, float* z,
               float* qkv, float* ffn, cudaStream_t st) const;
};

// DurationPredictor (tts_modules.py:98-112): n x [conv k SAME -> ReLU -> LayerNorm -> x nonpad], Linear -> 1 (padded to 4)
struct DurPredictorNet {
  std::vector<PackedConv> conv;
  std::vector<DevBuf> g, b;
  PackedConv lin;
  int P = 0;
  void load(WeightCursor& wc, int H, int P_, int k, int layers);
  // x [B][T][H] (read only) -> pred4 [B][T][4]; s0 / s1 / s2: scratch of B*T*max(H, P) floats
  void forward(const float* x, int H, int B, int T, const float* nonpad, float* s0, float* s1, float* s2, float* pred4,
               cudaStream_t st) const;
};

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
