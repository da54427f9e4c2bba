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
// utils/pitch_utils.py denorm_f0: 'standard' rounds the product and the sum separately, as torch does (no FMA)
__device__ __forceinline__ float denorm(float f, int norm, float mean, float std_) {
  if (norm == 1) f = __fadd_rn(__fmul_rn(f, std_), mean);   // 'standard'
  if (norm == 2) f = exp2f(f);                              // 'log': 2 ** f0
  return f;
}
// f0_to_coarse's f0_mel_min and f0_mel_max - f0_mel_min (f0 in [50, 1100] Hz), computed in double and rounded to fp32
inline float f0_mel_min() { return (float)(1127.0 * std::log(1.0 + 50.0 / 700.0)); }
inline float f0_mel_range() { return (float)(1127.0 * std::log(1.0 + 1100.0 / 700.0) - 1127.0 * std::log(1.0 + 50.0 / 700.0)); }

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

// ---- the element-wise kernels of fs2.cu, generspeech.cu and pe.cu, one launch each (the drivers and agpt_fs_probe
// call these).  norm: 0 none, 1 'standard', 2 'log'.
// add_pitch 'frame': pitch_pred [rows][2], f0d (uv and mel2ph == 0 -> 0), coarse; f0_in / uv_in may be null (predicted)
void fs2_pitch_frame(const float* pred4, const int* mel2ph, const float* f0_in, const float* uv_in, int use_uv, int norm, float mean,
                     float std_, float* pitch_pred, float* f0d, int* coarse, long rows, cudaStream_t st);
// add_pitch 'ph': per token, no uv; pitch_pred [rows]
void fs2_pitch_ph(const float* pred4, const float* f0_in, int norm, float mean, float std_, float* pitch_pred, float* f0d, int* coarse,
                  long rows, cudaStream_t st);
// add_energy: e_pred = pred4[..., 0]; bucket = clamp(floor(e * 256 / 4), 0, 255) of e_in (or e_pred when null)
void fs2_energy(const float* pred4, const float* e_in, float* e_pred, int* bucket, long rows, cudaStream_t st);
// out = (x + pE[pitch bin] + eE[bucket]) * tgt; pitch bin from pframe [B*Tm] or (ptok [B*Tt] through mel2ph); pE / eE may be null
void fs2_embed_add(const float* x, const float* tgt, const float* pE, const int* pframe, const int* ptok, const int* mel2ph,
                   const float* eE, const int* ebucket, float* out, int Tt, int Tm, long rows, int H, cudaStream_t st);
// out[r] = (x[r] + a[b] + e[b] (+ tab[idx[r]]) (+ s[r])) * mask[r], b = r / T
void gs_sum(const float* x, const float* a, const float* e, const float* tab, const int* idx, const float* s, const float* mask, float* out,
            int T, long rows, int H, cudaStream_t st);
// dst (+)= src over n floats (first: dst = src)
void gs_accum(float* dst, const float* src, long n, int first, cudaStream_t st);
// mask[r] = mel[r][0] != 0 (mel rows of 80 bins)
void gs_refmask(const float* mel, float* mask, long rows, cudaStream_t st);
// acts [rows][C] = tanh(a[:, :C]) * sigmoid(a[:, C:]), a [rows][2C]
void gs_wn_gate(const float* a, float* acts, long rows, int C, cudaStream_t st);
// out [B][nseg][C] = mean of h [B][T][C] over the frames with seg == s + 1 (0 for an empty segment)
void gs_segmean(const float* h, const int* seg, float* out, int B, int T, int nseg, int C, cudaStream_t st);
// VQ argmin over M codes from dots [rows][M] = x . e_m, enorm [M] = |e_m|^2; idx (may be null), q = x + (e - x) (may alias x)
void gs_vq(const float* x, const float* dots, const float* emb, const float* enorm, int* idx, float* q, long rows, int H, int M,
           cudaStream_t st);
// out [rows][2H] = cat[p, SinusoidalPositionalEmbedding(pos)]
void gs_catpos(const float* p, const int* pos, float* out, long rows, int H, cudaStream_t st);
// kpm[r] = x[r][0] == 0
void gs_kpm(const float* x, uint8_t* kpm, long rows, int H, cudaStream_t st);
// inpaint_pitch: pitch_pred = p1 + p2 (channels 0, 1 of [rows][4]); f0d = f0d_pred = denorm 'standard' (uv, mel2ph == 0 -> 0)
void gs_pitch(const float* p1, const float* p2, const int* mel2ph, float mean, float std_, float* pitch_pred, float* f0d, float* f0d_pred,
              int* coarse, long rows, cudaStream_t st);
// g [rows][M + 4H] = cat[mel [rows][M], dec [rows][H], spk [b][H], emo [b][H], pros [rows][H]], b = r / T
void gs_cond_cat(const float* mel, const float* dec, const float* spk, const float* emo, const float* pros, float* g, int T, long rows,
                 int M, int H, cudaStream_t st);
// x [B][T2][2M] = squeeze(z [B][M][Tz], 2) channels-last (Tz >= 2 T2)
void gs_squeeze(const float* z, float* x, int B, int Tz, int T2, int M, cudaStream_t st);
// one reverse post-flow step (coupling, InvConvNear, ActNorm) on x [rows][C2] in place; e = the end layer's [rows][C2];
// blk = winv[16], bias[C2], logs[C2]
void gs_flow_step(float* x, const float* e, const float* blk, long rows, int C2, cudaStream_t st);
// PitchExtractor: mask[r] = any(mel[r] != 0) over M bins (warp per row)
void pe_mask(const float* mel, float* mask, long rows, int M, cudaStream_t st);
// PitchExtractor: pitch_pred [rows][2] = pred4[..., :2]; f0 = denorm_f0(pred4[..., 0]) (uv, mask == 0 -> 0)
void pe_denorm(const float* pred4, const float* mask, float* pitch_pred, float* f0, long rows, int use_uv, int norm, float mean,
               float std_, cudaStream_t st);

}  // namespace agpt
