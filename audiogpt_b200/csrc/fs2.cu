// FastSpeech2 / FastSpeech2MIDI acoustic front-end on sm_90a: phoneme tokens -> durations -> mel2ph -> frame
// features (+ pitch / energy embeddings) -> FFT decoder -> mel.  Two calls: encode (token side; ends with the one
// device -> host copy, the B mel lengths, when durations are predicted) and decode (frame side, sized by those lengths).
// Reference: NeuralSeq/modules/fastspeech/fs2.py:22-226 (FastSpeech2), modules/diffsinger_midi/fs2.py:11-118
// (FastSpeech2MIDI), modules/fastspeech/tts_modules.py:59-143 (DurationPredictor), :179-214 (LengthRegulator),
// :217-264 (Pitch / EnergyPredictor), :276-384 (FFTBlocks, FastspeechEncoder / Decoder), modules/commons/
// common_layers.py:541-587 (EncSALayer), :485-521 (TransformerFFNLayer), :87-142 (SinusoidalPositionalEmbedding),
// modules/commons/espnet_positional_embedding.py:89-113 (RelPositionalEncoding), utils/pitch_utils.py:22-76.
// Every Linear / Conv1d is a tap-GEMM (tcconv5 on the tensor cores); self-attention is the masked attention kernel.
#include <cstring>
#include "common.cuh"
#include "tapconv.cuh"
#include "nn_kernels.h"
#include "models.h"
#include "fs_layers.cuh"

namespace agpt {

namespace {

constexpr int kRelMaxLen = 5000;    // RelPositionalEncoding's table length (positions run backwards from max_len - 1)

// x[b][t] = escale * E[tok] (+ midi_E[pitch_midi] + midi_dur * w + b + slur_E[is_slur]), then the encoder positions:
// pos_mode 1 = fairseq (x + table[make_positions(tokens)]), 2 = espnet rel_pos (x * sqrt(H) + pe[max(5000, T) - 1 - t]).
// Also the source masks: nonpad[b][t] = tok != 0, kpm[b][t] = tok == 0.  Grid (T, B); out-of-range ids are clamped.
__global__ void fs2_embed_kernel(const int* __restrict__ tok, const int* __restrict__ pmidi, const float* __restrict__ mdur,
                                 const int* __restrict__ slur, const float* __restrict__ E, const float* __restrict__ midiE,
                                 const float* __restrict__ mdw, const float* __restrict__ mdb, const float* __restrict__ slurE,
                                 int ntok, float escale, int pos_mode, const float* __restrict__ rel_div, float neg_emb, float xscale,
                                 float* __restrict__ x, float* __restrict__ nonpad, uint8_t* __restrict__ kpm, int T, int H) {
  const int t = blockIdx.x, b = blockIdx.y;
  const long r = (long)b * T + t;
  const int* tb = tok + (long)b * T;
  const int id = tb[t];
  int pos = 0;
  if (pos_mode == 1 && id != 0) {                        // make_positions: count of non-padding tokens in [0, t]
    for (int i0 = 0; i0 <= t; i0 += blockDim.x) {
      const int i = i0 + threadIdx.x;
      pos += __syncthreads_count(i <= t && tb[i] != 0);
    }
  }
  const int e = min(max(id, 0), ntok - 1);
  const int pm = pmidi ? min(max(pmidi[r], 0), 299) : 0;
  const int sl = slur ? min(max(slur[r], 0), 1) : 0;
  const float md = mdur ? mdur[r] : 0.f;
  const int half = H / 2;
  const int relpos = max(kRelMaxLen, T) - 1 - t;
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    float v = __fmul_rn(escale, E[(long)e * H + c]);
    if (pmidi) v = __fadd_rn(v, midiE[(long)pm * H + c]);
    if (mdur) v = __fadd_rn(v, __fadd_rn(__fmul_rn(md, mdw[c]), mdb[c]));
    if (slur) v = __fadd_rn(v, slurE[(long)sl * H + c]);
    if (pos_mode == 1 && pos != 0 && c < 2 * half) {
      const int k = c < half ? c : c - half;
      const float a = (float)pos * expf((float)k * neg_emb);
      v += c < half ? sinf(a) : cosf(a);
    } else if (pos_mode == 2) {
      const float a = __fmul_rn((float)relpos, rel_div[c >> 1]);
      v = __fadd_rn(__fmul_rn(v, xscale), (c & 1) ? cosf(a) : sinf(a));
    }
    x[r * H + c] = v;
  }
  if (threadIdx.x == 0) {
    nonpad[r] = id != 0 ? 1.f : 0.f;
    kpm[r] = id == 0 ? 1 : 0;
  }
}

// FFTBlocks' padding mask from the rows themselves: nonpad[r] = any(x[r] != 0), kpm[r] = !nonpad[r]  (warp per row)
__global__ void fs2_rowmask_kernel(const float* __restrict__ x, float* __restrict__ nonpad, uint8_t* __restrict__ kpm, long rows, int C) {
  const long r = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += fabsf(x[r * C + c]);
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) { nonpad[r] = s == 0.f ? 0.f : 1.f; kpm[r] = s == 0.f ? 1 : 0; }
}

// DurationPredictor.inference / LengthRegulator: xs = linear * nonpad -> dur[r]; dur_choice = clamp(round(exp(xs) - 1), 0)
// (round half to even, as torch.round), zero on padding tokens
__global__ void fs2_dur_kernel(const float* __restrict__ pred4, const float* __restrict__ nonpad, float* __restrict__ dur,
                               int* __restrict__ dch, long rows) {
  for (long r = (long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long)gridDim.x * blockDim.x) {
    const float xs = pred4[r * 4] * nonpad[r];
    dur[r] = xs;
    if (dch) dch[r] = nonpad[r] != 0.f ? (int)fmaxf(rintf(expf(xs) - 1.f), 0.f) : 0;
  }
}
// per utterance: inclusive cumsum of the durations, mel_len[b] = total frames
__global__ void fs2_lr_scan_kernel(const int* __restrict__ dch, int* __restrict__ cum, int* __restrict__ mel_len, int T) {
  if (threadIdx.x != 0) return;
  const int b = blockIdx.x;
  int run = 0;
  for (int t = 0; t < T; ++t) { run += dch[(long)b * T + t]; cum[(long)b * T + t] = run; }
  mel_len[b] = run;
}
// mel2ph[b][f] = 1 + (the token whose frame range [cum[t-1], cum[t]) holds f), 0 past the utterance's last frame
__global__ void fs2_lr_fill_kernel(const int* __restrict__ cum, const int* __restrict__ mel_len, int* __restrict__ mel2ph, int B,
                                   int Tt, int Tm) {
  const long total = (long)B * Tm;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int b = (int)(i / Tm), f = (int)(i - (long)b * Tm);
    int v = 0;
    if (f < mel_len[b]) {
      const int* c = cum + (long)b * Tt;
      int lo = 0, hi = Tt - 1;                             // first t with cum[t] > f
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (c[mid] > f) hi = mid; else lo = mid + 1; }
      v = lo + 1;
    }
    mel2ph[i] = v;
  }
}
// decoder_inp = gather(pad(encoder_out, 1 leading zero row), mel2ph); tgt_nonpad = mel2ph > 0
__global__ void fs2_gather_kernel(const float* __restrict__ enc, const int* __restrict__ mel2ph, float* __restrict__ out,
                                  float* __restrict__ tgt, int B, int Tt, int Tm, int H) {
  const long total = (long)B * Tm * H;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / H;
    const int c = (int)(i - r * H);
    const int b = (int)(r / Tm);
    const int m = min(mel2ph[r], Tt);
    out[i] = m > 0 ? enc[((long)b * Tt + m - 1) * H + c] : 0.f;
    if (c == 0) tgt[r] = m > 0 ? 1.f : 0.f;
  }
}

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
// add_pitch, pitch_type 'frame' (fs2.py:187-220): pitch_pred (channel 0 zeroed on padding frames when it is the f0 used, as
// the reference's in-place f0[pitch_padding] = 0 does through the view), f0_denorm (uv and padding -> 0), coarse bins
__global__ void fs2_pitch_frame_kernel(const float* __restrict__ pred4, const int* __restrict__ mel2ph, const float* __restrict__ f0_in,
                                       const float* __restrict__ uv_in, int use_uv, int norm, float mean, float std_, float mel_min,
                                       float mel_range, float* __restrict__ pitch_pred, float* __restrict__ f0d, int* __restrict__ coarse,
                                       long rows) {
  for (long r = (long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long)gridDim.x * blockDim.x) {
    const float p0 = pred4[r * 4], p1 = pred4[r * 4 + 1];
    const bool pad = mel2ph[r] == 0;
    float f = denorm(f0_in ? f0_in[r] : p0, norm, mean, std_);
    if (use_uv && (uv_in ? uv_in[r] > 0.f : p1 > 0.f)) f = 0.f;
    if (pad) f = 0.f;
    pitch_pred[r * 2] = (!f0_in && pad) ? 0.f : p0;
    pitch_pred[r * 2 + 1] = p1;
    f0d[r] = f;
    coarse[r] = f0_coarse(f, mel_min, mel_range);
  }
}
// add_pitch, pitch_type 'ph' (fs2.py:175-186): per token, no uv
__global__ void fs2_pitch_ph_kernel(const float* __restrict__ pred4, const float* __restrict__ f0_in, int norm, float mean, float std_,
                                    float mel_min, float mel_range, float* __restrict__ pitch_pred, float* __restrict__ f0d,
                                    int* __restrict__ coarse, long rows) {
  for (long r = (long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long)gridDim.x * blockDim.x) {
    const float p0 = pred4[r * 4];
    const float f = denorm(f0_in ? f0_in[r] : p0, norm, mean, std_);
    pitch_pred[r] = p0;
    f0d[r] = f;
    coarse[r] = f0_coarse(f, mel_min, mel_range);
  }
}
// add_energy (fs2.py:165-172): energy_pred = predictor[..., 0]; bucket = clamp(floor(e * 256 / 4), 0, 255)
__global__ void fs2_energy_kernel(const float* __restrict__ pred4, const float* __restrict__ e_in, float* __restrict__ e_pred,
                                  int* __restrict__ bucket, long rows) {
  for (long r = (long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long)gridDim.x * blockDim.x) {
    const float p = pred4[r * 4];
    e_pred[r] = p;
    const float e = e_in ? e_in[r] : p;
    bucket[r] = (int)fminf(fmaxf(floorf(__fmul_rn(e, 256.f) / 4.f), 0.f), 255.f);
  }
}
// decoder_inp = (gathered + pitch_embed[pitch] + energy_embed[energy]) * tgt_nonpad.  Pitch index per frame (frame mode)
// or per token through mel2ph (ph mode: F.pad(coarse, [1, 0]) then gather, so padding frames read bin 0).
__global__ void fs2_embed_add_kernel(const float* __restrict__ x, const float* __restrict__ tgt, const float* __restrict__ pE,
                                     const int* __restrict__ pframe, const int* __restrict__ ptok, const int* __restrict__ mel2ph,
                                     const float* __restrict__ eE, const int* __restrict__ ebucket, float* __restrict__ out, int Tt, int Tm,
                                     long total, int H) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / H;
    const int c = (int)(i - r * H);
    float v = x[i];
    if (pE) {
      int pi;
      if (ptok) { const int m = min(mel2ph[r], Tt); pi = m > 0 ? ptok[(r / Tm) * Tt + m - 1] : 0; }
      else pi = pframe[r];
      v = __fadd_rn(v, pE[(long)pi * H + c]);
    }
    if (eE) v = __fadd_rn(v, eE[(long)ebucket[r] * H + c]);
    out[i] = v * tgt[r];
  }
}

unsigned ew_grid(long total) { return (unsigned)std::min<long>(cdivl(total, 256), 2368); }
int* iptr(DevBuf& d) { return reinterpret_cast<int*>(d.p); }
uint8_t* bptr(DevBuf& d) { return reinterpret_cast<uint8_t*>(d.p); }

// EncSALayer (common_layers.py:541-587), norm 'ln', act 'gelu', padding 'SAME'
struct FftLayer {
  DevBuf ln1g, ln1b, ln2g, ln2b;
  PackedConv qkv, out, ffn1, ffn2;
  int k = 9;
};

struct FftStack {
  std::vector<FftLayer> layers;
  DevBuf lng, lnb;
};

}  // namespace

struct Fs2Net : Handle {
  agpt_fs2_cfg cfg;
  DevBuf E, midiE, mdw, mdb, slurE, rel_div, pitchE, energyE;
  FftStack enc, dec;
  float dec_alpha = 1.f;
  PackedConv mel_out;
  std::vector<PackedConv> dp_conv;
  std::vector<DevBuf> dp_g, dp_b;
  PackedConv dp_lin;
  PitchPredictorNet pitch_pp, energy_pp;
  // encode -> decode state
  int B = 0, Tt = 0, have_dur = 0;
  DevBuf enc_out, snp, skpm, dch, cum, mlen;
  // work buffers
  DevBuf x, y, z, qkv, ffn, s[3], pred4, dnp, dkpm, tnp, pos, ebkt;

  // FFTBlocks.forward after the input positions (tts_modules.py:307-332): x * nonpad, layers, last LayerNorm * nonpad.
  // xs [rows][H] is the work tensor (overwritten), the result goes to out (which may be y); uses y, z, qkv, ffn, which
  // ensure_work has sized (no buffer may grow once a pointer into it has been taken).
  void fft(FftStack& S, float* xs, float* out, int B_, int T, const float* nonpad, const uint8_t* kpm, cudaStream_t st) {
    const int H = cfg.hidden_size, heads = cfg.num_heads;
    const long rows = (long)B_ * T;
    fs_affine_mask(xs, nullptr, nullptr, nonpad, rows, H, st);
    for (auto& L : S.layers) {
      layernorm(xs, y.p, L.ln1g.p, L.ln1b.p, rows, H, 1e-5f, st);
      fs_conv(L.qkv, y.p, H, qkv.p, 3 * H, 1, (int)rows, EPI_BIAS, st);
      attention(qkv.p, 3 * H, qkv.p + H, 3 * H, qkv.p + 2 * H, 3 * H, y.p, H, B_, heads, H / heads, T, T, st, kpm);
      fs_conv(L.out, y.p, H, z.p, H, 1, (int)rows, EPI_RES, st, xs);                 // residual + attention
      fs_affine_mask(z.p, nullptr, nullptr, nonpad, rows, H, st);
      layernorm(z.p, y.p, L.ln2g.p, L.ln2b.p, rows, H, 1e-5f, st);
      fs_conv(L.ffn1, y.p, H, ffn.p, 4 * H, B_, T, EPI_GELU_SCALED, st, nullptr, (float)std::pow((double)L.k, -0.5));
      fs_conv(L.ffn2, ffn.p, 4 * H, xs, H, 1, (int)rows, EPI_RES, st, z.p);          // residual + FFN
      fs_affine_mask(xs, nullptr, nullptr, nonpad, rows, H, st);
    }
    layernorm(xs, out, S.lng.p, S.lnb.p, rows, H, 1e-5f, st);
    fs_affine_mask(out, nullptr, nullptr, nonpad, rows, H, st);
  }

  void ensure_work(long rows) {
    const int H = cfg.hidden_size, Cmax = std::max(H, cfg.predictor_hidden);
    for (auto& b : s) b.ensure((size_t)rows * Cmax);
    pred4.ensure(rows * 4);
    x.ensure(rows * H); y.ensure(rows * H); z.ensure(rows * H); qkv.ensure(rows * 3 * H); ffn.ensure(rows * 4 * H);
  }

  void encode(const int* tok, int B_, int T, const int* pmidi, const float* mdur, const int* slur, int predict, float* dur, int* dur_choice,
              int* mel_len_host, cudaStream_t st) {
    AGPT_CHECK(B_ >= 1 && T >= 1, "empty batch");
    AGPT_CHECK(!cfg.use_midi || pmidi, "FastSpeech2MIDI needs pitch_midi");
    const int H = cfg.hidden_size, P = cfg.predictor_hidden;
    const long rows = (long)B_ * T;
    B = B_; Tt = T; have_dur = 0;
    enc_out.ensure(rows * H); snp.ensure(rows); skpm.ensure(rows / 4 + 1); dch.ensure(rows); cum.ensure(rows); mlen.ensure(B_);
    ensure_work(rows);
    const int pos_mode = cfg.use_pos_embed ? (cfg.rel_pos ? 2 : 1) : 0;
    fs2_embed_kernel<<<dim3(T, B_), 128, 0, st>>>(tok, cfg.use_midi ? pmidi : nullptr, cfg.use_midi ? mdur : nullptr, cfg.use_midi ? slur : nullptr,
                                                  E.p, midiE.p, mdw.p, mdb.p, slurE.p, cfg.n_tokens, (float)std::sqrt((double)H), pos_mode,
                                                  rel_div.p, (float)(-(std::log(10000.0) / (double)(H / 2 - 1))), (float)std::sqrt((double)H),
                                                  x.p, snp.p, bptr(skpm), T, H);
    count_launch(1);
    fft(enc, x.p, enc_out.p, B_, T, snp.p, bptr(skpm), st);
    // ---- DurationPredictor (tts_modules.py:98-112): n x [conv k SAME -> ReLU -> LayerNorm -> x nonpad], Linear -> 1
    const float* cur = enc_out.p;
    int cin = H;
    for (size_t l = 0; l < dp_conv.size(); ++l) {
      float* o = s[1 + (l & 1)].p;
      fs_conv(dp_conv[l], cur, cin, s[0].p, P, B_, T, EPI_RELU, st);
      layernorm(s[0].p, o, dp_g[l].p, dp_b[l].p, rows, P, 1e-5f, st);
      fs_affine_mask(o, nullptr, nullptr, snp.p, rows, P, st);
      cur = o;
      cin = P;
    }
    fs_conv(dp_lin, cur, cin, pred4.p, 4, 1, (int)rows, EPI_BIAS, st);
    fs2_dur_kernel<<<ew_grid(rows), 256, 0, st>>>(pred4.p, snp.p, dur, predict ? iptr(dch) : nullptr, rows);
    count_launch(1);
    if (predict) {
      fs2_lr_scan_kernel<<<B_, 32, 0, st>>>(iptr(dch), iptr(cum), iptr(mlen), T);
      count_launch(1);
      if (dur_choice) AGPT_CUDA(cudaMemcpyAsync(dur_choice, dch.p, sizeof(int) * rows, cudaMemcpyDeviceToDevice, st));
      // the one device -> host transfer: the frame count sizes the decoder (the reference syncs on dur.sum(-1).max())
      AGPT_CUDA(cudaMemcpyAsync(mel_len_host, mlen.p, sizeof(int) * B_, cudaMemcpyDeviceToHost, st));
      AGPT_CUDA(cudaStreamSynchronize(st));
      have_dur = 1;
    }
    AGPT_CUDA(cudaGetLastError());
  }

  void decode(int Tm, const int* mel2ph_in, int* mel2ph_out, const float* f0_in, const float* uv_in, const float* e_in, int use_uv, int norm,
              float f0_mean, float f0_std, float* pitch_pred, float* f0d, int* coarse, float* e_pred, float* dec_inp, float* mel,
              cudaStream_t st) {
    AGPT_CHECK(B >= 1, "agpt_fs2_decode before agpt_fs2_encode");
    AGPT_CHECK(Tm >= 1, "no mel frames");
    AGPT_CHECK(mel2ph_in || have_dur, "mel2ph not given and durations not predicted by the last encode");
    AGPT_CHECK(!cfg.pitch_type || (pitch_pred && f0d && coarse), "pitch outputs required");
    AGPT_CHECK(!cfg.use_energy_embed || e_pred, "energy output required");
    AGPT_CHECK(dec_inp, "decoder_inp output required");
    const int H = cfg.hidden_size;
    const long rows = (long)B * Tm, trow = (long)B * Tt;
    tnp.ensure(rows); dnp.ensure(rows); dkpm.ensure(rows / 4 + 1); pos.ensure(rows); ebkt.ensure(rows);
    ensure_work(std::max(rows, trow));
    const int* m2p = mel2ph_in;
    if (!m2p) {
      AGPT_CHECK(mel2ph_out, "mel2ph output required when it is predicted");
      fs2_lr_fill_kernel<<<ew_grid(rows), 256, 0, st>>>(iptr(cum), iptr(mlen), mel2ph_out, B, Tt, Tm);
      count_launch(1);
      m2p = mel2ph_out;
    }
    fs2_gather_kernel<<<ew_grid(rows * H), 256, 0, st>>>(enc_out.p, m2p, x.p, tnp.p, B, Tt, Tm, H);
    count_launch(1);
    // pitch_inp = decoder_inp_origin * tgt_nonpad = x (gathered rows are zero where mel2ph == 0)
    const double mmin = 1127.0 * std::log(1.0 + 50.0 / 700.0), mmax = 1127.0 * std::log(1.0 + 1100.0 / 700.0);
    const float mel_min = (float)mmin, mel_range = (float)(mmax - mmin);
    const int* ptok = nullptr;
    const int* pframe = nullptr;
    if (cfg.pitch_type == 1) {
      pitch_pp.forward(x.p, H, B, Tm, s[0].p, s[1].p, s[2].p, pred4.p, st);
      fs2_pitch_frame_kernel<<<ew_grid(rows), 256, 0, st>>>(pred4.p, m2p, f0_in, uv_in, use_uv, norm, f0_mean, f0_std, mel_min, mel_range,
                                                            pitch_pred, f0d, coarse, rows);
      count_launch(1);
      pframe = coarse;
    } else if (cfg.pitch_type == 2) {
      pitch_pp.forward(enc_out.p, H, B, Tt, s[0].p, s[1].p, s[2].p, pred4.p, st);
      fs2_pitch_ph_kernel<<<ew_grid(trow), 256, 0, st>>>(pred4.p, f0_in, norm, f0_mean, f0_std, mel_min, mel_range, pitch_pred, f0d, coarse,
                                                         trow);
      count_launch(1);
      ptok = coarse;
    }
    if (cfg.use_energy_embed) {
      energy_pp.forward(x.p, H, B, Tm, s[0].p, s[1].p, s[2].p, pred4.p, st);
      fs2_energy_kernel<<<ew_grid(rows), 256, 0, st>>>(pred4.p, e_in, e_pred, iptr(ebkt), rows);
      count_launch(1);
    }
    fs2_embed_add_kernel<<<ew_grid(rows * H), 256, 0, st>>>(x.p, tnp.p, cfg.pitch_type ? pitchE.p : nullptr, pframe, ptok, m2p,
                                                            cfg.use_energy_embed ? energyE.p : nullptr, iptr(ebkt), dec_inp, Tt, Tm, rows * H, H);
    count_launch(1);
    if (!mel) { AGPT_CUDA(cudaGetLastError()); return; }        // skip_decoder
    // ---- FastspeechDecoder: padding mask and positions from decoder_inp itself (tts_modules.py:313-318)
    fs2_rowmask_kernel<<<(unsigned)cdivl(rows, 8), 256, 0, st>>>(dec_inp, dnp.p, bptr(dkpm), rows, H);
    count_launch(1);
    fs_positions(dec_inp, iptr(pos), B, Tm, H, st);
    fs_posemb_add(dec_inp, x.p, iptr(pos), dec_alpha, rows, H, st);
    fft(dec, x.p, y.p, B, Tm, dnp.p, bptr(dkpm), st);
    fs_conv(mel_out, y.p, H, mel, cfg.out_dims, 1, (int)rows, EPI_BIAS, st);
    fs_affine_mask(mel, nullptr, nullptr, tnp.p, rows, cfg.out_dims, st);
    AGPT_CUDA(cudaGetLastError());
  }
};

namespace {
void load_stack(FftStack& S, WeightCursor& wc, int H, int L, int k) {
  S.layers.resize(L);
  for (auto& l : S.layers) {
    l.k = k;
    { auto g = wc.next(); auto b = wc.next(); l.ln1g.upload(g, H); l.ln1b.upload(b, H); }
    pack_conv(l.qkv, wc.next(), nullptr, 3 * H, H, 1, false);        // in_proj_weight [3H][H], no bias
    pack_conv(l.out, wc.next(), nullptr, H, H, 1, false);            // out_proj.weight, no bias
    { auto g = wc.next(); auto b = wc.next(); l.ln2g.upload(g, H); l.ln2b.upload(b, H); }
    { auto w = wc.next(); auto b = wc.next(); pack_conv(l.ffn1, w, b, 4 * H, H, k, false); }
    { auto w = wc.next(); auto b = wc.next(); pack_conv(l.ffn2, w, b, H, 4 * H, 1, false); }
  }
  { auto g = wc.next(); auto b = wc.next(); S.lng.upload(g, H); S.lnb.upload(b, H); }
}
}  // namespace

Handle* fs2_create(const agpt_fs2_cfg* cfg, const float* const* W, int nW, int device) {
  DeviceGuard dg_(device);
  const int H = cfg->hidden_size, P = cfg->predictor_hidden;
  AGPT_CHECK(H % 16 == 0 && cfg->num_heads >= 1 && H % cfg->num_heads == 0 && P % 4 == 0 && cfg->out_dims % 4 == 0 &&
                 cfg->n_tokens >= 1 && cfg->enc_ffn_kernel % 2 == 1 && cfg->dec_ffn_kernel % 2 == 1 &&
                 cfg->enc_ffn_kernel <= kMaxTaps && cfg->dec_ffn_kernel <= kMaxTaps && cfg->dur_predictor_kernel % 2 == 1 &&
                 cfg->dur_predictor_kernel <= kMaxTaps && cfg->pitch_type >= 0 && cfg->pitch_type <= 2,
             "bad FastSpeech2 config");
  std::unique_ptr<Fs2Net> h(new Fs2Net());
  h->magic = kMagicFs2; h->device = device; h->cfg = *cfg;
  WeightCursor wc{W, nW};
  h->E.upload(wc.next(), (size_t)cfg->n_tokens * H);                // encoder_embed_tokens.weight
  wc.next();                                                      // encoder.embed_tokens.weight (the same tensor)
  if (!cfg->rel_pos) wc.next();                                   // encoder.embed_positions._float_tensor
  load_stack(h->enc, wc, H, cfg->enc_layers, cfg->enc_ffn_kernel);
  h->dec_alpha = wc.next()[0];                                    // decoder.pos_embed_alpha
  wc.next();                                                      // decoder.embed_positions._float_tensor
  load_stack(h->dec, wc, H, cfg->dec_layers, cfg->dec_ffn_kernel);
  { auto w = wc.next(); auto b = wc.next(); pack_conv(h->mel_out, w, b, cfg->out_dims, H, 1, false); }
  h->dp_conv.resize(cfg->dur_predictor_layers); h->dp_g.resize(cfg->dur_predictor_layers); h->dp_b.resize(cfg->dur_predictor_layers);
  int cin = H;
  for (int l = 0; l < cfg->dur_predictor_layers; ++l) {
    { auto w = wc.next(); auto b = wc.next(); pack_conv(h->dp_conv[l], w, b, P, cin, cfg->dur_predictor_kernel, false); }
    { auto g = wc.next(); auto b = wc.next(); h->dp_g[l].upload(g, P); h->dp_b[l].upload(b, P); }
    cin = P;
  }
  {  // Linear(P -> 1) padded to 4 output channels
    auto w = wc.next(); auto b = wc.next();
    std::vector<float> wp((size_t)4 * P, 0.f), bp(4, 0.f);
    memcpy(wp.data(), w, sizeof(float) * P);
    bp[0] = b[0];
    pack_conv(h->dp_lin, wp.data(), bp.data(), 4, P, 1, false);
  }
  if (cfg->pitch_type) {
    h->pitchE.upload(wc.next(), (size_t)300 * H);
    h->pitch_pp.load(wc, H, P, cfg->predictor_kernel, cfg->predictor_layers, cfg->pitch_type == 1 ? 2 : 1);
  }
  if (cfg->use_energy_embed) {
    h->energyE.upload(wc.next(), (size_t)256 * H);
    h->energy_pp.load(wc, H, P, cfg->predictor_kernel, cfg->predictor_layers, 1);
  }
  if (cfg->use_midi) {
    h->midiE.upload(wc.next(), (size_t)300 * H);
    h->mdw.upload(wc.next(), H);
    h->mdb.upload(wc.next(), H);
    h->slurE.upload(wc.next(), (size_t)2 * H);
  }
  wc.done();
  if (cfg->rel_pos) {   // espnet div_term: exp(arange(0, H, 2) * -(ln 10000 / H)) in fp32
    std::vector<float> d(H / 2);
    const float c = (float)(-(std::log(10000.0) / (double)H));
    for (int i = 0; i < H / 2; ++i) d[i] = (float)std::exp((double)((float)(2 * i) * c));
    h->rel_div.upload(d);
  }
  return h.release();
}

void fs2_encode(Handle* hh, const int* tok, int B, int T, const int* pmidi, const float* mdur, const int* slur, int predict, float* dur,
                int* dur_choice, int* mel_len_host, cudaStream_t st) {
  auto* h = static_cast<Fs2Net*>(hh);
  DeviceGuard dg_(h->device);
  h->encode(tok, B, T, pmidi, mdur, slur, predict, dur, dur_choice, mel_len_host, st);
}

void fs2_decode(Handle* hh, int Tm, const int* mel2ph_in, int* mel2ph_out, const float* f0, const float* uv, const float* energy, int use_uv,
                int norm, float f0_mean, float f0_std, float* pitch_pred, float* f0d, int* coarse, float* e_pred, float* dec_inp, float* mel,
                cudaStream_t st) {
  auto* h = static_cast<Fs2Net*>(hh);
  DeviceGuard dg_(h->device);
  h->decode(Tm, mel2ph_in, mel2ph_out, f0, uv, energy, use_uv, norm, f0_mean, f0_std, pitch_pred, f0d, coarse, e_pred, dec_inp, mel, st);
}

}  // namespace agpt
