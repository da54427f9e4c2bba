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

}  // namespace

void fs2_pitch_frame(const float* pred4, const int* mel2ph, const float* f0_in, const float* uv_in, int use_uv, int norm, float mean,
                     float std_, float* pitch_pred, float* f0d, int* coarse, long rows, cudaStream_t st) {
  fs2_pitch_frame_kernel<<<ew_grid(rows), 256, 0, st>>>(pred4, mel2ph, f0_in, uv_in, use_uv, norm, mean, std_, f0_mel_min(),
                                                        f0_mel_range(), pitch_pred, f0d, coarse, rows);
  count_launch(1);
}

void fs2_pitch_ph(const float* pred4, const float* f0_in, int norm, float mean, float std_, float* pitch_pred, float* f0d, int* coarse,
                  long rows, cudaStream_t st) {
  fs2_pitch_ph_kernel<<<ew_grid(rows), 256, 0, st>>>(pred4, f0_in, norm, mean, std_, f0_mel_min(), f0_mel_range(), pitch_pred, f0d,
                                                     coarse, rows);
  count_launch(1);
}

void fs2_energy(const float* pred4, const float* e_in, float* e_pred, int* bucket, long rows, cudaStream_t st) {
  fs2_energy_kernel<<<ew_grid(rows), 256, 0, st>>>(pred4, e_in, e_pred, bucket, rows);
  count_launch(1);
}

void fs2_embed_add(const float* x, const float* tgt, const float* pE, const int* pframe, const int* ptok, const int* mel2ph,
                   const float* eE, const int* ebucket, float* out, int Tt, int Tm, long rows, int H, cudaStream_t st) {
  fs2_embed_add_kernel<<<ew_grid(rows * H), 256, 0, st>>>(x, tgt, pE, pframe, ptok, mel2ph, eE, ebucket, out, Tt, Tm, rows * H, H);
  count_launch(1);
}

struct Fs2Net : Handle {
  agpt_fs2_cfg cfg;
  DevBuf E, midiE, mdw, mdb, slurE, rel_div, pitchE, energyE;
  FftStack enc, dec;
  float dec_alpha = 1.f;
  PackedConv mel_out;
  DurPredictorNet dp;
  PitchPredictorNet pitch_pp, energy_pp;
  // encode -> decode state
  int B = 0, Tt = 0, have_dur = 0;
  DevBuf enc_out, snp, skpm, dch, cum, mlen;
  // work buffers
  DevBuf x, y, z, qkv, ffn, s[3], pred4, dnp, dkpm, tnp, pos, ebkt;

  void fft(const FftStack& S, float* xs, float* out, int B_, int T, const float* nonpad, const uint8_t* kpm, cudaStream_t st) {
    S.forward(xs, out, B_, T, cfg.hidden_size, cfg.num_heads, nonpad, kpm, y.p, z.p, qkv.p, ffn.p, st);
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
    fs_embed_tokens(tok, cfg.use_midi ? pmidi : nullptr, cfg.use_midi ? mdur : nullptr, cfg.use_midi ? slur : nullptr, E.p, midiE.p, mdw.p,
                    mdb.p, slurE.p, cfg.n_tokens, (float)std::sqrt((double)H), pos_mode, rel_div.p,
                    (float)(-(std::log(10000.0) / (double)(H / 2 - 1))), (float)std::sqrt((double)H), x.p, snp.p, bptr(skpm), B_, T, H, st);
    fft(enc, x.p, enc_out.p, B_, T, snp.p, bptr(skpm), st);
    // ---- DurationPredictor (tts_modules.py:98-112) on the encoder output
    dp.forward(enc_out.p, H, B_, T, snp.p, s[0].p, s[1].p, s[2].p, pred4.p, st);
    fs_dur(pred4.p, snp.p, dur, predict ? iptr(dch) : nullptr, rows, st);
    if (predict) {
      fs_lr_scan(iptr(dch), iptr(cum), iptr(mlen), B_, T, st);
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
      fs_lr_fill(iptr(cum), iptr(mlen), mel2ph_out, B, Tt, Tm, st);
      m2p = mel2ph_out;
    }
    fs_gather(enc_out.p, m2p, x.p, tnp.p, B, Tt, Tm, H, st);
    // pitch_inp = decoder_inp_origin * tgt_nonpad = x (gathered rows are zero where mel2ph == 0)
    const int* ptok = nullptr;
    const int* pframe = nullptr;
    if (cfg.pitch_type == 1) {
      pitch_pp.forward(x.p, H, B, Tm, s[0].p, s[1].p, s[2].p, pred4.p, st);
      fs2_pitch_frame(pred4.p, m2p, f0_in, uv_in, use_uv, norm, f0_mean, f0_std, pitch_pred, f0d, coarse, rows, st);
      pframe = coarse;
    } else if (cfg.pitch_type == 2) {
      pitch_pp.forward(enc_out.p, H, B, Tt, s[0].p, s[1].p, s[2].p, pred4.p, st);
      fs2_pitch_ph(pred4.p, f0_in, norm, f0_mean, f0_std, pitch_pred, f0d, coarse, trow, st);
      ptok = coarse;
    }
    if (cfg.use_energy_embed) {
      energy_pp.forward(x.p, H, B, Tm, s[0].p, s[1].p, s[2].p, pred4.p, st);
      fs2_energy(pred4.p, e_in, e_pred, iptr(ebkt), rows, st);
    }
    fs2_embed_add(x.p, tnp.p, cfg.pitch_type ? pitchE.p : nullptr, pframe, ptok, m2p, cfg.use_energy_embed ? energyE.p : nullptr,
                  iptr(ebkt), dec_inp, Tt, Tm, rows, H, st);
    if (!mel) { AGPT_CUDA(cudaGetLastError()); return; }        // skip_decoder
    // ---- FastspeechDecoder: padding mask and positions from decoder_inp itself (tts_modules.py:313-318)
    fs_rowmask(dec_inp, dnp.p, bptr(dkpm), rows, H, st);
    fs_positions(dec_inp, iptr(pos), B, Tm, H, st);
    fs_posemb_add(dec_inp, x.p, iptr(pos), dec_alpha, rows, H, st);
    fft(dec, x.p, y.p, B, Tm, dnp.p, bptr(dkpm), st);
    fs_conv(mel_out, y.p, H, mel, cfg.out_dims, 1, (int)rows, EPI_BIAS, st);
    fs_affine_mask(mel, nullptr, nullptr, tnp.p, rows, cfg.out_dims, st);
    AGPT_CUDA(cudaGetLastError());
  }
};

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
  h->enc.load(wc, H, cfg->enc_layers, cfg->enc_ffn_kernel);
  h->dec_alpha = wc.next()[0];                                    // decoder.pos_embed_alpha
  wc.next();                                                      // decoder.embed_positions._float_tensor
  h->dec.load(wc, H, cfg->dec_layers, cfg->dec_ffn_kernel);
  { auto w = wc.next(); auto b = wc.next(); pack_conv(h->mel_out, w, b, cfg->out_dims, H, 1, false); }
  h->dp.load(wc, H, P, cfg->dur_predictor_kernel, cfg->dur_predictor_layers);
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
