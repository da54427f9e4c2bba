// Layers shared by the FastSpeech-family drivers (fs_layers.cuh).
// Reference: NeuralSeq/modules/fastspeech/tts_modules.py:217-264 (PitchPredictor / EnergyPredictor), :59-143
// (DurationPredictor), :179-214 (LengthRegulator), :276-384 (FFTBlocks), modules/fastspeech/fs2.py:141-163 (add_dur,
// expand_states),
// modules/commons/common_layers.py:87-142 (SinusoidalPositionalEmbedding), utils/__init__.py:145-157 (make_positions).
#include "fs_layers.cuh"
#include "models.h"
#include "nn_kernels.h"

namespace agpt {

static unsigned ew_grid(long total) { return (unsigned)std::min<long>(cdivl(total, 256), 2368); }

namespace {

// x[b][t] = escale * E[tok] (+ midi_E[pitch_midi] + midi_dur * w + b + slur_E[is_slur]), then the encoder positions:
// pos_mode 1 = fairseq (x + table[make_positions(tokens)]), 2 = espnet rel_pos (x * sqrt(H) + pe[max(5000, T) - 1 - t]).
// Also the source masks: nonpad[b][t] = tok != 0, kpm[b][t] = tok == 0.  Grid (T, B); out-of-range ids are clamped.
__global__ void fs_embed_tokens_kernel(const int* __restrict__ tok, const int* __restrict__ pmidi, const float* __restrict__ mdur,
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
__global__ void fs_rowmask_kernel(const float* __restrict__ x, float* __restrict__ nonpad, uint8_t* __restrict__ kpm, long rows, int C) {
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
__global__ void fs_dur_kernel(const float* __restrict__ pred4, const float* __restrict__ nonpad, float* __restrict__ dur,
                               int* __restrict__ dch, long rows) {
  for (long r = (long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long)gridDim.x * blockDim.x) {
    const float xs = pred4[r * 4] * nonpad[r];
    dur[r] = xs;
    if (dch) dch[r] = nonpad[r] != 0.f ? (int)fmaxf(rintf(expf(xs) - 1.f), 0.f) : 0;
  }
}
// per utterance: inclusive cumsum of the durations, mel_len[b] = total frames
__global__ void fs_lr_scan_kernel(const int* __restrict__ dch, int* __restrict__ cum, int* __restrict__ mel_len, int T) {
  if (threadIdx.x != 0) return;
  const int b = blockIdx.x;
  int run = 0;
  for (int t = 0; t < T; ++t) { run += dch[(long)b * T + t]; cum[(long)b * T + t] = run; }
  mel_len[b] = run;
}
// mel2ph[b][f] = 1 + (the token whose frame range [cum[t-1], cum[t]) holds f), 0 past the utterance's last frame
__global__ void fs_lr_fill_kernel(const int* __restrict__ cum, const int* __restrict__ mel_len, int* __restrict__ mel2ph, int B,
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
__global__ void fs_gather_kernel(const float* __restrict__ enc, const int* __restrict__ mel2ph, float* __restrict__ out,
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

}  // namespace

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

void fs_embed_tokens(const int* tok, const int* pmidi, const float* mdur, const int* slur, const float* E, const float* midiE,
                     const float* mdw, const float* mdb, const float* slurE, int ntok, float escale, int pos_mode, const float* rel_div,
                     float neg_emb, float xscale, float* x, float* nonpad, uint8_t* kpm, int B, int T, int H, cudaStream_t st) {
  fs_embed_tokens_kernel<<<dim3(T, B), 128, 0, st>>>(tok, pmidi, mdur, slur, E, midiE, mdw, mdb, slurE, ntok, escale, pos_mode, rel_div,
                                                     neg_emb, xscale, x, nonpad, kpm, T, H);
  count_launch(1);
}

void fs_rowmask(const float* x, float* nonpad, uint8_t* kpm, long rows, int C, cudaStream_t st) {
  fs_rowmask_kernel<<<(unsigned)cdivl(rows, 8), 256, 0, st>>>(x, nonpad, kpm, rows, C);
  count_launch(1);
}

void fs_dur(const float* pred4, const float* nonpad, float* dur, int* dch, long rows, cudaStream_t st) {
  fs_dur_kernel<<<ew_grid(rows), 256, 0, st>>>(pred4, nonpad, dur, dch, rows);
  count_launch(1);
}

void fs_lr_scan(const int* dch, int* cum, int* mel_len, int B, int T, cudaStream_t st) {
  fs_lr_scan_kernel<<<B, 32, 0, st>>>(dch, cum, mel_len, T);
  count_launch(1);
}

void fs_lr_fill(const int* cum, const int* mel_len, int* mel2ph, int B, int Tt, int Tm, cudaStream_t st) {
  fs_lr_fill_kernel<<<ew_grid((long)B * Tm), 256, 0, st>>>(cum, mel_len, mel2ph, B, Tt, Tm);
  count_launch(1);
}

void fs_gather(const float* enc, const int* mel2ph, float* out, float* tgt, int B, int Tt, int Tm, int H, cudaStream_t st) {
  fs_gather_kernel<<<ew_grid((long)B * Tm * H), 256, 0, st>>>(enc, mel2ph, out, tgt, B, Tt, Tm, H);
  count_launch(1);
}

void FftStack::load(WeightCursor& wc, int H, int L, int k) {
  layers.resize(L);
  for (auto& l : layers) {
    l.k = k;
    { auto g = wc.next(); auto b = wc.next(); l.ln1g.upload(g, H); l.ln1b.upload(b, H); }
    pack_conv(l.qkv, wc.next(), nullptr, 3 * H, H, 1, false);        // in_proj_weight [3H][H], no bias
    pack_conv(l.out, wc.next(), nullptr, H, H, 1, false);            // out_proj.weight, no bias
    { auto g = wc.next(); auto b = wc.next(); l.ln2g.upload(g, H); l.ln2b.upload(b, H); }
    { auto w = wc.next(); auto b = wc.next(); pack_conv(l.ffn1, w, b, 4 * H, H, k, false); }
    { auto w = wc.next(); auto b = wc.next(); pack_conv(l.ffn2, w, b, H, 4 * H, 1, false); }
  }
  { auto g = wc.next(); auto b = wc.next(); lng.upload(g, H); lnb.upload(b, H); }
}

void FftStack::forward(float* xs, float* out, int B, int T, int H, int heads, const float* nonpad, const uint8_t* kpm, float* y,
                       float* z, float* qkv, float* ffn, cudaStream_t st) const {
  const long rows = (long)B * T;
  fs_affine_mask(xs, nullptr, nullptr, nonpad, rows, H, st);
  for (auto& L : layers) {
    layernorm(xs, y, L.ln1g.p, L.ln1b.p, rows, H, 1e-5f, st);
    fs_conv(L.qkv, y, H, qkv, 3 * H, 1, (int)rows, EPI_BIAS, st);
    attention(qkv, 3 * H, qkv + H, 3 * H, qkv + 2 * H, 3 * H, y, H, B, heads, H / heads, T, T, st, kpm);
    fs_conv(L.out, y, H, z, H, 1, (int)rows, EPI_RES, st, xs);                 // residual + attention
    fs_affine_mask(z, nullptr, nullptr, nonpad, rows, H, st);
    layernorm(z, y, L.ln2g.p, L.ln2b.p, rows, H, 1e-5f, st);
    fs_conv(L.ffn1, y, H, ffn, 4 * H, B, T, EPI_GELU_SCALED, st, nullptr, (float)std::pow((double)L.k, -0.5));
    fs_conv(L.ffn2, ffn, 4 * H, xs, H, 1, (int)rows, EPI_RES, st, z);          // residual + FFN
    fs_affine_mask(xs, nullptr, nullptr, nonpad, rows, H, st);
  }
  layernorm(xs, out, lng.p, lnb.p, rows, H, 1e-5f, st);
  fs_affine_mask(out, nullptr, nullptr, nonpad, rows, H, st);
}

void DurPredictorNet::load(WeightCursor& wc, int H, int P_, int k, int layers) {
  P = P_;
  conv.resize(layers); g.resize(layers); b.resize(layers);
  int cin = H;
  for (int l = 0; l < layers; ++l) {
    { auto w = wc.next(); auto bb = wc.next(); pack_conv(conv[l], w, bb, P, cin, k, false); }
    { auto gg = wc.next(); auto bb = wc.next(); g[l].upload(gg, P); b[l].upload(bb, P); }
    cin = P;
  }
  {  // Linear(P -> 1) padded to 4 output channels
    auto w = wc.next(); auto bb = wc.next();
    std::vector<float> wp((size_t)4 * P, 0.f), bp(4, 0.f);
    memcpy(wp.data(), w, sizeof(float) * P);
    bp[0] = bb[0];
    pack_conv(lin, wp.data(), bp.data(), 4, P, 1, false);
  }
}

void DurPredictorNet::forward(const float* x, int H, int B, int T, const float* nonpad, float* s0, float* s1, float* s2, float* pred4,
                              cudaStream_t st) const {
  const long rows = (long)B * T;
  const float* cur = x;
  int cin = H;
  float* s12[2] = {s1, s2};
  for (size_t l = 0; l < conv.size(); ++l) {
    float* o = s12[l & 1];
    fs_conv(conv[l], cur, cin, s0, P, B, T, EPI_RELU, st);
    layernorm(s0, o, g[l].p, b[l].p, rows, P, 1e-5f, st);
    fs_affine_mask(o, nullptr, nullptr, nonpad, rows, P, st);
    cur = o;
    cin = P;
  }
  fs_conv(lin, cur, cin, pred4, 4, 1, (int)rows, EPI_BIAS, st);
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
