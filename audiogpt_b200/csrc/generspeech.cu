// GenerSpeech (the out-of-domain TTS tool's acoustic model) on sm_90a, inference path: FastSpeech2 encoder and durations
// with the speaker / emotion terms, three LocalStyleAdaptors (WN -> segment mean -> ConvBlocks -> VQ), positions + l1 +
// ProsodyAligner, the two pitch predictors, the FFT decoder, and the Glow post-flow in reverse.  Two calls, as fs2.cu:
// encode (token side; ends with the one device -> host copy of the mel lengths when durations are predicted) and forward.
// Reference: NeuralSeq/modules/GenerSpeech/model/generspeech.py:75-260, prosody_util.py:16-199, wavenet.py:14-78,
// glow_modules.py:68-192, 282-335, 496-592, 742-767, utils/tts_utils.py:357-371 (group_hidden_by_segs).
// Every Linear / Conv1d is a tap-GEMM (tcconv5 on the tensor cores); attention is the masked attention kernel.
#include <cstring>
#include <cmath>
#include "common.cuh"
#include "tapconv.cuh"
#include "nn_kernels.h"
#include "models.h"
#include "fs_layers.cuh"

namespace agpt {

namespace {

constexpr int kStyleC = 80;      // LocalStyleAdaptor: WN / ConvBlocks width
constexpr int kStyleWnLayers = 4;
constexpr int kStyleBlocks = 10; // ConvBlocks: 5 ResidualBlocks x 2 layers
constexpr int kAlignFfn = 2048;

unsigned ew_grid(long total) { return (unsigned)std::min<long>(cdivl(total, 256), 2368); }
int* iptr(DevBuf& d) { return reinterpret_cast<int*>(d.p); }
uint8_t* bptr(DevBuf& d) { return reinterpret_cast<uint8_t*>(d.p); }

// out[r] = (x[r] + a[b] + e[b] (+ tab[idx[r]]) (+ s[r])) * mask[r], b = r / T: the speaker / emotion / pitch / prosody
// sums of generspeech.py:87, 102, 106 (a, e: [B][H] per-utterance rows)
__global__ void gs_sum_kernel(const float* __restrict__ x, const float* __restrict__ a, const float* __restrict__ e,
                              const float* __restrict__ tab, const int* __restrict__ idx, const float* __restrict__ s,
                              const float* __restrict__ mask, float* __restrict__ out, int T, long total, int H) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / H;
    const int c = (int)(i - r * H);
    const long b = r / T;
    float v = __fadd_rn(__fadd_rn(x[i], a[b * H + c]), e[b * H + c]);
    if (tab) v = __fadd_rn(v, tab[(long)idx[r] * H + c]);
    if (s) v = __fadd_rn(v, s[i]);
    out[i] = v * mask[r];
  }
}

// dst (+)= src
__global__ void gs_accum_kernel(float* __restrict__ dst, const float* __restrict__ src, long n, int first) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    dst[i] = first ? src[i] : __fadd_rn(dst[i], src[i]);
}

// LocalStyleAdaptor's WN mask: ref_mels[..., 0] != 0
__global__ void gs_refmask_kernel(const float* __restrict__ mel, float* __restrict__ mask, long rows) {
  for (long r = (long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long)gridDim.x * blockDim.x)
    mask[r] = mel[r * kStyleC] != 0.f ? 1.f : 0.f;
}

// WN gate (wavenet.py:5-11): acts = tanh(a[:, :C]) * sigmoid(a[:, C:]), a [rows][2C] -> acts [rows][C]
__global__ void gs_wn_gate_kernel(const float* __restrict__ a, float* __restrict__ acts, long total, int C) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / C;
    const int c = (int)(i - r * C);
    const float t = tanhf(a[r * 2 * C + c]);
    const float g = a[r * 2 * C + C + c];
    acts[i] = t * (1.f / (1.f + expf(-g)));
  }
}

// group_hidden_by_segs: out[b][s] = mean of h[b][t] over the frames with seg[b][t] == s + 1 (0 for an empty segment).
// Grid (nseg, B), threads over channels.
__global__ void gs_segmean_kernel(const float* __restrict__ h, const int* __restrict__ seg, float* __restrict__ out, int T, int nseg, int C) {
  const int s = blockIdx.x + 1, b = blockIdx.y;
  const int* sb = seg + (long)b * T;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float sum = 0.f, cnt = 0.f;
    for (int t = 0; t < T; ++t)
      if (sb[t] == s) { sum += h[((long)b * T + t) * C + c]; cnt += 1.f; }
    out[((long)b * nseg + s - 1) * C + c] = sum / fmaxf(cnt, 1.f);
  }
}

// VQEmbeddingEMA.encode + straight-through: per row (one warp), d[m] = (|e_m|^2 + |x|^2) - 2 x.e_m from the GEMM's dots,
// argmin (ties -> lowest index, as torch.argmin), q = x + (e - x).  x / q may alias.
__global__ void gs_vq_kernel(const float* x, const float* __restrict__ dots, const float* __restrict__ emb,
                             const float* __restrict__ enorm, int* __restrict__ idx, float* q, long rows, int H, int M) {
  const long r = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  float xn = 0.f;
  for (int c = lane; c < H; c += 32) { const float v = x[r * H + c]; xn = fmaf(v, v, xn); }
#pragma unroll
  for (int o = 16; o; o >>= 1) xn += __shfl_xor_sync(0xffffffffu, xn, o);
  float best = INFINITY;
  int bi = 0x7fffffff;
  for (int m = lane; m < M; m += 32) {
    const float d = __fsub_rn(__fadd_rn(enorm[m], xn), 2.f * dots[r * M + m]);
    if (d < best) { best = d; bi = m; }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  if (lane == 0 && idx) idx[r] = bi;
  for (int c = lane; c < H; c += 32) {
    const float v = x[r * H + c];
    q[r * H + c] = __fadd_rn(v, __fsub_rn(emb[(long)bi * H + c], v));
  }
}

// l1_*'s input cat[prosody, positions]: positions of prosody[..., 0] (fairseq table, (H/2 - 1) divisor, row 0 = padding)
__global__ void gs_catpos_kernel(const float* __restrict__ p, const int* __restrict__ pos, float* __restrict__ out, long total, int H,
                                 float neg_emb) {
  const int half = H / 2;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / (2 * H);
    const int c = (int)(i - r * 2 * H);
    float v;
    if (c < H) v = p[r * H + c];
    else {
      const int k = c - H, ps = pos[r];
      v = 0.f;
      if (ps != 0 && k < 2 * half) {
        const int kk = k < half ? k : k - half;
        const float a = (float)ps * expf((float)kk * neg_emb);
        v = k < half ? sinf(a) : cosf(a);
      }
    }
    out[i] = v;
  }
}

// ProsodyAligner's key padding: kpm[r] = (prosody_embedding[r][0] == 0.0)
__global__ void gs_kpm_kernel(const float* __restrict__ x, uint8_t* __restrict__ kpm, long rows, int H) {
  for (long r = (long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long)gridDim.x * blockDim.x)
    kpm[r] = x[r * H] == 0.f ? 1 : 0;
}

// inpaint_pitch ('frame', use_uv, pitch_norm 'standard'): pitch_pred = p1 + p2; f0_denorm = f0_denorm_pred =
// denorm(pitch_pred[..., 0]) with uv (pitch_pred[..., 1] > 0) and padding frames -> 0; coarse bins
__global__ void gs_pitch_kernel(const float* __restrict__ p1, const float* __restrict__ p2, const int* __restrict__ mel2ph, float mean,
                                float std_, float mel_min, float mel_range, float* __restrict__ pitch_pred, float* __restrict__ f0d,
                                float* __restrict__ f0d_pred, int* __restrict__ coarse, long rows) {
  for (long r = (long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long)gridDim.x * blockDim.x) {
    const float a = __fadd_rn(p1[r * 4], p2[r * 4]), u = __fadd_rn(p1[r * 4 + 1], p2[r * 4 + 1]);
    float f = denorm(a, 1, mean, std_);
    if (u > 0.f || mel2ph[r] == 0) f = 0.f;
    pitch_pred[r * 2] = a;
    pitch_pred[r * 2 + 1] = u;
    f0d[r] = f;
    f0d_pred[r] = f;
    coarse[r] = f0_coarse(f, mel_min, mel_range);
  }
}

// the post-flow's conditioning g = cat[mel_out, decoder_inp, spk, emo, ref_prosody] per frame, channels-last [B][T][G]
__global__ void gs_cond_cat_kernel(const float* __restrict__ mel, const float* __restrict__ dec, const float* __restrict__ spk,
                                   const float* __restrict__ emo, const float* __restrict__ pros, float* __restrict__ g, int T, long total,
                                   int M, int H) {
  const int G = M + 4 * H;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / G;
    const int c = (int)(i - r * G);
    const long b = r / T;
    float v;
    if (c < M) v = mel[r * M + c];
    else if (c < M + H) v = dec[r * H + c - M];
    else if (c < M + 2 * H) v = spk[b * H + c - M - H];
    else if (c < M + 3 * H) v = emo[b * H + c - M - 2 * H];
    else v = pros[r * H + c - M - 3 * H];
    g[i] = v;
  }
}

// squeeze(z, 2) into the channels-last flow state: x[b][t][j * M + c] = z[b][c][2 t + j]  (z [B][M][Tz], Tz >= 2 T2)
__global__ void gs_squeeze_kernel(const float* __restrict__ z, float* __restrict__ x, int Tz, int T2, int M, long total) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / (2 * M);
    const int ch = (int)(i - r * 2 * M);
    const long b = r / T2;
    const int t = (int)(r - b * T2), j = ch / M, c = ch - j * M;
    x[i] = z[(b * M + c) * Tz + 2 * t + j];
  }
}

// One reverse step of a post-flow block on the squeezed state x [rows][C2] (C2 = 2 M), in place:
// CouplingBlock reverse (z1 = (x1 - m) * exp(-logs), m / logs = the end layer's output halves), then InvConvNear reverse
// (4 x 4 mix of the channels {a * C2/2 + 2 k + r}, group i = 2 a + r, for each k < C2/4), then ActNorm reverse.
// blk: winv[16], bias[C2], logs[C2].
__global__ void gs_flow_step_kernel(float* __restrict__ x, const float* __restrict__ e, const float* __restrict__ blk, long total, int C2) {
  const int half = C2 / 2, q = C2 / 4;
  const float* winv = blk;
  const float* bias = blk + 16;
  const float* logs = blk + 16 + C2;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / q;
    const int k = (int)(i - r * q);
    float* xr = x + r * C2;
    const float* er = e + r * C2;
    float v[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const int ch = (g >> 1) * half + 2 * k + (g & 1);
      v[g] = ch < half ? xr[ch] : __fmul_rn(__fsub_rn(xr[ch], er[ch - half]), expf(-er[ch]));
    }
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const int ch = (g >> 1) * half + 2 * k + (g & 1);
      float s = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) s = fmaf(winv[g * 4 + j], v[j], s);
      xr[ch] = __fmul_rn(__fsub_rn(s, bias[ch]), expf(-logs[ch]));
    }
  }
}

}  // namespace

void gs_sum(const float* x, const float* a, const float* e, const float* tab, const int* idx, const float* s, const float* mask, float* out,
            int T, long rows, int H, cudaStream_t st) {
  gs_sum_kernel<<<ew_grid(rows * H), 256, 0, st>>>(x, a, e, tab, idx, s, mask, out, T, rows * H, H);
  count_launch(1);
}

void gs_accum(float* dst, const float* src, long n, int first, cudaStream_t st) {
  gs_accum_kernel<<<ew_grid(n), 256, 0, st>>>(dst, src, n, first);
  count_launch(1);
}

void gs_refmask(const float* mel, float* mask, long rows, cudaStream_t st) {
  gs_refmask_kernel<<<ew_grid(rows), 256, 0, st>>>(mel, mask, rows);
  count_launch(1);
}

void gs_wn_gate(const float* a, float* acts, long rows, int C, cudaStream_t st) {
  gs_wn_gate_kernel<<<ew_grid(rows * C), 256, 0, st>>>(a, acts, rows * C, C);
  count_launch(1);
}

void gs_segmean(const float* h, const int* seg, float* out, int B, int T, int nseg, int C, cudaStream_t st) {
  gs_segmean_kernel<<<dim3(nseg, B), 128, 0, st>>>(h, seg, out, T, nseg, C);
  count_launch(1);
}

void gs_vq(const float* x, const float* dots, const float* emb, const float* enorm, int* idx, float* q, long rows, int H, int M,
           cudaStream_t st) {
  gs_vq_kernel<<<(unsigned)cdivl(rows, 8), 256, 0, st>>>(x, dots, emb, enorm, idx, q, rows, H, M);
  count_launch(1);
}

void gs_catpos(const float* p, const int* pos, float* out, long rows, int H, cudaStream_t st) {
  const float neg_emb = (float)(-(std::log(10000.0) / (double)(H / 2 - 1)));
  gs_catpos_kernel<<<ew_grid(rows * 2 * H), 256, 0, st>>>(p, pos, out, rows * 2 * H, H, neg_emb);
  count_launch(1);
}

void gs_kpm(const float* x, uint8_t* kpm, long rows, int H, cudaStream_t st) {
  gs_kpm_kernel<<<ew_grid(rows), 256, 0, st>>>(x, kpm, rows, H);
  count_launch(1);
}

void gs_pitch(const float* p1, const float* p2, const int* mel2ph, float mean, float std_, float* pitch_pred, float* f0d, float* f0d_pred,
              int* coarse, long rows, cudaStream_t st) {
  gs_pitch_kernel<<<ew_grid(rows), 256, 0, st>>>(p1, p2, mel2ph, mean, std_, f0_mel_min(), f0_mel_range(), pitch_pred, f0d, f0d_pred,
                                                 coarse, rows);
  count_launch(1);
}

void gs_cond_cat(const float* mel, const float* dec, const float* spk, const float* emo, const float* pros, float* g, int T, long rows,
                 int M, int H, cudaStream_t st) {
  gs_cond_cat_kernel<<<ew_grid(rows * (M + 4 * H)), 256, 0, st>>>(mel, dec, spk, emo, pros, g, T, rows * (M + 4 * H), M, H);
  count_launch(1);
}

void gs_squeeze(const float* z, float* x, int B, int Tz, int T2, int M, cudaStream_t st) {
  const long total = (long)B * T2 * 2 * M;
  gs_squeeze_kernel<<<ew_grid(total), 256, 0, st>>>(z, x, Tz, T2, M, total);
  count_launch(1);
}

void gs_flow_step(float* x, const float* e, const float* blk, long rows, int C2, cudaStream_t st) {
  gs_flow_step_kernel<<<ew_grid(rows * (C2 / 4)), 256, 0, st>>>(x, e, blk, rows * (C2 / 4), C2);
  count_launch(1);
}

namespace {

// A tap-GEMM on explicitly strided channels-last operands (squeezed views, column slices); epi as TapConvParams
void gs_conv(const PackedConv& pc, const float* in, int in_pitch, long in_gs, float* out, int out_pitch, long out_gs, int G, int L,
             int epi, cudaStream_t st, const float* res = nullptr, int res_pitch = 0, long res_gs = 0, int accumulate = 0,
             float scale = 1.f) {
  TapConvParams P = tapconv_params(pc, G, L, 0, 1);
  P.in = in; P.in_gstride = in_gs; P.in_pitch = in_pitch;
  P.out = out; P.out_gstride = out_gs; P.out_pitch = out_pitch;
  P.epi = epi; P.scale = scale; P.accumulate = accumulate;
  if (res) { P.res = res; P.res_gstride = res_gs; P.res_pitch = res_pitch; }
  tapconv_launch(P, st);
}

// folded weight-norm conv -> PackedConv; split rows [r0, r0 + n) of a [Cout][Cin][K] weight
void pack_rows(PackedConv& pc, const float* w, const float* b, int r0, int n, int Cin, int K) {
  pack_conv(pc, w + (size_t)r0 * Cin * K, b ? b + r0 : nullptr, n, Cin, K, false);
}

struct AlignLayer {
  PackedConv q, kv, o, f1, f2;
  DevBuf n1g, n1b, n2g, n2b;
};

struct Style {
  PackedConv wn_in[kStyleWnLayers], wn_res[kStyleWnLayers - 1], wn_skip[kStyleWnLayers];
  DevBuf lng[kStyleBlocks], lnb[kStyleBlocks];
  PackedConv c1[kStyleBlocks], c2[kStyleBlocks];
  DevBuf lastg, lastb;
  PackedConv post, vq_dot, l1;
  DevBuf emb, enorm;
  AlignLayer al[2];
};

struct GlowBlock {
  PackedConv start, end;
  std::vector<PackedConv> in, res, skip;   // filled on the blocks that own their WN layers
  DevBuf prm;                              // winv[16], ActNorm bias[C2], logs[C2]
};

}  // namespace

struct GsNet : Handle {
  agpt_gs_cfg cfg;
  // FastSpeech2 part
  DevBuf E, pitchE;
  FftStack enc, dec;
  float dec_alpha = 1.f;
  PackedConv mel_out, spk_proj, emo_proj;
  DurPredictorNet dp;
  PitchPredictorNet pp, ppi;
  Style style[3];
  PackedConv cond_all;                     // the eight blocks' cond_layers as one GEMM
  std::vector<GlowBlock> glow;
  // encode -> forward state
  int B = 0, Tt = 0, have_dur = 0;
  DevBuf enc_out, snp, skpm, dch, cum, mlen, spk, emo;
  // work
  DevBuf x, y, z, qkv, ffn, s[3], p4a, p4b, tnp, dnp, dkpm, pos, mpre;
  DevBuf rmask, sh, sa, sacts, so, sseg, cba, cbb, cbt, cnp, ckpm, dots, pq, cat, kv, kvp, kkpm, src, al_a, al_b, al_f;
  DevBuf gcond, cond, gh, ga, gacts, gskip, gend;

  const agpt_fs2_cfg& f() const { return cfg.fs2; }

  void fft(const FftStack& S, float* xs, float* out, int B_, int T, const float* nonpad, const uint8_t* kpm, cudaStream_t st) {
    S.forward(xs, out, B_, T, f().hidden_size, f().num_heads, nonpad, kpm, y.p, z.p, qkv.p, ffn.p, st);
  }

  void ensure_work(long rows) {
    const int H = f().hidden_size;
    for (auto& b : s) b.ensure((size_t)rows * std::max(H, f().predictor_hidden));
    p4a.ensure(rows * 4); p4b.ensure(rows * 4);
    x.ensure(rows * H); y.ensure(rows * H); z.ensure(rows * H); qkv.ensure(rows * 3 * H); ffn.ensure(rows * 4 * H);
  }

  void encode(const int* tok, int B_, int T, const float* spk_in, const float* emo_in, int predict, float* dur, int* dur_choice,
              int* mel_len_host, float* spk_out, float* emo_out, cudaStream_t st) {
    AGPT_CHECK(B_ >= 1 && T >= 1, "empty batch");
    const int H = f().hidden_size;
    const long rows = (long)B_ * T;
    B = B_; Tt = T; have_dur = 0;
    enc_out.ensure(rows * H); snp.ensure(rows); skpm.ensure(rows / 4 + 1); dch.ensure(rows); cum.ensure(rows); mlen.ensure(B_);
    spk.ensure((size_t)B_ * H); emo.ensure((size_t)B_ * H);
    ensure_work(rows);
    fs_embed_tokens(tok, nullptr, nullptr, nullptr, E.p, nullptr, nullptr, nullptr, nullptr, f().n_tokens, (float)std::sqrt((double)H), 1,
                    nullptr, (float)(-(std::log(10000.0) / (double)(H / 2 - 1))), 1.f, x.p, snp.p, bptr(skpm), B_, T, H, st);
    fft(enc, x.p, enc_out.p, B_, T, snp.p, bptr(skpm), st);
    fs_conv(spk_proj, spk_in, 256, spk.p, H, 1, B_, EPI_BIAS, st);
    fs_conv(emo_proj, emo_in, 256, emo.p, H, 1, B_, EPI_BIAS, st);
    if (spk_out) AGPT_CUDA(cudaMemcpyAsync(spk_out, spk.p, sizeof(float) * B_ * H, cudaMemcpyDeviceToDevice, st));
    if (emo_out) AGPT_CUDA(cudaMemcpyAsync(emo_out, emo.p, sizeof(float) * B_ * H, cudaMemcpyDeviceToDevice, st));
    // dur_inp = (encoder_out + spk + emo) * src_nonpadding (generspeech.py:87)
    gs_sum(enc_out.p, spk.p, emo.p, nullptr, nullptr, nullptr, snp.p, x.p, T, rows, H, st);
    dp.forward(x.p, H, B_, T, snp.p, s[0].p, s[1].p, s[2].p, p4a.p, st);
    fs_dur(p4a.p, snp.p, dur, predict ? iptr(dch) : nullptr, rows, st);
    if (predict) {
      fs_lr_scan(iptr(dch), iptr(cum), iptr(mlen), B_, T, st);
      if (dur_choice) AGPT_CUDA(cudaMemcpyAsync(dur_choice, dch.p, sizeof(int) * rows, cudaMemcpyDeviceToDevice, st));
      AGPT_CUDA(cudaMemcpyAsync(mel_len_host, mlen.p, sizeof(int) * B_, cudaMemcpyDeviceToHost, st));
      AGPT_CUDA(cudaStreamSynchronize(st));
      have_dur = 1;
    }
    AGPT_CUDA(cudaGetLastError());
  }

  // WN (wavenet.py:54-78) on h [rows][C] in place, skip sum -> out [rows][C]; cond (column offset into [rows][cond_pitch])
  // or null; mask or null (= ones).  a [rows][2C], acts [rows][C] scratch.
  void wn(PackedConv* in, PackedConv* res, PackedConv* skip, int layers, float* h, int C, float* out, const float* cond, int cond_pitch,
          const float* mask, int G, int L, float* a, float* acts, cudaStream_t st) {
    const long rows = (long)G * L;
    for (int i = 0; i < layers; ++i) {
      if (cond) gs_conv(in[i], h, C, (long)L * C, a, 2 * C, (long)L * 2 * C, G, L, EPI_RES, st, cond + (size_t)i * 2 * C, cond_pitch,
                        (long)L * cond_pitch);
      else gs_conv(in[i], h, C, (long)L * C, a, 2 * C, (long)L * 2 * C, G, L, EPI_BIAS, st);
      gs_wn_gate(a, acts, rows, C, st);
      if (i < layers - 1) {
        gs_conv(res[i], acts, C, (long)L * C, h, C, (long)L * C, G, L, EPI_ACC, st, nullptr, 0, 0, 1);
        if (mask) fs_affine_mask(h, nullptr, nullptr, mask, rows, C, st);
      }
      gs_conv(skip[i], acts, C, (long)L * C, out, C, (long)L * C, G, L, EPI_ACC, st, nullptr, 0, 0, i > 0);
    }
    if (mask) fs_affine_mask(out, nullptr, nullptr, mask, rows, C, st);
  }

  // LocalStyleAdaptor + positions + l1 + ProsodyAligner of one level; adds the aligned prosody [B][Tm][H] into psum
  // (first: writes it).  Returns Tk (the prosody sequence length).
  void style_level(int lvl, const float* ref, int Tr, const int* seg, int nseg, int Tm, const float* dec0, float* psum, int first,
                   float* q_out, int* idx_out, cudaStream_t st) {
    Style& S = style[lvl];
    const int H = f().hidden_size, C = kStyleC, M = cfg.n_vq;
    const long rr = (long)B * Tr;
    AGPT_CUDA(cudaMemcpyAsync(sh.p, ref, sizeof(float) * rr * C, cudaMemcpyDeviceToDevice, st));
    wn(S.wn_in, S.wn_res, S.wn_skip, kStyleWnLayers, sh.p, C, so.p, nullptr, 0, rmask.p, B, Tr, sa.p, sacts.p, st);
    int Tk = Tr;
    float* cb_in = so.p;
    if (seg) {
      Tk = nseg;
      gs_segmean(so.p, seg, sseg.p, B, Tr, nseg, C, st);
      cb_in = sseg.p;
    }
    const long rk = (long)B * Tk;
    // ConvBlocks (prosody_util.py:298-335): nonpadding of the input rows; 5 x 2 [LN -> conv k5 -> x 5^-0.5 -> GELU -> 1x1]
    fs_rowmask(cb_in, cnp.p, bptr(ckpm), rk, C, st);
    float* cur = cb_in;
    float* nxt = cba.p;
    for (int l = 0; l < kStyleBlocks; ++l) {
      layernorm(cur, cbt.p, S.lng[l].p, S.lnb[l].p, rk, C, 1e-5f, st);
      fs_conv(S.c1[l], cbt.p, C, sa.p, 2 * C, B, Tk, EPI_GELU_SCALED, st, nullptr, (float)std::pow(5.0, -0.5));
      fs_conv(S.c2[l], sa.p, 2 * C, nxt, C, 1, (int)rk, EPI_RES, st, cur);
      fs_affine_mask(nxt, nullptr, nullptr, cnp.p, rk, C, st);
      cur = nxt;
      nxt = nxt == cba.p ? cbb.p : cba.p;
    }
    layernorm(cur, cbt.p, S.lastg.p, S.lastb.p, rk, C, 1e-5f, st);
    fs_affine_mask(cbt.p, nullptr, nullptr, cnp.p, rk, C, st);
    float* q = q_out ? q_out : pq.p;
    fs_conv(S.post, cbt.p, C, q, H, B, Tk, EPI_BIAS, st);
    fs_affine_mask(q, nullptr, nullptr, cnp.p, rk, H, st);
    // VQ: x . e^T on the tap-GEMM, then argmin + gather
    fs_conv(S.vq_dot, q, H, dots.p, M, 1, (int)rk, EPI_BIAS, st);
    gs_vq(q, dots.p, S.emb.p, S.enorm.p, idx_out, q, rk, H, M, st);
    // positions of prosody[..., 0], l1(cat[prosody, positions]), key padding of its output
    fs_positions(q, iptr(pos), B, Tk, H, st);
    gs_catpos(q, iptr(pos), cat.p, rk, H, st);
    fs_conv(S.l1, cat.p, 2 * H, kv.p, H, 1, (int)rk, EPI_BIAS, st);
    gs_kpm(kv.p, bptr(kkpm), rk, H, st);
    // ProsodyAligner: 2 post-norm cross-attention layers, queries = the frame-level decoder input
    const long rq = (long)B * Tm;
    const float* sq = dec0;
    for (int i = 0; i < 2; ++i) {
      AlignLayer& A = S.al[i];
      float* outp = (i == 1 && first) ? psum : src.p;
      fs_conv(A.q, sq, H, qkv.p, H, 1, (int)rq, EPI_BIAS, st);
      fs_conv(A.kv, kv.p, H, kvp.p, 2 * H, 1, (int)rk, EPI_BIAS, st);
      attention(qkv.p, H, kvp.p, 2 * H, kvp.p + H, 2 * H, y.p, H, B, 2, H / 2, Tm, Tk, st, bptr(kkpm));
      fs_conv(A.o, y.p, H, al_a.p, H, 1, (int)rq, EPI_RES, st, sq);
      layernorm(al_a.p, al_b.p, A.n1g.p, A.n1b.p, rq, H, 1e-5f, st);
      fs_conv(A.f1, al_b.p, H, al_f.p, kAlignFfn, 1, (int)rq, EPI_RELU, st);
      fs_conv(A.f2, al_f.p, kAlignFfn, al_a.p, H, 1, (int)rq, EPI_RES, st, al_b.p);
      layernorm(al_a.p, outp, A.n2g.p, A.n2b.p, rq, H, 1e-5f, st);
      sq = outp;
    }
    if (!first) {
      gs_accum(psum, src.p, rq * H, 0, st);
    }
  }

  void forward(int Tm, const int* mel2ph_in, int* mel2ph_out, const float* ref, int Tr, const int* ref_mel2ph, int nseg_ph,
               const int* ref_mel2word, int nseg_word, const float* znoise, float f0_mean, float f0_std, float* pitch_pred, float* f0d,
               float* f0d_pred, int* coarse, float* dec_inp, float* ref_prosody, float* mel, const agpt_gs_taps* taps, cudaStream_t st) {
    AGPT_CHECK(B >= 1, "agpt_gs_forward before agpt_gs_encode");
    AGPT_CHECK(Tm >= 2, "the post-flow needs at least 2 mel frames");
    AGPT_CHECK(Tr >= 1 && nseg_ph >= 1 && nseg_word >= 1, "empty reference");
    AGPT_CHECK(mel2ph_in || have_dur, "mel2ph not given and durations not predicted by the last encode");
    AGPT_CHECK(ref && ref_mel2ph && ref_mel2word && znoise && pitch_pred && f0d && f0d_pred && coarse && dec_inp && ref_prosody && mel,
               "null argument");
    const int H = f().hidden_size, C = kStyleC, M = cfg.n_vq, Mo = f().out_dims;
    const long rows = (long)B * Tm, trow = (long)B * Tt;
    const long rr = (long)B * Tr, rk = (long)B * std::max(Tr, std::max(nseg_ph, nseg_word));
    const int T2 = Tm / 2, hid = cfg.glow_hidden, L = cfg.glow_layers, NB = cfg.glow_blocks;
    const int Gc = Mo + 4 * H, CC = NB * 2 * hid * L;
    const long r2 = (long)B * T2;
    // every buffer is sized before any pointer into one is taken
    tnp.ensure(rows); dnp.ensure(rows); dkpm.ensure(rows / 4 + 1); pos.ensure(std::max(rows, rk));
    ensure_work(std::max(rows, trow));
    rmask.ensure(rr); sh.ensure(rr * C); so.ensure(rr * C); sa.ensure(std::max(rr, rk) * 2 * C); sacts.ensure(rr * C);
    sseg.ensure(rk * C); cba.ensure(rk * C); cbb.ensure(rk * C); cbt.ensure(rk * C); cnp.ensure(rk); ckpm.ensure(rk / 4 + 1);
    dots.ensure(rk * M); pq.ensure(rk * H); cat.ensure(rk * 2 * H); kv.ensure(rk * H); kvp.ensure(rk * 2 * H); kkpm.ensure(rk / 4 + 1);
    src.ensure(rows * H); al_a.ensure(rows * H); al_b.ensure(rows * H); al_f.ensure(rows * kAlignFfn);
    gcond.ensure(rows * Gc); cond.ensure(r2 * CC); gh.ensure(r2 * hid); ga.ensure(r2 * 2 * hid); gacts.ensure(r2 * hid);
    gskip.ensure(r2 * hid); gend.ensure(r2 * 2 * Mo); mpre.ensure(rows * Mo);
    float* melpre = taps && taps->mel_pre_flow ? taps->mel_pre_flow : mpre.p;

    const int* m2p = mel2ph_in;
    if (!m2p) {
      AGPT_CHECK(mel2ph_out, "mel2ph output required when it is predicted");
      fs_lr_fill(iptr(cum), iptr(mlen), mel2ph_out, B, Tt, Tm, st);
      m2p = mel2ph_out;
    }
    fs_gather(enc_out.p, m2p, x.p, tnp.p, B, Tt, Tm, H, st);      // decoder_inp after expand_states (MixStyle: identity)
    // ---- the three prosody levels (generspeech.py:96-98)
    gs_refmask(ref, rmask.p, rr, st);
    const int* segs[3] = {nullptr, ref_mel2ph, ref_mel2word};
    const int nsegs[3] = {Tr, nseg_ph, nseg_word};
    for (int l = 0; l < 3; ++l)
      style_level(l, ref, Tr, segs[l], nsegs[l], Tm, x.p, ref_prosody, l == 0, taps ? taps->prosody[l] : nullptr,
                  taps ? taps->vq_idx[l] : nullptr, st);
    // ---- pitch (inpaint_pitch): pitch_predictor(decoder_inp * tgt) + pitch_inpainter((decoder_inp + spk + emo + prosody) * tgt)
    pp.forward(x.p, H, B, Tm, s[0].p, s[1].p, s[2].p, p4a.p, st);
    gs_sum(x.p, spk.p, emo.p, nullptr, nullptr, ref_prosody, tnp.p, y.p, Tm, rows, H, st);
    ppi.forward(y.p, H, B, Tm, s[0].p, s[1].p, s[2].p, p4b.p, st);
    gs_pitch(p4a.p, p4b.p, m2p, f0_mean, f0_std, pitch_pred, f0d, f0d_pred, coarse, rows, st);
    // ---- decoder_inp = (decoder_inp + spk + emo + pitch_embed + prosody) * tgt, FFT decoder, mel_out
    gs_sum(x.p, spk.p, emo.p, pitchE.p, coarse, ref_prosody, tnp.p, dec_inp, Tm, rows, H, st);
    fs_rowmask(dec_inp, dnp.p, bptr(dkpm), rows, H, st);
    fs_positions(dec_inp, iptr(pos), B, Tm, H, st);
    fs_posemb_add(dec_inp, x.p, iptr(pos), dec_alpha, rows, H, st);
    fft(dec, x.p, y.p, B, Tm, dnp.p, bptr(dkpm), st);
    fs_conv(mel_out, y.p, H, melpre, Mo, 1, (int)rows, EPI_BIAS, st);
    fs_affine_mask(melpre, nullptr, nullptr, tnp.p, rows, Mo, st);
    // ---- Glow post-flow, reverse (generspeech.py:233-260): the squeezed views are strided reads of [B][Tm][*]
    gs_cond_cat(melpre, dec_inp, spk.p, emo.p, ref_prosody, gcond.p, Tm, rows, Mo, H, st);
    gs_conv(cond_all, gcond.p, 2 * Gc, (long)Tm * Gc, cond.p, CC, (long)T2 * CC, B, T2, EPI_BIAS, st);
    gs_squeeze(znoise, mel, B, Tm, T2, Mo, st);
    const int C2 = 2 * Mo;
    for (int b = NB - 1; b >= 0; --b) {
      GlowBlock& G = glow[b];
      GlowBlock& W = glow[b - b % std::max(cfg.share_wn_layers, 1)];
      gs_conv(G.start, mel, C2, (long)T2 * C2, gh.p, hid, (long)T2 * hid, B, T2, EPI_BIAS, st);
      wn(W.in.data(), W.res.data(), W.skip.data(), L, gh.p, hid, gskip.p, cond.p + (size_t)b * 2 * hid * L, CC, nullptr, B, T2, ga.p,
         gacts.p, st);
      gs_conv(G.end, gskip.p, hid, (long)T2 * hid, gend.p, C2, (long)T2 * C2, B, T2, EPI_BIAS, st);
      gs_flow_step(mel, gend.p, G.prm.p, r2, C2, st);
    }
    AGPT_CUDA(cudaGetLastError());
  }
};

Handle* gs_create(const agpt_gs_cfg* cfg, const float* const* W, int nW, int device) {
  DeviceGuard dg_(device);
  const agpt_fs2_cfg& c = cfg->fs2;
  const int H = c.hidden_size, P = c.predictor_hidden, C = kStyleC, M = cfg->n_vq, Mo = c.out_dims;
  AGPT_CHECK(H % 16 == 0 && c.num_heads >= 1 && H % c.num_heads == 0 && H % 2 == 0 && P % 4 == 0 && Mo == 80 && c.n_tokens >= 1 &&
                 c.enc_ffn_kernel % 2 == 1 && c.dec_ffn_kernel % 2 == 1 && c.enc_ffn_kernel <= kMaxTaps && c.dec_ffn_kernel <= kMaxTaps &&
                 c.dur_predictor_kernel % 2 == 1 && c.dur_predictor_kernel <= kMaxTaps && c.predictor_kernel % 2 == 1 &&
                 c.predictor_kernel <= kMaxTaps && c.pitch_type == 1 && !c.use_energy_embed && !c.use_midi && !c.rel_pos &&
                 c.use_pos_embed && M >= 2 && cfg->glow_hidden % 4 == 0 && cfg->glow_kernel % 2 == 1 && cfg->glow_kernel <= kMaxTaps &&
                 cfg->glow_blocks >= 1 && cfg->glow_layers >= 1 && cfg->share_wn_layers >= 0,
             "bad GenerSpeech config");
  std::unique_ptr<GsNet> h(new GsNet());
  h->magic = kMagicGs; h->device = device; h->cfg = *cfg;
  WeightCursor wc{W, nW};
  // the FastSpeech2 keys, in specs.fs2_param_shapes order
  h->E.upload(wc.next(), (size_t)c.n_tokens * H);
  wc.next();                                                      // encoder.embed_tokens.weight (the same tensor)
  wc.next();                                                      // encoder.embed_positions._float_tensor
  h->enc.load(wc, H, c.enc_layers, c.enc_ffn_kernel);
  h->dec_alpha = wc.next()[0];
  wc.next();                                                      // decoder.embed_positions._float_tensor
  h->dec.load(wc, H, c.dec_layers, c.dec_ffn_kernel);
  { auto w = wc.next(); auto b = wc.next(); pack_conv(h->mel_out, w, b, Mo, H, 1, false); }
  h->dp.load(wc, H, P, c.dur_predictor_kernel, c.dur_predictor_layers);
  h->pitchE.upload(wc.next(), (size_t)300 * H);
  h->pp.load(wc, H, P, c.predictor_kernel, c.predictor_layers, 2);
  { auto w = wc.next(); auto b = wc.next(); pack_conv(h->spk_proj, w, b, H, 256, 1, false); }
  { auto w = wc.next(); auto b = wc.next(); pack_conv(h->emo_proj, w, b, H, 256, 1, false); }
  for (auto& S : h->style) {
    for (int i = 0; i < kStyleWnLayers; ++i) { auto w = wc.next(); auto b = wc.next(); pack_conv(S.wn_in[i], w, b, 2 * C, C, 3, false); }
    for (int i = 0; i < kStyleWnLayers; ++i) {
      auto w = wc.next(); auto b = wc.next();
      if (i < kStyleWnLayers - 1) { pack_rows(S.wn_res[i], w, b, 0, C, C, 1); pack_rows(S.wn_skip[i], w, b, C, C, C, 1); }
      else pack_rows(S.wn_skip[i], w, b, 0, C, C, 1);
    }
    for (int l = 0; l < kStyleBlocks; ++l) {
      { auto g = wc.next(); auto b = wc.next(); S.lng[l].upload(g, C); S.lnb[l].upload(b, C); }
      { auto w = wc.next(); auto b = wc.next(); pack_conv(S.c1[l], w, b, 2 * C, C, 5, false); }
      { auto w = wc.next(); auto b = wc.next(); pack_conv(S.c2[l], w, b, C, 2 * C, 1, false); }
    }
    { auto g = wc.next(); auto b = wc.next(); S.lastg.upload(g, C); S.lastb.upload(b, C); }
    { auto w = wc.next(); auto b = wc.next(); pack_conv(S.post, w, b, H, C, 3, false); }
    {  // codebook [M][H]: the distance GEMM's weight, the gather table and |e|^2 (torch.sum(e ** 2, 1) in fp32)
      const float* e = wc.next();
      pack_conv(S.vq_dot, e, nullptr, M, H, 1, false);
      S.emb.upload(e, (size_t)M * H);
      std::vector<float> n(M);
      for (int m = 0; m < M; ++m) { float a = 0.f; for (int k = 0; k < H; ++k) a += e[(size_t)m * H + k] * e[(size_t)m * H + k]; n[m] = a; }
      S.enorm.upload(n);
    }
    { auto w = wc.next(); auto b = wc.next(); pack_conv(S.l1, w, b, H, 2 * H, 1, false); }
    for (auto& A : S.al) {
      auto w = wc.next(); auto b = wc.next();
      pack_rows(A.q, w, b, 0, H, H, 1);
      pack_rows(A.kv, w, b, H, 2 * H, H, 1);
      { auto ow = wc.next(); auto ob = wc.next(); pack_conv(A.o, ow, ob, H, H, 1, false); }
      { auto fw = wc.next(); auto fb = wc.next(); pack_conv(A.f1, fw, fb, kAlignFfn, H, 1, false); }
      { auto g = wc.next(); auto bb = wc.next(); A.n1g.upload(g, H); A.n1b.upload(bb, H); }
      { auto fw = wc.next(); auto fb = wc.next(); pack_conv(A.f2, fw, fb, H, kAlignFfn, 1, false); }
      { auto g = wc.next(); auto bb = wc.next(); A.n2g.upload(g, H); A.n2b.upload(bb, H); }
    }
  }
  h->ppi.load(wc, H, H, c.predictor_kernel, 3, 2);
  const int hid = cfg->glow_hidden, L = cfg->glow_layers, NB = cfg->glow_blocks, C2 = 2 * Mo, Gc = Mo + 4 * H;
  { auto w = wc.next(); auto b = wc.next(); pack_conv(h->cond_all, w, b, NB * 2 * hid * L, 2 * Gc, 1, false); }
  h->glow.resize(NB);
  for (int b = 0; b < NB; ++b) {
    GlowBlock& G = h->glow[b];
    { auto w = wc.next(); auto bb = wc.next(); pack_conv(G.start, w, bb, hid, Mo, 1, false); }
    { auto w = wc.next(); auto bb = wc.next(); pack_conv(G.end, w, bb, C2, hid, 1, false); }
    { auto wi = wc.next(); auto bi = wc.next(); auto lg = wc.next();
      std::vector<float> prm(16 + 2 * C2);
      memcpy(prm.data(), wi, sizeof(float) * 16);
      memcpy(prm.data() + 16, bi, sizeof(float) * C2);
      memcpy(prm.data() + 16 + C2, lg, sizeof(float) * C2);
      G.prm.upload(prm); }
    if (cfg->share_wn_layers == 0 || b % cfg->share_wn_layers == 0) {
      G.in.resize(L); G.res.resize(L > 1 ? L - 1 : 1); G.skip.resize(L);
      for (int i = 0; i < L; ++i) { auto w = wc.next(); auto bb = wc.next(); pack_conv(G.in[i], w, bb, 2 * hid, hid, cfg->glow_kernel, false); }
      for (int i = 0; i < L; ++i) {
        auto w = wc.next(); auto bb = wc.next();
        if (i < L - 1) { pack_rows(G.res[i], w, bb, 0, hid, hid, 1); pack_rows(G.skip[i], w, bb, hid, hid, hid, 1); }
        else pack_rows(G.skip[i], w, bb, 0, hid, hid, 1);
      }
    }
  }
  wc.done();
  return h.release();
}

void gs_encode(Handle* hh, const int* tok, int B, int T, const float* spk, const float* emo, int predict, float* dur, int* dur_choice,
               int* mel_len_host, float* spk_out, float* emo_out, cudaStream_t st) {
  auto* h = static_cast<GsNet*>(hh);
  DeviceGuard dg_(h->device);
  h->encode(tok, B, T, spk, emo, predict, dur, dur_choice, mel_len_host, spk_out, emo_out, st);
}

void gs_forward(Handle* hh, int Tm, const int* mel2ph, int* mel2ph_out, const float* ref_mels, int Tr, const int* ref_mel2ph, int nseg_ph,
                const int* ref_mel2word, int nseg_word, const float* z, float f0_mean, float f0_std, float* pitch_pred, float* f0d,
                float* f0d_pred, int* coarse, float* dec_inp, float* ref_prosody, float* mel, const agpt_gs_taps* taps, cudaStream_t st) {
  auto* h = static_cast<GsNet*>(hh);
  DeviceGuard dg_(h->device);
  h->forward(Tm, mel2ph, mel2ph_out, ref_mels, Tr, ref_mel2ph, nseg_ph, ref_mel2word, nseg_word, z, f0_mean, f0_std, pitch_pred, f0d,
             f0d_pred, coarse, dec_inp, ref_prosody, mel, taps, st);
}

}  // namespace agpt
