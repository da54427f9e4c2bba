// Sound extraction on sm_90a: LASSNet (the SoundExtraction tool's text-queried separation network) and the tool's
// conv-STFT / inverse STFT.
// Reference: sound_extraction/model/LASSNet.py, text_encoder.py (bert-mini, [CLS] row -> Linear(256, 256) + ReLU),
// resunet_film.py (UNetRes_FiLM), modules.py:169-214 (EncoderBlockRes2BCond / DecoderBlockRes2BCond), :326-379
// (ConvBlockResCond), film.py; sound_extraction/utils/stft.py:53-147 (STFT transform / inverse, window_sumsquare).
//
// Activations are channels-last rows [B][T][F][C].  Every contraction is a tap-GEMM (tcconv5 on the tensor cores; the
// 511-, 255- and 127-wide maps in strip mode, as the VAE's wide maps):
// - ConvBlockResCond, eval BatchNorm: h = conv1(lrelu(bn1(x))) + film1 only feeds bn2, so bn2 is folded into conv1
//   (weights x s2, EPI_ADDVEC vector s2 film1 + t2) and conv2 reads it through PRO_LRELU; bn1(x) is written by a
//   per-channel affine pass (the conv's zero padding then stays zero under PRO_LRELU), which also writes the residual
//   x + film2 of the identity blocks.  The shortcut blocks' 1x1 conv adds film_res + film2 in its EPI_ADDVEC epilogue,
//   so conv2 always ends in a plain EPI_RES.  The first block's single input channel is padded to 4: channel 0 carries
//   bn1(x) for conv1, channel 1 the raw x for the shortcut.
// - FiLM: the 63 Film MLPs depend on the text condition only; they run once per request as one GEMM for every first
//   Linear (EPI_RELU) and one grouped kernel for the second Linears that writes each block's two vectors pre-combined.
// - ConvTranspose2d(k3, s2, p0) + prune: output phase (a, b) of input pixel (m, n) is a sum over the 2 x 2 input
//   neighbourhood {m, m - 1} x {n, n - 1}; one im2col pass (with the decoder's BatchNorm and ReLU applied) feeds one
//   GEMM with 4 C_in -> 4 C_out channels (9 of its 16 weight blocks are non-zero), and one pass shuffles the phases
//   into the concat buffer next to the encoder's skip: 2h rows (the prune) by 2w + 1 columns.
// - after_conv2 (1x1 + bias), the two-bin pad, the T crop and the sigmoid are one store.
// STFT: both directions are 2-tap GEMMs over hop-sample rows (filter_length = 2 hop): transform = reflect-padded signal
// [rows][hop] x forward_basis halves -> [re | im], then magnitude / phase; inverse = [mag cos | mag sin] frames x
// inverse_basis halves at row offsets {0, -1} -> the overlap-added signal, divided by the window sum where it exceeds
// fp32 tiny, times filter_length / hop, cropped.
#include <cmath>
#include <limits>
#include "common.cuh"
#include "tapconv.cuh"
#include "nn_kernels.h"
#include "models.h"
#include "clap.cuh"
#include "audio_front.cuh"
#include "an_kernels.cuh"

namespace agpt {

namespace {

constexpr int kLevels = 6;
constexpr int kEncCh[kLevels] = {32, 64, 128, 256, 384, 384};
constexpr int kCond = 256;
constexpr float kBnEps = 1e-5f;
constexpr float kSlope = 0.01f;   // F.leaky_relu_(..., negative_slope=0.01)

unsigned ew_blocks(long n) { return (unsigned)std::min<long>(cdivl(n, 256), 8192); }

// img[b][t][f][0..3] = {s x + sh, x, 0, 0}, x = mag[b, t, f] for t < T (zero in the padded rows t >= T), f < W
__global__ void lass_input_kernel(const float* __restrict__ mag, long sb, long st, long sf, int T, int Tp, int W, float s,
                                  float sh, float4* __restrict__ img, long total) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long bt = i / W;
    const int f = (int)(i - bt * W);
    const long b = bt / Tp;
    const int t = (int)(bt - b * Tp);
    const float x = t < T ? mag[b * sb + (long)t * st + (long)f * sf] : 0.f;
    img[i] = make_float4(fmaf(x, s, sh), x, 0.f, 0.f);
  }
}

// a = x * s[c] + t[c]; r (optional) = x + vec[b][c], b = row / rows_per_sample.  C % 4 == 0.
__global__ void lass_affine_kernel(const float4* __restrict__ x, const float4* __restrict__ s, const float4* __restrict__ t,
                                   float4* __restrict__ a, float4* __restrict__ r, const float* __restrict__ vec, int vec_len,
                                   long rows_per_sample, int C4, long total) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    const float4 v = x[i], sc = s[c], sh = t[c];
    a[i] = make_float4(fmaf(v.x, sc.x, sh.x), fmaf(v.y, sc.y, sh.y), fmaf(v.z, sc.z, sh.z), fmaf(v.w, sc.w, sh.w));
    if (r) {
      const long b = (i / C4) / rows_per_sample;
      const float4 e = reinterpret_cast<const float4*>(vec + b * vec_len)[c];
      r[i] = make_float4(v.x + e.x, v.y + e.y, v.z + e.z, v.w + e.w);
    }
  }
}

// col[b][m][n][k C + c] = relu(y[b][m + dh_k][n + dw_k][c] s[c] + t[c]) (zero outside the h x w map), n in [0, w]:
// the transposed conv's 2 x 2 neighbourhood, taps k = (0, 0), (0, -1), (-1, 0), (-1, -1)
__global__ void lass_upcol_kernel(const float4* __restrict__ y, const float4* __restrict__ s, const float4* __restrict__ t, int h,
                                  int w, int C4, float4* __restrict__ col, long total) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    long q = i / C4;
    const int k = (int)(q % 4);
    q /= 4;
    const int n = (int)(q % (w + 1));
    q /= (w + 1);
    const int m = (int)(q % h);
    const long b = q / h;
    const int mm = m - (k >> 1), nn = n - (k & 1);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (mm >= 0 && nn >= 0 && nn < w) {
      const float4 x = y[((b * h + mm) * w + nn) * C4 + c], sc = s[c], sh = t[c];
      v = make_float4(fmaxf(fmaf(x.x, sc.x, sh.x), 0.f), fmaxf(fmaf(x.y, sc.y, sh.y), 0.f), fmaxf(fmaf(x.z, sc.z, sh.z), 0.f),
                      fmaxf(fmaf(x.w, sc.w, sh.w), 0.f));
    }
    col[i] = v;
  }
}

// cat[b][r][c'] (2h x (2w + 1) map, 2 C channels): c' < C from phase (r & 1, col & 1) of up[b][r / 2][col / 2],
// c' >= C from the encoder's skip [b][r][col][c' - C]
__global__ void lass_shuffle_kernel(const float4* __restrict__ up, const float4* __restrict__ skip, int h, int w, int C4,
                                    float4* __restrict__ cat, long total) {
  const int W2 = 2 * w + 1;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % (2 * C4));
    const long p = i / (2 * C4);            // pixel of the 2h x W2 map
    if (c >= C4) { cat[i] = skip[p * C4 + (c - C4)]; continue; }
    const int col = (int)(p % W2);
    const long br = p / W2;
    const int r = (int)(br % (2 * h));
    const long b = br / (2 * h);
    const int ph = (r & 1) * 2 + (col & 1);
    cat[i] = up[(((b * h + (r >> 1)) * (w + 1) + (col >> 1)) * 4 + ph) * C4 + c];
  }
}

// The FiLM second Linears, one warp per (sample, job): film(o) = relu(w2[o] . hid[o's slice] + b2[o]);
// vec[b][dst] = alpha film(A) + beta (+ film(B))
__global__ void lass_film_kernel(const float* __restrict__ hid, int hid_len, const float* __restrict__ w2, FilmJobs J, int nj,
                                 int B, float* __restrict__ vec, int vec_len) {
  const int warp = (int)(((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (warp >= nj * B) return;
  const int b = warp / nj, j = warp - b * nj;
  const float* hb = hid + (long)b * hid_len;
  auto film = [&](int o) {
    const float* wr = w2 + J.woff[o];
    const float* hr = hb + J.hoff[o];
    float s = 0.f;
    for (int k = lane; k < J.nin[o]; k += 32) s = fmaf(wr[k], hr[k], s);
    for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
    return fmaxf(s + J.b2[o], 0.f);
  };
  float v = fmaf(J.alpha[j], film(J.ja[j]), J.beta[j]);
  if (J.jb[j] >= 0) v += film(J.jb[j]);
  if (lane == 0) vec[(long)b * vec_len + J.dst[j]] = v;
}

// after_conv2 + F.pad(x, (0, 2)) + crop to T + sigmoid: x [B][Tp][W][32] -> mask / logits [B][T][F], F = W + 2
__global__ void lass_head_kernel(const float* __restrict__ x, const float* __restrict__ wb, int T, int Tp, int W, int F,
                                 float* __restrict__ mask, float* __restrict__ logits, long total) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long bt = i / F;
    const int f = (int)(i - bt * F);
    const long b = bt / T;
    const int t = (int)(bt - b * T);
    float v = 0.f;
    if (f < W) {
      const float4* r = reinterpret_cast<const float4*>(x + ((b * Tp + t) * W + f) * 32);
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float4 a = r[k];
        s = fmaf(a.x, wb[4 * k], s); s = fmaf(a.y, wb[4 * k + 1], s); s = fmaf(a.z, wb[4 * k + 2], s); s = fmaf(a.w, wb[4 * k + 3], s);
      }
      v = s + wb[32];
    }
    mask[i] = 1.f / (1.f + expf(-v));
    if (logits) logits[i] = v;
  }
}

// rows[b][r][j] = padded sample r * hop + j of wav b (reflect-padded by n / 2 on each side, zero past the end)
__global__ void stft_rows_kernel(const float* __restrict__ wav, long N, int half, int hop, long R, float* __restrict__ rows, long total) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long b = i / (R * hop);
    const long s = i - b * R * hop;
    float v = 0.f;
    if (s < N + 2 * half) {
      long k = s - half;
      k = k < 0 ? -k : (k >= N ? 2 * (N - 1) - k : k);
      v = wav[b * N + k];
    }
    rows[i] = v;
  }
}

// spec [B][R][pitch] ([re | im] per frame) -> magnitude / phase [B][nb][T]
__global__ void stft_magphase_kernel(const float* __restrict__ spec, long R, int pitch, int nb, int T, float* __restrict__ mag,
                                     float* __restrict__ phase, long total) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int t = (int)(i % T);
    const long bf = i / T;
    const int f = (int)(bf % nb);
    const long b = bf / nb;
    const float* p = spec + (b * R + t) * pitch;
    const float re = p[f], im = p[nb + f];
    mag[i] = sqrtf(__fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im)));
    phase[i] = atan2f(im, re);
  }
}

// X[b][t][c] (T + 1 rows, the last zero; pitch channels, zero past 2 nb) = [mag cos(phase) | mag sin(phase)]
__global__ void istft_frames_kernel(const float* __restrict__ mag, const float* __restrict__ phase, int nb, int T, int pitch,
                                    float* __restrict__ X, long total) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % pitch);
    const long bt = i / pitch;
    const int t = (int)(bt % (T + 1));
    const long b = bt / (T + 1);
    float v = 0.f;
    if (t < T && c < 2 * nb) {
      const int f = c < nb ? c : c - nb;
      const long k = (b * nb + f) * T + t;
      v = __fmul_rn(mag[k], c < nb ? cosf(phase[k]) : sinf(phase[k]));
    }
    X[i] = v;
  }
}

// out[b][i] = y[b][i + half] / ws[i + half] (where ws > tiny) * scale, i < (T - 1) hop
__global__ void istft_finish_kernel(const float* __restrict__ y, long ylen, const float* __restrict__ ws, int half, float scale,
                                    long n_out, float* __restrict__ out, long total) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long b = i / n_out;
    const long s = i - b * n_out + half;
    float v = y[b * ylen + s];
    const float w = ws[s];
    if (w > std::numeric_limits<float>::min()) v = __fdiv_rn(v, w);
    out[i] = __fmul_rn(v, scale);
  }
}

}  // namespace

void lass_affine(const float* x, const float* s, const float* t, float* a, float* r, const float* vec, int vec_len, int vec_off,
                 long rows, long rows_per_sample, int C, cudaStream_t st) {
  AGPT_CHECK(C >= 4 && C % 4 == 0, "LASS affine: C % 4 == 0 (float4 rows)");
  AGPT_CHECK(rows >= 1 && rows_per_sample >= 1, "LASS affine: rows >= 1 and rows_per_sample >= 1");
  AGPT_CHECK(!r || (vec_off >= 0 && (long)vec_off + C <= vec_len), "LASS affine: the vector slice must fit in vec_len");
  AGPT_CHECK(!r || (vec_off % 4 == 0 && vec_len % 4 == 0), "LASS affine: vec_off and vec_len must be multiples of 4 (float4 reads)");
  const long tot = rows * (C / 4);
  lass_affine_kernel<<<ew_blocks(tot), 256, 0, st>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<const float4*>(s), reinterpret_cast<const float4*>(t),
      reinterpret_cast<float4*>(a), reinterpret_cast<float4*>(r), vec ? vec + vec_off : nullptr, vec_len, rows_per_sample, C / 4,
      tot);
  count_launch(1);
}

void lass_upcol(const float* y, const float* s, const float* t, int B, int h, int w, int C, float* col, cudaStream_t st) {
  AGPT_CHECK(C >= 4 && C % 4 == 0, "LASS upcol: C % 4 == 0 (float4 rows)");
  AGPT_CHECK(B >= 1 && h >= 1 && w >= 1, "LASS upcol: B, h, w >= 1");
  const long tot = (long)B * h * (w + 1) * 4 * (C / 4);
  lass_upcol_kernel<<<ew_blocks(tot), 256, 0, st>>>(reinterpret_cast<const float4*>(y), reinterpret_cast<const float4*>(s),
                                                   reinterpret_cast<const float4*>(t), h, w, C / 4, reinterpret_cast<float4*>(col),
                                                   tot);
  count_launch(1);
}

void lass_shuffle(const float* up, const float* skip, int B, int h, int w, int C, float* cat, cudaStream_t st) {
  AGPT_CHECK(C >= 4 && C % 4 == 0, "LASS shuffle: C % 4 == 0 (float4 rows)");
  AGPT_CHECK(B >= 1 && h >= 1 && w >= 1, "LASS shuffle: B, h, w >= 1");
  const long tot = (long)B * (2 * h) * (2 * w + 1) * 2 * (C / 4);
  lass_shuffle_kernel<<<ew_blocks(tot), 256, 0, st>>>(reinterpret_cast<const float4*>(up), reinterpret_cast<const float4*>(skip),
                                                     h, w, C / 4, reinterpret_cast<float4*>(cat), tot);
  count_launch(1);
}

void lass_film(const float* hid, int hid_len, const float* w2, const FilmJobs& J, int nj, int B, float* vec, int vec_len,
               cudaStream_t st) {
  AGPT_CHECK(nj >= 1 && B >= 1 && hid_len >= 1 && vec_len >= 1, "LASS FiLM: nj, B, hid_len, vec_len >= 1");
  const long warps = (long)nj * B;
  lass_film_kernel<<<(unsigned)cdivl(warps * 32, 256), 256, 0, st>>>(hid, hid_len, w2, J, nj, B, vec, vec_len);
  count_launch(1);
}

void lass_input(const float* mag, long sb, long stt, long sf, int B, int T, int Tp, int W, float s, float sh, float* img,
                cudaStream_t st) {
  AGPT_CHECK(B >= 1 && T >= 1 && Tp >= T && W >= 1, "LASS input: bad sizes");
  const long tot = (long)B * Tp * W;
  lass_input_kernel<<<ew_blocks(tot), 256, 0, st>>>(mag, sb, stt, sf, T, Tp, W, s, sh, reinterpret_cast<float4*>(img), tot);
  count_launch(1);
}

void lass_head(const float* x, const float* wb, int B, int T, int Tp, int W, float* mask, float* logits, cudaStream_t st) {
  AGPT_CHECK(B >= 1 && T >= 1 && Tp >= T && W >= 1, "LASS head: bad sizes");
  const int F = W + 2;
  const long tot = (long)B * T * F;
  lass_head_kernel<<<ew_blocks(tot), 256, 0, st>>>(x, wb, T, Tp, W, F, mask, logits, tot);
  count_launch(1);
}

void stft_rows(const float* wav, int B, long N, int n, int hop, float* rows, cudaStream_t st) {
  AGPT_CHECK(B >= 1 && n >= 2 && hop >= 1, "STFT rows: bad sizes");
  if (N <= n / 2)
    throw Error("STFT: " + std::to_string(N) + " samples are too few for the reflect padding of " + std::to_string(n / 2));
  const long R = cdivl(N + n, hop);
  stft_rows_kernel<<<ew_blocks((long)B * R * hop), 256, 0, st>>>(wav, N, n / 2, hop, R, rows, (long)B * R * hop);
  count_launch(1);
}

void stft_magphase(const float* spec, int B, long R, int pitch, int nb, int T, float* mag, float* phase, cudaStream_t st) {
  AGPT_CHECK(B >= 1 && T >= 1 && T <= R && nb >= 1 && pitch >= 2 * nb, "STFT magnitude / phase: bad sizes");
  const long tot = (long)B * nb * T;
  stft_magphase_kernel<<<ew_blocks(tot), 256, 0, st>>>(spec, R, pitch, nb, T, mag, phase, tot);
  count_launch(1);
}

void istft_frames(const float* mag, const float* phase, int B, int nb, int T, int pitch, float* X, cudaStream_t st) {
  AGPT_CHECK(B >= 1 && T >= 2, "the inverse STFT needs at least two frames");
  AGPT_CHECK(nb >= 1 && pitch >= 2 * nb, "inverse STFT frames: bad sizes");
  const long tot = (long)B * (T + 1) * pitch;
  istft_frames_kernel<<<ew_blocks(tot), 256, 0, st>>>(mag, phase, nb, T, pitch, X, tot);
  count_launch(1);
}

void istft_finish(const float* y, const float* ws, int B, int T, int n, int hop, float* out, cudaStream_t st) {
  AGPT_CHECK(B >= 1 && T >= 2, "the inverse STFT needs at least two frames");
  AGPT_CHECK(hop >= 1 && n == 2 * hop, "inverse STFT: filter_length = 2 hop_length");
  const long n_out = (long)(T - 1) * hop;
  istft_finish_kernel<<<ew_blocks((long)B * n_out), 256, 0, st>>>(y, (long)(T + 1) * hop, ws, n / 2, (float)n / (float)hop, n_out,
                                                                  out, (long)B * n_out);
  count_launch(1);
}

namespace {

// Every ConvBlockResCond of the UNet; vector offsets index the per-sample FiLM vector buffer
struct LBlock {
  int cin = 0, cout = 0;
  bool sc = false;
  DevBuf s1, t1;                 // bn1 as a per-channel affine (not used by the first block)
  PackedConv conv1, conv2, shortcut;
  int e1 = 0, r2 = 0;            // offsets of s2 film1 + t2 and of film2 (+ film_res)
};
struct LDec {
  int cin = 0, cout = 0;
  DevBuf s, t;                   // bn1 of the decoder block
  PackedConv up;                 // [4 C_in] -> [4 C_out]: the four output phases of the transposed conv
};

void bn_fold(WeightCursor& wc, int c, std::vector<float>& s, std::vector<float>& t) {
  const float* g = wc.next(); const float* be = wc.next(); const float* rm = wc.next(); const float* rv = wc.next();
  s.resize(c); t.resize(c);
  for (int i = 0; i < c; ++i) { s[i] = g[i] / sqrtf(rv[i] + kBnEps); t[i] = be[i] - rm[i] * s[i]; }
}

}  // namespace

struct LassNet : Handle {
  agpt_lass_cfg cfg;
  ClapNet bert;
  PackedConv lin, film1;
  std::vector<LBlock> blocks;       // 26, in forward order
  LDec dec[kLevels];
  float in_s = 1.f, in_t = 0.f;     // the first block's bn1 (one channel)
  DevBuf head;                      // after_conv2: 32 weights, then the bias
  // FiLM: host tables while loading, then device
  std::vector<float> h_w1, h_b1, h_w2, h_b2, h_alpha, h_beta;
  std::vector<int> h_woff, h_hoff, h_nin, h_dst, h_ja, h_jb;
  int hid_len = 0, vec_len = 0, njobs = 0;
  DevBuf w2, ftab, hid, vec, zeros, lin_out;
  DevBuf bx, bo, ba, bh, br, cat, col, upb, skip[kLevels];

  // one Film (Linear(256, 2c) -> ReLU -> Linear(2c, c) -> ReLU): returns the index of its first output
  int load_film(WeightCursor& wc, int c) {
    const float* w1 = wc.next(); const float* b1 = wc.next(); const float* wt = wc.next(); const float* b2 = wc.next();
    const int h0 = hid_len, o0 = (int)h_b2.size();
    h_w1.insert(h_w1.end(), w1, w1 + (size_t)2 * c * kCond);
    h_b1.insert(h_b1.end(), b1, b1 + 2 * c);
    for (int o = 0; o < c; ++o) {
      h_woff.push_back((int)h_w2.size() + o * 2 * c);
      h_hoff.push_back(h0); h_nin.push_back(2 * c); h_b2.push_back(b2[o]);
    }
    h_w2.insert(h_w2.end(), wt, wt + (size_t)2 * c * c);
    hid_len += 2 * c;
    return o0;
  }
  void add_jobs(int dst, int a, int b, const std::vector<float>& al, const std::vector<float>& be, int c) {
    for (int i = 0; i < c; ++i) {
      h_dst.push_back(dst + i); h_ja.push_back(a + i); h_jb.push_back(b < 0 ? -1 : b + i);
      h_alpha.push_back(al.empty() ? 1.f : al[i]); h_beta.push_back(be.empty() ? 0.f : be[i]);
    }
  }

  // ConvBlockResCond in state-dict order: bn1, bn2, conv1, film1, conv2, film2 [, shortcut, film_res]
  void load_block(WeightCursor& wc, int cin, int cout) {
    blocks.emplace_back();
    LBlock& b = blocks.back();
    const bool first = cin == 1;
    const int cin_p = first ? 4 : cin;
    b.cin = cin_p; b.cout = cout; b.sc = cin != cout;
    std::vector<float> s1, t1, s2, t2;
    bn_fold(wc, cin, s1, t1);
    bn_fold(wc, cout, s2, t2);
    if (first) { in_s = s1[0]; in_t = t1[0]; }
    else { b.s1.upload(s1); b.t1.upload(t1); }
    {  // conv1 with bn2 folded: weights x s2 (per output channel); first block: input channel 0 of 4
      const float* w = wc.next();
      std::vector<float> wf((size_t)cout * cin_p * 9, 0.f);
      for (int co = 0; co < cout; ++co)
        for (int ci = 0; ci < cin; ++ci)
          for (int k = 0; k < 9; ++k) wf[((size_t)co * cin_p + ci) * 9 + k] = w[((size_t)co * cin + ci) * 9 + k] * s2[co];
      pack_conv(b.conv1, wf.data(), nullptr, cout, cin_p, 9, true);
    }
    const int f1 = load_film(wc, cout);
    pack_conv(b.conv2, wc.next(), nullptr, cout, cout, 9, true);
    const int f2 = load_film(wc, cout);
    int fr = -1;
    if (b.sc) {  // shortcut 1x1 (+ bias); first block: reads the raw x in input channel 1
      const float* w = wc.next(); const float* bias = wc.next();
      std::vector<float> wf((size_t)cout * cin_p, 0.f);
      for (int co = 0; co < cout; ++co)
        for (int ci = 0; ci < cin; ++ci) wf[(size_t)co * cin_p + ci + (first ? 1 : 0)] = w[(size_t)co * cin + ci];
      pack_conv(b.shortcut, wf.data(), bias, cout, cin_p, 1, false);
      fr = load_film(wc, cout);
    }
    b.e1 = vec_len; vec_len += cout;
    b.r2 = vec_len; vec_len += cout;
    add_jobs(b.e1, f1, -1, s2, t2, cout);
    add_jobs(b.r2, f2, fr, {}, {}, cout);
  }

  // decoder_block{j}.conv1 (ConvTranspose2d [C_in][C_out][3][3]) and bn1
  void load_dec(WeightCursor& wc, LDec& d, int cin, int cout) {
    d.cin = cin; d.cout = cout;
    const float* w = wc.next();
    std::vector<float> s, t;
    bn_fold(wc, cin, s, t);
    d.s.upload(s); d.t.upload(t);
    // phase ph = (a, b) of output channel block ph, tap k = (dh, dw) of input channel block k: kernel element
    // (a + 2 [dh = -1], b + 2 [dw = -1]) when both are <= 2
    std::vector<float> wg((size_t)4 * cout * 4 * cin, 0.f);
    for (int ph = 0; ph < 4; ++ph)
      for (int k = 0; k < 4; ++k) {
        const int kh = (ph >> 1) + ((k >> 1) ? 2 : 0), kw = (ph & 1) + ((k & 1) ? 2 : 0);
        if (kh > 2 || kw > 2) continue;
        for (int co = 0; co < cout; ++co)
          for (int ci = 0; ci < cin; ++ci)
            wg[(size_t)(ph * cout + co) * 4 * cin + k * cin + ci] = w[(((size_t)ci * cout + co) * 3 + kh) * 3 + kw];
      }
    pack_conv(d.up, wg.data(), nullptr, 4 * cout, 4 * cin, 1, false);
    d.up.useful = 9.f / 16.f;
  }

  void finish_films() {
    pack_conv(film1, h_w1.data(), h_b1.data(), hid_len, kCond, 1, false);
    w2.upload(h_w2);
    njobs = (int)h_dst.size();
    const int nout = (int)h_b2.size();
    std::vector<float> tab;
    auto put_i = [&](const std::vector<int>& v) { const size_t o = tab.size(); tab.resize(o + v.size()); memcpy(&tab[o], v.data(), sizeof(int) * v.size()); };
    auto put_f = [&](const std::vector<float>& v) { tab.insert(tab.end(), v.begin(), v.end()); };
    put_i(h_woff); put_i(h_hoff); put_i(h_nin); put_f(h_b2);
    put_i(h_dst); put_i(h_ja); put_i(h_jb); put_f(h_alpha); put_f(h_beta);
    ftab.upload(tab);
    AGPT_CHECK((int)h_woff.size() == nout, "film table");
    std::vector<float>().swap(h_w1); std::vector<float>().swap(h_w2);
  }
  FilmJobs jobs() const {
    const int nout = (int)h_b2.size();
    const float* p = ftab.p;
    FilmJobs J;
    J.woff = reinterpret_cast<const int*>(p); J.hoff = J.woff + nout; J.nin = J.hoff + nout;
    J.b2 = p + 3 * (size_t)nout;
    J.dst = reinterpret_cast<const int*>(J.b2 + nout); J.ja = J.dst + njobs; J.jb = J.ja + njobs;
    J.alpha = reinterpret_cast<const float*>(J.jb + njobs); J.beta = J.alpha + njobs;
    return J;
  }

  // text_embedder: BertModel(input_ids, attention_mask)[0][:, 0] -> Linear + ReLU -> cond [N][256]
  void text(const int* ids, const int* mask, int N, int L, float* cond, cudaStream_t st) {
    AGPT_CHECK(N >= 1 && L >= 1, "empty batch");
    zeros.ensure((size_t)N * L);
    AGPT_CUDA(cudaMemsetAsync(zeros.p, 0, sizeof(float) * N * L, st));   // token_type_ids: zeros
    bert.encode_hidden(ids, reinterpret_cast<const int*>(zeros.p), mask, N, L, st);
    TapConvParams P = tapconv_params(lin, 1, N, 0, 1);
    P.in = bert.x.p; P.in_pitch = L * cfg.hidden_size;     // the [CLS] row of sequence n is row n * L
    P.out = cond; P.out_pitch = kCond;
    P.epi = EPI_RELU;
    tapconv_launch(P, st);
  }

  static int pick_strip(int W) {   // VaeBase::pick_strip's rule: strips of at most 78 columns on maps wider than 79
    if (W <= 79) return 0;
    const int n = cdiv(W, 78);
    return cdiv(W, n);
  }
  void conv3x3(const PackedConv& pc, const float* in, float* out, int B, int H, int W, int epi, const float* evec,
               const float* res, cudaStream_t st) {
    TapConvParams P = tapconv_params(pc, B, H * W, W, 1);
    const int sw = pick_strip(W);
    if (sw) tapconv_set_strips(P, sw);
    P.in = in; P.in_gstride = (long)H * W * pc.Cin; P.in_pitch = pc.Cin;
    P.out = out; P.out_gstride = (long)H * W * pc.Cout; P.out_pitch = pc.Cout;
    P.pro = PRO_LRELU; P.slope = kSlope;
    P.epi = epi;
    P.evec = evec; P.evec_gstride = vec_len;
    P.res = res; P.res_gstride = (long)H * W * pc.Cout; P.res_pitch = pc.Cout;
    tapconv_launch(P, st);
  }

  // ConvBlockResCond: x [B][H][W][cin] -> out [B][H][W][cout]; the first block's x is the 4-channel input image
  void run_block(const LBlock& b, const float* x, float* out, int B, int H, int W, cudaStream_t st) {
    const long rows = (long)B * H * W;
    const float* a = x;
    if (b.s1.p) {
      lass_affine(x, b.s1.p, b.t1.p, ba.p, b.sc ? nullptr : br.p, vec.p, vec_len, b.r2, rows, (long)H * W, b.cin, st);
      a = ba.p;
    }
    if (b.sc) {   // shortcut(x) + bias + film_res + film2
      TapConvParams P = tapconv_params(b.shortcut, B, H * W, 0, 1);
      P.in = x; P.in_gstride = (long)H * W * b.cin; P.in_pitch = b.cin;
      P.out = br.p; P.out_gstride = (long)H * W * b.cout; P.out_pitch = b.cout;
      P.epi = EPI_ADDVEC; P.evec = vec.p + b.r2; P.evec_gstride = vec_len;
      tapconv_launch(P, st);
    }
    conv3x3(b.conv1, a, bh.p, B, H, W, EPI_ADDVEC, vec.p + b.e1, nullptr, st);
    conv3x3(b.conv2, bh.p, out, B, H, W, EPI_RES, nullptr, br.p, st);
  }

  // the FiLM vectors of a request: cond [B][256] -> film1 (EPI_RELU) into hid, lass_film -> v [B][vec_len]
  void film_vec(const float* cond, int B, float* v, cudaStream_t st) {
    hid.ensure((size_t)B * hid_len);
    TapConvParams P = tapconv_params(film1, 1, B, 0, 1);
    P.in = cond; P.in_pitch = kCond;
    P.out = hid.p; P.out_pitch = hid_len;
    P.epi = EPI_RELU;
    tapconv_launch(P, st);
    lass_film(hid.p, hid_len, w2.p, jobs(), njobs, B, v, vec_len, st);
  }

  // decoder d's bn1, ReLU and ConvTranspose2d(k3, s2) + prune on y [B][h][w][d.cin], next to the skip [B][2h][2w + 1]
  // [d.cout] -> cat [B][2h][2w + 1][2 d.cout]: lass_upcol, the packed 4 C_in -> 4 C_out GEMM, lass_shuffle
  void up(const LDec& d, const float* y, const float* skp, int B, int h, int w, float* out, cudaStream_t st) {
    col.ensure((size_t)B * h * (w + 1) * 4 * d.cin);
    upb.ensure((size_t)B * h * (w + 1) * 4 * d.cout);
    lass_upcol(y, d.s.p, d.t.p, B, h, w, d.cin, col.p, st);
    TapConvParams P = tapconv_params(d.up, 1, B * h * (w + 1), 0, 1);
    P.in = col.p; P.in_pitch = 4 * d.cin;
    P.out = upb.p; P.out_pitch = 4 * d.cout;
    P.epi = EPI_BIAS;
    tapconv_launch(P, st);
    lass_shuffle(upb.p, skp, B, h, w, d.cout, out, st);
  }

  void mask(const float* mag, int B, int T, int F, long sb, long stt, long sf, const float* cond, float* out_mask,
            float* out_logits, cudaStream_t st) {
    AGPT_CHECK(B >= 1 && T >= 1, "empty input");
    const int W0 = F - 2;
    if (W0 < 127 || W0 % 64 != 63)
      throw Error("LASSNet: F = " + std::to_string(F) + " frequency bins do not fit UNetRes_FiLM: F - 2 must be 63 mod 64 "
                  "and at least 127 (513 for a 1024-point STFT)");
    const int Tp = cdiv(T, 64) * 64;
    int Hs[kLevels + 1], Ws[kLevels + 1];
    Hs[0] = Tp; Ws[0] = W0;
    for (int k = 1; k <= kLevels; ++k) { Hs[k] = Hs[k - 1] / 2; Ws[k] = Ws[k - 1] / 2; }
    // buffers: the largest map per role
    size_t mx = (size_t)Tp * W0 * 4, mcat = 0, mcol = 0, mup = 0;
    for (int k = 0; k < kLevels; ++k) {
      const size_t px = (size_t)Hs[k] * Ws[k];
      mx = std::max(mx, px * 2 * kEncCh[k]);
      mcat = std::max(mcat, px * 2 * kEncCh[k]);
      const size_t pin = (size_t)Hs[k + 1] * (Ws[k + 1] + 1);
      mcol = std::max(mcol, pin * 4 * dec[k].cin);
      mup = std::max(mup, pin * 4 * dec[k].cout);
      skip[k].ensure((size_t)B * px * kEncCh[k]);
    }
    mx = std::max(mx, (size_t)Hs[kLevels] * Ws[kLevels] * 384);
    for (DevBuf* d : {&bx, &bo, &ba, &bh, &br}) d->ensure(mx * B);
    cat.ensure(mcat * B); col.ensure(mcol * B); upb.ensure(mup * B);
    vec.ensure((size_t)B * vec_len);
    film_vec(cond, B, vec.p, st);     // FiLM vectors of the whole request
    lass_input(mag, sb, stt, sf, B, T, Tp, W0, in_s, in_t, bx.p, st);
    // encoder: two blocks per level, the second one's output is the skip; then 2x2 average pool (floor)
    int bi = 0;
    for (int k = 0; k < kLevels; ++k) {
      run_block(blocks[bi++], bx.p, bo.p, B, Hs[k], Ws[k], st);
      run_block(blocks[bi++], bo.p, skip[k].p, B, Hs[k], Ws[k], st);
      avgpool2(skip[k].p, bx.p, B, Hs[k], Ws[k], kEncCh[k], st);
    }
    run_block(blocks[bi++], bx.p, bo.p, B, Hs[kLevels], Ws[kLevels], st);     // conv_block7
    float* y = bo.p;
    for (int k = kLevels - 1; k >= 0; --k) {
      const LDec& d = dec[k];
      const int h = Hs[k + 1], w = Ws[k + 1];
      AGPT_CHECK(Hs[k] == 2 * h && Ws[k] == 2 * w + 1, "decoder shape");
      up(d, y, skip[k].p, B, h, w, cat.p, st);
      run_block(blocks[bi++], cat.p, bx.p, B, Hs[k], Ws[k], st);
      run_block(blocks[bi++], bx.p, bo.p, B, Hs[k], Ws[k], st);
      y = bo.p;
    }
    run_block(blocks[bi++], bo.p, bx.p, B, Tp, W0, st);                       // after_conv_block1
    lass_head(bx.p, head.p, B, T, Tp, W0, out_mask, out_logits, st);
    AGPT_CUDA(cudaGetLastError());
  }
};

Handle* lass_create(const agpt_lass_cfg* cfg, const float* const* W, int nW, int device) {
  DeviceGuard dg_(device);
  const int H = cfg->hidden_size;
  AGPT_CHECK(cfg->vocab_size >= 1 && cfg->max_position_embeddings >= 1 && cfg->type_vocab_size >= 1 && cfg->num_layers >= 0 &&
                 cfg->num_heads >= 1 && H % cfg->num_heads == 0 && cfg->intermediate_size % 4 == 0 && H == kCond &&
                 cfg->layer_norm_eps > 0.f,
             "bad LASSNet config (the text encoder's Linear is 256 -> 256: hidden_size must be 256)");
  std::unique_ptr<LassNet> h(new LassNet());
  h->magic = kMagicLass; h->device = device; h->cfg = *cfg;
  agpt_clap_cfg& b = h->bert.cfg;
  memset(&b, 0, sizeof(b));
  b.vocab_size = cfg->vocab_size; b.max_position_embeddings = cfg->max_position_embeddings; b.type_vocab_size = cfg->type_vocab_size;
  b.hidden_size = H; b.num_layers = cfg->num_layers; b.num_heads = cfg->num_heads; b.intermediate_size = cfg->intermediate_size;
  b.layer_norm_eps = cfg->layer_norm_eps;
  WeightCursor wc{W, nW};
  h->bert.load_bert(wc);
  { auto w = wc.next(); auto bb = wc.next(); pack_conv(h->lin, w, bb, kCond, H, 1, false); }
  for (int k = 0; k < kLevels; ++k) {
    const int ci = k == 0 ? 1 : kEncCh[k - 1], co = kEncCh[k];
    h->load_block(wc, ci, co);
    h->load_block(wc, co, co);
  }
  h->load_block(wc, 384, 384);
  for (int j = 0; j < kLevels; ++j) {
    const int k = kLevels - 1 - j, cout = kEncCh[k], cin = kEncCh[std::min(k + 1, kLevels - 1)];
    h->load_dec(wc, h->dec[k], cin, cout);
    h->load_block(wc, 2 * cout, cout);
    h->load_block(wc, cout, cout);
  }
  h->load_block(wc, 32, 32);
  {
    const float* w = wc.next(); const float* bb = wc.next();
    std::vector<float> hw(w, w + 32);
    hw.push_back(bb[0]);
    h->head.upload(hw);
  }
  wc.done();
  h->finish_films();
  return h.release();
}

void lass_text(Handle* hh, const int* ids, const int* mask, int N, int L, float* cond, cudaStream_t st) {
  auto* h = static_cast<LassNet*>(hh);
  DeviceGuard dg_(h->device);
  h->text(ids, mask, N, L, cond, st);
}

void lass_mask(Handle* hh, const float* mag, int B, int T, int F, long sb, long stt, long sf, const float* cond, float* mask,
               float* logits, cudaStream_t st) {
  auto* h = static_cast<LassNet*>(hh);
  DeviceGuard dg_(h->device);
  h->mask(mag, B, T, F, sb, stt, sf, cond, mask, logits, st);
}

int lass_film_vec(Handle* hh, const float* cond, int B, float* vec, cudaStream_t st) {
  auto* h = static_cast<LassNet*>(hh);
  DeviceGuard dg_(h->device);
  if (vec) {
    AGPT_CHECK(B >= 1 && cond, "LASS FiLM vectors: B >= 1 and a condition");
    h->film_vec(cond, B, vec, st);
  }
  return h->vec_len;
}

void lass_up(Handle* hh, int level, const float* y, const float* skip, int B, int h, int w, float* cat, cudaStream_t st) {
  auto* net = static_cast<LassNet*>(hh);
  DeviceGuard dg_(net->device);
  AGPT_CHECK(level >= 0 && level < kLevels, "LASS up: the decoder level must be in [0, 6)");
  net->up(net->dec[level], y, skip, B, h, w, cat, st);
}

struct StftNet : Handle {
  int n = 0, hop = 0, nb = 0;
  PackedConv fwd, inv;
  DevBuf rows, spec, X, Y, ws;
  int ws_T = -1;

  void transform(const float* wav, int B, long N, float* mag, float* phase, cudaStream_t st) {
    AGPT_CHECK(B >= 1, "empty batch");
    if (N <= n / 2)
      throw Error("STFT: " + std::to_string(N) + " samples are too few for the reflect padding of " + std::to_string(n / 2));
    const int T = (int)(N / hop + 1);
    const long R = cdivl(N + n, hop);
    rows.ensure((size_t)B * R * hop);
    stft_rows(wav, B, N, n, hop, rows.p, st);
    spec.ensure((size_t)B * R * fwd.cout_pad);
    TapConvParams P = tapconv_params(fwd, B, (int)R, 0, 1);
    P.in = rows.p; P.in_gstride = R * hop; P.in_pitch = hop;
    P.out = spec.p; P.out_gstride = R * fwd.cout_pad; P.out_pitch = fwd.cout_pad;
    P.epi = EPI_BIAS;
    tapconv_launch(P, st);
    stft_magphase(spec.p, B, R, fwd.cout_pad, nb, T, mag, phase, st);
    AGPT_CUDA(cudaGetLastError());
  }

  // stft.py window_sumsquare (norm None) for T frames: each frame's float64 squared periodic Hann window added in
  // float64 to the fp32 envelope
  void window_sum(int T) {
    if (T == ws_T) return;
    const long len = (long)n + (long)hop * (T - 1);
    std::vector<float> x(len, 0.f);
    std::vector<double> wsq(n);
    const double pi = 3.14159265358979323846, step = 2.0 * pi / n;
    for (int k = 0; k < n; ++k) {   // scipy get_window('hann', n, fftbins=True): 0.5 + 0.5 cos(k step - pi)
      const double w = 0.5 + 0.5 * cos(k * step + -pi);
      wsq[k] = w * w;
    }
    for (int i = 0; i < T; ++i)
      for (int k = 0; k < n && (long)i * hop + k < len; ++k) x[(long)i * hop + k] = (float)((double)x[(long)i * hop + k] + wsq[k]);
    ws.upload(x);
    ws_T = T;
  }

  void inverse(const float* mag, const float* phase, int B, int T, float* out, cudaStream_t st) {
    AGPT_CHECK(B >= 1 && T >= 2, "the inverse STFT needs at least two frames");
    const int pitch = inv.cin_pad;
    X.ensure((size_t)B * (T + 1) * pitch);
    istft_frames(mag, phase, B, nb, T, pitch, X.p, st);
    Y.ensure((size_t)B * (T + 1) * hop);
    TapConvParams P = tapconv_params(inv, B, T + 1, 0, 1);
    P.in = X.p; P.in_gstride = (long)(T + 1) * pitch; P.in_pitch = pitch;
    P.out = Y.p; P.out_gstride = (long)(T + 1) * hop; P.out_pitch = hop;
    P.epi = EPI_BIAS;
    tapconv_launch(P, st);
    window_sum(T);
    istft_finish(Y.p, ws.p, B, T, n, hop, out, st);
    AGPT_CUDA(cudaGetLastError());
  }
};

Handle* stft_create(int filter_length, int hop_length, const float* fwd_basis, const float* inv_basis, int device) {
  DeviceGuard dg_(device);
  AGPT_CHECK(filter_length == 2 * hop_length && hop_length >= 8 && hop_length % 8 == 0 && fwd_basis && inv_basis,
             "the STFT engine runs filter_length = 2 hop_length (hop a multiple of 8)");
  std::unique_ptr<StftNet> h(new StftNet());
  h->magic = kMagicStft; h->device = device;
  const int n = filter_length, hop = hop_length, nb = n / 2 + 1, C = 2 * nb;
  h->n = n; h->hop = hop; h->nb = nb;
  {  // forward_basis [C][1][n]: tap 0 (row r) = columns [0, hop), tap 1 (row r + 1) = [hop, n)
    std::vector<float> w((size_t)C * hop * 2);
    for (int c = 0; c < C; ++c)
      for (int j = 0; j < hop; ++j)
        for (int k = 0; k < 2; ++k) w[((size_t)c * hop + j) * 2 + k] = fwd_basis[(size_t)c * n + k * hop + j];
    pack_conv(h->fwd, w.data(), nullptr, C, hop, 2, false);   // tap offsets {0, +1}
  }
  {  // inverse_basis [C][1][n] as conv_transpose1d: output row r = X[r] . basis[:, :hop] + X[r - 1] . basis[:, hop:]
    std::vector<float> w((size_t)hop * C * 2);
    for (int j = 0; j < hop; ++j)
      for (int c = 0; c < C; ++c) {
        w[((size_t)j * C + c) * 2 + 0] = inv_basis[(size_t)c * n + hop + j];   // tap offset -1
        w[((size_t)j * C + c) * 2 + 1] = inv_basis[(size_t)c * n + j];         // tap offset 0
      }
    pack_conv(h->inv, w.data(), nullptr, hop, C, 2, false);
    h->inv.tap_off_1d[0] = -1; h->inv.tap_off_1d[1] = 0;
  }
  return h.release();
}

void stft_transform(Handle* hh, const float* wav, int B, long n_samples, float* mag, float* phase, cudaStream_t st) {
  auto* h = static_cast<StftNet*>(hh);
  DeviceGuard dg_(h->device);
  h->transform(wav, B, n_samples, mag, phase, st);
}

void stft_inverse(Handle* hh, const float* mag, const float* phase, int B, int T, float* wav, cudaStream_t st) {
  auto* h = static_cast<StftNet*>(hh);
  DeviceGuard dg_(h->device);
  h->inverse(mag, phase, B, T, wav, st);
}

}  // namespace agpt
