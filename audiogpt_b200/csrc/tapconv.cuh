// tapconv: the one contraction primitive of the hot path (fp32 FMA version).
//
//   out[g, p, co] = epi( bias[co] + sum_tap sum_ci  pro(in[g, p (+) off_tap, ci]) * W[tap][ci][co] )
//
// Activations are CHANNELS-LAST rows ([G][L][C], C contiguous), so a conv tap is a
// row shift, a Linear is the 1-tap case, a 3x3 conv is 9 taps over a "virtual"
// flat grid of width W+1 (one shared zero column => no per-tap masks), and
// ConvTranspose1d(k=2u, stride u) is a 3-tap conv producing u*Cout channels whose
// [L][u*Cout] output *is* the [u*L][Cout] upsampled tensor.
//
// Replaces (reference call sites): F.conv1d / F.conv_transpose1d in
// NeuralSeq/modules/hifigan/hifigan.py:54-61,151-167 and modules/diff/net.py:66-78,107-130;
// F.conv2d / F.linear in ldm/modules/diffusionmodules/openaimodel.py:255-275,711-744 and
// ldm/modules/attention.py:37-64,170-193,250-261.
//
// Tiling: CTA = 128 rows x BN cols (BN in {32,64,128}), 8x8 register micro-tile per
// thread, K-loop over (8-channel chunk) x tap.  The activation tile (+halo) is staged
// ONCE per chunk in shared memory in four row-shifted copies so that every tap is read
// with aligned 128-bit LDS; weight slabs [8][BN] stream through a cp.async double buffer.
#pragma once
#include <cuda_fp16.h>
#include "common.cuh"
#include "../../include/agpt_b200.h"   // AGPT_TC_KERN_*, the kernel family a launch records

namespace agpt {

constexpr int kMaxTaps = 12;
constexpr int TC_BM = 128;
constexpr int TC_KC = 8;

enum Pro : int { PRO_NONE = 0, PRO_LRELU = 1, PRO_ADDVEC = 2, PRO_SILU = 3 };
enum Epi : int {
  EPI_BIAS = 0,     // v + bias
  EPI_RES = 1,      // v + bias + res[g,p,co]
  EPI_ACC = 2,      // out = (accumulate ? out : 0) + scale * (v + bias + res)
  EPI_RELU = 3,     // relu(v + bias)
  EPI_ADDVEC = 4,   // v + bias + evec[g,co]
  EPI_GATE = 5,     // interleaved (gate,filter) pairs: sigmoid(g)*tanh(f), + aux[g,p,co] before; out has Cout/2 channels
  EPI_GEGLU = 6,    // interleaved (a,gate) pairs: a*gelu(gate); out has Cout/2 channels
  EPI_DIFFOUT = 7,  // co<csplit: out=(out+v)*rsqrt2 in place ; else out2 (+)= v
  EPI_STORE_CF = 8, // channels-first store out[g][co][p]
  EPI_TANH = 9,     // tanh(v + bias)
  EPI_MISH = 10,    // mish(v + bias) = x * tanh(softplus(x))   (NeuralSeq/modules/diff/diffusion.py:68-70)
  EPI_SILU = 11,    // silu(v + bias)
  EPI_GELU_SCALED = 12,   // gelu_erf(scale * (v + bias))   (TransformerFFNLayer: conv * k^-0.5, then F.gelu)
};

struct TapConvParams {
  const float* in; long in_gstride; int in_pitch;
  const float* w;      // packed [ntaps][cin_pad][cout_pad]
  const float* bias;   // [cout_pad] or nullptr
  float* out; long out_gstride; int out_pitch;
  int G, L, Wreal, Cin, cin_pad, Cout, cout_pad;
  int ntaps; int tap_off[kMaxTaps];
  int lo_al, R;
  int pro; float slope; const float* pvec; int pvec_gstride;
  int epi; const float* res; long res_gstride; int res_pitch; float scale; int accumulate;
  const float* evec; int evec_gstride;
  float* out2; long out2_gstride; int out2_pitch; int csplit;
  const float* w_h; const float* w_h64; const float* w_h96; int tc_chunks_h; float tc_descale;   // fp16 hi/lo image (tcconv5.cu): 64-channel chunks, weights pre-scaled by 1/tc_descale
  const float* w_hk;   // 128 -> 128 channels: the same weights in 32-channel half-stages (tcpair_pipe_kernel's ring)
  int tc_bn, tc_na, tc_nw, tc_nr;   // tc_bn == 0 => FMA only
  float flops_scale;   // useful fraction of the MACs (zero-padded polyphase taps); 0 => 1
  // 2-D convs on WIDE images (the VAE decoder's 80x624 maps): the image is cut into `strips` vertical strips of
  // `strip_w` columns; grid slice gz = g * strips + s works on the virtual grid [H][strip_w + 2] of strip s
  // (column j <-> image column s*strip_w + j - 1: one halo column on each side, zero outside the image), so
  // the halo of a 128-row tile stays 2*(strip_w+2)+2 rows whatever the image width is.  strips == 0: one virtual
  // grid [H][W + 1] per sample (one shared zero column), as the UNet's 10x78 maps use.
  int strips, strip_w;
  // optional operand-plane copy of the GATE / GEGLU epilogue's output (fp16 hi/lo [L][pl_pitch], G == 1): the
  // consumer (UNet ff2, a 4C-deep 1-tap GEMM) is then plane-fed; with out == nullptr the fp32 tensor is not written
  __half* pl_hi; __half* pl_lo; int pl_pitch;
  // 1: the tensor-core kernels may run 256-row tiles (tc5_tall in tcconv5.cu decides per launch); set by the HiFi-GAN
  // driver.
  int tc_tall;
  // Operand planes of the leaky-ReLU tap-GEMMs (HiFi-GAN driver; tensor-core kernels only).
  // A plane is two fp16 tensors laid out like the fp32 one (same pitch and sample stride, in elements):
  //   hi = fp16(lrelu(x, slope)),  lo = fp16(lrelu(x, slope) - hi)
  // bit for bit the operands the kernels' own fp32 transform makes.  pi_*: the input is read from this plane (TMA)
  // instead of `in`.  po_*: the epilogue also writes the plane of the value it stores (po_slope: the consumer's
  // slope); with out == nullptr only the plane is written.
  const __half* pi_hi; const __half* pi_lo;
  __half* po_hi; __half* po_lo; float po_slope;
  // 1: a fused ResBlock pair (tcpair_launch) may run as two 128-row CTAs per SM (tcpair2_kernel); set by the HiFi-GAN
  // driver unless AGPT_PAIR_DUAL=0.
  int tc_dual;
  // 1: a C = 128 fused pair may run on tcpair_pipe_kernel (two tiles in flight per CTA), its input and residual
  // staged by TMA; 2: the same pipeline with one data warpgroup loading them per thread.  Set by the HiFi-GAN driver
  // unless AGPT_PAIR_PIPE=0 (2 with AGPT_PAIR_PIPE_STAGE=0).
  int tc_pipe;
  // 1: a narrow fused pair that tc_dual allows may run on tcpair_narrow_kernel (persistent, several tiles in flight
  // per CTA) before tcpair2_kernel; set by the HiFi-GAN driver unless AGPT_NARROW_PIPE=0.
  int tc_narrow_pipe;
  // 1: a plane-fed launch at BN = 128 over 1-D rows may run on tcconv_pipe_pl_kernel (persistent, one tile's epilogue
  // beside the next tile's wgmmas); set by the HiFi-GAN driver unless AGPT_CONV_PIPE=0.
  int tc_conv_pipe;
};

__host__ __device__ inline int tc_wv(const TapConvParams& P) { return P.Wreal > 0 ? (P.strips > 0 ? P.strip_w + 2 : P.Wreal + 1) : 0; }
__host__ __device__ inline int tc_lv(const TapConvParams& P) { const int wv = tc_wv(P); return wv ? (P.L / P.Wreal) * wv : P.L; }
__host__ __device__ inline int tc_groups(const TapConvParams& P) { return P.strips > 0 ? P.G * P.strips : P.G; }
__host__ __device__ inline int tc_sample(const TapConvParams& P, int gz) { return P.strips > 0 ? gz / P.strips : gz; }
// virtual row q of grid slice gz -> row index inside the sample's [L][C] tensor, or -1 (zero padding / no output)
__host__ __device__ inline int tc_row_in(const TapConvParams& P, int gz, int q, int Wv, int Lv) {
  if (q < 0 || q >= Lv) return -1;
  if (!Wv) return q;
  const int h = q / Wv, j = q - h * Wv;
  if (P.strips > 0) {
    const int w = (gz % P.strips) * P.strip_w + j - 1;
    return (w >= 0 && w < P.Wreal) ? h * P.Wreal + w : -1;
  }
  return j < P.Wreal ? h * P.Wreal + j : -1;
}
__host__ __device__ inline int tc_row_out(const TapConvParams& P, int gz, int q, int Wv, int Lv) {
  if (q < 0 || q >= Lv) return -1;
  if (!Wv) return q;
  const int h = q / Wv, j = q - h * Wv;
  if (P.strips > 0) {
    if (j < 1 || j > P.strip_w) return -1;
    const int w = (gz % P.strips) * P.strip_w + j - 1;
    return w < P.Wreal ? h * P.Wreal + w : -1;
  }
  return j < P.Wreal ? h * P.Wreal + j : -1;
}


// ---------------------------------------------------------------- host side
struct PackedConv {
  DevBuf w, b, w_h, w_h64, w_h96, w_hk;
  int tc_bn = 0, h_chunks = 0;
  float h_descale = 1.f;
  int Cin = 0, cin_pad = 0, Cout = 0, cout_pad = 0, ntaps = 0;
  int tap_off_1d[kMaxTaps] = {0};   // for 1-D convs: row offsets; 2-D convs derive offsets from W at launch
  bool is2d = false;
  bool has_bias = false;
  float useful = 1.f;   // fraction of packed taps that are algorithmic work
};

inline int tc_pick_bn(int cout) {
  if (cout <= 32) return 32;
  if (cout <= 64) return 64;
  const int w128 = round_up(cout, 128), w64 = round_up(cout, 64);
  return (w128 <= w64) ? 128 : 64;
}

struct PackedConv;
// Fill geometry-dependent fields (offsets, halo, smem rows) and launch (tapconv.cu).
void tapconv_launch(TapConvParams P, cudaStream_t st);
void tcconv_launch(TapConvParams P, cudaStream_t st);          // tensor-core dispatcher (tcconv.cu)
bool tcconv5_launch(TapConvParams P, cudaStream_t st);
bool tcpair_launch(TapConvParams c1, TapConvParams c2, cudaStream_t st);   // fused ResBlock1 pair (tcconv5.cu)
struct HTile { int bn; const float* w; long ntiles; int mt; };
HTile pick_h_tile(const TapConvParams& P, int sms);   // tile width and height of the fp16 tensor-core kernel (tcconv5.cu)
void pack_h_weights(struct PackedConv& pc, const std::vector<float>& h);
bool tcconv_supported(const TapConvParams& P);
void pack_tc_weights(struct PackedConv& pc, const std::vector<float>& h);
void tc_set_enabled(int on);
bool tc_enabled();
void profile_enable(int on);
void* profile_begin(const TapConvParams& P, bool tc, double bytes_override, cudaStream_t st);
void* profile_begin_pair(const TapConvParams& c1, const TapConvParams& c2, cudaStream_t st);
void profile_end(void* rec, cudaStream_t st);
void profile_count_tall();            // a tensor-core launch with 256-row tiles (counted while profiling)
long long profile_tall_launches();
void profile_count_dual();            // a launch of narrow pairs with overlapped tiles (counted while profiling)
long long profile_dual_launches();
void profile_count_pipe();            // a fused-pair launch of tcpair_pipe_kernel (counted while profiling)
long long profile_pipe_launches();
void profile_count_narrow_pipe();     // a fused-pair launch of tcpair_narrow_kernel (counted while profiling)
long long profile_narrow_pipe_launches();
void profile_count_conv_pipe();       // a plane-fed launch of tcconv_pipe_pl_kernel (counted while profiling)
long long profile_conv_pipe_launches();
void profile_count_plane();           // a plane-fed tensor-core launch (counted while profiling)
long long profile_plane_launches();
// The variant of the most recent tap-GEMM launch on this host thread, {1 tensor-core | 0 fp32-FMA, tile width, tile
// height, 1 plane-fed, kernel family AGPT_TC_KERN_*}, recorded where a kernel is actually launched
// (agpt_tapconv_probe reports it); -1s before any.
void tapconv_note_launch(int tc, int bn, int mt, int plane, int kern);
void tapconv_last_launch(int ran[5]);
// fp32 [n] -> operand plane hi / lo of lrelu(x, slope) (TapConvParams::pi_hi), n a multiple of 4 (tcconv5.cu)
void plane_split(const float* x, __half* hi, __half* lo, long n, float slope, cudaStream_t st);
void profile_collect(double* ms, double* flops, double* bytes, long long* launches);
long profile_dump(char* out, long cap);
double fma_peak_tflops();

// Common setup from a PackedConv; caller fills in/out/pro/epi afterwards.
inline TapConvParams tapconv_params(const PackedConv& pc, int G, int L, int Wreal, int dil) {
  TapConvParams P;
  memset(&P, 0, sizeof(P));
  P.w = pc.w.p;
  P.bias = pc.has_bias ? pc.b.p : nullptr;
  P.G = G; P.L = L; P.Wreal = Wreal;
  P.Cin = pc.Cin; P.cin_pad = pc.cin_pad; P.Cout = pc.Cout; P.cout_pad = pc.cout_pad;
  P.ntaps = pc.ntaps;
  if (pc.is2d) {
    AGPT_CHECK(pc.ntaps == 9 && Wreal > 0, "2d conv needs W");
    const int Wv = Wreal + 1;
    for (int dh = -1, t = 0; dh <= 1; ++dh)
      for (int dw = -1; dw <= 1; ++dw, ++t) P.tap_off[t] = dh * Wv + dw;
  } else {
    for (int t = 0; t < pc.ntaps; ++t) P.tap_off[t] = pc.tap_off_1d[t] * dil;
  }
  P.scale = 1.f;
  P.flops_scale = pc.useful;
  P.tc_bn = pc.tc_bn;
  P.w_h = pc.w_h.p; P.w_h64 = pc.w_h64.p; P.w_h96 = pc.w_h96.p; P.w_hk = pc.w_hk.p; P.tc_chunks_h = pc.h_chunks; P.tc_descale = pc.h_descale;
  return P;
}

// Switch a 3x3 launch to strip mode (see TapConvParams::strips): strips of at most `strip_w` columns.
inline void tapconv_set_strips(TapConvParams& P, int strip_w) {
  AGPT_CHECK(P.Wreal > 0 && P.ntaps == 9 && strip_w >= 8, "strip mode is for 3x3 convs");
  P.strips = cdiv(P.Wreal, strip_w);
  P.strip_w = strip_w;
  const int Wv = strip_w + 2;
  for (int dh = -1, t = 0; dh <= 1; ++dh)
    for (int dw = -1; dw <= 1; ++dw, ++t) P.tap_off[t] = dh * Wv + dw;
}

// ---- host-side weight packing (reference layouts -> [tap][cin_pad][cout_pad]) ----
// Conv1d / Conv2d weight [Cout][Cin][K...] (torch layout), "same" padding, odd K.
inline void pack_conv(PackedConv& pc, const float* w, const float* b, int Cout, int Cin, int K, bool is2d,
                      float wscale = 1.f) {
  pc.Cin = Cin; pc.Cout = Cout; pc.cin_pad = round_up(Cin, TC_KC); pc.cout_pad = round_up(Cout, 32);
  pc.ntaps = K; pc.is2d = is2d;
  std::vector<float> h((size_t)K * pc.cin_pad * pc.cout_pad, 0.f);
  for (int co = 0; co < Cout; ++co)
    for (int ci = 0; ci < Cin; ++ci)
      for (int k = 0; k < K; ++k)
        h[((size_t)k * pc.cin_pad + ci) * pc.cout_pad + co] = w[((size_t)co * Cin + ci) * K + k] * wscale;
  pc.w.upload(h);
  pack_tc_weights(pc, h);
  if (!is2d) {
    const int c = (K - 1) / 2;
    for (int k = 0; k < K; ++k) pc.tap_off_1d[k] = k - c;
  }
  pc.has_bias = b != nullptr;
  std::vector<float> hb(pc.cout_pad, 0.f);
  if (b) for (int co = 0; co < Cout; ++co) hb[co] = b[co];
  pc.b.upload(hb);
}

// Conv1d (dilation 1, "same" padding) on g CONSECUTIVE TIME STEPS AT ONCE: the [L][C] tensor is read as [L/g][g*C]
// (the same memory), so a k-tap conv over C channels becomes a conv over g*C channels with block-Toeplitz weights
//   W'[s][(i, ci)][(j, co)] = w[co][ci][g*s + i - j + c],   c = (k-1)/2,  s = floor((j + t - c) / g)
// over super-taps s.  Narrow layers (C = 32 / 64) are bound by the NUMBER of MMA instructions -- each one
// re-reads its A slice from shared memory whatever N is -- and this raises N per instruction from C to
// g*C = 128: k = 11, C = 32, g = 4 needs 5 super-taps x 8 k-steps per 512 time steps instead of 11 x 2 per 128
// (2.2x fewer MMAs); the zero blocks of W' cost 1.45x the algorithmic MACs, which the tensor pipe has to spare.
inline void pack_conv_grouped(PackedConv& pc, const float* w, const float* b, int C, int K, int g) {
  const int c = (K - 1) / 2;
  auto fdiv = [](int a, int d) { return a >= 0 ? a / d : -((-a + d - 1) / d); };
  const int smin = fdiv(-c, g), smax = fdiv(g - 1 + K - 1 - c, g);
  const int nt = smax - smin + 1;
  AGPT_CHECK(nt <= kMaxTaps, "grouped conv: too many super-taps");
  const int Cg = g * C;
  std::vector<float> wg((size_t)Cg * Cg * nt, 0.f), bg(Cg, 0.f);
  for (int j = 0; j < g; ++j)
    for (int co = 0; co < C; ++co) {
      if (b) bg[j * C + co] = b[co];
      for (int i = 0; i < g; ++i)
        for (int ci = 0; ci < C; ++ci)
          for (int s = smin; s <= smax; ++s) {
            const int t = g * s + i - j + c;
            if (t < 0 || t >= K) continue;
            wg[((size_t)(j * C + co) * Cg + (i * C + ci)) * nt + (s - smin)] = w[((size_t)co * C + ci) * K + t];
          }
    }
  pack_conv(pc, wg.data(), b ? bg.data() : nullptr, Cg, Cg, nt, false);
  for (int t = 0; t < nt; ++t) pc.tap_off_1d[t] = smin + t;
  pc.useful = (float)K / (float)(nt * g);
}

// Same, but output channels interleaved (co -> 2*(co % half) + co / half): used where the
// epilogue consumes (first-half, second-half) channel pairs (DiffNet gate/filter, GEGLU).
inline void pack_conv_pairs(PackedConv& pc, const float* w, const float* b, int Cout, int Cin, int K) {
  const int half = Cout / 2;
  std::vector<float> w2((size_t)Cout * Cin * K), b2(Cout, 0.f);
  for (int co = 0; co < Cout; ++co) {
    const int dst = 2 * (co % half) + co / half;
    memcpy(&w2[(size_t)dst * Cin * K], &w[(size_t)co * Cin * K], sizeof(float) * Cin * K);
    if (b) b2[dst] = b[co];
  }
  pack_conv(pc, w2.data(), b ? b2.data() : nullptr, Cout, Cin, K, false);
}

// ConvTranspose1d weight [Cin][Cout][K], stride u, padding pad  ->  taps d in {..-1,0,+1..}
// over INPUT rows with u*Cout output channels (polyphase form; SURVEY.md 8a kernel cheat sheet).
inline void pack_convtranspose(PackedConv& pc, const float* w, const float* b, int Cin, int Cout, int K, int u, int pad) {
  std::vector<int> deltas;
  for (int d = -8; d <= 8; ++d) {
    bool any = false;
    for (int r = 0; r < u && !any; ++r) {
      const int k = r + pad - d * u;
      if (k >= 0 && k < K) any = true;
    }
    if (any) deltas.push_back(d);
  }
  AGPT_CHECK((int)deltas.size() <= kMaxTaps, "convtranspose taps");
  pc.Cin = Cin; pc.Cout = u * Cout; pc.cin_pad = round_up(Cin, TC_KC); pc.cout_pad = round_up(u * Cout, 32);
  pc.ntaps = (int)deltas.size(); pc.is2d = false;
  std::vector<float> h((size_t)pc.ntaps * pc.cin_pad * pc.cout_pad, 0.f);
  for (int t = 0; t < pc.ntaps; ++t) {
    pc.tap_off_1d[t] = deltas[t];
    for (int r = 0; r < u; ++r) {
      const int k = r + pad - deltas[t] * u;
      if (k < 0 || k >= K) continue;
      for (int ci = 0; ci < Cin; ++ci)
        for (int co = 0; co < Cout; ++co)
          h[((size_t)t * pc.cin_pad + ci) * pc.cout_pad + r * Cout + co] = w[((size_t)ci * Cout + co) * K + k];
    }
  }
  pc.w.upload(h);
  pack_tc_weights(pc, h);
  pc.useful = (float)(K / (double)u) / (float)pc.ntaps;
  pc.has_bias = b != nullptr;
  std::vector<float> hb(pc.cout_pad, 0.f);
  if (b) for (int r = 0; r < u; ++r) for (int co = 0; co < Cout; ++co) hb[r * Cout + co] = b[co];
  pc.b.upload(hb);
}

}  // namespace agpt
