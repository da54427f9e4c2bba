// Launchers of the small kernels of the vocoder and diffusion-step back end, shared by the drivers (hifigan.cu:
// Hifigan::forward, diffnet.cu: Diffnet::eps and gd_sample_loop) and the conformance probe (microbench.cu:
// agpt_voc_probe).  Each one launches its kernel with the production grid and block size and counts the launch; none
// synchronises.  Each one checks the preconditions its kernel's indexing relies on and throws before launching when
// they fail.  (cf_to_cl's launcher, launch_cf_to_cl, is declared in models.h.)
#pragma once
#include "common.cuh"

namespace agpt {

// conv_post: out [B][c_out][L] = tanh(b + Conv1d(k 7, pad 3) over lrelu(in, slope)), in [B][L][C] rows, w [c_out][7][C].
// Runs conv_post32_kernel (rows staged once in shared memory) when C == 32 and the weights take at most 8 KB, else the
// generic kernel; both accumulate in the same order.  C % 4 == 0 (float4 rows) and c_out 7 C 4 bytes <= 48 KB (dynamic
// shared memory without an opt-in).  Returns true when conv_post32_kernel ran.
bool launch_conv_post(const float* in, const float* w, const float* b, float* out, int B, int L, int C, int c_out,
                      float slope, cudaStream_t st);
// BigVGAN's Activation1d(Snake | SnakeBeta) on rows [B][L][C]: x -> y, a [C] = alpha (exp'd when log-scaled), inv_b [C]
// = 1 / (beta + 1e-9), taps [12] (HOST) = the Kaiser-sinc filter buffer.  L >= 1.
void aa_snake(const float* x, float* y, const float* a, const float* inv_b, const float* taps, int B, int L, int C,
              cudaStream_t st);
// NSF noise conv added in place: x [B][L][C] += bias[c] + sum_k w [C][K] har[b][p st - pad + k] over har [B][Lh]
// (taps outside [0, Lh) read zero).  K >= 1, st >= 1.
void nsf_add(float* x, const float* har, const float* w, const float* bias, int B, int L, int C, int Lh, int K, int stride,
             int pad, cudaStream_t st);
// SinusoidalPosEmb (NeuralSeq/modules/diff/net.py:37-44): out [B][C] = sin(t e) || cos(t e), e_i = exp(-i ln(1e4) /
// (C/2 - 1)), t_host [B] (HOST, passed by value in the kernel's parameters: B <= 256).  C even, C/2 > 1.
void diff_step_embed(const int* t_host, float* out, int B, int C, cudaStream_t st);
// The same with t_dev [N] on the device (the sampling loop embeds every step at once).  C even, C/2 > 1.
void diff_step_embed_dev(const int* t_dev, float* out, int N, int C, cudaStream_t st);
// The graph-replayed ancestral step: k = *ctr, coefficient row coef_tab[k] = {A, Bc, c1, c2, s} and
// x [B][n] <- c1 clamp(A x - Bc eps) + c2 x + s noise, noise = (*noises_pp) + (nsteps - 1 - k) noise_stride (none when
// *noises_pp is null); clamp to [-1, 1] only when clip.  B >= 1, n >= 1, nsteps >= 1.
void p_sample_tab(float* x, const float* eps, const float* const* noises_pp, long noise_stride, const float* coef_tab,
                  const int* ctr, int nsteps, int clip, int B, long n, cudaStream_t st);

}  // namespace agpt
