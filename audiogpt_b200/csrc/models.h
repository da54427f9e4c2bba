// Internal C++ entry points behind the C ABI (include/agpt_b200.h).
#pragma once
#include "../../include/agpt_b200.h"
#include "common.cuh"

namespace agpt {

void count_launch(long n);
long long launch_count_now();
bool profile_enabled();

void launch_cf_to_cl(const float* in, float* out, int B, int C, int T, cudaStream_t st);

Handle* hifigan_create(const agpt_hifigan_cfg* cfg, const float* const* W, int nW, int device);
void hifigan_forward(Handle* h, const float* mel, const float* har, int B, int T, float* wav, cudaStream_t st);
void hifigan_vocode_host(Handle* h, const float* mel_host, const float* har_host, int B, int T, float* wav_host);

void nsf_source(const float* f0, int B, int L, int dim, float sr, const float* lin_w_host, float lin_b,
                const float* rand_ini, const float* noise, float sine_amp, float noise_std, float thr, float* har,
                cudaStream_t st);

Handle* diffnet_create(const agpt_diffnet_cfg* cfg, const float* const* W, int nW, int device);
void diffnet_set_cond(Handle* h, const float* cond, int B, int T, cudaStream_t st);
void diffnet_eps(Handle* h, const float* x, const int* t_host, float* eps, cudaStream_t st);
void gd_p_sample(Handle* h_or_null, const float* x, const float* eps_or_null, const int* t_host, const float* coef_host,
                 const float* noise, int clip, int B, long n, float* x_out, cudaStream_t st);
void gd_sample_loop(Handle* h, float* x_io, int t_hi, int t_lo, const float* coef_host, const float* noises,
                    long noise_stride, int clip, cudaStream_t st);
long diffnet_launches_per_step(Handle* h);
void axpby5(const float* x, const float* e0, const float* e1, const float* e2, const float* e3,
            const float* coef_host, int B, long n, float* out, cudaStream_t st);

Handle* unet_create(const agpt_unet_cfg* cfg, const float* const* W, int nW, int device);
void unet_set_context(Handle* h, const float* ctx, int N, int S, cudaStream_t st);
void unet_set_concat(Handle* h, const float* c, int N, int C, int H, int W, cudaStream_t st);
void unet_forward(Handle* h, const float* x, const int* t_host, int N, int H, int W, float* eps, cudaStream_t st);
void unet_ddim_sample(Handle* h, const float* x_T, int B, int H, int W, int S, const int* t_steps,
                      const float* a_t, const float* a_prev, const float* sigma, const float* sqrt_om,
                      float cfg_scale, float* x_out, float* pred_x0_out, cudaStream_t st);
long unet_launches_per_step(Handle* h);

Handle* vae_create(const agpt_vae_cfg* cfg, const float* const* W, int nW, int device);
void vae_decode(Handle* h, const float* z, int B, int H, int W, float* out, cudaStream_t st);
Handle* vae_encoder_create(const agpt_vae_cfg* cfg, int in_channels, const float* const* W, int nW, int device);
void vae_encode(Handle* h, const float* x, int B, int H, int W, float* moments, cudaStream_t st);

Handle* pe_create(const agpt_pe_cfg* cfg, const float* const* W, int nW, int device);
void pe_forward(Handle* h, const float* mel, int B, int T, float* pitch_pred, float* f0, int use_uv, int norm_mode,
                float f0_mean, float f0_std, cudaStream_t st);

Handle* fs2_create(const agpt_fs2_cfg* cfg, const float* const* W, int nW, int device);
void fs2_encode(Handle* h, const int* tok, int B, int T, const int* pmidi, const float* mdur, const int* slur, int predict, float* dur,
                int* dur_choice, int* mel_len_host, cudaStream_t st);
void fs2_decode(Handle* h, int Tm, const int* mel2ph_in, int* mel2ph_out, const float* f0, const float* uv, const float* energy, int use_uv,
                int norm, float f0_mean, float f0_std, float* pitch_pred, float* f0d, int* coarse, float* e_pred, float* dec_inp, float* mel,
                cudaStream_t st);

Handle* clap_create(const agpt_clap_cfg* cfg, const float* const* W, int nW, int device);
void clap_encode(Handle* h, const int* ids, int N, int L, float* z, cudaStream_t st);
void clap_encode_cls(Handle* h, const int* ids, const int* type_ids, const int* mask, int N, int L, float* out, cudaStream_t st);
void clap_similarity(const float* a, int Na, const float* t, int Nt, int D, float scale, float* out, cudaStream_t st);

Handle* cnn14_create(const agpt_cnn14_cfg* cfg, const float* const* W, int nW, int device);
void cnn14_set_resample(Handle* h, int orig, int nw, int width, const float* table, int clip);
void cnn14_embed(Handle* h, const float* wav, long n_samples, int B, const int* start_host, float* out, cudaStream_t st);

void bench_tapconv(int G, int L, int Cin, int Cout, int K, int dil, int Wreal, int epi_res, int use_tc, int reps,
                   double* out, double* dbg_avg);
void tapconv_probe(const agpt_tapconv_probe_args& a, int ran[4], cudaStream_t st);

}  // namespace agpt
