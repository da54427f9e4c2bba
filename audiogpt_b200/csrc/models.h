// Internal C++ entry points behind the C ABI (include/agpt_b200.h).
#pragma once
#include "../../include/agpt_b200.h"
#include <cuda_fp16.h>
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

Handle* gs_create(const agpt_gs_cfg* cfg, const float* const* W, int nW, int device);
void gs_encode(Handle* h, const int* tok, int B, int T, const float* spk, const float* emo, int predict, float* dur, int* dur_choice,
               int* mel_len_host, float* spk_out, float* emo_out, cudaStream_t st);
void gs_forward(Handle* h, int Tm, const int* mel2ph, int* mel2ph_out, const float* ref_mels, int Tr, const int* ref_mel2ph, int nseg_ph,
                const int* ref_mel2word, int nseg_word, const float* z, float f0_mean, float f0_std, float* pitch_pred, float* f0d,
                float* f0d_pred, int* coarse, float* dec_inp, float* ref_prosody, float* mel, const agpt_gs_taps* taps, cudaStream_t st);

Handle* clap_create(const agpt_clap_cfg* cfg, const float* const* W, int nW, int device);
void clap_encode(Handle* h, const int* ids, int N, int L, float* z, cudaStream_t st);
void clap_encode_cls(Handle* h, const int* ids, const int* type_ids, const int* mask, int N, int L, float* out, cudaStream_t st);
void clap_similarity(const float* a, int Na, const float* t, int Nt, int D, float scale, float* out, cudaStream_t st);

Handle* cnn14_create(const agpt_cnn14_cfg* cfg, const float* const* W, int nW, int device);
void cnn14_set_resample(Handle* h, int orig, int nw, int width, const float* table, int clip);
void cnn14_embed(Handle* h, const float* wav, long n_samples, int B, const int* start_host, float* out, cudaStream_t st);

Handle* lass_create(const agpt_lass_cfg* cfg, const float* const* W, int nW, int device);
void lass_text(Handle* h, const int* ids, const int* mask, int N, int L, float* cond, cudaStream_t st);
void lass_mask(Handle* h, const float* mag, int B, int T, int F, long sb, long st_, long sf, const float* cond, float* mask,
               float* logits, cudaStream_t st);
// the probe's view of a LASSNet handle: its FiLM vectors for cond [B][256] into vec [B][vec_len] (vec null: nothing
// runs), returning vec_len; and decoder level `level`'s up path (LassNet::up) on caller-owned maps
int lass_film_vec(Handle* h, const float* cond, int B, float* vec, cudaStream_t st);
void lass_up(Handle* h, int level, const float* y, const float* skip, int B, int hh, int w, float* cat, cudaStream_t st);
Handle* stft_create(int filter_length, int hop_length, const float* fwd_basis, const float* inv_basis, int device);
void stft_transform(Handle* h, const float* wav, int B, long n_samples, float* mag, float* phase, cudaStream_t st);
void stft_inverse(Handle* h, const float* mag, const float* phase, int B, int T, float* wav, cudaStream_t st);

Handle* pvt_create(const agpt_pvt_cfg* cfg, const float* const* W, int nW, int device);
void pvt_frames(const agpt_pvt_cfg* cfg, long n_samples, int grid_hw[4][2]);
void pvt_forward(Handle* h, const float* wav, int B, long n_samples, float* framewise, float* clipwise, float* logits, cudaStream_t st);
void pvt_patch7(const float* img, const float* w, const float* bias, const float* gamma, const float* beta, float eps, int B, int H,
                int W, int C, float* out, cudaStream_t st);
void pvt_sr_gather(const float* x, int B, int H, int W, int C, int sr, float* out, cudaStream_t st);
void pvt_dwconv_gelu(const float* x, const float* w, const float* bias, int B, int H, int W, int C, float* out, __half* phi, __half* plo,
                     cudaStream_t st);
void pvt_head(const float* x, const float* w, const float* bias, int B, int H, int W, int C, int classes, int ratio, float* framewise,
              float* clipwise, float* logits, cudaStream_t st);

Handle* tsd_create(const agpt_tsd_cfg* cfg, const float* const* W, int nW, int device);
void tsd_frames(const agpt_tsd_cfg* cfg, int T, int Tr, int frames[3]);
void tsd_forward(Handle* h, const float* x, const float* ref, int B, int T, int Tr, float* decision, float* decision_up, cudaStream_t st);
constexpr int kTsdStages = 6;   // agpt_tsd_stage_events: the stage boundaries one forward records
void tsd_stage_events(Handle* h, void* const* events, int n);
void tsd_stem(const float* mel, const float* w, const float* b, int B, int T, int ph, float* out, cudaStream_t st);
void tsd_avgpool(const float* in, int B, int H, int W, int C, int ph, int pw, float* out, cudaStream_t st);
void tsd_gru(const float* whh, const float* bhh, const float* xp, int B, int T, float* out, cudaStream_t st);
void tsd_enhance(const float* p1, int B, int Td, int O, const float* Emix, int Te, const float* emb, int top, float tao,
                 const float* const wts[8], float* me, float* wmix, int* idx, float* val, cudaStream_t st);

Handle* binaural_create(const agpt_binaural_cfg* cfg, const float* const* W, int nW, int device);
void binaural_forward(Handle* h, const float* mono, const float* view, const agpt_binaural_row* rows, int n, float* out, int clamp,
                      cudaStream_t st);
void binaural_frames(Handle* h, const float* view, const agpt_binaural_row* rows, int n, float* field, cudaStream_t st);
void binaural_warp(Handle* h, const float* field, const float* mono, const agpt_binaural_row* rows, int n, float* out, int clamp,
                   cudaStream_t st);

Handle* w2v_create(const agpt_w2v_cfg* cfg, const float* const* W, int nW, int device);
void w2v_lengths(const agpt_w2v_cfg* cfg, long S, int* frames);
void w2v_logits(Handle* h, const float* x, int B, long S, float* logits, cudaStream_t st);
void w2v_features(Handle* h, const float* x, int B, long S, float* feats, cudaStream_t st);
void w2v_pos_conv(Handle* h, const float* x, int B, int T, float* y, cudaStream_t st);

Handle* emo_create(const agpt_emo_cfg* cfg, const float* const* W, int nW, int device);
void emo_partials(long n_samples, int partial_frames, double min_pad_coverage, double overlap, int* n_partials, int* frame_step,
                  long* padded);
void emo_mel(Handle* h, const float* wav, long n, float* mel, cudaStream_t st);
void emo_lstm(const float* whh, const float* xp, int N, int T, long seq_stride, float* h_seq, float* h_last, cudaStream_t st);
void emo_hidden(Handle* h, const float* frames, int N, int T, float* hidden, cudaStream_t st);
void emo_forward(Handle* h, const float* frames, int N, int T, float* embeds, cudaStream_t st);
void emo_embed(Handle* h, const float* wav, long n, int partial_frames, double min_pad_coverage, double overlap, float* embed,
               float* partials, cudaStream_t st);

void tapconv_probe(const agpt_tapconv_probe_args& a, const agpt_tapconv_pipes& sw, int ran[5], cudaStream_t st);
void nn_probe(const agpt_nn_probe_args& a, cudaStream_t st);
void fs_probe(const agpt_fs_probe_args& a, cudaStream_t st);
void audio_probe(const agpt_audio_probe_args& a, cudaStream_t st);
void voc_probe(const agpt_voc_probe_args& a, cudaStream_t st);
void an_probe(const agpt_an_probe_args& a, Handle* lass, cudaStream_t st);

}  // namespace agpt
