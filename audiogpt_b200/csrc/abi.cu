// extern "C" boundary of libagpt_b200.so (declared in include/agpt_b200.h).
#include <atomic>
#include "models.h"
#include "nn_kernels.h"
#include "tapconv.cuh"

namespace agpt {
static thread_local std::string g_last_error;
static std::atomic<long long> g_launches{0};
void set_last_error(const std::string& msg) { g_last_error = msg; }
void count_launch(long n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
long long launch_count_now() { return g_launches.load(std::memory_order_relaxed); }

template <typename F>
static int guarded(F&& f) {
  try {
    f();
    return 0;
  } catch (const std::exception& e) {
    set_last_error(e.what());
    return 1;
  } catch (...) {
    set_last_error("unknown C++ exception");
    return 2;
  }
}

static Handle* as(agpt_handle h, uint32_t magic, const char* what) {
  auto* p = reinterpret_cast<Handle*>(h);
  if (!p || p->magic != magic) throw Error(std::string("invalid handle: expected ") + what);
  return p;
}
}  // namespace agpt

using namespace agpt;

extern "C" {

const char* agpt_last_error(void) { return g_last_error.c_str(); }
int agpt_version(void) { return 100; }
long long agpt_launch_count(void) { return g_launches.load(); }

int agpt_profile_enable(int on) { return guarded([&] { profile_enable(on); }); }
long agpt_profile_dump(char* out, long cap) {
  long n = -1;
  guarded([&] { n = profile_dump(out, cap); });
  return n;
}
int agpt_profile_collect(double ms[4], double flops[4], double bytes[4], long long launches[4]) {
  return guarded([&] { profile_collect(ms, flops, bytes, launches); });
}
long long agpt_profile_tall_launches(void) { return profile_tall_launches(); }
long long agpt_profile_plane_launches(void) { return profile_plane_launches(); }
long long agpt_profile_dual_launches(void) { return profile_dual_launches(); }
long long agpt_profile_pipe_launches(void) { return profile_pipe_launches(); }
long long agpt_profile_narrow_pipe_launches(void) { return profile_narrow_pipe_launches(); }
long long agpt_profile_conv_pipe_launches(void) { return profile_conv_pipe_launches(); }
int agpt_set_tensor_cores(int on) { return guarded([&] { tc_set_enabled(on); }); }
int agpt_set_attention_tc(int on) { return guarded([&] { attention_set_tc(on); }); }
int agpt_attention(const float* q, int q_pitch, const float* k, int k_pitch, const float* v, int v_pitch, float* o,
                   int o_pitch, int N, int heads, int d, int Lq, int Lk, void* stream) {
  return guarded([&] {
    AGPT_CHECK(q && k && v && o && N >= 1 && heads >= 1 && Lq >= 1 && Lk >= 1, "bad argument");
    attention(q, q_pitch, k, k_pitch, v, v_pitch, o, o_pitch, N, heads, d, Lq, Lk, (cudaStream_t)stream);
  });
}
double agpt_fma_peak_tflops(void) {
  double v = -1.0;
  guarded([&] { v = fma_peak_tflops(); });
  return v;
}

void agpt_destroy(agpt_handle h) {
  auto* p = reinterpret_cast<Handle*>(h);
  if (!p) return;
  int prev = -1;
  cudaGetDevice(&prev);
  cudaSetDevice(p->device);
  cudaDeviceSynchronize();
  p->magic = 0;
  delete p;
  if (prev >= 0) cudaSetDevice(prev);
}

int agpt_hifigan_create(const agpt_hifigan_cfg* cfg, const float* const* host_weights, int n_weights,
                        int device, agpt_handle* out) {
  return guarded([&] {
    AGPT_CHECK(cfg && host_weights && out, "null argument");
    *out = reinterpret_cast<agpt_handle>(hifigan_create(cfg, host_weights, n_weights, device));
  });
}

int agpt_hifigan_forward(agpt_handle h, const float* mel, const float* har_source, int B, int T, float* wav,
                         void* stream) {
  return guarded([&] {
    AGPT_CHECK(mel && wav, "null tensor");
    hifigan_forward(as(h, kMagicHifigan, "hifigan"), mel, har_source, B, T, wav, (cudaStream_t)stream);
  });
}

int agpt_hifigan_vocode_host(agpt_handle h, const float* mel_host, const float* har_host, int B, int T,
                             float* wav_host) {
  return guarded([&] {
    AGPT_CHECK(mel_host && wav_host, "null tensor");
    hifigan_vocode_host(as(h, kMagicHifigan, "hifigan"), mel_host, har_host, B, T, wav_host);
  });
}

int agpt_nsf_source(const float* f0, int B, int L, int dim, float sampling_rate, const float* lin_w_host, float lin_b,
                    const float* rand_ini_or_null, const float* noise_or_null, float sine_amp, float noise_std,
                    float voiced_threshold, float* har_source, void* stream) {
  return guarded([&] {
    AGPT_CHECK(f0 && lin_w_host && har_source, "null argument");
    nsf_source(f0, B, L, dim, sampling_rate, lin_w_host, lin_b, rand_ini_or_null, noise_or_null, sine_amp, noise_std,
               voiced_threshold, har_source, (cudaStream_t)stream);
  });
}

int agpt_diffnet_create(const agpt_diffnet_cfg* cfg, const float* const* host_weights, int n_weights, int device,
                        agpt_handle* out) {
  return guarded([&] {
    AGPT_CHECK(cfg && host_weights && out, "null argument");
    *out = reinterpret_cast<agpt_handle>(diffnet_create(cfg, host_weights, n_weights, device));
  });
}

int agpt_diffnet_set_cond(agpt_handle h, const float* cond, int B, int T, void* stream) {
  return guarded([&] { diffnet_set_cond(as(h, kMagicDiffnet, "diffnet"), cond, B, T, (cudaStream_t)stream); });
}

int agpt_diffnet_eps(agpt_handle h, const float* x, const int* t_host, float* eps, void* stream) {
  return guarded([&] {
    AGPT_CHECK(x && t_host && eps, "null argument");
    diffnet_eps(as(h, kMagicDiffnet, "diffnet"), x, t_host, eps, (cudaStream_t)stream);
  });
}

int agpt_gd_p_sample(agpt_handle h_or_null, const float* x, const float* eps_or_null, const int* t_host,
                     const float* coef_host, const float* noise_or_null, int clip_denoised, int B,
                     long n_per_sample, float* x_out, void* stream) {
  return guarded([&] {
    AGPT_CHECK(x && coef_host && x_out && B >= 1, "null argument");
    Handle* hh = nullptr;
    if (!eps_or_null) { AGPT_CHECK(t_host, "t_host required when eps is computed internally"); hh = as(h_or_null, kMagicDiffnet, "diffnet"); }
    gd_p_sample(hh, x, eps_or_null, t_host, coef_host, noise_or_null, clip_denoised, B, n_per_sample, x_out,
                (cudaStream_t)stream);
  });
}

int agpt_gd_sample_loop(agpt_handle h, float* x_io, int t_hi, int t_lo, const float* coef_host, const float* noises_or_null,
                        long noise_step_stride, int clip_denoised, void* stream) {
  return guarded([&] {
    AGPT_CHECK(x_io && coef_host, "null argument");
    gd_sample_loop(as(h, kMagicDiffnet, "diffnet"), x_io, t_hi, t_lo, coef_host, noises_or_null, noise_step_stride,
                   clip_denoised, (cudaStream_t)stream);
  });
}

long agpt_diffnet_launches_per_step(agpt_handle h) {
  long n = -1;
  guarded([&] { n = diffnet_launches_per_step(as(h, kMagicDiffnet, "diffnet")); });
  return n;
}

int agpt_axpby5(const float* x, const float* e0, const float* e1, const float* e2, const float* e3,
                const float* coef_host, int B, long n_per_sample, float* out, void* stream) {
  return guarded([&] {
    AGPT_CHECK(x && coef_host && out && B >= 1, "null argument");
    axpby5(x, e0, e1, e2, e3, coef_host, B, n_per_sample, out, (cudaStream_t)stream);
  });
}

int agpt_unet_create(const agpt_unet_cfg* cfg, const float* const* host_weights, int n_weights, int device,
                     agpt_handle* out) {
  return guarded([&] {
    AGPT_CHECK(cfg && host_weights && out, "null argument");
    *out = reinterpret_cast<agpt_handle>(unet_create(cfg, host_weights, n_weights, device));
  });
}

int agpt_unet_set_context(agpt_handle h, const float* context, int N, int S, void* stream) {
  return guarded([&] {
    AGPT_CHECK(context, "null context");
    unet_set_context(as(h, kMagicUnet, "unet"), context, N, S, (cudaStream_t)stream);
  });
}

int agpt_unet_set_concat(agpt_handle h, const float* c, int N, int C, int H, int W, void* stream) {
  return guarded([&] {
    AGPT_CHECK(c, "null conditioning");
    unet_set_concat(as(h, kMagicUnet, "unet"), c, N, C, H, W, (cudaStream_t)stream);
  });
}

int agpt_unet_forward(agpt_handle h, const float* x, const int* t_host, int N, int H, int W, float* eps, void* stream) {
  return guarded([&] {
    AGPT_CHECK(x && t_host && eps, "null argument");
    unet_forward(as(h, kMagicUnet, "unet"), x, t_host, N, H, W, eps, (cudaStream_t)stream);
  });
}

int agpt_ddim_update(const float* x, const float* eps2, int eps2_is_single, float cfg_scale, float a_t, float a_prev,
                     float sigma_t, float sqrt_one_minus_at, const float* noise, float temperature, int B,
                     long n_per_sample, float* x_prev, float* pred_x0_or_null, void* stream) {
  return guarded([&] {
    AGPT_CHECK(x && eps2 && x_prev && B >= 1, "null argument");
    ddim_update(x, eps2, eps2_is_single, cfg_scale, a_t, a_prev, sigma_t, sqrt_one_minus_at, noise, temperature, B,
                n_per_sample, x_prev, pred_x0_or_null, (cudaStream_t)stream);
  });
}

int agpt_unet_ddim_sample(agpt_handle h, const float* x_T, int B, int H, int W, int S, const int* t_steps_host,
                          const float* a_t, const float* a_prev, const float* sigma, const float* sqrt_om,
                          float cfg_scale, float* x_out, float* pred_x0_or_null, void* stream) {
  return guarded([&] {
    AGPT_CHECK(x_T && t_steps_host && a_t && a_prev && sigma && sqrt_om && x_out && S >= 1 && B >= 1, "null argument");
    unet_ddim_sample(as(h, kMagicUnet, "unet"), x_T, B, H, W, S, t_steps_host, a_t, a_prev, sigma, sqrt_om, cfg_scale,
                     x_out, pred_x0_or_null, (cudaStream_t)stream);
  });
}

long agpt_unet_launches_per_step(agpt_handle h) {
  long n = -1;
  guarded([&] { n = unet_launches_per_step(as(h, kMagicUnet, "unet")); });
  return n;
}

int agpt_vae_create(const agpt_vae_cfg* cfg, const float* const* host_weights, int n_weights, int device,
                    agpt_handle* out) {
  return guarded([&] {
    AGPT_CHECK(cfg && host_weights && out, "null argument");
    *out = reinterpret_cast<agpt_handle>(vae_create(cfg, host_weights, n_weights, device));
  });
}

int agpt_vae_decode(agpt_handle h, const float* z, int B, int H, int W, float* out, void* stream) {
  return guarded([&] {
    AGPT_CHECK(z && out, "null argument");
    vae_decode(as(h, kMagicVae, "vae"), z, B, H, W, out, (cudaStream_t)stream);
  });
}

int agpt_vae_encoder_create(const agpt_vae_cfg* cfg, int in_channels, const float* const* host_weights, int n_weights,
                            int device, agpt_handle* out) {
  return guarded([&] {
    AGPT_CHECK(cfg && host_weights && out, "null argument");
    *out = reinterpret_cast<agpt_handle>(vae_encoder_create(cfg, in_channels, host_weights, n_weights, device));
  });
}

int agpt_vae_encode(agpt_handle h, const float* x, int B, int H, int W, float* moments, void* stream) {
  return guarded([&] {
    vae_encode(as(h, kMagicVaeEnc, "vae encoder"), x, B, H, W, moments, (cudaStream_t)stream);
  });
}

int agpt_pe_create(const agpt_pe_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out) {
  return guarded([&] {
    AGPT_CHECK(cfg && host_weights && out, "null argument");
    *out = reinterpret_cast<agpt_handle>(pe_create(cfg, host_weights, n_weights, device));
  });
}

int agpt_pe_forward(agpt_handle h, const float* mel, int B, int T, float* pitch_pred, float* f0_denorm, int use_uv,
                    int pitch_norm, float f0_mean, float f0_std, void* stream) {
  return guarded([&] {
    AGPT_CHECK(mel && pitch_pred && f0_denorm, "null argument");
    pe_forward(as(h, kMagicPe, "pitch extractor"), mel, B, T, pitch_pred, f0_denorm, use_uv, pitch_norm, f0_mean, f0_std,
               (cudaStream_t)stream);
  });
}

int agpt_attention_masked(const float* q, int q_pitch, const float* k, int k_pitch, const float* v, int v_pitch,
                          const uint8_t* key_padding_mask, float* o, int o_pitch, int N, int heads, int d, int Lq, int Lk, void* stream) {
  return guarded([&] {
    AGPT_CHECK(q && k && v && o && key_padding_mask && N >= 1 && heads >= 1 && Lq >= 1 && Lk >= 1, "bad argument");
    attention(q, q_pitch, k, k_pitch, v, v_pitch, o, o_pitch, N, heads, d, Lq, Lk, (cudaStream_t)stream, key_padding_mask);
  });
}

int agpt_fs2_create(const agpt_fs2_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out) {
  return guarded([&] {
    AGPT_CHECK(cfg && host_weights && out, "null argument");
    *out = reinterpret_cast<agpt_handle>(fs2_create(cfg, host_weights, n_weights, device));
  });
}

int agpt_fs2_encode(agpt_handle h, const int* txt_tokens, int B, int T_txt, const int* pitch_midi, const float* midi_dur,
                    const int* is_slur, int predict_dur, float* dur, int* dur_choice, int* mel_len_host, void* stream) {
  return guarded([&] {
    AGPT_CHECK(txt_tokens && dur && (!predict_dur || mel_len_host), "null argument");
    fs2_encode(as(h, kMagicFs2, "fastspeech2"), txt_tokens, B, T_txt, pitch_midi, midi_dur, is_slur, predict_dur, dur, dur_choice,
               mel_len_host, (cudaStream_t)stream);
  });
}

int agpt_fs2_decode(agpt_handle h, int T_mel, const int* mel2ph, int* mel2ph_out, const float* f0, const float* uv, const float* energy,
                    int use_uv, int pitch_norm, float f0_mean, float f0_std, float* pitch_pred, float* f0_denorm, int* pitch_coarse,
                    float* energy_pred, float* decoder_inp, float* mel_out, void* stream) {
  return guarded([&] {
    fs2_decode(as(h, kMagicFs2, "fastspeech2"), T_mel, mel2ph, mel2ph_out, f0, uv, energy, use_uv, pitch_norm, f0_mean, f0_std, pitch_pred,
               f0_denorm, pitch_coarse, energy_pred, decoder_inp, mel_out, (cudaStream_t)stream);
  });
}

int agpt_gs_create(const agpt_gs_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out) {
  return guarded([&] {
    AGPT_CHECK(cfg && host_weights && out, "null argument");
    *out = reinterpret_cast<agpt_handle>(gs_create(cfg, host_weights, n_weights, device));
  });
}

int agpt_gs_encode(agpt_handle h, const int* txt_tokens, int B, int T_txt, const float* spk_embed, const float* emo_embed, int predict_dur,
                   float* dur, int* dur_choice, int* mel_len_host, float* spk_out, float* emo_out, void* stream) {
  return guarded([&] {
    AGPT_CHECK(txt_tokens && spk_embed && emo_embed && dur && (!predict_dur || mel_len_host), "null argument");
    gs_encode(as(h, kMagicGs, "generspeech"), txt_tokens, B, T_txt, spk_embed, emo_embed, predict_dur, dur, dur_choice, mel_len_host,
              spk_out, emo_out, (cudaStream_t)stream);
  });
}

int agpt_gs_forward(agpt_handle h, int T_mel, const int* mel2ph, int* mel2ph_out, const float* ref_mels, int T_ref, const int* ref_mel2ph,
                    int n_seg_ph, const int* ref_mel2word, int n_seg_word, const float* z, float f0_mean, float f0_std, float* pitch_pred,
                    float* f0_denorm, float* f0_denorm_pred, int* pitch_coarse, float* decoder_inp, float* ref_prosody, float* mel_out,
                    const agpt_gs_taps* taps, void* stream) {
  return guarded([&] {
    gs_forward(as(h, kMagicGs, "generspeech"), T_mel, mel2ph, mel2ph_out, ref_mels, T_ref, ref_mel2ph, n_seg_ph, ref_mel2word, n_seg_word, z,
               f0_mean, f0_std, pitch_pred, f0_denorm, f0_denorm_pred, pitch_coarse, decoder_inp, ref_prosody, mel_out, taps,
               (cudaStream_t)stream);
  });
}

int agpt_clap_create(const agpt_clap_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out) {
  return guarded([&] {
    AGPT_CHECK(cfg && host_weights && out, "null argument");
    *out = reinterpret_cast<agpt_handle>(clap_create(cfg, host_weights, n_weights, device));
  });
}

int agpt_clap_encode(agpt_handle h, const int* input_ids, int N, int L, float* z, void* stream) {
  return guarded([&] {
    AGPT_CHECK(input_ids && z, "null argument");
    clap_encode(as(h, kMagicClap, "clap"), input_ids, N, L, z, (cudaStream_t)stream);
  });
}

int agpt_clap_encode_cls(agpt_handle h, const int* input_ids, const int* token_type_ids, const int* attention_mask, int N,
                         int L, float* out, void* stream) {
  return guarded([&] {
    AGPT_CHECK(input_ids && token_type_ids && attention_mask && out, "null argument");
    clap_encode_cls(as(h, kMagicClap, "clap"), input_ids, token_type_ids, attention_mask, N, L, out, (cudaStream_t)stream);
  });
}

int agpt_clap_similarity(const float* a, int Na, const float* t, int Nt, int D, float scale, float* out, void* stream) {
  return guarded([&] {
    AGPT_CHECK(a && t && out, "null argument");
    clap_similarity(a, Na, t, Nt, D, scale, out, (cudaStream_t)stream);
  });
}

int agpt_cnn14_create(const agpt_cnn14_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out) {
  return guarded([&] {
    AGPT_CHECK(cfg && host_weights && out, "null argument");
    *out = reinterpret_cast<agpt_handle>(cnn14_create(cfg, host_weights, n_weights, device));
  });
}

int agpt_cnn14_set_resample(agpt_handle h, int orig_freq, int new_freq, int width, const float* table_host, int clip_samples) {
  return guarded([&] {
    cnn14_set_resample(as(h, kMagicCnn14, "cnn14"), orig_freq, new_freq, width, table_host, clip_samples);
  });
}

int agpt_cnn14_embed(agpt_handle h, const float* wav, long n_samples, int B, const int* start_or_tile_host, float* out_emb,
                     void* stream) {
  return guarded([&] {
    AGPT_CHECK(wav && start_or_tile_host && out_emb, "null argument");
    cnn14_embed(as(h, kMagicCnn14, "cnn14"), wav, n_samples, B, start_or_tile_host, out_emb, (cudaStream_t)stream);
  });
}

int agpt_lass_create(const agpt_lass_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out) {
  return guarded([&] {
    AGPT_CHECK(cfg && host_weights && out, "null argument");
    *out = reinterpret_cast<agpt_handle>(lass_create(cfg, host_weights, n_weights, device));
  });
}

int agpt_lass_text(agpt_handle h, const int* input_ids, const int* attention_mask, int N, int L, float* cond, void* stream) {
  return guarded([&] {
    AGPT_CHECK(input_ids && attention_mask && cond, "null argument");
    lass_text(as(h, kMagicLass, "lass"), input_ids, attention_mask, N, L, cond, (cudaStream_t)stream);
  });
}

int agpt_lass_mask(agpt_handle h, const float* mag, int B, int T, int F, long stride_b, long stride_t, long stride_f,
                   const float* cond, float* mask, float* logits, void* stream) {
  return guarded([&] {
    AGPT_CHECK(mag && cond && mask, "null argument");
    lass_mask(as(h, kMagicLass, "lass"), mag, B, T, F, stride_b, stride_t, stride_f, cond, mask, logits, (cudaStream_t)stream);
  });
}

int agpt_stft_create(int filter_length, int hop_length, const float* const* host_weights, int n_weights, int device,
                     agpt_handle* out) {
  return guarded([&] {
    AGPT_CHECK(host_weights && out, "null argument");
    AGPT_CHECK(n_weights == 2, "the STFT takes forward_basis and inverse_basis");
    *out = reinterpret_cast<agpt_handle>(stft_create(filter_length, hop_length, host_weights[0], host_weights[1], device));
  });
}

int agpt_stft_transform(agpt_handle h, const float* wav, int B, long n_samples, float* magnitude, float* phase, void* stream) {
  return guarded([&] {
    AGPT_CHECK(wav && magnitude && phase, "null argument");
    stft_transform(as(h, kMagicStft, "stft"), wav, B, n_samples, magnitude, phase, (cudaStream_t)stream);
  });
}

int agpt_stft_inverse(agpt_handle h, const float* magnitude, const float* phase, int B, int T, float* wav, void* stream) {
  return guarded([&] {
    AGPT_CHECK(magnitude && phase && wav, "null argument");
    stft_inverse(as(h, kMagicStft, "stft"), magnitude, phase, B, T, wav, (cudaStream_t)stream);
  });
}

int agpt_pvt_create(const agpt_pvt_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out) {
  return guarded([&] {
    AGPT_CHECK(cfg && host_weights && out, "null argument");
    *out = reinterpret_cast<agpt_handle>(pvt_create(cfg, host_weights, n_weights, device));
  });
}

int agpt_pvt_frames(const agpt_pvt_cfg* cfg, long n_samples, int grid_hw[4][2]) {
  return guarded([&] {
    AGPT_CHECK(cfg && grid_hw, "null argument");
    pvt_frames(cfg, n_samples, grid_hw);
  });
}

int agpt_pvt_forward(agpt_handle h, const float* wav, int B, long n_samples, float* framewise, float* clipwise, float* logits,
                     void* stream) {
  return guarded([&] {
    AGPT_CHECK(wav && framewise && clipwise, "null argument");
    pvt_forward(as(h, kMagicPvt, "pvt"), wav, B, n_samples, framewise, clipwise, logits, (cudaStream_t)stream);
  });
}

int agpt_pvt_dwconv_gelu(const float* x, const float* w, const float* bias, int B, int H, int W, int C, float* out, void* plane_hi,
                         void* plane_lo, void* stream) {
  return guarded([&] {
    AGPT_CHECK(x && w && bias, "null argument");
    pvt_dwconv_gelu(x, w, bias, B, H, W, C, out, static_cast<__half*>(plane_hi), static_cast<__half*>(plane_lo), (cudaStream_t)stream);
  });
}

int agpt_pvt_patch7(const float* img, const float* w, const float* bias, const float* gamma, const float* beta, float eps, int B,
                    int H, int W, int C, float* out, void* stream) {
  return guarded([&] {
    AGPT_CHECK(img && w && bias && gamma && beta && out, "null argument");
    pvt_patch7(img, w, bias, gamma, beta, eps, B, H, W, C, out, (cudaStream_t)stream);
  });
}

int agpt_pvt_sr_gather(const float* x, int B, int H, int W, int C, int sr, float* out, void* stream) {
  return guarded([&] {
    AGPT_CHECK(x && out, "null argument");
    pvt_sr_gather(x, B, H, W, C, sr, out, (cudaStream_t)stream);
  });
}

int agpt_pvt_head(const float* x, const float* w, const float* bias, int B, int H, int W, int C, int classes, int ratio,
                  float* framewise, float* clipwise, float* logits, void* stream) {
  return guarded([&] {
    AGPT_CHECK(x && w && bias && framewise && clipwise, "null argument");
    pvt_head(x, w, bias, B, H, W, C, classes, ratio, framewise, clipwise, logits, (cudaStream_t)stream);
  });
}

int agpt_tsd_create(const agpt_tsd_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out) {
  return guarded([&] {
    AGPT_CHECK(cfg && host_weights && out, "null argument");
    *out = reinterpret_cast<agpt_handle>(tsd_create(cfg, host_weights, n_weights, device));
  });
}

int agpt_tsd_frames(const agpt_tsd_cfg* cfg, int T, int Tr, int frames[3]) {
  return guarded([&] {
    AGPT_CHECK(cfg && frames, "null argument");
    tsd_frames(cfg, T, Tr, frames);
  });
}

int agpt_tsd_forward(agpt_handle h, const float* x, const float* ref, int B, int T, int Tr, float* decision, float* decision_up,
                     void* stream) {
  return guarded([&] {
    AGPT_CHECK(x && ref && decision && decision_up, "null argument");
    tsd_forward(as(h, kMagicTsd, "tsd"), x, ref, B, T, Tr, decision, decision_up, (cudaStream_t)stream);
  });
}

int agpt_tsd_stage_events(agpt_handle h, void* events, int n) {
  return guarded([&] {
    AGPT_CHECK(n == 0 || events, "null argument");
    tsd_stage_events(as(h, kMagicTsd, "tsd"), static_cast<void* const*>(events), n);
  });
}

int agpt_tsd_stem(const float* mel, const float* w, const float* b, int B, int T, int ph, float* out, void* stream) {
  return guarded([&] {
    AGPT_CHECK(mel && w && b && out, "null argument");
    tsd_stem(mel, w, b, B, T, ph, out, (cudaStream_t)stream);
  });
}

int agpt_tsd_avgpool(const float* in, int B, int H, int W, int C, int ph, int pw, float* out, void* stream) {
  return guarded([&] {
    AGPT_CHECK(in && out, "null argument");
    tsd_avgpool(in, B, H, W, C, ph, pw, out, (cudaStream_t)stream);
  });
}

int agpt_tsd_gru(const float* w_hh, const float* b_hh, const float* xproj, int B, int T, float* out, void* stream) {
  return guarded([&] {
    AGPT_CHECK(w_hh && b_hh && xproj && out, "null argument");
    tsd_gru(w_hh, b_hh, xproj, B, T, out, (cudaStream_t)stream);
  });
}

int agpt_tsd_enhance(const float* p1, int B, int Td, int O, const float* mix_emb, int Te, const float* emb, int top, float tao,
                     const float* const* weights8, float* me, float* wmix, int* topk_idx, float* topk_val, void* stream) {
  return guarded([&] {
    AGPT_CHECK(p1 && mix_emb && emb && weights8 && me && wmix && topk_idx, "null argument");
    for (int i = 0; i < 8; ++i) AGPT_CHECK(weights8[i], "null weight");
    tsd_enhance(p1, B, Td, O, mix_emb, Te, emb, top, tao, weights8, me, wmix, topk_idx, topk_val, (cudaStream_t)stream);
  });
}

int agpt_binaural_create(const agpt_binaural_cfg* cfg, const float* const* host_weights, int n_weights, int device,
                         agpt_handle* out) {
  return guarded([&] {
    AGPT_CHECK(cfg && host_weights && out, "null argument");
    *out = reinterpret_cast<agpt_handle>(binaural_create(cfg, host_weights, n_weights, device));
  });
}

int agpt_binaural_forward(agpt_handle h, const float* mono, const float* view, const agpt_binaural_row* rows, int n_rows,
                          float* out, int clamp, void* stream) {
  return guarded([&] {
    AGPT_CHECK(mono && view && out, "null argument");
    binaural_forward(as(h, kMagicBinaural, "binaural"), mono, view, rows, n_rows, out, clamp, (cudaStream_t)stream);
  });
}

int agpt_binaural_frames(agpt_handle h, const float* view, const agpt_binaural_row* rows, int n_rows, float* field, void* stream) {
  return guarded([&] {
    AGPT_CHECK(view && field, "null argument");
    binaural_frames(as(h, kMagicBinaural, "binaural"), view, rows, n_rows, field, (cudaStream_t)stream);
  });
}

int agpt_binaural_warp(agpt_handle h, const float* field, const float* mono, const agpt_binaural_row* rows, int n_rows,
                       float* out, int clamp, void* stream) {
  return guarded([&] {
    AGPT_CHECK(field && mono && out, "null argument");
    binaural_warp(as(h, kMagicBinaural, "binaural"), field, mono, rows, n_rows, out, clamp, (cudaStream_t)stream);
  });
}

int agpt_w2v_create(const agpt_w2v_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out) {
  return guarded([&] {
    AGPT_CHECK(cfg && host_weights && out, "null argument");
    *out = reinterpret_cast<agpt_handle>(w2v_create(cfg, host_weights, n_weights, device));
  });
}

int agpt_w2v_frames(const agpt_w2v_cfg* cfg, long n_samples, int* frames) {
  return guarded([&] {
    AGPT_CHECK(cfg && frames, "null argument");
    AGPT_CHECK(cfg->conv_layers >= 1 && cfg->conv_layers <= AGPT_W2V_MAX_CONV, "conv_layers must be 1..8");
    for (int i = 0; i < cfg->conv_layers; ++i) AGPT_CHECK(cfg->conv_kernel[i] >= 1 && cfg->conv_stride[i] >= 1, "bad conv geometry");
    w2v_lengths(cfg, n_samples, frames);
  });
}

int agpt_w2v_logits(agpt_handle h, const float* input_values, int B, long n_samples, float* logits, void* stream) {
  return guarded([&] {
    AGPT_CHECK(input_values && logits, "null argument");
    w2v_logits(as(h, kMagicW2v, "w2v"), input_values, B, n_samples, logits, (cudaStream_t)stream);
  });
}

int agpt_w2v_features(agpt_handle h, const float* input_values, int B, long n_samples, float* features, void* stream) {
  return guarded([&] {
    AGPT_CHECK(input_values && features, "null argument");
    w2v_features(as(h, kMagicW2v, "w2v"), input_values, B, n_samples, features, (cudaStream_t)stream);
  });
}

int agpt_w2v_pos_conv(agpt_handle h, const float* hidden, int B, int T, float* out, void* stream) {
  return guarded([&] {
    AGPT_CHECK(hidden && out, "null argument");
    w2v_pos_conv(as(h, kMagicW2v, "w2v"), hidden, B, T, out, (cudaStream_t)stream);
  });
}

int agpt_emo_create(const agpt_emo_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out) {
  return guarded([&] {
    AGPT_CHECK(cfg && host_weights && out, "null argument");
    *out = reinterpret_cast<agpt_handle>(emo_create(cfg, host_weights, n_weights, device));
  });
}

int agpt_emo_partials(long n_samples, int partial_frames, double min_pad_coverage, double overlap, int* n_partials, int* frame_step,
                      long* padded) {
  return guarded([&] {
    AGPT_CHECK(n_partials && frame_step && padded, "null argument");
    emo_partials(n_samples, partial_frames, min_pad_coverage, overlap, n_partials, frame_step, padded);
  });
}

int agpt_emo_embed(agpt_handle h, const float* wav, long n_samples, int partial_frames, double min_pad_coverage, double overlap,
                   float* embed, float* partials, void* stream) {
  return guarded([&] {
    AGPT_CHECK(wav && embed, "null argument");
    emo_embed(as(h, kMagicEmo, "emotion"), wav, n_samples, partial_frames, min_pad_coverage, overlap, embed, partials,
              (cudaStream_t)stream);
  });
}

int agpt_emo_hidden(agpt_handle h, const float* frames, int N, int T, float* hidden, void* stream) {
  return guarded([&] {
    AGPT_CHECK(frames && hidden, "null argument");
    emo_hidden(as(h, kMagicEmo, "emotion"), frames, N, T, hidden, (cudaStream_t)stream);
  });
}

int agpt_emo_forward(agpt_handle h, const float* frames, int N, int T, float* embeds, void* stream) {
  return guarded([&] {
    AGPT_CHECK(frames && embeds, "null argument");
    emo_forward(as(h, kMagicEmo, "emotion"), frames, N, T, embeds, (cudaStream_t)stream);
  });
}

int agpt_emo_mel(agpt_handle h, const float* wav, long n_samples, float* mel, void* stream) {
  return guarded([&] {
    AGPT_CHECK(wav && mel, "null argument");
    emo_mel(as(h, kMagicEmo, "emotion"), wav, n_samples, mel, (cudaStream_t)stream);
  });
}

int agpt_emo_lstm(const float* w_hh, const float* xproj, int N, int T, long seq_stride, float* h_seq, float* h_last, void* stream) {
  return guarded([&] {
    AGPT_CHECK(w_hh && xproj, "null argument");
    emo_lstm(w_hh, xproj, N, T, seq_stride, h_seq, h_last, (cudaStream_t)stream);
  });
}

int agpt_tapconv_probe(const agpt_tapconv_probe_args* args, int ran[4], void* stream) {
  return guarded([&] {
    AGPT_CHECK(args && ran, "null argument");
    int r[5];
    for (int i = 0; i < 4; ++i) ran[i] = -1;
    tapconv_probe(*args, agpt_tapconv_pipes{}, r, (cudaStream_t)stream);
    for (int i = 0; i < 4; ++i) ran[i] = r[i];
  });
}

int agpt_tapconv_probe_pipes(const agpt_tapconv_probe_args* args, const agpt_tapconv_pipes* pipes, int ran[5],
                             void* stream) {
  return guarded([&] {
    AGPT_CHECK(args && pipes && ran, "null argument");
    tapconv_probe(*args, *pipes, ran, (cudaStream_t)stream);
  });
}

int agpt_nn_probe(const agpt_nn_probe_args* args, void* stream) {
  return guarded([&] {
    AGPT_CHECK(args, "null argument");
    nn_probe(*args, (cudaStream_t)stream);
  });
}

int agpt_fs_probe(const agpt_fs_probe_args* args, void* stream) {
  return guarded([&] {
    AGPT_CHECK(args, "null argument");
    fs_probe(*args, (cudaStream_t)stream);
  });
}

int agpt_audio_probe(const agpt_audio_probe_args* args, void* stream) {
  return guarded([&] {
    AGPT_CHECK(args, "null argument");
    audio_probe(*args, (cudaStream_t)stream);
  });
}

int agpt_voc_probe(const agpt_voc_probe_args* args, void* stream) {
  return guarded([&] {
    AGPT_CHECK(args, "null argument");
    voc_probe(*args, (cudaStream_t)stream);
  });
}

int agpt_an_probe(const agpt_an_probe_args* args, void* stream) {
  return guarded([&] {
    AGPT_CHECK(args, "null argument");
    const bool handle_op = args->op == AGPT_AN_LASS_FILM_VEC || args->op == AGPT_AN_LASS_UP;
    an_probe(*args, handle_op ? as(reinterpret_cast<agpt_handle>(args->h), kMagicLass, "lass") : nullptr,
             (cudaStream_t)stream);
  });
}

}  // extern "C"
