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

int agpt_bench_tapconv(int G, int L, int Cin, int Cout, int K, int dil, int Wreal, int epi_res, int use_tc, int reps,
                       double* out2, double* dbg8_or_null) {
  return guarded([&] {
    AGPT_CHECK(out2, "null argument");
    bench_tapconv(G, L, Cin, Cout, K, dil, Wreal, epi_res, use_tc, reps, out2, dbg8_or_null);
  });
}

int agpt_tapconv_probe(const agpt_tapconv_probe_args* args, int ran[4], void* stream) {
  return guarded([&] {
    AGPT_CHECK(args && ran, "null argument");
    tapconv_probe(*args, ran, (cudaStream_t)stream);
  });
}

}  // extern "C"
