/* libagpt_b200 -- C ABI of the H100 (sm_90a) AudioGPT generative back-end.
 *
 * The reference (AIGC-Audio/AudioGPT) is pure Python: it has no FFI layer, its
 * "plugin boundary" is the Python class surface listed in SURVEY.md 8(b).  The
 * drop-in Python classes in audiogpt_b200/ bind these entry points through
 * ctypes (audiogpt_b200/_lib.py); INTEGRATION.md shows the stub.  Each entry
 * point cites the reference interface it replaces.
 *
 * Conventions: every function returns 0 on success, non-zero on error with a
 * thread-local message retrievable through agpt_last_error().  Device pointers
 * are plain fp32 arrays, valid for the stream-ordered duration of the call;
 * `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 * Weights are copied and re-laid-out at create time (the handle owns them).
 * One handle per device; a handle is not re-entrant.  There is no CPU fallback.
 */
#ifndef AGPT_B200_H
#define AGPT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct agpt_handle_s* agpt_handle;

const char* agpt_last_error(void);
int agpt_version(void);
/* number of kernels launched by this library in this process so far (bench.py's gpu_launches) */
long long agpt_launch_count(void);
void agpt_destroy(agpt_handle h);
/* Measurement helpers (bench.py): per-launch CUDA-event timing of the tapconv kernel,
 * summed per variant v = {0,1,2: fp32-FMA tiles BN=128/64/32; 3: wgmma tensor-core version}; an fp32-FMA
 * saturation probe returning the measured TFLOP/s of the current device.       */
int agpt_profile_enable(int on);
int agpt_profile_collect(double ms[4], double flops[4], double bytes[4], long long launches[4]);
/* recorded wgmma launches that ran 256-row tiles (narrow HiFi-GAN / BigVGAN convs) since profiling was enabled */
long long agpt_profile_tall_launches(void);
/* recorded wgmma launches whose input was a pre-split fp16 operand plane (HiFi-GAN) since profiling was enabled */
long long agpt_profile_plane_launches(void);
/* dev tooling: one text line per recorded launch ("variant G L Cin Cout ntaps span epi Wreal ms flops"); returns bytes written or -1 */
long agpt_profile_dump(char* out, long cap);
double agpt_fma_peak_tflops(void);
/* 1 (default): contractions run on the tensor cores (wgmma) with error-compensated fp16 parts
 * ("3xfp16": x = hi + lo, products hi*hi + lo*hi + hi*lo, fp32 accumulation; weights pre-scaled
 * by a power of two per layer); 0: the fp32-FMA kernels only.  Environment: AGPT_TENSOR_CORES.        */
int agpt_set_tensor_cores(int on);
/* Multi-head attention softmax_j(q_i . k_j * d^-0.5) v_j, heads outermost in the channel dim ('b n (h d)'),
 * CrossAttention.forward (ldm/modules/attention.py:170-193): q [N][Lq][q_pitch], k / v [N][Lk][pitch] device rows with
 * head h at channels [h*d, (h+1)*d); o [N][Lq][o_pitch].  Default: QK^T and PV on the tensor cores (wgmma,
 * error-compensated fp16 parts, fp32 accumulation, exact online softmax; d in {8,16,32,40,64,80});
 * agpt_set_attention_tc(0) / AGPT_ATTN_TC=0 selects the fp32-FMA kernel, -1 = environment / default.            */
int agpt_attention(const float* q, int q_pitch, const float* k, int k_pitch, const float* v, int v_pitch, float* o,
                   int o_pitch, int N, int heads, int d, int Lq, int Lk, void* stream);
int agpt_set_attention_tc(int on);
/* Same with a key-padding mask (fairseq MultiheadAttention's key_padding_mask, modules/commons/common_layers.py:235-364):
 * key_padding_mask [N][Lk] bytes, 1 = padding key (need not be a suffix).  d in {8,16,32,40,64,80,128}.  A query whose
 * keys are all padding gets zeros (the reference gets NaN there).                                                 */
int agpt_attention_masked(const float* q, int q_pitch, const float* k, int k_pitch, const float* v, int v_pitch,
                          const uint8_t* key_padding_mask, float* o, int o_pitch, int N, int heads, int d, int Lq, int Lk,
                          void* stream);
/* Micro-benchmark of one tapconv layer (random data): out2 = {ms per launch, algorithmic TFLOP/s}; dbg8
 * (tensor-core kernel only) = average per-CTA phase cycles {setup, first activation tile, MMA issue loop, drain,
 * epilogue, total, wait-on-activations, wait-on-weights}.  Wreal > 0 selects a 3x3 conv on an (L/Wreal) x Wreal
 * image.                                                                                                       */
int agpt_bench_tapconv(int G, int L, int Cin, int Cout, int K, int dil, int Wreal, int epi_res, int use_tc,
                       int reps, double* out2, double* dbg8_or_null);

/* Conformance entry of the tap-GEMM primitive (tests/test_tapconv_gpu.py): ONE launch of the production path --
 * the production weight packer, tapconv_launch (or the fused pair launch) -- on caller-owned device tensors.
 * Weights and bias are fp32 HOST arrays in the torch layouts; everything else passes through to the launch
 * parameters as given (pitches and sample strides in elements).                                               */
typedef struct agpt_tapconv_probe_args {
  int kind;        /* 0 Conv1d w [Cout][Cin][K] (dilation dil), "same" padding
                      1 Conv2d w [Cout][Cin][3][3] on (L / Wreal) x Wreal images, padding 1; strip_w > 0: strip mode
                      2 ConvTranspose1d w [Cin][Cout][K], stride u, padding pad: the output [L][u*Cout] is [L*u][Cout]
                      3 Conv1d (dilation 1) over g time steps at once: the [L][C] tensors are viewed as [L/g][g*C]
                        (pitches must equal C), Cin == Cout == C
                      4 Conv1d with (first half, second half) output channels interleaved, for EPI_GATE / EPI_GEGLU:
                        the epilogue's res operand is in the interleaved order                                    */
  int Cin, Cout, K, dil, Wreal, strip_w, u, pad, g;
  const float* w;  /* host */
  const float* b;  /* host, NULL = no bias */
  int G, L;
  const float* in; long in_gstride; int in_pitch;
  float* out; long out_gstride; int out_pitch;          /* out may be NULL when a plane output is set */
  const float* res; long res_gstride; int res_pitch;
  float* out2; long out2_gstride; int out2_pitch;
  int pro; float slope; const float* pvec; int pvec_gstride;
  int epi; float scale; int accumulate; int csplit; const float* evec; int evec_gstride;
  int tc_tall;
  int plane_in;    /* split `in` into fp16 hi / lo operand planes (probe-owned) and feed the launch from them;
                      PRO_LRELU only (the split applies the slope), tensor cores only                           */
  void* po_hi; void* po_lo; float po_slope;            /* output operand plane (fp16), NULL = none */
  void* pl_hi; void* pl_lo; int pl_pitch;              /* EPI_GATE / EPI_GEGLU output plane (fp16), NULL = none */
  int fma;         /* 1: force the fp32-FMA kernel (the tensor-core setting is restored afterwards) */
  int pair;        /* 1: fused ResBlock pair out = epi(c2(lrelu(c1(lrelu(in))))) in one launch: c1 = (w, b, K, dil),
                      Cin == Cout; c2 = (w2, b2, K2, dil2) Conv1d [Cout][Cout][K2]; the epilogue fields are c2's.
                      An error when the pair launch is not taken.                                                */
  const float* w2; const float* b2; int K2, dil2;
} agpt_tapconv_probe_args;
/* ran = what actually launched: {1 tensor-core | 0 fp32-FMA, tile width BN, tile height MT, 1 plane-fed}.
 * Synchronises `stream` before returning.                                                                   */
int agpt_tapconv_probe(const agpt_tapconv_probe_args* args, int ran[4], void* stream);

/* ------------------------------------------------------------------ HiFi-GAN
 * Replaces HifiGanGenerator.__init__/forward/remove_weight_norm
 * (NeuralSeq/modules/hifigan/hifigan.py:104-178) and the twin
 * text_to_audio/Make_An_Audio/vocoder/hifigan/modules.py:86-136.            */
#define AGPT_MAX_UPS 8
#define AGPT_MAX_RBK 8
#define AGPT_MAX_DIL 8
typedef struct {
  int n_mels;                  /* 80 */
  int c_out;                   /* 1 */
  int upsample_initial_channel;
  int num_upsamples;
  int upsample_rates[AGPT_MAX_UPS];
  int upsample_kernel_sizes[AGPT_MAX_UPS];
  int resblock_type;           /* 1 = ResBlock1 (hifigan.py:30-67), 2 = ResBlock2 (:70-91) */
  int num_kernels;
  int resblock_kernel_sizes[AGPT_MAX_RBK];
  int resblock_num_dilations[AGPT_MAX_RBK];
  int resblock_dilations[AGPT_MAX_RBK][AGPT_MAX_DIL];
  int use_nsf;                 /* h['use_pitch_embed']: noise_convs present (hifigan.py:111-132) */
  /* BigVGAN (text_to_audio/Make_An_Audio/vocoder/bigvgan/models.py:133-203) is the same generator with
   * anti-aliased periodic activations (Activation1d(Snake|SnakeBeta)) instead of leaky-relu:
   * activation 0 = leaky-relu (HiFi-GAN), 1 = 'snake', 2 = 'snakebeta'; snake_logscale = h.snake_logscale.
   * With activation != 0 the weight list is: conv_pre w,b; ups w,b ...; per resblock: convs1 w,b x nd,
   * convs2 w,b x nd, then alpha[, beta] for activations.0 .. (2 nd - 1); activation_post alpha[, beta];
   * conv_post w,b; the 12 filter taps (Activation1d's registered buffer).                          */
  int activation;
  int snake_logscale;
} agpt_hifigan_cfg;

/* host_weights: fp32 HOST arrays in the key order of
 * audiogpt_b200.specs.hifigan_param_shapes(h) (weight-norm already folded;
 * m_source.l_linear.* entries are skipped by the library).                   */
int agpt_hifigan_create(const agpt_hifigan_cfg* cfg, const float* const* host_weights,
                        int n_weights, int device, agpt_handle* out);
/* mel [B,n_mels,T] (device) -> wav [B,c_out,T*prod(rates)] (device).
 * har_source: NULL or the merged NSF excitation [B,1,T*prod(rates)] (device),
 * i.e. SourceModuleHnNSF's first output (hifigan.py:145-149).                */
int agpt_hifigan_forward(agpt_handle h, const float* mel, const float* har_source,
                         int B, int T, float* wav, void* stream);
/* Same through HOST buffers: H2D copy, forward, D2H copy, synchronise.
 * This is what HifiGAN.spec2wav (NeuralSeq/vocoders/hifigan.py:55-69) calls. */
int agpt_hifigan_vocode_host(agpt_handle h, const float* mel_host, const float* har_host,
                             int B, int T, float* wav_host);

/* NSF harmonic source: replaces SineGen.forward + SourceModuleHnNSF.forward
 * (NeuralSeq/modules/parallel_wavegan/models/source.py:311-441,484-532; call site hifigan.py:145-149).
 * f0 [B][L] device, ALREADY upsampled to the sample rate (hifigan.py:147 f0_upsamp); dim = harmonic_num + 1 (<= 16);
 * lin_w_host [dim], lin_b: m_source.l_linear; rand_ini [B][dim] (torch.rand, entry 0 ignored) and noise [B][L][dim]
 * (torch.randn_like(sines)) are drawn by the caller in the reference's order, NULL = zeros.
 * har_source [B][L] = tanh(l_linear(sines * uv + noise_amp * noise)): the array agpt_hifigan_forward takes.
 * The phase prefix sum over the whole utterance is a three-level scan in fp64.                            */
int agpt_nsf_source(const float* f0, int B, int L, int dim, float sampling_rate, const float* lin_w_host, float lin_b,
                    const float* rand_ini_or_null, const float* noise_or_null, float sine_amp, float noise_std,
                    float voiced_threshold, float* har_source, void* stream);

/* ------------------------------------------------------------------ DiffNet + GaussianDiffusion
 * Replaces DiffNet.forward (NeuralSeq/modules/diff/net.py:107-130) and the
 * elementwise part of GaussianDiffusion.p_sample / p_sample_plms
 * (NeuralSeq/modules/diff/shallow_diffusion_tts.py:134-204).                 */
typedef struct {
  int in_dims;                 /* 80 mel bins */
  int hidden_size;             /* encoder_hidden: channels of cond */
  int residual_layers;
  int residual_channels;
  int dilation_cycle_length;
} agpt_diffnet_cfg;

int agpt_diffnet_create(const agpt_diffnet_cfg* cfg, const float* const* host_weights,
                        int n_weights, int device, agpt_handle* out);
/* Hoist the step-invariant conditioner projections of all layers
 * (net.py:68: conditioner_projection(cond)) for cond [B,hidden,T] (device).  */
int agpt_diffnet_set_cond(agpt_handle h, const float* cond, int B, int T, void* stream);
/* eps [B,1,M,T] = DiffNet(x [B,1,M,T], t [B] (host ints), cond set above)    */
int agpt_diffnet_eps(agpt_handle h, const float* x, const int* t_host, float* eps, void* stream);
/* x_out = p_sample(x, t, noise): eps is taken from `eps` when non-NULL (any
 * denoise_fn), else computed by the DiffNet handle `h` (cond set above).
 * coef_host[b] = {sqrt_recip_ac[t], sqrt_recipm1_ac[t], post_mean_coef1[t],
 * post_mean_coef2[t], exp(0.5*post_log_var[t]) * (t!=0)} gathered on the host
 * from the fp32 tables (shallow_diffusion_tts.py:108-123,159-166).  clip: clamp
 * x0 to [-1,1] (:153-154).  n_per_sample = M*T.  x_out may alias x.           */
int agpt_gd_p_sample(agpt_handle h_or_null, const float* x, const float* eps_or_null, const int* t_host,
                     const float* coef_host /*[B][5]*/, const float* noise_or_null, int clip_denoised,
                     int B, long n_per_sample, float* x_out, void* stream);
/* The whole ancestral loop of GaussianDiffusion.forward(infer=True) (shallow_diffusion_tts.py:263-272) on the
 * device: for t = t_hi-1 .. t_lo: x_io <- p_sample(x_io, t, noises[t - t_lo]) with every sample at the same t, the
 * DiffNet handle `h` (cond set by agpt_diffnet_set_cond) predicting eps.  coef_host [t_hi-t_lo][5]: the rows of
 * agpt_gd_p_sample in SAMPLING order (row k belongs to t = t_hi-1-k).  noises_or_null: device
 * [t_hi-t_lo][noise_step_stride] floats, pre-drawn by the caller in the reference's RNG call order.  The
 * step-embedding MLP and the per-layer diffusion projections run once for all steps; step 0 runs as plain
 * launches, then ONE captured step (CUDA graph + device-side step counter) is replayed.  AGPT_GRAPH=0 disables. */
int agpt_gd_sample_loop(agpt_handle h, float* x_io, int t_hi, int t_lo, const float* coef_host,
                        const float* noises_or_null, long noise_step_stride, int clip_denoised, void* stream);
long agpt_diffnet_launches_per_step(agpt_handle h);
/* generic elementwise: out = a0*x + a1*e0 + a2*e1 + a3*e2 + a4*e3 (per-sample
 * coefficient rows coef_host[B][5]; NULL e_i are skipped) -- the PLMS
 * combinations of shallow_diffusion_tts.py:174-204.                          */
int agpt_axpby5(const float* x, const float* e0, const float* e1, const float* e2, const float* e3,
                const float* coef_host, int B, long n_per_sample, float* out, void* stream);

/* ------------------------------------------------------------------ UNet + DDIM
 * Replaces UNetModel.forward (ldm/modules/diffusionmodules/openaimodel.py:711-744)
 * and DDIMSampler.p_sample_ddim's arithmetic (ldm/models/diffusion/ddim.py:168-225). */
#define AGPT_MAX_LEVELS 8
typedef struct {
  int in_channels, out_channels, model_channels;
  int num_res_blocks;
  int num_levels;
  int channel_mult[AGPT_MAX_LEVELS];
  int attn_at_level[AGPT_MAX_LEVELS];   /* 1 if ds=2^level is in attention_resolutions */
  int num_heads;                        /* -1 => use num_head_channels */
  int num_head_channels;
  int transformer_depth;
  int context_dim;
  int use_spatial_transformer;          /* 1: SpatialTransformer blocks (cross-attention on a context);
                                           0: AttentionBlock (self-attention only, no context) */
  int resblock_updown;                  /* 1: down/up-sampling ResBlocks (avg-pool / nearest) instead of
                                           the strided / upsampling convs */
  int attention_order;                  /* AttentionBlock qkv channel order: 0 legacy per-head [q_h;k_h;v_h]
                                           (QKVAttentionLegacy), 1 [Q|K|V] (use_new_attention_order) */
} agpt_unet_cfg;

int agpt_unet_create(const agpt_unet_cfg* cfg, const float* const* host_weights,
                     int n_weights, int device, agpt_handle* out);
/* Hoist the step-invariant to_k/to_v(context) of every cross-attention
 * (attention.py:174-176) for context [N,S,context_dim] (device).             */
int agpt_unet_set_context(agpt_handle h, const float* context, int N, int S, void* stream);
/* Concat conditioning of agpt_unet_ddim_sample for a UNet with in_channels > out_channels
 * (DiffusionWrapper 'concat', ddpm.py:1404-1406): c [N, in_channels - out_channels, H, W] (device) is
 * appended to the latent's channels at every step.  It is read once here and put into the kernel
 * layout once; the loop state stays the out_channels latent.                                       */
int agpt_unet_set_concat(agpt_handle h, const float* c, int N, int C, int H, int W, void* stream);
/* eps [N,Cout,H,W] = UNet(x [N,Cin,H,W], t [N] host ints, context set above) */
int agpt_unet_forward(agpt_handle h, const float* x, const int* t_host, int N, int H, int W,
                      float* eps, void* stream);
/* One DDIM step with classifier-free guidance on a doubled batch
 * (ddim.py:177-225): eps2 = [e_uncond ; e_cond] (2B samples), e = e_u + s*(e_c-e_u);
 * pred_x0 = (x - sqrt_om*e)/sqrt(a_t); x_prev = sqrt(a_prev)*pred_x0 +
 * sqrt(1-a_prev-sigma^2)*e + sigma*noise*temperature.  If eps2_is_single != 0
 * eps2 holds B samples and no guidance is applied.                           */
int agpt_ddim_update(const float* x, const float* eps2, int eps2_is_single, float cfg_scale,
                     float a_t, float a_prev, float sigma_t, float sqrt_one_minus_at,
                     const float* noise, float temperature, int B, long n_per_sample,
                     float* x_prev, float* pred_x0_or_null, void* stream);
/* Whole DDIM loop on device (ddim.py:117-166, eta = 0) with CFG; context = [uncond ; cond]
 * set through agpt_unet_set_context (2B rows) or B rows when cfg_scale == 1.  A UNet with
 * in_channels > out_channels samples x_T [B, out_channels, H, W] with the conditioning of
 * agpt_unet_set_concat (B rows, same H and W, cfg_scale 1).
 * tables: host arrays of length S in *sampling order* (index S-1 first).  The time-embedding
 * MLP and the ResBlock embedding projections run once for all S timesteps; step 0 runs as plain
 * launches, then ONE captured step (CUDA graph, device-side step counter and coefficient tables)
 * is replayed S-1 times; the step's x_prev update reads its scalars from the table (no host sync,
 * no per-step H2D).  pred_x0_or_null receives the last step's pred_x0 (ddim.py:216).
 * AGPT_GRAPH=0 in the environment replaces the replays by plain launches.                     */
int agpt_unet_ddim_sample(agpt_handle h, const float* x_T, int B, int H, int W, int S,
                          const int* t_steps_host, const float* a_t, const float* a_prev,
                          const float* sigma, const float* sqrt_om, float cfg_scale,
                          float* x_out, float* pred_x0_or_null, void* stream);
/* kernels launched per DDIM step by the last agpt_unet_ddim_sample call (bench.py reports it) */
long agpt_unet_launches_per_step(agpt_handle h);

/* ------------------------------------------------------------------ AutoencoderKL.decode (first stage)
 * Replaces AutoencoderKL.decode = post_quant_conv -> Decoder.forward
 * (text_to_audio/Make_An_Audio/ldm/models/autoencoder.py:351-354,
 *  ldm/modules/diffusionmodules/model.py:462-568; ResnetBlock :121-143, AttnBlock :150-203, Upsample :43-49):
 * the step between DDIMSampler.sample and the vocoder on every text-to-audio call
 * (ddpm.py decode_first_stage; audio-chatgpt.py:174).                                                  */
typedef struct {
  int embed_dim, z_channels;            /* 4, 4 */
  int ch, out_ch;                       /* 128, 1 */
  int num_levels;                       /* len(ch_mult) */
  int ch_mult[AGPT_MAX_LEVELS];
  int num_res_blocks;                   /* the decoder uses num_res_blocks + 1 blocks per level */
  int attn_at_level[AGPT_MAX_LEVELS];   /* 1 if resolution / 2^level is in attn_resolutions (model.py:481,517) */
} agpt_vae_cfg;
/* host_weights: fp32 HOST arrays in the key order of audiogpt_b200.specs.vae_decoder_param_shapes(cfg). */
int agpt_vae_create(const agpt_vae_cfg* cfg, const float* const* host_weights, int n_weights, int device,
                    agpt_handle* out);
/* z [B, embed_dim, H, W] (device) -> out [B, out_ch, H * 2^(levels-1), W * 2^(levels-1)] (device) */
int agpt_vae_decode(agpt_handle h, const float* z, int B, int H, int W, float* out, void* stream);

/* ------------------------------------------------------------------ AutoencoderKL.encode (first stage, encoder side)
 * Replaces the arithmetic of AutoencoderKL.encode = quant_conv(Encoder.forward(x)) (autoencoder.py:345-349,
 * model.py:368-459; Downsample :60-79): the masked-mel encoding of the Inpaint tool (audio-chatgpt.py:507) and the
 * first half of AutoencoderKL.forward.  The posterior (DiagonalGaussianDistribution) is built by the caller.
 * cfg: the same agpt_vae_cfg as the decoder (num_res_blocks blocks per level, attn_at_level as there);
 * in_channels: ddconfig in_channels (1 for mel images).
 * host_weights: fp32 HOST arrays in the key order of audiogpt_b200.specs.vae_encoder_param_shapes(cfg) (encoder.*,
 * then quant_conv.*).                                                                                             */
int agpt_vae_encoder_create(const agpt_vae_cfg* cfg, int in_channels, const float* const* host_weights, int n_weights,
                            int device, agpt_handle* out);
/* x [B, in_channels, H, W] (device) -> moments [B, 2 * embed_dim, H >> (levels-1), W >> (levels-1)] (device):
 * mean then logvar (before the clamp).  H and W below 2^(levels-1) are rejected.                                  */
int agpt_vae_encode(agpt_handle h, const float* x, int B, int H, int W, float* moments, void* stream);

/* ------------------------------------------------------------------ PitchExtractor
 * Replaces PitchExtractor.forward (NeuralSeq/modules/fastspeech/pe.py:119-148: Prenet :7-42, ConvStacks :82-116,
 * PitchPredictor modules/fastspeech/tts_modules.py:217-260, denorm_f0 utils/pitch_utils.py:63-76): F0 from a generated
 * mel for the NSF vocoder (inference/svs/base_svs_infer.py run_vocoder).                                          */
typedef struct {
  int n_mel_bins;          /* 80 */
  int hidden_size;         /* hparams['hidden_size'] */
  int conv_layers;         /* ConvStacks layers (2) */
  int predictor_hidden;    /* hparams['predictor_hidden'] or hidden_size */
  int predictor_layers;    /* 5 */
  int predictor_kernel;    /* hparams['predictor_kernel'] */
} agpt_pe_cfg;
/* host_weights: fp32 HOST arrays in the key order of audiogpt_b200.specs.pe_param_shapes(cfg) (state-dict order incl. the
 * BatchNorm buffers; num_batches_tracked and embed_positions._float_tensor are passed and ignored).               */
int agpt_pe_create(const agpt_pe_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out);
/* mel [B][T][n_mel_bins] (device, channels-last as the reference passes it) -> pitch_pred [B][T][2], f0_denorm [B][T].
 * pitch_norm: 0 none, 1 'standard' (f0 * std + mean), 2 'log' (2 ** f0); use_uv: zero F0 where pitch_pred[..., 1] > 0;
 * all-zero mel frames (padding) give F0 = 0.                                                                      */
int agpt_pe_forward(agpt_handle h, const float* mel, int B, int T, float* pitch_pred, float* f0_denorm, int use_uv,
                    int pitch_norm, float f0_mean, float f0_std, void* stream);

/* ------------------------------------------------------------------ FastSpeech2 / FastSpeech2MIDI
 * Replaces FastSpeech2.forward (NeuralSeq/modules/fastspeech/fs2.py:79-226) and FastSpeech2MIDI.forward
 * (modules/diffsinger_midi/fs2.py:55-118) for encoder_type = decoder_type = 'fft', ffn_act 'gelu', ffn_padding 'SAME',
 * dur_loss 'mse', no speaker conditioning: the acoustic front-end of the TTS and text-to-singing paths.           */
typedef struct {
  int hidden_size, num_heads;
  int enc_layers, dec_layers;
  int enc_ffn_kernel, dec_ffn_kernel;
  int n_tokens;                /* len(dictionary) */
  int out_dims;                /* audio_num_mel_bins */
  int predictor_hidden;        /* resolved: hparams['predictor_hidden'] or hidden_size */
  int dur_predictor_layers, dur_predictor_kernel;
  int predictor_layers, predictor_kernel;
  int use_pos_embed;           /* encoder positions (the decoder always has them) */
  int rel_pos;                 /* 0: fairseq sinusoidal table; 1: espnet RelPositionalEncoding (x * sqrt(H) + pe) */
  int pitch_type;              /* 0: use_pitch_embed off; 1: 'frame'; 2: 'ph' */
  int use_energy_embed;
  int use_midi;                /* FastSpeech2MIDI: midi_embed / midi_dur_layer / is_slur_embed in the encoder input */
} agpt_fs2_cfg;
/* host_weights: fp32 HOST arrays in the key order of audiogpt_b200.specs.fs2_param_shapes(cfg) (both names of the shared
 * token embedding and the _float_tensor marker buffers are passed; the duplicates and markers are ignored).       */
int agpt_fs2_create(const agpt_fs2_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out);
/* Token side: txt_tokens [B][T_txt] int32 (0 = padding); pitch_midi / is_slur int32 and midi_dur fp32 [B][T_txt] (MIDI
 * model; midi_dur / is_slur may be NULL).  dur [B][T_txt] = the duration predictor's log-domain output.  predict_dur != 0:
 * dur_choice [B][T_txt] int32 (may be NULL) = clamp(round(exp(dur) - 1), 0), and mel_len_host [B] (HOST) = frames per
 * utterance -- the call synchronises the stream for this one device -> host copy.  The encoder output stays in the
 * handle for agpt_fs2_decode.                                                                                       */
int agpt_fs2_encode(agpt_handle h, const int* txt_tokens, int B, int T_txt, const int* pitch_midi, const float* midi_dur,
                    const int* is_slur, int predict_dur, float* dur, int* dur_choice, int* mel_len_host, void* stream);
/* Frame side, T_mel frames: mel2ph [B][T_mel] int32 (teacher-forced) or NULL = expand the durations predicted by the last
 * encode into mel2ph_out.  f0 / uv / energy: teacher-forced values or NULL (f0 is [B][T_txt] for pitch_type 'ph').
 * pitch_norm 1 'standard', 2 'log'.  Outputs (device): pitch_pred ([B][T_mel][2] 'frame', [B][T_txt][1] 'ph'), f0_denorm
 * and pitch_coarse (int32) on the same grid; energy_pred [B][T_mel]; decoder_inp [B][T_mel][H]; mel_out
 * [B][T_mel][out_dims] or NULL to skip the decoder.                                                                */
int agpt_fs2_decode(agpt_handle h, int T_mel, const int* mel2ph, int* mel2ph_out, const float* f0, const float* uv,
                    const float* energy, int use_uv, int pitch_norm, float f0_mean, float f0_std, float* pitch_pred,
                    float* f0_denorm, int* pitch_coarse, float* energy_pred, float* decoder_inp, float* mel_out, void* stream);

/* ------------------------------------------------------------------ CLAP text encoder
 * Replaces FrozenCLAPEmbedder.encode after tokenization (text_to_audio/Make_An_Audio/ldm/modules/encoders/modules.py:
 * 205-212): BERT (HF BertModel called with input_ids only, so every position attends to every position, padding
 * included; token type 0) then CLAP's Projection (ldm/modules/encoders/CLAP/clap.py:8-20, dropout off):
 * z = LayerNorm(e1 + linear2(gelu(e1))), e1 = linear1(last_hidden_state).  The conditioning of every Make-An-Audio
 * text-to-audio call (get_learned_conditioning).  Unlike the other configs this one carries floats, so it is a
 * tagged struct.                                                                                                 */
typedef struct agpt_clap_cfg {
  int vocab_size;              /* BertConfig.vocab_size (30522) */
  int max_position_embeddings; /* 512: the longest sequence */
  int type_vocab_size;         /* 2 (only type 0 is read) */
  int hidden_size;             /* 768 */
  int num_layers;              /* 12 */
  int num_heads;               /* 12 */
  int intermediate_size;       /* 3072 */
  int d_proj;                  /* 1024: the UNet's context_dim */
  float layer_norm_eps;        /* BERT's LayerNorms (1e-12) */
  float proj_layer_norm_eps;   /* Projection.layer_norm (1e-5) */
} agpt_clap_cfg;
/* host_weights: fp32 HOST arrays in the key order of audiogpt_b200.specs.clap_param_shapes(cfg) (the reference's
 * state-dict keys under caption_encoder.base.* and caption_encoder.projection.*); the pooler, which encode never
 * uses, is passed and ignored.                                                                                      */
int agpt_clap_create(const agpt_clap_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out);
/* input_ids [N][L] int32 (device) -> z [N][L][d_proj] (device).  L <= max_position_embeddings; ids outside
 * [0, vocab_size) are clamped to it (callers are expected to reject them first).                                  */
int agpt_clap_encode(agpt_handle h, const int* input_ids, int N, int L, float* z, void* stream);

/* ------------------------------------------------------------------ CLAP candidate scorer
 * Replaces the arithmetic of wav_evaluation.models.CLAPWrapper (text_to_audio/Make_An_Audio/wav_evaluation/models/
 * CLAPWrapper.py:119-215, clap.py, audio.py:107-179): get_text_embeddings / get_audio_embeddings / compute_similarity,
 * with which T2A.select_best_audio (audio-chatgpt.py:185-199) picks the best of its candidate clips.
 *
 * Text tower: an agpt_clap_create handle built from the scorer checkpoint's caption_encoder.* weights.  BERT is
 * called with token_type_ids and attention_mask (padding keys masked out); only the [CLS] row goes through the
 * Projection.  input_ids / token_type_ids / attention_mask [N][L] int32 (device); ids and type ids outside the tables
 * are clamped (callers are expected to reject them first).  out [N][d_proj] (device): the embedding divided by its
 * norm twice, as the reference does.  The plain agpt_clap_encode path is unchanged.                              */
int agpt_clap_encode_cls(agpt_handle h, const int* input_ids, const int* token_type_ids, const int* attention_mask, int N,
                         int L, float* out, void* stream);
/* out [Na][Nt] = scale * a t^T (a [Na][D], t [Nt][D], device; fp32 FMA dots): compute_similarity's (t @ a.T).T, scale
 * = logit_scale.exp() or 1 (use_logit_scale=False).                                                               */
int agpt_clap_similarity(const float* a, int Na, const float* t, int Nt, int D, float scale, float* out, void* stream);

/* Audio tower: Cnn14 (torchlibrosa Spectrogram n_fft = win = window_size, hop_size, periodic Hann, center + reflect,
 * power 2; LogmelFilterBank ref 1, amin 1e-10, no top_db; bn0; six ConvBlocks 1 -> 64 -> ... -> 2048 with 2x2 average
 * pools after blocks 1-5; mean over mel, max + mean over time; relu(fc1)) and the audio Projection, eval mode.
 * A tagged struct, as agpt_clap_cfg.                                                                            */
typedef struct agpt_cnn14_cfg {
  int window_size;   /* 1024 */
  int hop_size;      /* 320 */
  int mel_bins;      /* 64 (Cnn14's bn0 is BatchNorm2d(64)) */
  int out_emb;       /* 2048: fc1's width */
  int d_proj;        /* 1024 */
} agpt_cnn14_cfg;
/* host_weights: fp32 HOST arrays in the key order of audiogpt_b200.specs.cnn14_engine_keys(cfg): the checkpoint's
 * audio_encoder.* keys without fc_audioset.* and num_batches_tracked.  BatchNorms are folded (eps 1e-5).          */
int agpt_cnn14_create(const agpt_cnn14_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out);
/* The resampler and clip length of the following agpt_cnn14_embed calls: torchaudio.transforms.Resample's polyphase
 * filter table_host [new_freq][2 width + orig_freq] (HOST, rates reduced by their gcd; 1 / 1 / 0 with the table {1}
 * is no resampling) and clip_samples = duration * the INPUT rate (resample_and_duration's target length).          */
int agpt_cnn14_set_resample(agpt_handle h, int orig_freq, int new_freq, int width, const float* table_host, int clip_samples);
/* wav [B][n_samples] (device, at the input rate) -> out_emb [B][d_proj] (device): resampled (R = ceil(new * n /
 * orig) samples), fitted to clip_samples -- start_or_tile_host[b] (HOST) is the crop start in [0, R - clip) when R >
 * clip, and -1 (tile: repeat, then cut) otherwise -- then Cnn14, Projection and the two L2 normalisations.        */
int agpt_cnn14_embed(agpt_handle h, const float* wav, long n_samples, int B, const int* start_or_tile_host, float* out_emb,
                     void* stream);

#ifdef __cplusplus
}
#endif
#endif /* AGPT_B200_H */
