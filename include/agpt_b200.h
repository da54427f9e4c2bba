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
/* recorded launches of narrow pairs with overlapped tiles (HiFi-GAN's C <= 64 stages) since profiling was enabled */
long long agpt_profile_dual_launches(void);
/* recorded fused-pair launches that ran two tiles in flight per CTA (HiFi-GAN's C = 128 stage) since profiling was enabled */
long long agpt_profile_pipe_launches(void);
/* recorded narrow fused-pair launches on the persistent tile pipeline (HiFi-GAN's C <= 64 stages) since profiling was enabled */
long long agpt_profile_narrow_pipe_launches(void);
/* recorded plane-fed single tap-GEMM launches on the persistent tile pipeline (HiFi-GAN's C = 256 convs, ups[0] / ups[1]) since profiling was enabled */
long long agpt_profile_conv_pipe_launches(void);
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
                      kind 0, or kind 3 (both convs time-grouped by g, dil = dil2 = 1).
                      An error when the pair launch is not taken.                                                */
  const float* w2; const float* b2; int K2, dil2;
} agpt_tapconv_probe_args;
/* ran = what actually launched: {1 tensor-core | 0 fp32-FMA, tile width BN, tile height MT, 1 plane-fed}.
 * Synchronises `stream` before returning.                                                                   */
int agpt_tapconv_probe(const agpt_tapconv_probe_args* args, int ran[4], void* stream);
/* The HiFi-GAN driver's pipeline switches (TapConvParams::tc_*): set on the launch and, for a pair, on c1; 0 keeps
 * the launch off that pipeline.  Tensor cores only (an error with fma = 1).                                    */
typedef struct agpt_tapconv_pipes {
  int tc_dual, tc_pipe, tc_narrow_pipe, tc_conv_pipe;
} agpt_tapconv_pipes;
/* ran[4] of agpt_tapconv_probe_pipes: the kernel family of the launch.  TILE covers the FMA kernel, tcconv5[_pl]
 * and tcpair, which ran[0..3] tell apart; the others are the persistent / two-CTA pipelines the switches allow.   */
enum { AGPT_TC_KERN_TILE = 0, AGPT_TC_KERN_DUAL, AGPT_TC_KERN_PAIR_PIPE, AGPT_TC_KERN_NARROW_PIPE, AGPT_TC_KERN_CONV_PIPE };
/* agpt_tapconv_probe with the pipeline switches `pipes`; ran = {the four fields of agpt_tapconv_probe, kernel
 * family AGPT_TC_KERN_*}.  Synchronises `stream` before returning.                                           */
int agpt_tapconv_probe_pipes(const agpt_tapconv_probe_args* args, const agpt_tapconv_pipes* pipes, int ran[5],
                             void* stream);
/* Conformance entry of the non-contraction kernels (nn_kernels.cu, tests/test_nn_kernels_gpu.py): ONE call of the
 * production launcher selected by `op` on caller-owned device tensors, with the arguments as given.  All tensors are
 * fp32 device arrays unless marked host; the fields each op reads:
 *   GROUPNORM      groupnorm_ex: x [N][rows][C] -> y, gamma / beta [C], G, eps, act (0 none, 1 SiLU, 2 ReLU),
 *                  x2 = residual added after the activation (NULL = none)
 *   LAYERNORM      layernorm: x [rows][C] -> y, gamma / beta [C], eps
 *   SOFTMAX_ROWS   softmax_rows: y [rows][pitch] in place, softmax over the first cols after scaling by scale
 *   TRANSPOSE_PAD  transpose_pad: x [rows][pitch] (cols used) -> y [cols][rows_pad]
 *   COPY_PAD_ROWS  copy_pad_rows: x [rows][pitch] (cols used) -> y [rows_pad][cols]
 *   CONCAT         concat_channels: x [rows][C], x2 [rows][C2] -> y [rows][C + C2]
 *   UPSAMPLE2      upsample_nearest2: x [N][H][W][C] -> y [N][2H][2W][C]
 *   AVGPOOL2       avgpool2: x [N][H][W][C] -> y [N][H/2][W/2][C]
 *   IM2COL_S2      im2col_stride2: x [N][H][W][C] -> y [N][Ho][Wo][9][C]; pad 1: Ho = (H - 1) / 2 + 1 (Conv2d k3 s2
 *                  p1), pad 0: Ho = H / 2 (the VAE encoder's pad-after Downsample); likewise Wo
 *   CF_TO_CL_PAD   cf_to_cl_pad: x [Nsrc][C][H*W] -> y [N][H*W][pitch], sample n reads source n % Nsrc (0 = N)
 *   TIMESTEP       timestep_embedding: t HOST [N] -> y [N][C]
 *   TIMESTEP_DEV   timestep_embedding_dev: t device [N] -> y [N][C]
 *   DDIM_TAB       select_row(sel_table [..][sel_cols] -> sel_out), ddim_update_tab(x [N][rows], x2 = eps [N or 2N][rows],
 *                  single, table = coefficients [steps][6] at *step) -> y = x_prev (may be x), y2 = pred_x0 (NULL = none),
 *                  then step_inc(step)
 *   CONV_OUT_DDIM  conv_out_ddim: x = normalised activation [N or 2N][H*W][C], w [9][C][4], b [4], y = the latent
 *                  [N][4][H*W] updated in place, y2 = pred_x0 (NULL = none), single, table / step as DDIM_TAB
 * Synchronises `stream` before returning.                                                                      */
enum {
  AGPT_NN_GROUPNORM = 0, AGPT_NN_LAYERNORM, AGPT_NN_SOFTMAX_ROWS, AGPT_NN_TRANSPOSE_PAD, AGPT_NN_COPY_PAD_ROWS,
  AGPT_NN_CONCAT, AGPT_NN_UPSAMPLE2, AGPT_NN_AVGPOOL2, AGPT_NN_IM2COL_S2, AGPT_NN_CF_TO_CL_PAD, AGPT_NN_TIMESTEP,
  AGPT_NN_TIMESTEP_DEV, AGPT_NN_DDIM_TAB, AGPT_NN_CONV_OUT_DDIM
};
typedef struct agpt_nn_probe_args {
  int op;
  const float* x; const float* x2;
  float* y; float* y2;
  const float* gamma; const float* beta;
  const float* w; const float* b;
  const float* table; int* step;
  const float* sel_table; float* sel_out; int sel_cols;
  const int* t;
  int N, H, W, C, C2, G, act, pad, Nsrc, single;
  long rows; int cols, pitch, rows_pad;
  float eps, scale;
} agpt_nn_probe_args;
int agpt_nn_probe(const agpt_nn_probe_args* args, void* stream);
/* Conformance entry of the FastSpeech-family element-wise kernels (fs_layers.cu, fs2.cu, generspeech.cu, pe.cu;
 * tests/test_fs_kernels_gpu.py): ONE call of the production launcher selected by `op` on caller-owned device tensors,
 * with the arguments as given.  Tensors are fp32 (x*, E*, w, b, y*), int32 (tok, midi, slur, idx*, mel2ph, iy*) or
 * uint8 (kpm) device arrays; null where an op allows it.  norm: 0 none, 1 'standard', 2 'log'.  The fields each op reads:
 *   EMBED_TOKENS  fs_embed_tokens: tok [B][T] -> y = x [B][T][H], y2 = nonpad, kpm; E [ntok][H] * escale (+ midi [B][T] rows
 *                 of E2 [300][H], + x = midi_dur * w + b, + slur rows of E3 [2][H]: each of the three null = off); pos_mode
 *                 0 none, 1 fairseq (neg_emb), 2 rel_pos (x2 = div_term [H/2], xscale)
 *   ROWMASK       fs_rowmask: x [rows][C] -> y = nonpad [rows], kpm
 *   DUR           fs_dur: x = pred4 [rows][4], x2 = nonpad -> y = dur, iy = dur_choice (null = none)
 *   LR_SCAN       fs_lr_scan: idx = dur_choice [B][T] -> iy = cum [B][T], iy2 = mel_len [B]
 *   LR_FILL       fs_lr_fill: idx = cum [B][T], idx2 = mel_len [B] -> iy = mel2ph [B][T2]
 *   GATHER        fs_gather: x = enc [B][T][H], mel2ph [B][T2] -> y [B][T2][H], y2 = tgt [B][T2]
 *   AFFINE_MASK   fs_affine_mask: y [rows][C] in place, w = a [C], b [C] (both null: mask only), x = mask [rows]
 *   POSITIONS     fs_positions: x [B][T][C] -> iy = pos [B][T]
 *   POSEMB_ADD    fs_posemb_add: x [rows][C], idx = pos [rows], alpha -> y (may be x)
 *   PITCH_FRAME   fs2_pitch_frame: x = pred4 [rows][4], mel2ph, x2 = f0 / x3 = uv (null = predicted), use_uv, norm, mean,
 *                 std_ -> y = pitch_pred [rows][2], y2 = f0_denorm, iy = coarse
 *   PITCH_PH      fs2_pitch_ph: x = pred4, x2 = f0 (null = predicted), norm, mean, std_ -> y = pitch_pred [rows], y2, iy
 *   ENERGY        fs2_energy: x = pred4, x2 = energy (null = predicted) -> y = energy_pred, iy = bucket
 *   EMBED_ADD     fs2_embed_add: x [B*T2][H], x2 = tgt, E = pitch table (null = none) with idx = bins [B*T2] or idx2 = bins
 *                 [B][T] through mel2ph [B][T2], E2 = energy table (null = none) with idx3 = buckets -> y; rows = B*T2
 *   GS_SUM        gs_sum: x [rows][H], x2 = spk / x3 = emo [rows / T][H], E (null = none) with idx, x4 (null = none),
 *                 x5 = mask [rows] -> y
 *   GS_ACCUM      gs_accum: y (+)= x over rows floats (first: y = x)
 *   GS_REFMASK    gs_refmask: x = ref mel [rows][80] -> y [rows]
 *   GS_WN_GATE    gs_wn_gate: x [rows][2C] -> y [rows][C]
 *   GS_SEGMEAN    gs_segmean: x [B][T][C], idx = seg [B][T] -> y [B][nseg][C]
 *   GS_VQ         gs_vq: x [rows][H], x2 = dots [rows][M], E = codebook [M][H], x3 = |e|^2 [M] -> iy (null = none),
 *                 y = quantised (may be x)
 *   GS_CATPOS     gs_catpos: x [rows][H], idx = pos [rows] -> y [rows][2H]
 *   GS_KPM        gs_kpm: x [rows][H] -> kpm
 *   GS_PITCH      gs_pitch: x / x2 = the two predictors' [rows][4], mel2ph, mean, std_ -> y = pitch_pred [rows][2],
 *                 y2 = f0_denorm, y3 = f0_denorm_pred, iy = coarse
 *   GS_COND_CAT   gs_cond_cat: x = mel [rows][M], x2 = dec [rows][H], x3 / x4 = spk / emo [rows / T][H], x5 = prosody
 *                 [rows][H] -> y [rows][M + 4H]
 *   GS_SQUEEZE    gs_squeeze: x = z [B][M][T] -> y [B][T2][2M] (T >= 2 T2)
 *   GS_FLOW_STEP  gs_flow_step: y [rows][C] in place, x = the end layer's output [rows][C], w = winv[16] bias[C] logs[C]
 *   PE_MASK       pe_mask: x = mel [rows][M] -> y [rows]
 *   PE_DENORM     pe_denorm: x = pred4 [rows][4], x2 = mask, use_uv, norm, mean, std_ -> y = pitch_pred [rows][2], y2 = f0
 * Synchronises `stream` before returning.                                                                          */
enum {
  AGPT_FS_EMBED_TOKENS = 0, AGPT_FS_ROWMASK, AGPT_FS_DUR, AGPT_FS_LR_SCAN, AGPT_FS_LR_FILL, AGPT_FS_GATHER, AGPT_FS_AFFINE_MASK,
  AGPT_FS_POSITIONS, AGPT_FS_POSEMB_ADD, AGPT_FS_PITCH_FRAME, AGPT_FS_PITCH_PH, AGPT_FS_ENERGY, AGPT_FS_EMBED_ADD, AGPT_FS_GS_SUM,
  AGPT_FS_GS_ACCUM, AGPT_FS_GS_REFMASK, AGPT_FS_GS_WN_GATE, AGPT_FS_GS_SEGMEAN, AGPT_FS_GS_VQ, AGPT_FS_GS_CATPOS, AGPT_FS_GS_KPM,
  AGPT_FS_GS_PITCH, AGPT_FS_GS_COND_CAT, AGPT_FS_GS_SQUEEZE, AGPT_FS_GS_FLOW_STEP, AGPT_FS_PE_MASK, AGPT_FS_PE_DENORM
};
typedef struct agpt_fs_probe_args {
  int op;
  const int* tok; const int* midi; const int* slur; const int* idx; const int* idx2; const int* idx3; const int* mel2ph;
  const float* x; const float* x2; const float* x3; const float* x4; const float* x5;
  const float* E; const float* E2; const float* E3; const float* w; const float* b;
  float* y; float* y2; float* y3;
  int* iy; int* iy2;
  uint8_t* kpm;
  int B, T, T2, H, C, M, nseg, ntok, pos_mode, use_uv, norm, first;
  long rows;
  float escale, neg_emb, xscale, alpha, mean, std_;
} agpt_fs_probe_args;
int agpt_fs_probe(const agpt_fs_probe_args* args, void* stream);
/* Conformance entry of the kernels that touch audio samples and spectrogram bins (logmel front end, emotion power mel,
 * STFT / inverse STFT, LASS's mask input and output stores, Cnn14's resampler and pooling head, the CLAP scorer's L2
 * norms and similarity, wav2vec2's conv stem; tests/test_audio_kernels_gpu.py): ONE call of the production launcher
 * selected by `op` on caller-owned device tensors, with the arguments as given.  Tensors are fp32 device arrays except
 * `starts` (int32, HOST), `cnt` (int32) and the stem workspaces `part` (double2) / `stat` (float2).  The launcher's
 * preconditions are checked first; a violation returns an error with nothing launched.  The fields each op reads:
 *   FRAMES        x [B][N] -> y [B][N / hop + 1][n]; N > n / 2
 *   LOGMEL        x = spec [rows][pitch] ([re | im], nb bins each), w = melW [nb][nm], g = bn0 scale [nm], b = bn0
 *                 shift [nm], ch (1 or 4) -> y [rows][nm][ch]
 *   POWMEL        x = spec [rows][pitch] (201 bins each), w = melW [201][40] -> y [rows][40]
 *   STFT_ROWS     x = wav [B][N], n, hop -> y [B][ceil((N + n) / hop)][hop]; N > n / 2
 *   MAGPHASE      x = spec [B][R][pitch], nb, T -> y = mag, y2 = phase [B][nb][T]
 *   ISTFT_FRAMES  x = mag, x2 = phase [B][nb][T], pitch -> y [B][T + 1][pitch]; T >= 2
 *   ISTFT_FINISH  x = overlap-added y [B][(T + 1) hop], x2 = window sum [(T + 1) hop], n = 2 hop -> y [B][(T - 1) hop];
 *                 T >= 2
 *   RESAMPLE      x [B][N], w = kernel [nw][2 width + orig], orig, nw, width, starts [B] (host), clip -> y [B][clip]
 *   CNN14_HEAD    x [B][T][F][C] -> y [B][C]
 *   L2NORM2       x [rows][D] -> y [rows][D]
 *   SIMILARITY    x = a [Na][D], x2 = t [Nt][D], scale -> y [Na][Nt]
 *   LASS_INPUT    x = mag at element strides sb / stt / sf, B, T, W, scale, shift -> y [B][64 ceil(T / 64)][W][4]
 *   LASS_HEAD     x [B][64 ceil(T / 64)][W][32], w = after_conv2 [33] (32 weights, bias) -> y = mask, y2 = logits (null =
 *                 none) [B][T][W + 2]
 *   W2V_STEM      x [B][N], w = conv0 [C][k0], s0, g = gamma [C], b = beta [C], eps, s1 (the next conv's stride; 0 = no
 *                 zero rows), part, stat, cnt (zero) -> y [B][R][C]; T0 = (N - k0) / s0 + 1 rows plus
 *                 round_up(T0, s1) - T0 zero rows; k0 <= 16, C <= 1024
 * Synchronises `stream` before returning.                                                                          */
enum {
  AGPT_AU_FRAMES = 0, AGPT_AU_LOGMEL, AGPT_AU_POWMEL, AGPT_AU_STFT_ROWS, AGPT_AU_MAGPHASE, AGPT_AU_ISTFT_FRAMES,
  AGPT_AU_ISTFT_FINISH, AGPT_AU_RESAMPLE, AGPT_AU_CNN14_HEAD, AGPT_AU_L2NORM2, AGPT_AU_SIMILARITY, AGPT_AU_LASS_INPUT,
  AGPT_AU_LASS_HEAD, AGPT_AU_W2V_STEM
};
typedef struct agpt_audio_probe_args {
  int op;
  const float* x; const float* x2; const float* w; const float* g; const float* b;
  const int* starts;
  float* y; float* y2;
  void* part; void* stat; int* cnt;
  int B, T, F, C, D, W, n, hop, nb, nm, ch, pitch, Na, Nt, k0, s0, s1, orig, nw, width, clip;
  long rows, N, R, sb, stt, sf;
  float scale, shift, eps;
} agpt_audio_probe_args;
int agpt_audio_probe(const agpt_audio_probe_args* args, void* stream);
/* Conformance entry of the vocoder and diffusion-step kernels that no other entry reaches on their own (HiFi-GAN /
 * BigVGAN layout, conv_post, BigVGAN's anti-aliased Snake, the NSF excitation add, DiffNet's step embedding and the
 * graph-replayed p_sample step; tests/test_vocoder_kernels_gpu.py): ONE call of the production launcher selected by
 * `op` on caller-owned device tensors, with the arguments as given.  Tensors are fp32 device arrays except `taps`
 * (fp32, HOST), `t` (int32: HOST for STEP_EMBED, device for STEP_EMBED_DEV), `ctr` (int32, device), `noises_pp` (a
 * device slot holding a device pointer) and `ran` (int32, HOST).  The launcher's preconditions are checked first; a
 * violation returns an error with nothing launched.  The fields each op reads:
 *   CF_TO_CL        x [B][C][L] -> y [B][L][C]
 *   CONV_POST       x [B][L][C], w [c_out][7][C], b [c_out], slope -> y [B][c_out][L]; ran (null = not reported) <- 1
 *                   when conv_post32_kernel ran, 0 for the generic kernel; C % 4 == 0, c_out 7 C 4 bytes <= 48 KB
 *   AA_SNAKE        x [B][L][C], a [C], inv_b [C], taps [12] -> y [B][L][C]; L >= 1
 *   NSF_ADD         y [B][L][C] in place, x = har [B][Lh], w [C][K], b [C], K, st, pad; K >= 1, st >= 1
 *   STEP_EMBED      t [B] (host) -> y [B][C]; B <= 256, C even, C / 2 > 1
 *   STEP_EMBED_DEV  t [B] (device) -> y [B][C]; C even, C / 2 > 1
 *   P_SAMPLE_TAB    y = x [B][n] in place, x = eps [B][n], w = coefficient table [nsteps][5], ctr [1], nsteps,
 *                   noises_pp, noise_stride, clip; nsteps >= 1
 * Synchronises `stream` before returning.                                                                          */
enum {
  AGPT_VC_CF_TO_CL = 0, AGPT_VC_CONV_POST, AGPT_VC_AA_SNAKE, AGPT_VC_NSF_ADD, AGPT_VC_STEP_EMBED, AGPT_VC_STEP_EMBED_DEV,
  AGPT_VC_P_SAMPLE_TAB
};
typedef struct agpt_voc_probe_args {
  int op;
  const float* x; const float* w; const float* b; const float* a; const float* inv_b; const float* taps;
  const int* t; const int* ctr;
  const float* const* noises_pp;
  float* y;
  int* ran;
  int B, L, C, c_out, Lh, K, st, pad, nsteps, clip;
  long n, noise_stride;
  float slope;
} agpt_voc_probe_args;
int agpt_voc_probe(const agpt_voc_probe_args* args, void* stream);
/* Conformance entry of the analysis models' kernels outside the GEMMs (LASSNet's FiLM ResUNet, RaDur's detection tail,
 * the BERT embeddings, the emotion encoder's tail; tests/test_an_kernels_gpu.py): ONE call of the production launcher
 * selected by `op` on caller-owned device tensors, with the arguments as given.  Tensors are fp32 device arrays except
 * the int32 device arrays ids, type_ids, mask and the FiLM tables (woff .. jb), kpm (uint8_t, device) and info (int32,
 * HOST); h is an agpt_handle.  The launcher's preconditions are checked first; a violation returns an error with nothing
 * launched.  Rows are channels-last; the map sizes h, w below are the fields hh, ww.  The fields each op reads:
 *   LASS_AFFINE      x [rows][C], s [C], t [C], vec [B][vec_len], vec_off, rows, rows_per_sample -> y = fmaf(x, s, t)
 *                    [rows][C], y2 (null = none) = x + vec[row / rows_per_sample][vec_off + c]; C % 4 == 0,
 *                    rows, rows_per_sample >= 1; with y2: vec_off + C <= vec_len, vec_off and vec_len multiples of 4
 *   LASS_UPCOL       x [B][h][w][C], s [C], t [C] -> y [B][h][w + 1][4][C]; C % 4 == 0, h, w >= 1
 *   LASS_SHUFFLE     x = up [B][h][w + 1][4][C], x2 = skip [B][2h][2w + 1][C] -> y [B][2h][2w + 1][2C]; C % 4 == 0
 *   LASS_FILM        x = hid [B][hid_len], w2 [..], woff / hoff / nin [outputs], b2 [outputs], dst / ja / jb / alpha /
 *                    beta [nj] -> y = vec [B][vec_len] (only the dst entries are written)
 *   LASS_FILM_VEC    h (LASSNet), x = cond [B][256] -> y = the FiLM vectors [B][vec_len] (y null: nothing runs);
 *                    info[0] <- vec_len
 *   LASS_UP          h (LASSNet), level in [0, 6), x [B][h][w][cin], x2 = skip [B][2h][2w + 1][cout] -> y = the
 *                    decoder's concat [B][2h][2w + 1][2 cout] (bn1, ReLU, ConvTranspose2d(3, 2) pruned, skip);
 *                    info[0] <- vec_len
 *   TSD_PAD4         x [rows] -> y [rows][4]
 *   TSD_FUSE         x = f2 [B][Td][C n], x2 = e1 [B][C n], n -> y [B][Td][C]; n >= 1
 *   TSD_REFEMB       x = E [B][T][128], att_pool, w = q weight [128][128], b = q bias, w2 = k weight, b2 = k bias,
 *                    scratch [B][T] -> y [B][128]; T >= 1, scratch required when att_pool
 *   TSD_HEAD         x [rows][1024], w [O][1024], b [O] -> y [rows][O]; 1 <= O <= 16
 *   TSD_MIX_INTERP   x = p1 [B][Td][O], x2 = p2 (null = one pass), vec = wmix [B] -> y = decision [B][Td], y2 = the
 *                    interpolated [B][T][O]; 1 <= O <= 16
 *   CLAP_EMBED       ids [N][L], w = word [vocab][H], x = pos [L][H], x2 = type row [H] -> y [N][L][H]
 *   CLAP_EMBED_TYPED ids, type_ids, mask [N][L], w = word, x = pos, x2 = types [ntypes][H] -> y [N][L][H], kpm [N][L]
 *   CLAP_GELU        x [rows], max_blocks -> y [rows]
 *   EMO_MEAN_NORM    x [N][256] -> y [256]; N >= 1
 *   EMO_LINEAR_NORM  x [N][256], w [E][256], b [E] -> y [N][E]; E >= 1, (E + 288) floats <= 48 KB
 * Synchronises `stream` before returning.                                                                          */
enum {
  AGPT_AN_LASS_AFFINE = 0, AGPT_AN_LASS_UPCOL, AGPT_AN_LASS_SHUFFLE, AGPT_AN_LASS_FILM, AGPT_AN_LASS_FILM_VEC, AGPT_AN_LASS_UP,
  AGPT_AN_TSD_PAD4, AGPT_AN_TSD_FUSE, AGPT_AN_TSD_REFEMB, AGPT_AN_TSD_HEAD, AGPT_AN_TSD_MIX_INTERP, AGPT_AN_CLAP_EMBED,
  AGPT_AN_CLAP_EMBED_TYPED, AGPT_AN_CLAP_GELU, AGPT_AN_EMO_MEAN_NORM, AGPT_AN_EMO_LINEAR_NORM
};
typedef struct agpt_an_probe_args {
  int op;
  void* h;
  const float* x; const float* x2; const float* s; const float* t; const float* w; const float* b; const float* w2;
  const float* b2; const float* vec; const float* alpha; const float* beta;
  const int* ids; const int* type_ids; const int* mask;
  const int* woff; const int* hoff; const int* nin; const int* dst; const int* ja; const int* jb;
  float* y; float* y2; float* scratch;
  uint8_t* kpm;
  int* info;
  int B, C, hh, ww, level, nj, hid_len, vec_len, vec_off, Td, T, O, n, att_pool, N, L, H, E, vocab, ntypes, max_blocks;
  long rows, rows_per_sample;
} agpt_an_probe_args;
int agpt_an_probe(const agpt_an_probe_args* args, void* stream);

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
 * launches, then ONE captured step (CUDA graph + device-side step counter) is replayed; while agpt_profile_enable
 * is on, every step runs as plain launches.                                                                 */
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
 * While agpt_profile_enable is on, every step runs as plain launches.                          */
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

/* ------------------------------------------------------------------ GenerSpeech
 * Replaces GenerSpeech.forward (NeuralSeq/modules/GenerSpeech/model/generspeech.py:75-260) as GenerSpeechInfer.forward_model
 * calls it (infer=True, global_steps past `forcing`): the FastSpeech2 encoder / durations / decoder of agpt_fs2_cfg (pitch_type
 * 'frame', pitch_norm 'standard' with uv, fairseq positions, no energy / MIDI) with the 256 -> H speaker and emotion
 * projections, three LocalStyleAdaptors (utterance, phoneme, word: WN, segment mean, ConvBlocks, VQ) feeding ProsodyAligners
 * (2 heads), the pitch inpainter, and the Glow post-flow (n_sqz 2, n_split 4, post_share_cond_layers off, sigmoid_scale
 * off, use_txt_cond on) run in reverse.  The training diagnostics (VQ losses, perplexities, guided-attention losses and
 * maps) are not computed.                                                                                         */
typedef struct agpt_gs_cfg {   /* tagged, as agpt_clap_cfg: it nests agpt_fs2_cfg */
  agpt_fs2_cfg fs2;
  int n_vq;                    /* hparams['nVQ'] */
  int glow_hidden, glow_kernel, glow_blocks, glow_layers;   /* post_glow_hidden / _kernel_size / _n_blocks / _n_block_layers */
  int share_wn_layers;         /* blocks b - b % share_wn_layers share their WN in_layers / res_skip_layers (0: none) */
} agpt_gs_cfg;
/* Optional stage outputs of agpt_gs_forward (any pointer may be NULL): the decoder's mel before the post-flow
 * [B][T_mel][80]; per level (utterance, phoneme, word) the quantised prosody [B][T_k][H] and its code indices [B][T_k]
 * int32, T_k = T_ref, n_seg_ph, n_seg_word.                                                                         */
typedef struct agpt_gs_taps {
  float* mel_pre_flow;
  float* prosody[3];
  int* vq_idx[3];
} agpt_gs_taps;
/* host_weights: fp32 HOST arrays in the order of audiogpt_b200.modules.GenerSpeech.model.generspeech.GenerSpeech
 * .engine_weights() (weight norm folded, each InvConvNear's inverse computed, the eight cond_layers concatenated).  */
int agpt_gs_create(const agpt_gs_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out);
/* Token side, as agpt_fs2_encode: txt_tokens [B][T_txt] int32, spk_embed / emo_embed [B][256] fp32 (device).  dur = the
 * duration predictor's output on (encoder_out + spk + emo) * nonpadding.  predict_dur != 0: dur_choice (may be NULL) and
 * mel_len_host [B] (HOST; the call synchronises the stream for this one copy).  spk_out / emo_out [B][H] (may be NULL):
 * spk_embed_proj(spk_embed), emo_embed_proj(emo_embed).                                                            */
int agpt_gs_encode(agpt_handle h, const int* txt_tokens, int B, int T_txt, const float* spk_embed, const float* emo_embed,
                   int predict_dur, float* dur, int* dur_choice, int* mel_len_host, float* spk_out, float* emo_out, void* stream);
/* Frame side, T_mel >= 2 frames: mel2ph [B][T_mel] int32 (teacher-forced) or NULL = the durations of the last encode,
 * expanded into mel2ph_out.  ref_mels [B][T_ref][80] (frames whose channel 0 is exactly 0 are padding); ref_mel2ph /
 * ref_mel2word [B][T_ref] int32 segment ids (0 = none), n_seg_* = their maximum over the batch.  z [B][80][T_mel]: the
 * post-flow's input noise, already scaled by noise_scale.  Outputs (device): pitch_pred [B][T_mel][2], f0_denorm,
 * f0_denorm_pred [B][T_mel], pitch_coarse [B][T_mel] int32, decoder_inp and ref_prosody [B][T_mel][H], mel_out
 * [B][2 (T_mel / 2)][80] (the post-flow truncates an odd T_mel).                                                    */
int agpt_gs_forward(agpt_handle h, int T_mel, const int* mel2ph, int* mel2ph_out, const float* ref_mels, int T_ref,
                    const int* ref_mel2ph, int n_seg_ph, const int* ref_mel2word, int n_seg_word, const float* z, float f0_mean,
                    float f0_std, float* pitch_pred, float* f0_denorm, float* f0_denorm_pred, int* pitch_coarse, float* decoder_inp,
                    float* ref_prosody, float* mel_out, const agpt_gs_taps* taps, void* stream);

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

/* ------------------------------------------------------------------ Sound extraction
 * The SoundExtraction tool (audio-chatgpt.py:675-710): sound_extraction/model/LASSNet.py -- bert-mini on the query
 * ([CLS] row -> Linear(256, 256) -> ReLU = cond), then UNetRes_FiLM (resunet_film.py, modules.py:169-379, film.py;
 * eval BatchNorm, eps 1e-5) conditioned on cond, then a sigmoid -- and sound_extraction/utils/stft.py's STFT.
 * A tagged struct, as agpt_clap_cfg (it carries a float).                                                          */
typedef struct agpt_lass_cfg {
  int vocab_size;              /* bert-mini: 30522 */
  int max_position_embeddings; /* 512 */
  int type_vocab_size;         /* 2 (only type 0 is read) */
  int hidden_size;             /* 256 (the Linear after BERT is 256 -> 256) */
  int num_layers;              /* 4 */
  int num_heads;               /* 4 */
  int intermediate_size;       /* 1024 */
  float layer_norm_eps;        /* 1e-12 */
} agpt_lass_cfg;
/* host_weights: fp32 HOST arrays in the key order of audiogpt_b200.specs.lass_engine_keys(cfg): LASSNet's state dict
 * without num_batches_tracked (and without the position_ids buffer).                                              */
int agpt_lass_create(const agpt_lass_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out);
/* input_ids / attention_mask [N][L] int32 (device; ids clamped to the table, callers reject them first) -> cond
 * [N][256] (device): relu(Linear(BertModel(input_ids, attention_mask)[0][:, 0])), padding keys masked out.       */
int agpt_lass_text(agpt_handle h, const int* input_ids, const int* attention_mask, int N, int L, float* cond, void* stream);
/* mag: the magnitude [B][T][F] (device) at element strides stride_b / stride_t / stride_f (the tool passes a transposed
 * view); cond [B][256] (device) -> mask [B][T][F] = sigmoid(UNetRes_FiLM(mag, cond, cond)) and, when logits is not
 * NULL, the pre-sigmoid values (0 in the two top bins).  F - 2 must be 63 mod 64 and at least 127; any T >= 1.     */
int agpt_lass_mask(agpt_handle h, const float* mag, int B, int T, int F, long stride_b, long stride_t, long stride_f,
                   const float* cond, float* mask, float* logits, void* stream);
/* STFT(filter_length, hop_length, win_length = filter_length, window 'hann') with filter_length = 2 hop_length:
 * host_weights: the module's buffers forward_basis, inverse_basis [filter_length + 2][1][filter_length] (HOST).   */
int agpt_stft_create(int filter_length, int hop_length, const float* const* host_weights, int n_weights, int device,
                     agpt_handle* out);
/* STFT.transform: wav [B][n_samples] (device, n_samples > filter_length / 2) -> magnitude / phase
 * [B][filter_length / 2 + 1][n_samples / hop + 1] (device).                                                         */
int agpt_stft_transform(agpt_handle h, const float* wav, int B, long n_samples, float* magnitude, float* phase, void* stream);
/* STFT.inverse: magnitude / phase [B][filter_length / 2 + 1][T] (device, T >= 2) -> wav [B][(T - 1) hop] (device).   */
int agpt_stft_inverse(agpt_handle h, const float* magnitude, const float* phase, int B, int T, float* wav, void* stream);

/* ------------------------------------------------------------------ Sound event detection
 * The SoundDetection tool (audio-chatgpt.py:612-673): audio_detection/audio_infer/pytorch/models.py:141-237 PVT, eval
 * mode -- torchlibrosa Spectrogram / LogmelFilterBank / bn0 (as Cnn14's), PyramidVisionTransformerV2 (:832-927: four
 * stages of OverlapPatchEmbed + Blocks of spatial-reduction attention and a depthwise-conv Mlp; no positional
 * embedding, so any clip length), mean over the mel axis, fc_audioset, sigmoid.  A tagged struct, as agpt_clap_cfg.   */
typedef struct agpt_pvt_cfg {
  int window_size;        /* 1024 */
  int hop_size;           /* 320 */
  int mel_bins;           /* 64 (bn0 is BatchNorm2d(64)) */
  int classes_num;        /* 527 */
  int embed_dims[4];      /* 64, 128, 320, 512; embed_dims[i] = 64 * num_heads[i] */
  int depths[4];          /* 3, 4, 6, 3 */
  int num_heads[4];       /* 1, 2, 5, 8 */
  int mlp_ratios[4];      /* 8, 8, 4, 4 */
  int sr_ratios[4];       /* 8, 4, 2, 1: Attention.sr = Conv2d(C, C, sr, stride sr) when > 1 */
  int interpolate_ratio;  /* 32: each framewise row is repeated this many times */
  float layer_norm_eps;   /* 1e-6: Block.norm1 / norm2 and the stage norms (the norm_layer partial) */
  float embed_norm_eps;   /* 1e-5: OverlapPatchEmbed.norm and Attention.norm (plain nn.LayerNorm) */
} agpt_pvt_cfg;
/* host_weights: fp32 HOST arrays in the key order of audiogpt_b200.specs.pvt_engine_keys(cfg): PVT's state dict without
 * bn0.num_batches_tracked.  bn0 is folded (eps 1e-5).                                                             */
int agpt_pvt_create(const agpt_pvt_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out);
/* Host only: the token grid (rows = time, columns = mel) of each stage for a clip of n_samples, from the conv
 * arithmetic T = n / hop + 1; H1 = (T - 3) / 4 + 1, W1 = (mel_bins - 3) / 4 + 1; H(i+1) = (Hi - 1) / 2 + 1, likewise W.
 * Fails when n_samples <= window_size / 2 (reflect padding), when a grid is empty or when a stage's grid is smaller
 * than its sr_ratio in either direction (no key would be left).  With the shipped config the shortest clip is
 * 30 * hop = 9600 samples (0.3 s at 32 kHz): H1 = 8 needs T >= 31.                                                 */
int agpt_pvt_frames(const agpt_pvt_cfg* cfg, long n_samples, int grid_hw[4][2]);
/* wav [B][n_samples] (device) -> framewise [B][interpolate_ratio * H4][classes_num] and clipwise [B][classes_num]
 * (device; H4 from agpt_pvt_frames).  logits, when not NULL: the pre-sigmoid values [B][H4][classes_num].          */
int agpt_pvt_forward(agpt_handle h, const float* wav, int B, long n_samples, float* framewise, float* clipwise, float* logits,
                     void* stream);
/* One launch of each PVT kernel on caller-owned device tensors (the unit tests' entry points).
 * dwconv_gelu: x [B][H * W][C] -> gelu(depthwise 3 x 3 conv, padding 1, w [C][3][3] and bias [C] on the device) as fp32
 * (out) or as fp16 hi / lo operand planes (out NULL).  C % 4 == 0.                                                  */
int agpt_pvt_dwconv_gelu(const float* x, const float* w, const float* bias, int B, int H, int W, int C, float* out, void* plane_hi,
                         void* plane_lo, void* stream);
/* patch7: img [B][H][W] -> LayerNorm(Conv2d(1, C, 7, stride 4, padding 2)) as tokens [B][Ho * Wo][C]; w [C][49], bias,
 * gamma, beta [C] on the device; C in {32, 64, 96, 128}.                                                           */
int agpt_pvt_patch7(const float* img, const float* w, const float* bias, const float* gamma, const float* beta, float eps, int B,
                    int H, int W, int C, float* out, void* stream);
/* sr_gather: x [B][H * W][C] -> out [B][(H / sr) * (W / sr)][sr * sr * C], patch rows in (ky, kx, c) order.        */
int agpt_pvt_sr_gather(const float* x, int B, int H, int W, int C, int sr, float* out, void* stream);
/* head: x [B][H * W][C], fc weight [classes][C] and bias on the device -> framewise [B][ratio * H][classes], clipwise
 * [B][classes], logits [B][H][classes] or NULL.                                                                    */
int agpt_pvt_head(const float* x, const float* w, const float* bias, int B, int H, int W, int C, int classes, int ratio,
                  float* framewise, float* clipwise, float* logits, void* stream);

/* ------------------------------------------------------------------ Target sound detection
 * The TargetSoundDetection tool (audio-chatgpt.py:775-875): audio_detection/target_sound_detection/src/models.py:1109-1291
 * RaDur_fusion, eval mode -- Cnn14 (mel input, no front end) embeds the reference clip, Cnn10_mul_scale (a 1 x 1 /
 * 3 x 3 / 5 x 5 GLU stem, then three ConvBlocks) and Fusion(128, 512, 2) feed a bidirectional GRU(512, 512), fc,
 * outputlayer and a softmax; with enhancement the first decision's top-k frames select mixture embeddings that make a
 * second fused embedding and a second GRU pass, and the two decisions are mixed.  A tagged struct, as agpt_clap_cfg.  */
typedef struct agpt_tsd_cfg {
  int time_resolution;    /* 125 / 250 / 500 / other: Cnn10_mul_scale(8 / 4 / 2 / 0), which sets the pool sizes */
  int att_pool;           /* 1: attention-pool the reference embeddings (after RaDur_fusion.bn); 0: their plain mean */
  int enhancement;        /* 1: run orcal_EE (the second, top-k enhanced pass) */
  int top;                /* >= 1: frames in the top-k (all T' frames when T' < top) */
  float tao;              /* the top-k score gate (the tool sets 0.6) */
  int mel_bins;           /* 64 */
  int outputdim;          /* 2 (1..16) */
} agpt_tsd_cfg;
/* host_weights: fp32 HOST arrays in the key order of audiogpt_b200.specs.tsd_engine_keys(cfg): RaDur_fusion's state dict
 * without the encoder's unused front end (spectrogram_extractor, logmel_extractor, bn0), fc_audioset and
 * num_batches_tracked.  BatchNorm eps 1e-5.                                                                         */
int agpt_tsd_create(const agpt_tsd_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out);
/* Host only: frames[0] = T', the detection frames of a T-frame clip (the stem keeps min(floor((T + 2) / ph), 500,
 * floor(T / ph), floor((T - 2) / ph) + 1) rows, then the three pools divide by their row sizes); frames[1] = Tr / 8,
 * the reference encoder's frames; frames[2] = T / 8 with enhancement, else 0.  Fails when any of them would be 0.    */
int agpt_tsd_frames(const agpt_tsd_cfg* cfg, int T, int Tr, int frames[3]);
/* x [B][T][64], ref [B][Tr][64] log-mels (device) -> decision [B][T'] (the final decision's class 0) and decision_up
 * [B][T][outputdim] (the final decision linearly interpolated to T, align_corners = False).  With enhancement and
 * T' > T / 8 (time_resolution other than 125), a top-k frame past T / 8 is refused, as the reference's gather fails.   */
int agpt_tsd_forward(agpt_handle h, const float* x, const float* ref, int B, int T, int Tr, float* decision, float* decision_up,
                     void* stream);
/* Timing: events points to n = 7 cudaEvent_t (or n = 0 to stop) that every later forward records at its stage
 * boundaries: start, after the reference embedding, after the mixture's Cnn14 (enhancement), after the detection
 * features, after the first GRU pass, after the enhancement and second pass, end.                                  */
int agpt_tsd_stage_events(agpt_handle h, void* events, int n);
/* One launch of each new RaDur_fusion kernel on caller-owned device tensors (the unit tests' entry points).
 * stem: mel [B][T][64] -> [B][m][32][96] (m as in agpt_tsd_frames); w [3][64][25] (branch k = 1, 3, 5: the k * k
 * taps of each output channel first) and b [3][64] are the convs with BatchNorm folded; ph (1 or 2) the row pool.    */
int agpt_tsd_stem(const float* mel, const float* w, const float* b, int B, int T, int ph, float* out, void* stream);
/* avgpool: F.avg_pool2d(kernel = stride = (ph, pw)) on channels-last in [B][H][W][C] -> out [B][H / ph][W / pw][C].  */
int agpt_tsd_avgpool(const float* in, int B, int H, int W, int C, int ph, int pw, float* out, void* stream);
/* gru: the recurrence of a bidirectional GRU(512, 512): w_hh [2][1536][512], b_hh [2][1536] (forward, reverse), xproj
 * [B][T][3072] = the input projections W_ih x + b_ih (forward r, z, n | reverse r, z, n) -> out [B][T][1024].        */
int agpt_tsd_gru(const float* w_hh, const float* b_hh, const float* xproj, int B, int T, float* out, void* stream);
/* enhance: the tail of orcal_EE.  p1 [B][Td][O] the first decision (softmax), mix_emb [B][Te][128] bn(Cnn14(x)), emb
 * [B][128]; weights (device) q_ee.weight [128][128], q_ee.bias, k_ee.weight, k_ee.bias, EE_fusion.fuse_layer1.conv
 * weight [512][128] and bias, fuse_layer2 weight and bias -> me [B][128] (EE_fusion's output), wmix [B] (the second
 * decision's weight), topk_idx [B][k] int32 and topk_val [B][k] (may be NULL), k = min(top, Td), Td <= 500.           */
int agpt_tsd_enhance(const float* p1, int B, int Td, int O, const float* mix_emb, int Te, const float* emb, int top, float tao,
                     const float* const* weights8, float* me, float* wmix, int* topk_idx, float* topk_val, void* stream);

/* ------------------------------------------------------------------ Binaural
 * The Binaural tool (audio-chatgpt.py:713-773): mono2binaural/src/models.py BinauralNetwork -> Warpnet, eval mode.  A
 * warpnet of `layers` causal convs (F.pad([1, 0]), Conv1d(k = 2), ReLU; 7 -> C, then C -> C) and a 1 x 1 Conv1d C -> 2
 * plus a geometric warp from the mouth-to-ear distance give each view frame a warp per ear; it is selected per sample
 * as F.interpolate(mode = 'nearest') does, clipped to <= 0, added to the sample index, clamped to [0, T - 1], made
 * monotone by a running max, and the mono signal is read there by linear interpolation, for each ear.          */
typedef struct agpt_binaural_cfg {
  int layers;             /* warpnet_layers: 1..4 (the tool ships 4) */
  int channels;           /* warpnet_channels: a multiple of 8 in [8, 64] (the tool ships 64) */
} agpt_binaural_cfg;
/* One row: one BinauralNetwork forward of T samples and K view frames.  mono[mono_off + t], t < T; view channel c of
 * frame k at view[view_off + c * view_stride + k]; samples t >= keep of ear e go to out[out_off + e * out_stride + t -
 * keep].  A batch is B rows of one shape; the tool's chunk loop is one row per chunk, each writing its kept tail.   */
typedef struct agpt_binaural_row {
  int64_t mono_off, T, view_off, view_stride, K, keep, out_off, out_stride;
} agpt_binaural_row;
/* host_weights: fp32 HOST arrays in the order of audiogpt_b200.specs.binaural_param_shapes(cfg): warper.layers.{l}
 * .weight [C][cin][2] and .bias [C] for each layer, then warper.linear.weight [2][C][1] and .bias [2].             */
int agpt_binaural_create(const agpt_binaural_cfg* cfg, const float* const* host_weights, int n_weights, int device,
                         agpt_handle* out);
/* mono and view (device) -> out (device) for n_rows rows (a HOST array): three launches whatever the rows, no host
 * synchronisation.  clamp = 1 clamps every output sample to [-1, 1] (the tool's final clamp).  Every row needs
 * 1 <= T <= 2^24, K >= 1 and 0 <= keep < T.  The frame field, tile maxima and row table are workspaces of the handle:
 * calls on one handle must be ordered on one stream (calls from two streams at once race on them).               */
int agpt_binaural_forward(agpt_handle h, const float* mono, const float* view, const agpt_binaural_row* rows, int n_rows,
                          float* out, int clamp, void* stream);
/* The two stages apart (the unit tests' entry points).  frames: view -> the frame field, rows packed one after the
 * other, each [2][K]: f[e][k] = ((-d_e) / 343) * 48000 + n_e[k], d_e the mouth-to-ear distance, n the warpnet output.
 * warp: a frame field in that layout and mono -> out, as agpt_binaural_forward does after its frame stage.          */
int agpt_binaural_frames(agpt_handle h, const float* view, const agpt_binaural_row* rows, int n_rows, float* field, void* stream);
int agpt_binaural_warp(agpt_handle h, const float* field, const float* mono, const agpt_binaural_row* rows, int n_rows,
                       float* out, int clamp, void* stream);

/* ------------------------------------------------------------------ Reference-audio ASR (wav2vec2 CTC)
 * GenerSpeechInfer.preprocess_input transcribes the reference clip with transformers' Wav2Vec2ForCTC
 * (facebook/wav2vec2-base-960h; NeuralSeq/inference/tts/base_tts_infer.py:38-42, 83-101), eval mode, no attention mask:
 * the conv feature encoder (conv0 + GroupNorm(C groups) + GELU, then stride-s convs + GELU, no conv bias), the feature
 * projection (LayerNorm + Linear), the weight-normed grouped positional conv (padding K / 2, SamePad, GELU) added to it,
 * LayerNorm, post-LN encoder layers (exact GELU) and lm_head.  Only that layout is covered ("group" feature-extractor
 * norm, no stable layer norm); the drop-in rejects the others.  A tagged struct, as agpt_clap_cfg.                 */
#define AGPT_W2V_MAX_CONV 8
typedef struct agpt_w2v_cfg {
  int conv_layers;                    /* 7 */
  int conv_dim;                       /* 512: the width of every conv (a multiple of 32, at most 1024) */
  int conv_kernel[AGPT_W2V_MAX_CONV]; /* 10, 3, 3, 3, 3, 2, 2 (conv_kernel[0] <= 16) */
  int conv_stride[AGPT_W2V_MAX_CONV]; /* 5, 2, 2, 2, 2, 2, 2 */
  int hidden_size;                    /* 768 */
  int num_layers;                     /* 12 */
  int num_heads;                      /* 12: head dim 64 */
  int intermediate_size;              /* 3072 */
  int num_conv_pos_embeddings;        /* 128: the positional conv's taps (<= 128) */
  int num_conv_pos_embedding_groups;  /* 16: hidden_size = 48 * groups */
  int vocab_size;                     /* 32: lm_head's width */
  float layer_norm_eps;               /* 1e-5 (the GroupNorm's eps is nn.GroupNorm's 1e-5) */
} agpt_w2v_cfg;
/* host_weights: fp32 HOST arrays in the order of audiogpt_b200.specs.w2v_engine_weights(cfg, state_dict): conv0 weight,
 * GroupNorm weight / bias, conv 1.. as super-row weights [C][s C][ceil(k / s)], the projection's LayerNorm and Linear,
 * the positional conv's folded weight g v / |v| [H][48][K] and bias, encoder.layer_norm, each layer's q, k, v, out_proj,
 * layer_norm, intermediate_dense, output_dense, final_layer_norm (weight, bias each), lm_head weight / bias.           */
int agpt_w2v_create(const agpt_w2v_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out);
/* Host only: the frames an input of n_samples yields (the conv lengths (T - k) / s + 1 in turn; 0 when a layer has none). */
int agpt_w2v_frames(const agpt_w2v_cfg* cfg, long n_samples, int* frames);
/* input_values [B][n_samples] (device) -> logits [B][frames][vocab_size] (device).  frames >= 1.  Work buffers belong
 * to the handle: calls on one handle must be ordered on one stream.                                                 */
int agpt_w2v_logits(agpt_handle h, const float* input_values, int B, long n_samples, float* logits, void* stream);
/* The stages apart (the unit tests' entry points).  features: the conv feature encoder's output, channels last
 * [B][frames][conv_dim].  pos_conv: hidden [B][T][H] -> out = hidden + gelu(pos_conv(hidden)) [B][T][H] (not aliased;
 * hidden 16-byte and out 8-byte aligned).                                                                            */
int agpt_w2v_features(agpt_handle h, const float* input_values, int B, long n_samples, float* features, void* stream);
int agpt_w2v_pos_conv(agpt_handle h, const float* hidden, int B, int T, float* out, void* stream);

/* ------------------------------------------------------------------ Emotion encoder
 * The TTS_OOD tool's emo_embed (NeuralSeq/inference/tts/GenerSpeech.py:37,58): data_gen/tts/emotion/inference.py
 * embed_utterance -- the partial-utterance slices of compute_partial_slices, librosa's power mel of the zero-padded wav
 * (n_fft 400 = win, hop 160, periodic Hann, center with reflect padding, power 2, 40 Slaney bands 0..8 kHz, no log),
 * EmotionEncoder.inference (model.py: nn.LSTM(40, 256, num_layers, batch_first) from h0 = c0 = 0, the last layer's
 * final h) per partial, their mean and its L2 norm.  A tagged struct, as agpt_clap_cfg.                              */
typedef struct agpt_emo_cfg {
  int input_size;      /* 40: mel_n_channels */
  int hidden_size;     /* 256 */
  int num_layers;      /* 3 (1..16) */
  int embedding_size;  /* 256: EmotionEncoder.linear's width (forward only; 1..4096) */
} agpt_emo_cfg;
/* host_weights: fp32 HOST arrays in the order of audiogpt_b200.specs.emo_engine_weights(cfg, state_dict): per layer
 * lstm.weight_ih_l{k} [1024][in], lstm.weight_hh_l{k} [1024][256], bias_ih_l{k} + bias_hh_l{k} [1024]; linear.weight
 * [E][256] and bias [E]; the DFT rows of the periodic-Hann window, real and imaginary [201][400] each; the Slaney mel
 * matrix transposed, [201][40].                                                                                     */
int agpt_emo_create(const agpt_emo_cfg* cfg, const float* const* host_weights, int n_weights, int device, agpt_handle* out);
/* Host only: compute_partial_slices(n_samples, partial_frames, min_pad_coverage, overlap) in frames of 160 samples ->
 * the partial count, the frame step between partials (partial p is mel frames step p .. step p + partial_frames - 1)
 * and the length embed_utterance zero-pads the wav to (wav_slices[-1].stop when that is at least n_samples, else
 * n_samples).                                                                                                        */
int agpt_emo_partials(long n_samples, int partial_frames, double min_pad_coverage, double overlap, int* n_partials, int* frame_step,
                      long* padded);
/* wav [n_samples] (device, not padded) -> embed [256] (device): embed_utterance.  partial_frames >= 1: the slices of
 * agpt_emo_partials, and partials [n_partials][256] (device, may be NULL) receives each partial's hidden[-1];
 * partial_frames = 0: using_partials=False, the whole mel as one sequence (then the embedding is hidden[-1] itself,
 * not normalised, as the reference returns it).  The mel needs at least 201 samples after padding.  Work buffers
 * belong to the handle: calls on one handle must be ordered on one stream.                                           */
int agpt_emo_embed(agpt_handle h, const float* wav, long n_samples, int partial_frames, double min_pad_coverage, double overlap,
                   float* embed, float* partials, void* stream);
/* frames [N][T][40] (device) -> hidden [N][256]: EmotionEncoder.inference (the last layer's final h).              */
int agpt_emo_hidden(agpt_handle h, const float* frames, int N, int T, float* hidden, void* stream);
/* frames [N][T][40] (device) -> embeds [N][E]: EmotionEncoder.forward, relu(linear(hidden[-1])) / its L2 norm.      */
int agpt_emo_forward(agpt_handle h, const float* frames, int N, int T, float* embeds, void* stream);
/* The stages apart (the unit tests' entry points).  mel: wav [n_samples] (device, n_samples >= 201) -> mel
 * [n_samples / 160 + 1][40], wav_to_mel_spectrogram.  lstm: one layer's recurrence, no handle: w_hh [1024][256], xproj
 * [.][1024] the input projections W_ih x + b_ih + b_hh, sequence n's step t at row n * seq_stride + t -> h_seq
 * [N][T][256] every step's h and h_last [N][256] the final h (either may be NULL, not both).                          */
int agpt_emo_mel(agpt_handle h, const float* wav, long n_samples, float* mel, void* stream);
int agpt_emo_lstm(const float* w_hh, const float* xproj, int N, int T, long seq_stride, float* h_seq, float* h_last, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* AGPT_B200_H */
