// Launchers of the kernels that touch audio samples and spectrogram bins, shared by the drivers (clap_score.cu, pvt.cu,
// emotion.cu, lass.cu, w2v.cu) and the conformance probe (microbench.cu: agpt_audio_probe).  Each one launches its
// kernel(s) with the production grid and block size and counts the launches; none synchronises.  Each one checks the
// preconditions its kernel's indexing relies on and throws before launching when they fail.
#pragma once
#include "common.cuh"

namespace agpt {

// fr [B][T][n] = x_b[reflect(t hop + j - n / 2)], T = clip / hop + 1 (center=True, pad_mode='reflect'); clip > n / 2
void cnn14_frames(const float* x, int clip, int B, int hop, int n, float* fr, cudaStream_t st);
// one block per frame of spec [frames][pitch] ([re | im], nb bins each): re^2 + im^2 -> melW [nb][nm] projection ->
// 10 log10(max(., 1e-10)) -> bn0 (folded scale bn_s / shift bn_t per mel bin) -> img [frames][nm][ch], ch = 1 or 4
// (channels 1..3 zero: Cnn14's first conv reads a 4-channel padded input)
void cnn14_logmel(const float* spec, int pitch, int nb, const float* melW, int nm, const float* bn_s, const float* bn_t, float* img,
                  long frames, int ch, cudaStream_t st);
// the emotion encoder's power mel: mel [frames][40] = sum_k (re_k^2 + im_k^2) melW [k][40] over spec [frames][pitch]
// ([re | im], 201 bins each; no log)
void emo_powmel(const float* spec, int pitch, const float* melW, float* mel, long frames, cudaStream_t st);

// out [B][clip]: out[b][i] = y_b[(start_b + i) mod R], y_b = torchaudio's polyphase resampling of x_b [L] (ker [nw][taps],
// taps = 2 width + orig), R = ceil(nw L / orig).  start_host [B] holds a crop start in [0, R - clip) when R > clip and -1
// (tile) otherwise; it is validated, then copied to start_dev (grown to B ints) on the stream.
void cnn14_resample(const float* x, long L, int B, const float* ker, int orig, int nw, int width, const int* start_host,
                    DevBuf& start_dev, int clip, float* out, cudaStream_t st);
// Cnn14's pooling tail: out [B][C] = max_t mean_f x + mean_t mean_f x over x [B][T][F][C]
void cnn14_head(const float* x, int B, int T, int F, int C, float* out, cudaStream_t st);

// rows [B][R][hop], R = ceil((N + n) / hop): padded sample r hop + j of wav_b [N] (reflect-padded by n / 2 on each
// side, zero past N + n); N > n / 2
void stft_rows(const float* wav, int B, long N, int n, int hop, float* rows, cudaStream_t st);
// spec [B][R][pitch] ([re | im] per frame, nb bins each; frames 0 .. T - 1) -> mag, phase [B][nb][T]
void stft_magphase(const float* spec, int B, long R, int pitch, int nb, int T, float* mag, float* phase, cudaStream_t st);
// X [B][T + 1][pitch] = [mag cos(phase) | mag sin(phase)] of mag, phase [B][nb][T]; row T and channels >= 2 nb are zero
void istft_frames(const float* mag, const float* phase, int B, int nb, int T, int pitch, float* X, cudaStream_t st);
// out [B][(T - 1) hop] = y_b[i + n / 2] / ws[i + n / 2] (where ws > FLT_MIN) * (n / hop), y [B][(T + 1) hop]
void istft_finish(const float* y, const float* ws, int B, int T, int n, int hop, float* out, cudaStream_t st);

// LASS's input image img [B][Tp][W][4] = {s x + sh, x, 0, 0}, x = mag[b sb + t stt + f sf] for t < T, 0 for the padded
// rows T <= t < Tp
void lass_input(const float* mag, long sb, long stt, long sf, int B, int T, int Tp, int W, float s, float sh, float* img,
                cudaStream_t st);
// after_conv2 (wb: 32 weights, then the bias) over x [B][Tp][W][32], F.pad(., (0, 2)), crop to T, sigmoid -> mask [B][T][W + 2],
// logits (may be null) the same
void lass_head(const float* x, const float* wb, int B, int T, int Tp, int W, float* mask, float* logits, cudaStream_t st);

// wav2vec2's conv0 (1 -> C, k0 taps, stride s0, no bias) + GroupNorm(C, C, eps) + GELU over x [B][S] (T0 rows per
// sample) -> out [B][R][C], rows T0 .. T0 + zpad - 1 zero; two launches (statistics, then apply).  Workspaces: part
// [B][ceil(T0 / 128)][C] double2, stat [B][C] float2, cnt [B] int (zero on entry, zero again when the first launch ends).
// k0 <= 16, C <= 1024.
void w2v_stem(const float* x, long S, int B, int T0, int zpad, int C, const float* w0, int k0, int s0, const float* gamma,
              const float* beta, float eps, void* part, void* stat, int* cnt, float* out, long R, cudaStream_t st);

}  // namespace agpt
