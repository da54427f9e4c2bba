// Launchers of the hand-written kernels of the analysis models outside the GEMMs: LASSNet's FiLM ResUNet (lass.cu:
// LassNet::run_block, LassNet::film_vec, LassNet::up), RaDur's detection tail (tsd.cu: TsdNet::encode, pass, forward),
// the BERT embeddings (clap.cu: ClapNet::encode, encode_hidden) and the emotion encoder's tail (emotion.cu), shared by
// the drivers and the conformance probe (microbench.cu: agpt_an_probe).  Each one launches its kernel with the
// production grid and block size and counts the launch; none synchronises.  Each one checks the preconditions its
// kernel's indexing relies on and throws before launching when they fail.  (The CLAP Projection's GELU, clap_gelu, is
// declared in clap.cuh.)
#pragma once
#include <cstdint>
#include "common.cuh"

namespace agpt {

// ---- LASSNet (lass.cu).  Rows are channels-last, C % 4 == 0 (float4 rows).
// a [rows][C] = fmaf(x, s[c], t[c]); r (null = none) [rows][C] = x + vec[b][vec_off + c], b = row / rows_per_sample, at
// a pitch of vec_len floats per sample.  rows, rows_per_sample >= 1; with r: 0 <= vec_off, vec_off + C <= vec_len, and
// vec_off, vec_len multiples of 4.
void lass_affine(const float* x, const float* s, const float* t, float* a, float* r, const float* vec, int vec_len, int vec_off,
                 long rows, long rows_per_sample, int C, cudaStream_t st);
// col [B][h][w + 1][4][C] = relu(fmaf(y[b][m + dh][n + dw][c], s[c], t[c])) for the taps (dh, dw) = (0, 0), (0, -1),
// (-1, 0), (-1, -1) of the transposed conv's 2 x 2 neighbourhood, zero outside the h x w map.  B, h, w >= 1.
void lass_upcol(const float* y, const float* s, const float* t, int B, int h, int w, int C, float* col, cudaStream_t st);
// cat [B][2h][2w + 1][2C]: channels < C from phase (r & 1, col & 1) of up [B][h][w + 1][4][C] at (r / 2, col / 2),
// channels >= C from skip [B][2h][2w + 1][C].  B, h, w >= 1.
void lass_shuffle(const float* up, const float* skip, int B, int h, int w, int C, float* cat, cudaStream_t st);
// The FiLM second Linears, one warp per (sample, job j < nj): film(o) = relu(w2[woff[o]:] . hid[b][hoff[o]:] (nin[o]
// terms) + b2[o]); vec[b][dst[j]] = fmaf(alpha[j], film(ja[j]), beta[j]) (+ film(jb[j]) when jb[j] >= 0).  Every table is
// a device array.
struct FilmJobs { const int *woff, *hoff, *nin, *dst, *ja, *jb; const float *b2, *alpha, *beta; };
void lass_film(const float* hid, int hid_len, const float* w2, const FilmJobs& J, int nj, int B, float* vec, int vec_len,
               cudaStream_t st);

// ---- RaDur (tsd.cu)
// img [n][4] = (mel[i], 0, 0, 0).  n >= 1.
void tsd_pad4(const float* mel, float* img, long n, cudaStream_t st);
// Fusion's product and pool: out [B][Td][C] = mean_q e1[b][j n + q] f2[b][t][j n + q], q < n.  B, Td, C, n >= 1.
void tsd_fuse(const float* f2, const float* e1, int B, int Td, int C, int n, float* out, cudaStream_t st);
// The reference embedding from E [B][Trr][128]: m = mean_t E; att_pool 0: emb = m; att_pool 1: q = qw m + qb, scores
// (kw^T q) . E_t / 11.3 + q . kb / 11.3, softmax over t into scratch [B][Trr] (device), emb = sum_t p_t E_t.  Trr >= 1;
// scratch is required when att_pool.
void tsd_refemb(const float* E, int B, int Trr, int att_pool, const float* qw, const float* qb, const float* kw, const float* kb,
                float* scratch, float* emb, cudaStream_t st);
// detection.fc -> outputlayer folded (w [O][1024], bias [O]) and the softmax over O: h [rows][1024] -> p [rows][O].
// 1 <= O <= 16, rows >= 1.
void tsd_head(const float* h, const float* w, const float* bias, int O, long rows, float* p, cudaStream_t st);
// fin = p1 (1 - wmix[b]) + wmix[b] p2 (p2 null: fin = p1), p1 / p2 [B][Td][O]; decision [B][Td] = fin[..., 0]; up
// [B][T][O] = interpolate(fin, T, 'linear', align_corners=False).  B, Td, T >= 1, 1 <= O <= 16.
void tsd_mix_interp(const float* p1, const float* p2, const float* wmix, int B, int Td, int T, int O, float* decision, float* up,
                    cudaStream_t st);

// ---- the BERT embeddings (clap.cu): x [N][L][H] = (word[id] + type) + pos[l], ids clamped to [0, vocab - 1].
// clap_embed: type = type0 [H] (token type 0).  clap_embed_typed: type = types[type_id] (type ids clamped to
// [0, ntypes - 1]) and kpm [N][L] = (mask == 0).  N, L, H, vocab, ntypes >= 1.
void clap_embed(const int* ids, const float* word, const float* pos, const float* type0, float* x, int N, int L, int H, int vocab,
                cudaStream_t st);
void clap_embed_typed(const int* ids, const int* type_ids, const int* mask, const float* word, const float* pos,
                      const float* types, float* x, uint8_t* kpm, int N, int L, int H, int vocab, int ntypes, cudaStream_t st);

// ---- the emotion encoder's tail (emotion.cu), rows of 256
// embed [256] = raw / ||raw||, raw = mean of h [N][256].  N >= 1.
void emo_mean_norm(const float* h, int N, float* embed, cudaStream_t st);
// out [N][E] = e / ||e||, e = relu(W h + b), W [E][256].  N, E >= 1, and E floats of dynamic shared memory next to the
// kernel's static 288 fit in 48 KB.
void emo_linear_norm(const float* h, const float* W, const float* bias, int N, int E, float* out, cudaStream_t st);

}  // namespace agpt
