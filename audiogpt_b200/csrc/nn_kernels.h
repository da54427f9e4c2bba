// Host launchers of the non-contraction kernels (nn_kernels.cu).
#pragma once
#include <cuda_fp16.h>
#include "common.cuh"

namespace agpt {

void groupnorm(const float* x, float* y, const float* gamma, const float* beta, int N, int HW, int C, int G,
               float eps, bool silu, double* scratch, cudaStream_t st, __half* phi = nullptr, __half* plo = nullptr);
void groupnorm_ex(const float* x, float* y, const float* gamma, const float* beta, int N, int HW, int C, int G,
                  float eps, int act, const float* res, cudaStream_t st, __half* phi = nullptr, __half* plo = nullptr);
size_t groupnorm_scratch_doubles(int N, int C);
// phi / plo given: the result is written as fp16 hi/lo operand planes [rows][C] INSTEAD of the fp32 tensor y
void layernorm(const float* x, float* y, const float* gamma, const float* beta, long rows, int C, float eps,
               cudaStream_t st, __half* phi = nullptr, __half* plo = nullptr);
// kpm: optional key-padding mask [N][Lk] bytes (1 = padding key); a query whose keys are all padding gets zeros
void attention(const float* q, int q_pitch, const float* k, int k_pitch, const float* v, int v_pitch,
               float* o, int o_pitch, int N, int heads, int d, int Lq, int Lk, cudaStream_t st, const uint8_t* kpm = nullptr);
void transpose_pad(const float* in, int in_pitch, int rows, int cols, float* out, int rows_pad, cudaStream_t st);
void copy_pad_rows(const float* in, int in_pitch, int rows, int cols, float* out, int rows_pad, cudaStream_t st);
void softmax_rows(float* x, int pitch, long rows, int cols, float scale, cudaStream_t st);
// tensor-core version (attention_tc.cu); false = unsupported head dim / alignment
bool attention_tc(const float* q, int q_pitch, const float* k, int k_pitch, const float* v, int v_pitch,
                  float* o, int o_pitch, int N, int heads, int d, int Lq, int Lk, cudaStream_t st, const uint8_t* kpm = nullptr);
void attention_set_tc(int on);
bool attention_tc_enabled();   // 1 (default) wgmma kernel, 0 fp32 kernel, -1 environment (AGPT_ATTN_TC)
void timestep_embedding(float* out, const int* t_host, int N, int dim, cudaStream_t st);
void concat_channels(const float* a, int Ca, const float* b, int Cb, float* out, long rows, cudaStream_t st);
void upsample_nearest2(const float* in, float* out, int N, int H, int W, int C, cudaStream_t st);
// 2x2 average pool, stride 2, floor: out [N][H/2][W/2][C]  (AvgPool2d(2, 2))
void avgpool2(const float* in, float* out, int N, int H, int W, int C, cudaStream_t st);
// pad: rows / columns of zeros before the image (1: Conv2d padding=1; 0: the encoder's Downsample, pad after only)
void im2col_stride2(const float* in, float* col, int N, int H, int W, int C, int Ho, int Wo, int pad, cudaStream_t st);
void cf_to_cl_pad(const float* in, float* out, int N, int C, int Cpad, int HW, cudaStream_t st, int Nsrc = 0);
void timestep_embedding_dev(float* out, const int* t_dev, int rows, int dim, cudaStream_t st);
void select_row(const float* table, const int* step_dev, float* out, int ncols, cudaStream_t st);
void step_inc(int* step_dev, cudaStream_t st);
void ddim_update_tab(const float* x, const float* eps2, int single, const float* coef_dev, const int* step_dev, int B, long n,
                     float* x_prev, float* pred_x0, cudaStream_t st);
void conv_out_ddim(const float* hn, const float* w9c4, const float* bias4, float* x_io, float* pred_x0, const float* coef_dev,
                   const int* step_dev, int B, int H, int W, int C, int single, cudaStream_t st);
void ddim_update(const float* x, const float* eps2, int single, float cfg_scale, float a_t, float a_prev,
                 float sigma_t, float sqrt_om, const float* noise, float temperature, int B, long n,
                 float* x_prev, float* pred_x0, cudaStream_t st);

}  // namespace agpt
