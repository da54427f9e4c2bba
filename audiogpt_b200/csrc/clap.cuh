// Pieces shared by the two CLAP towers of the candidate scorer (clap.cu: the masked BERT text tower, clap_score.cu:
// the Cnn14 audio tower).
#pragma once
#include "common.cuh"
#include "tapconv.cuh"

namespace agpt {

// CLAP's Projection (wav_evaluation/models/clap.py:8-20) followed by the scorer's two L2 normalisations
struct ClapProjection {
  PackedConv lin1, lin2;
  DevBuf lng, lnb, e1, g1, e12, z;
  float eps = 1e-5f;
  // consumes linear1.weight, linear2.weight, layer_norm.weight, layer_norm.bias
  void load(WeightCursor& wc, int d_in, int d_out, float eps_);
  // x: rows of d_in floats at pitch in_pitch (device) -> out [rows][d_out] (device), unit rows
  void run(const float* x, int in_pitch, int rows, float* out, cudaStream_t st);
};

// out[r] = in[r] / |in[r]|, applied twice (in may equal out)
void clap_l2norm2(const float* in, float* out, int rows, int D, cudaStream_t st);

}  // namespace agpt
