// Pieces shared by the two CLAP towers of the candidate scorer (clap.cu: the masked BERT text tower, clap_score.cu:
// the Cnn14 audio tower), and the BERT trunk LASSNet's text encoder (lass.cu) and wav2vec2's encoder (w2v.cu) run.
#pragma once
#include "common.cuh"
#include "tapconv.cuh"
#include "models.h"

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

// BertLayer: BertSelfAttention (query / key / value packed into one [3H][H] GEMM), BertSelfOutput, BertIntermediate,
// BertOutput
struct ClapLayer {
  PackedConv qkv, attn_out, inter, out;
  DevBuf ln1g, ln1b, ln2g, ln2b;
};

// HF BertModel (embeddings + encoder layers) and CLAP's Projection (clap.cu)
struct ClapNet : Handle {
  agpt_clap_cfg cfg;
  DevBuf word, pos, types, elng, elnb;   // types: every token_type_embeddings row (encode reads row 0)
  std::vector<ClapLayer> layers;
  ClapProjection proj;                            // Projection weights (encode_cls also runs its L2 norms)
  DevBuf x, y, qkv, ctx, ffn, e1, g1, e12, kpm;   // work buffers, grown to the largest N * L seen

  // consumes the BertModel keys of embeddings.* and encoder.layer.* (the clap_param_shapes order) for cfg
  void load_bert(WeightCursor& wc);
  // consumes the embeddings LayerNorm and the encoder layers only (load_bert's tail; wav2vec2's encoder in w2v.cu)
  void load_trunk(WeightCursor& wc);
  void ensure_work(long rows);
  void encode(const int* ids, int N, int L, float* z, cudaStream_t st);
  // TextEncoder.forward of the scorer: BertModel(input_ids, token_type_ids, attention_mask)[0][:, 0] -> Projection,
  // then divided by its norm twice -> out [N][d_proj]
  void encode_cls(const int* ids, const int* type_ids, const int* mask, int N, int L, float* out, cudaStream_t st);
  // BertModel(input_ids, token_type_ids, attention_mask)[0] -> x [N * L][hidden] (padding keys masked out)
  void encode_hidden(const int* ids, const int* type_ids, const int* mask, int N, int L, cudaStream_t st);
  // embeddings LayerNorm (y -> x) and the encoder layers; x holds the last hidden state
  void trunk(int N, int L, const uint8_t* kpm_, cudaStream_t st);
};

// the Projection's exact GELU, out [n] = gelu_erf(in [n]), on a grid-stride grid of at most max_blocks blocks of 256
// (clap.cu).  n >= 1, max_blocks >= 1.
void clap_gelu(const float* in, float* out, long n, int max_blocks, cudaStream_t st);

// out[r] = in[r] / |in[r]|, applied twice (in may equal out)
void clap_l2norm2(const float* in, float* out, int rows, int D, cudaStream_t st);

}  // namespace agpt
