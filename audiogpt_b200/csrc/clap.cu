// CLAP text encoder of Make-An-Audio on sm_90a: token ids -> BERT-base -> CLAP Projection -> the [N][L][d_proj]
// cross-attention context of the text-to-audio UNet.
// Reference: text_to_audio/Make_An_Audio/ldm/modules/encoders/modules.py:173-212 (FrozenCLAPEmbedder.encode),
// ldm/modules/encoders/CLAP/clap.py:8-20 (Projection), :42-46 (TextEncoder), and HF transformers' BertModel
// (BertEmbeddings, BertLayer: post-LN self-attention and GELU FFN; called without an attention mask, so padding
// positions are attended like any other).
// Every Linear is a tap-GEMM (tcconv5 on the tensor cores), self-attention is the unmasked attention kernel.
// The CLAP candidate scorer's text tower (wav_evaluation/models/CLAPWrapper.py:166-196, clap.py:42-53) runs the same
// BERT with token types and its attention mask (encode_cls: padding keys masked through the kernel's key-padding
// mask) and projects the [CLS] rows only.
#include "common.cuh"
#include "tapconv.cuh"
#include "nn_kernels.h"
#include "models.h"
#include "fs_layers.cuh"
#include "clap.cuh"

namespace agpt {

namespace {

// x[n][l] = (word[id] + type[0]) + position[l]  (BertEmbeddings' order of the adds); out-of-range ids are clamped so
// the table is never read out of bounds.  One block per row.
__global__ void clap_embed_kernel(const int* __restrict__ ids, const float* __restrict__ word, const float* __restrict__ pos,
                                  const float* __restrict__ type0, float* __restrict__ x, int L, int H, int vocab) {
  const long r = blockIdx.x;
  const int l = (int)(r % L);
  const int id = min(max(ids[r], 0), vocab - 1);
  const float* w = word + (long)id * H;
  const float* p = pos + (long)l * H;
  for (int c = threadIdx.x; c < H; c += blockDim.x) x[r * H + c] = __fadd_rn(__fadd_rn(w[c], type0[c]), p[c]);
}

// x[n][l] = (word[id] + type[type_id]) + position[l], kpm[n][l] = (attention_mask == 0): the scorer's tokenizer rows.
// Ids and type ids outside their tables are clamped.
__global__ void clap_embed_typed_kernel(const int* __restrict__ ids, const int* __restrict__ type_ids, const int* __restrict__ mask,
                                        const float* __restrict__ word, const float* __restrict__ pos, const float* __restrict__ types,
                                        float* __restrict__ x, uint8_t* __restrict__ kpm, int L, int H, int vocab, int ntypes) {
  const long r = blockIdx.x;
  const int l = (int)(r % L);
  const int id = min(max(ids[r], 0), vocab - 1);
  const int ty = min(max(type_ids[r], 0), ntypes - 1);
  const float* w = word + (long)id * H;
  const float* tt = types + (long)ty * H;
  const float* p = pos + (long)l * H;
  for (int c = threadIdx.x; c < H; c += blockDim.x) x[r * H + c] = __fadd_rn(__fadd_rn(w[c], tt[c]), p[c]);
  if (threadIdx.x == 0) kpm[r] = mask[r] == 0 ? 1 : 0;
}

// Projection's gelu(e1) into its own buffer: e1 itself is linear2's residual
__global__ void clap_gelu_kernel(const float* __restrict__ in, float* __restrict__ out, long n) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) out[i] = gelu_erf(in[i]);
}

// BertLayer: BertSelfAttention (query / key / value packed into one [3H][H] GEMM), BertSelfOutput, BertIntermediate,
// BertOutput
struct ClapLayer {
  PackedConv qkv, attn_out, inter, out;
  DevBuf ln1g, ln1b, ln2g, ln2b;
};

}  // namespace

struct ClapNet : Handle {
  agpt_clap_cfg cfg;
  DevBuf word, pos, types, elng, elnb;   // types: every token_type_embeddings row (encode reads row 0)
  std::vector<ClapLayer> layers;
  ClapProjection proj;                            // Projection weights (encode_cls also runs its L2 norms)
  DevBuf x, y, qkv, ctx, ffn, e1, g1, e12, kpm;   // work buffers, grown to the largest N * L seen

  void ensure_work(long rows) {
    const int H = cfg.hidden_size, I = cfg.intermediate_size;
    x.ensure(rows * H); y.ensure(rows * H); qkv.ensure(rows * 3 * H); ctx.ensure(rows * H); ffn.ensure(rows * I);
  }

  void encode(const int* ids, int N, int L, float* z, cudaStream_t st) {
    AGPT_CHECK(N >= 1 && L >= 1, "empty batch");
    AGPT_CHECK(L <= cfg.max_position_embeddings, "sequence longer than max_position_embeddings");
    const int H = cfg.hidden_size, D = cfg.d_proj;
    const long rows = (long)N * L;
    ensure_work(rows);
    e1.ensure(rows * D); g1.ensure(rows * D); e12.ensure(rows * D);
    clap_embed_kernel<<<(unsigned)rows, 128, 0, st>>>(ids, word.p, pos.p, types.p, y.p, L, H, cfg.vocab_size);
    count_launch(1);
    trunk(N, L, nullptr, st);
    // Projection: LayerNorm(e1 + linear2(gelu(e1))), both Linears without bias
    fs_conv(proj.lin1, x.p, H, e1.p, D, 1, (int)rows, EPI_BIAS, st);
    clap_gelu_kernel<<<(unsigned)std::min<long>(cdivl(rows * D, 256), 2368), 256, 0, st>>>(e1.p, g1.p, rows * D);
    count_launch(1);
    fs_conv(proj.lin2, g1.p, D, e12.p, D, 1, (int)rows, EPI_RES, st, e1.p);
    layernorm(e12.p, z, proj.lng.p, proj.lnb.p, rows, D, cfg.proj_layer_norm_eps, st);
    AGPT_CUDA(cudaGetLastError());
  }

  // TextEncoder.forward of the scorer: BertModel(input_ids, token_type_ids, attention_mask)[0][:, 0] -> Projection,
  // then divided by its norm twice -> out [N][d_proj]
  void encode_cls(const int* ids, const int* type_ids, const int* mask, int N, int L, float* out, cudaStream_t st) {
    AGPT_CHECK(N >= 1 && L >= 1, "empty batch");
    AGPT_CHECK(L <= cfg.max_position_embeddings, "sequence longer than max_position_embeddings");
    const int H = cfg.hidden_size;
    const long rows = (long)N * L;
    ensure_work(rows);
    uint8_t* m = reinterpret_cast<uint8_t*>(kpm.ensure(cdivl(rows, 4)));
    clap_embed_typed_kernel<<<(unsigned)rows, 128, 0, st>>>(ids, type_ids, mask, word.p, pos.p, types.p, y.p, m, L, H,
                                                            cfg.vocab_size, cfg.type_vocab_size);
    count_launch(1);
    trunk(N, L, m, st);
    proj.run(x.p, L * H, N, out, st);          // the [CLS] row of sequence n is row n * L
    AGPT_CUDA(cudaGetLastError());
  }

  // embeddings LayerNorm (y -> x) and the encoder layers; x holds the last hidden state
  void trunk(int N, int L, const uint8_t* kpm_, cudaStream_t st) {
    const int H = cfg.hidden_size, I = cfg.intermediate_size;
    const long rows = (long)N * L;
    layernorm(y.p, x.p, elng.p, elnb.p, rows, H, cfg.layer_norm_eps, st);
    for (auto& Ly : layers) {
      fs_conv(Ly.qkv, x.p, H, qkv.p, 3 * H, 1, (int)rows, EPI_BIAS, st);
      attention(qkv.p, 3 * H, qkv.p + H, 3 * H, qkv.p + 2 * H, 3 * H, ctx.p, H, N, cfg.num_heads, H / cfg.num_heads, L, L, st,
                kpm_);
      fs_conv(Ly.attn_out, ctx.p, H, y.p, H, 1, (int)rows, EPI_RES, st, x.p);          // dense + bias + residual
      layernorm(y.p, x.p, Ly.ln1g.p, Ly.ln1b.p, rows, H, cfg.layer_norm_eps, st);
      fs_conv(Ly.inter, x.p, H, ffn.p, I, 1, (int)rows, EPI_GELU_SCALED, st, nullptr, 1.f);   // exact GELU
      fs_conv(Ly.out, ffn.p, I, y.p, H, 1, (int)rows, EPI_RES, st, x.p);
      layernorm(y.p, x.p, Ly.ln2g.p, Ly.ln2b.p, rows, H, cfg.layer_norm_eps, st);
    }
  }
};

Handle* clap_create(const agpt_clap_cfg* cfg, const float* const* W, int nW, int device) {
  DeviceGuard dg_(device);
  const int H = cfg->hidden_size, I = cfg->intermediate_size, D = cfg->d_proj;
  AGPT_CHECK(cfg->vocab_size >= 1 && cfg->max_position_embeddings >= 1 && cfg->type_vocab_size >= 1 && cfg->num_layers >= 0 &&
                 cfg->num_heads >= 1 && H % cfg->num_heads == 0 && H % 4 == 0 && I % 4 == 0 && D % 4 == 0 && H > 0 && I > 0 &&
                 D > 0 && cfg->layer_norm_eps > 0.f && cfg->proj_layer_norm_eps > 0.f,
             "bad CLAP config");
  std::unique_ptr<ClapNet> h(new ClapNet());
  h->magic = kMagicClap; h->device = device; h->cfg = *cfg;
  WeightCursor wc{W, nW};
  h->word.upload(wc.next(), (size_t)cfg->vocab_size * H);
  h->pos.upload(wc.next(), (size_t)cfg->max_position_embeddings * H);
  h->types.upload(wc.next(), (size_t)cfg->type_vocab_size * H);
  { auto g = wc.next(); auto b = wc.next(); h->elng.upload(g, H); h->elnb.upload(b, H); }
  h->layers.resize(cfg->num_layers);
  for (auto& Ly : h->layers) {
    std::vector<float> w((size_t)3 * H * H), b((size_t)3 * H);
    for (int j = 0; j < 3; ++j) {                                 // query, key, value -> [Q | K | V]
      memcpy(w.data() + (size_t)j * H * H, wc.next(), sizeof(float) * H * H);
      memcpy(b.data() + (size_t)j * H, wc.next(), sizeof(float) * H);
    }
    pack_conv(Ly.qkv, w.data(), b.data(), 3 * H, H, 1, false);
    { auto ww = wc.next(); auto bb = wc.next(); pack_conv(Ly.attn_out, ww, bb, H, H, 1, false); }
    { auto g = wc.next(); auto bb = wc.next(); Ly.ln1g.upload(g, H); Ly.ln1b.upload(bb, H); }
    { auto ww = wc.next(); auto bb = wc.next(); pack_conv(Ly.inter, ww, bb, I, H, 1, false); }
    { auto ww = wc.next(); auto bb = wc.next(); pack_conv(Ly.out, ww, bb, H, I, 1, false); }
    { auto g = wc.next(); auto bb = wc.next(); Ly.ln2g.upload(g, H); Ly.ln2b.upload(bb, H); }
  }
  wc.next(); wc.next();                                           // pooler.dense weight / bias: encode never uses them
  h->proj.load(wc, H, D, cfg->proj_layer_norm_eps);
  wc.done();
  return h.release();
}

void clap_encode(Handle* hh, const int* ids, int N, int L, float* z, cudaStream_t st) {
  auto* h = static_cast<ClapNet*>(hh);
  DeviceGuard dg_(h->device);
  h->encode(ids, N, L, z, st);
}

void clap_encode_cls(Handle* hh, const int* ids, const int* type_ids, const int* mask, int N, int L, float* out, cudaStream_t st) {
  auto* h = static_cast<ClapNet*>(hh);
  DeviceGuard dg_(h->device);
  h->encode_cls(ids, type_ids, mask, N, L, out, st);
}

}  // namespace agpt
