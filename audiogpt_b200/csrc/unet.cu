// Make-An-Audio UNet (ResBlock + SpatialTransformer or AttentionBlock) and the DDIM loop on sm_90a.
// Reference: ldm/modules/diffusionmodules/openaimodel.py:443-744 (ctor + forward),
//            :255-275 (ResBlock._forward, with the up/down variants), :91-160 (Up/Downsample),
//            :278-406 (AttentionBlock, QKVAttentionLegacy / QKVAttention);
//            ldm/modules/attention.py:37-64,152-261; ldm/models/diffusion/ddim.py:117-225.
// Activations are channels-last token rows [N][H*W][C]; every contraction is a tapconv.
// Parity: tests/test_ldm_gpu.py against oracle/ldm_ref.py and tests/golden/ldm_*.npz.
#include "common.cuh"
#include "tapconv.cuh"
#include "nn_kernels.h"
#include "models.h"

namespace agpt {

struct ResW {
  int cin = 0, cout = 0;
  DevBuf gn1_g, gn1_b, gn2_g, gn2_b;
  PackedConv conv1, conv2, skip;
  bool has_skip = false;
  int emb_off = 0;  // channel offset inside the batched emb projection
  int updown = 0;   // resblock_updown: 1 down (2x2 average pool), 2 up (nearest x2), applied to h after GN+SiLU and to x
};

// AttentionBlock: GN (no SiLU) -> qkv 1x1 -> self-attention over H*W tokens -> proj_out 1x1 + x
struct AttnW {
  int ch = 0, heads = 0, dhead = 0;
  DevBuf gn_g, gn_b;
  PackedConv qkv, proj_out;   // qkv rows in [Q | K | V] order, heads outermost inside each
};

struct XfBlockW {
  DevBuf ln1_g, ln1_b, ln2_g, ln2_b, ln3_g, ln3_b;
  PackedConv qkv1, out1, q2, out2, ff1, ff2;
  int kv_off = 0;  // channel offset of this block's [K|V] inside the hoisted context projection
};

struct StW {
  int ch = 0, heads = 0, dhead = 0, inner = 0;
  DevBuf gn_g, gn_b;
  PackedConv proj_in, proj_out;
  std::vector<XfBlockW> blocks;
};

enum LayerKind { L_CONV_IN, L_RES, L_ST, L_ATTN, L_DOWN, L_UP };
struct Layer {
  LayerKind kind;
  int idx;   // index into res / st / attn / misc conv vectors
  int ch;    // channels (down/up)
};
struct Block { std::vector<Layer> layers; };

struct Unet : Handle {
  agpt_unet_cfg cfg;
  int mc = 0, temb = 0, ctx_dim = 0, final_ch = 0;
  PackedConv time0, time2, emb_all, ctx_kv_all, conv_in, conv_down, conv_up, conv_out;
  std::vector<PackedConv> down_convs, up_convs;
  DevBuf out_gn_g, out_gn_b;
  DevBuf out_w9c4, out_b4;      // the `out` conv as [9][C][4] fp32 for the fused conv_out + CFG + DDIM-update kernel
  std::vector<ResW> res;
  std::vector<StW> st;
  std::vector<AttnW> attn;
  std::vector<Block> in_blocks, out_blocks;
  Block mid;
  int emb_total = 0, kv_total = 0, cin_pad = 0;

  // per-call state
  int ctxN = 0, ctxS = 0;
  DevBuf ctx_kv;                // hoisted cross-attention K / V of the context
  int catN = 0, catH = 0, catW = 0;
  DevBuf cat_cl;                // concat conditioning [N][H*W][cin_pad - out_channels], zero-padded channels
  DevBuf arena;
  size_t arena_off = 0, arena_cap = 0;
  DevBuf ddim_eps, ddim_x, ddim_p0;
  // denoising-loop state: per-step tables on the device, a device step counter, one captured step (CUDA graph)
  DevBuf emb_table, emb_cur, coef_table, tsteps_dev, step_ctr;
  int emb_gstride = 0;            // row stride of the per-sample ResBlock embedding vectors (0: all samples share one row)
  cudaGraphExec_t step_graph = nullptr;
  cudaStream_t cap_stream = nullptr;
  struct GraphKey {
    int N = 0, H = 0, W = 0, single = 0;
    const void *arena = nullptr, *ctx = nullptr, *x = nullptr, *cat = nullptr;
    int ctxS = 0;
  } gkey;
  long launches_per_step = 0;

  ~Unet() override {
    if (step_graph) cudaGraphExecDestroy(step_graph);
    if (cap_stream) cudaStreamDestroy(cap_stream);
  }

  float* alloc(size_t n) {
    n = (n + 63) & ~(size_t)63;
    AGPT_CHECK(arena_off + n <= arena_cap, "UNet activation arena exhausted");
    float* p = arena.p + arena_off;
    arena_off += n;
    return p;
  }

  void set_context(const float* ctx, int N, int S, cudaStream_t s) {
    ctxN = N; ctxS = S;
    ctx_kv.ensure((size_t)N * S * kv_total);
    TapConvParams P = tapconv_params(ctx_kv_all, 1, N * S, 0, 1);
    P.in = ctx; P.in_gstride = 0; P.in_pitch = ctx_dim;
    P.out = ctx_kv.p; P.out_gstride = 0; P.out_pitch = kv_total;
    P.epi = EPI_BIAS;
    tapconv_launch(P, s);
  }

  // the step-invariant conditioning channels of the concat loop, in the kernel layout once per sampling call
  void set_concat(const float* c, int N, int C, int H, int W, cudaStream_t s) {
    const int oc = cfg.out_channels;
    AGPT_CHECK(C == cfg.in_channels - oc && C >= 1, "concat conditioning must have in_channels - out_channels channels");
    AGPT_CHECK(oc % 4 == 0, "concat conditioning needs out_channels to be a multiple of 4");
    AGPT_CHECK(N >= 1 && H >= 1 && W >= 1, "empty concat conditioning");
    cat_cl.ensure((size_t)N * H * W * (cin_pad - oc));
    cf_to_cl_pad(c, cat_cl.p, N, C, cin_pad - oc, H * W, s);
    catN = N; catH = H; catW = W;
  }

  // ---- building blocks --------------------------------------------------------------
  void conv3x3(const PackedConv& pc, const float* in, float* out, int N, int H, int W, int epi,
               const float* res_, const float* evec, int evec_stride, cudaStream_t s) {
    TapConvParams P = tapconv_params(pc, N, H * W, W, 1);
    P.in = in; P.in_gstride = (long)H * W * pc.Cin; P.in_pitch = pc.Cin;
    P.out = out; P.out_gstride = (long)H * W * pc.Cout; P.out_pitch = pc.Cout;
    P.epi = epi;
    P.res = res_; P.res_gstride = (long)H * W * pc.Cout; P.res_pitch = pc.Cout;
    P.evec = evec; P.evec_gstride = evec_stride;
    tapconv_launch(P, s);
  }
  void linear(const PackedConv& pc, const float* in, int in_pitch, float* out, int out_pitch, long rows, int epi,
              const float* res_, int res_pitch, cudaStream_t s, int pro = PRO_NONE) {
    TapConvParams P = tapconv_params(pc, 1, (int)rows, 0, 1);
    P.in = in; P.in_pitch = in_pitch;
    P.out = out; P.out_pitch = out_pitch;
    P.epi = epi; P.pro = pro;
    P.res = res_; P.res_pitch = res_pitch;
    tapconv_launch(P, s);
  }

  // H / W are updated to the output resolution of an up / down ResBlock
  float* run_res(const ResW& r, const float* x, const float* emb_out, int N, int& H, int& W, cudaStream_t s) {
    float* h1 = alloc((size_t)N * H * W * r.cin);
    groupnorm(x, h1, r.gn1_g.p, r.gn1_b.p, N, H * W, r.cin, 32, 1e-5f, true, nullptr, s);
    if (r.updown) {   // openaimodel.py:256-261: h_upd(in_rest(x)), x_upd(x), then in_conv at the new resolution
      const bool down = r.updown == 1;
      const int Ho = down ? H / 2 : 2 * H, Wo = down ? W / 2 : 2 * W;
      float* hr = alloc((size_t)N * Ho * Wo * r.cin);
      float* xr = alloc((size_t)N * Ho * Wo * r.cin);
      if (down) { avgpool2(h1, hr, N, H, W, r.cin, s); avgpool2(x, xr, N, H, W, r.cin, s); }
      else { upsample_nearest2(h1, hr, N, H, W, r.cin, s); upsample_nearest2(x, xr, N, H, W, r.cin, s); }
      h1 = hr; x = xr; H = Ho; W = Wo;
    }
    const int HW = H * W;
    float* h2 = alloc((size_t)N * HW * r.cout);
    conv3x3(r.conv1, h1, h2, N, H, W, EPI_ADDVEC, nullptr, emb_out + r.emb_off, emb_gstride, s);
    float* h3 = alloc((size_t)N * HW * r.cout);
    groupnorm(h2, h3, r.gn2_g.p, r.gn2_b.p, N, HW, r.cout, 32, 1e-5f, true, nullptr, s);
    const float* sk = x;
    if (r.has_skip) {
      float* skb = alloc((size_t)N * HW * r.cout);
      linear(r.skip, x, r.cin, skb, r.cout, (long)N * HW, EPI_BIAS, nullptr, 0, s);
      sk = skb;
    }
    float* out = alloc((size_t)N * HW * r.cout);
    conv3x3(r.conv2, h3, out, N, H, W, EPI_RES, sk, nullptr, 0, s);
    return out;
  }

  float* run_st(const StW& t, const float* x, int N, int H, int W, cudaStream_t s) {
    const int HW = H * W;
    const long rows = (long)N * HW;
    const int C = t.inner;
    float* xn = alloc(rows * t.ch);
    groupnorm(x, xn, t.gn_g.p, t.gn_b.p, N, HW, t.ch, 32, 1e-6f, false, nullptr, s);
    float* h = alloc(rows * C);
    linear(t.proj_in, xn, t.ch, h, C, rows, EPI_BIAS, nullptr, 0, s);
    float* a = alloc(rows * C);
    float* qkv = alloc(rows * 3 * C);
    float* att = alloc(rows * C);
    float* ff = alloc(rows * 4 * C);
    for (const XfBlockW& b : t.blocks) {
      // self-attention
      layernorm(h, a, b.ln1_g.p, b.ln1_b.p, rows, C, 1e-5f, s);
      linear(b.qkv1, a, C, qkv, 3 * C, rows, EPI_BIAS, nullptr, 0, s);
      attention(qkv, 3 * C, qkv + C, 3 * C, qkv + 2 * C, 3 * C, att, C, N, t.heads, t.dhead, HW, HW, s);
      float* h2 = alloc(rows * C);
      linear(b.out1, att, C, h2, C, rows, EPI_RES, h, C, s);
      // cross-attention on the hoisted K/V of the context
      AGPT_CHECK(ctxN == N, "context batch (agpt_unet_set_context) differs from the UNet batch");
      layernorm(h2, a, b.ln2_g.p, b.ln2_b.p, rows, C, 1e-5f, s);
      linear(b.q2, a, C, qkv, C, rows, EPI_BIAS, nullptr, 0, s);
      attention(qkv, C, ctx_kv.p + b.kv_off, kv_total, ctx_kv.p + b.kv_off + C, kv_total, att, C, N, t.heads, t.dhead,
                HW, ctxS, s);
      float* h3 = alloc(rows * C);
      linear(b.out2, att, C, h3, C, rows, EPI_RES, h2, C, s);
      // GEGLU feed-forward
      layernorm(h3, a, b.ln3_g.p, b.ln3_b.p, rows, C, 1e-5f, s);
      linear(b.ff1, a, C, ff, 4 * C, rows, EPI_GEGLU, nullptr, 0, s);
      float* h4 = alloc(rows * C);
      linear(b.ff2, ff, 4 * C, h4, C, rows, EPI_RES, h3, C, s);
      h = h4;
    }
    float* out = alloc(rows * t.ch);
    linear(t.proj_out, h, C, out, t.ch, rows, EPI_RES, x, t.ch, s);
    return out;
  }

  // AttentionBlock._forward (openaimodel.py:318-324); the d^-1/4 scale of q and of k is applied once as d^-1/2
  float* run_attn(const AttnW& a, const float* x, int N, int H, int W, cudaStream_t s) {
    const int HW = H * W, C = a.ch;
    const long rows = (long)N * HW;
    float* xn = alloc(rows * C);
    groupnorm(x, xn, a.gn_g.p, a.gn_b.p, N, HW, C, 32, 1e-5f, false, nullptr, s);
    float* qkv = alloc(rows * 3 * C);
    linear(a.qkv, xn, C, qkv, 3 * C, rows, EPI_BIAS, nullptr, 0, s);
    float* att = alloc(rows * C);
    attention(qkv, 3 * C, qkv + C, 3 * C, qkv + 2 * C, 3 * C, att, C, N, a.heads, a.dhead, HW, HW, s);
    float* out = alloc(rows * C);
    linear(a.proj_out, att, C, out, C, rows, EPI_RES, x, C, s);
    return out;
  }

  struct Act { float* p; int C, H, W; };

  Act run_block(const Block& blk, Act a, const float* emb_out, int N, cudaStream_t s) {
    for (const Layer& l : blk.layers) {
      switch (l.kind) {
        case L_CONV_IN: {
          float* o = alloc((size_t)N * a.H * a.W * mc);
          conv3x3(conv_in, a.p, o, N, a.H, a.W, EPI_BIAS, nullptr, nullptr, 0, s);
          a = {o, mc, a.H, a.W};
          break;
        }
        case L_RES: {
          const ResW& r = res[l.idx];
          AGPT_CHECK(a.C == r.cin, "ResBlock input channels");
          int H = a.H, W = a.W;
          float* o = run_res(r, a.p, emb_out, N, H, W, s);
          a = {o, r.cout, H, W};
          break;
        }
        case L_ST:
          a = {run_st(st[l.idx], a.p, N, a.H, a.W, s), a.C, a.H, a.W};
          break;
        case L_ATTN:
          a = {run_attn(attn[l.idx], a.p, N, a.H, a.W, s), a.C, a.H, a.W};
          break;
        case L_DOWN: {
          const int Ho = (a.H - 1) / 2 + 1, Wo = (a.W - 1) / 2 + 1;
          float* col = alloc((size_t)N * Ho * Wo * 9 * a.C);
          im2col_stride2(a.p, col, N, a.H, a.W, a.C, Ho, Wo, 1, s);
          float* o = alloc((size_t)N * Ho * Wo * a.C);
          linear(down_convs[l.idx], col, 9 * a.C, o, a.C, (long)N * Ho * Wo, EPI_BIAS, nullptr, 0, s);
          a = {o, a.C, Ho, Wo};
          break;
        }
        case L_UP: {
          float* up = alloc((size_t)N * 4 * a.H * a.W * a.C);
          upsample_nearest2(a.p, up, N, a.H, a.W, a.C, s);
          float* o = alloc((size_t)N * 4 * a.H * a.W * a.C);
          conv3x3(up_convs[l.idx], up, o, N, 2 * a.H, 2 * a.W, EPI_BIAS, nullptr, nullptr, 0, s);
          a = {o, a.C, 2 * a.H, 2 * a.W};
          break;
        }
      }
    }
    return a;
  }

  size_t arena_need(int N, int H, int W) const {
    // generous upper bound: every tensor of a forward lives in the bump arena
    size_t per_res = 0, per_st = 0;
    const size_t hw = (size_t)H * W;
    size_t maxc = 0;
    for (auto& r : res) maxc = std::max(maxc, (size_t)std::max(r.cin, r.cout));
    per_res = 5 * hw * maxc;
    per_st = 30 * hw * maxc;
    const size_t nblocks = in_blocks.size() + out_blocks.size() + 1;
    return (size_t)N * (nblocks * (2 * per_res + per_st + 3 * hw * maxc * 3)) + (1 << 20);
  }

  // time-embedding MLP + all ResBlock emb projections as ONE GEMM over `rows` timesteps (openaimodel.py:725-726,264):
  // te [rows][mc] -> out [rows][emb_total].  Scratch comes from the arena (call before the blocks).
  void embed_rows(const float* te, int rows, float* out, cudaStream_t s) {
    float* e1 = alloc((size_t)rows * temb);
    linear(time0, te, mc, e1, temb, rows, EPI_SILU, nullptr, 0, s);
    float* emb = alloc((size_t)rows * temb);
    linear(time2, e1, temb, emb, temb, rows, EPI_BIAS, nullptr, 0, s);
    linear(emb_all, emb, temb, out, emb_total, rows, EPI_BIAS, nullptr, 0, s, PRO_SILU);
  }

  void prepare(int N, int H, int W) {
    AGPT_CHECK(N >= 1 && N <= 256 && H >= 1 && W >= 1, "bad UNet input shape");
    const size_t need = arena_need(N, H, W);
    if (need > arena_cap) { arena.ensure(need); arena_cap = need; }
  }

  // everything after the embedding: x [Nsrc][C][H][W] (sample n reads n % Nsrc) -> eps [N][Cout][H][W]
  // eps == nullptr selects the FUSED tail of the sampling loop: out-conv + guidance + DDIM update in one kernel
  // (conv_out_ddim: x_io = ddim_x updated in place, coefficients from coef_table[*step_ctr])
  // cat != nullptr: x holds only the out_channels latent; the conditioning channels come from cat [N][H*W][..]
  void forward_core(const float* x, int Nsrc, const float* emb_out, int N, int H, int W, float* eps, cudaStream_t s,
                    const float* cat = nullptr) {
    float* x_cl = alloc((size_t)N * H * W * cin_pad);
    if (cat) {
      const int oc = cfg.out_channels;
      float* lat = alloc((size_t)N * H * W * oc);
      cf_to_cl_pad(x, lat, N, oc, oc, H * W, s, Nsrc);
      concat_channels(lat, oc, cat, cin_pad - oc, x_cl, (long)N * H * W, s);
    } else {
      cf_to_cl_pad(x, x_cl, N, cfg.in_channels, cin_pad, H * W, s, Nsrc);
    }
    Act a{x_cl, cin_pad, H, W};
    std::vector<Act> hs;
    for (const Block& b : in_blocks) { a = run_block(b, a, emb_out, N, s); hs.push_back(a); }
    a = run_block(mid, a, emb_out, N, s);
    for (const Block& b : out_blocks) {
      const Act sk = hs.back(); hs.pop_back();
      AGPT_CHECK(sk.H == a.H && sk.W == a.W, "skip/upsample spatial mismatch (H and W must be divisible by 2^(levels-1))");
      float* cat = alloc((size_t)N * a.H * a.W * (a.C + sk.C));
      concat_channels(a.p, a.C, sk.p, sk.C, cat, (long)N * a.H * a.W, s);
      a = run_block(b, Act{cat, a.C + sk.C, a.H, a.W}, emb_out, N, s);
    }
    float* hn = alloc((size_t)N * a.H * a.W * a.C);
    groupnorm(a.p, hn, out_gn_g.p, out_gn_b.p, N, a.H * a.W, a.C, 32, 1e-5f, true, nullptr, s);
    if (!eps) {
      conv_out_ddim(hn, out_w9c4.p, out_b4.p, ddim_x.p, ddim_p0.p, coef_table.p, reinterpret_cast<const int*>(step_ctr.p),
                    Nsrc, a.H, a.W, a.C, N == Nsrc ? 1 : 0, s);
      return;
    }
    {
      TapConvParams P = tapconv_params(conv_out, N, a.H * a.W, a.W, 1);
      P.in = hn; P.in_gstride = (long)a.H * a.W * a.C; P.in_pitch = a.C;
      P.out = eps; P.out_gstride = (long)cfg.out_channels * a.H * a.W; P.out_pitch = 0;
      P.epi = EPI_STORE_CF;
      tapconv_launch(P, s);
    }
  }

  void forward(const float* x, const int* t_host, int N, int H, int W, float* eps, cudaStream_t s) {
    prepare(N, H, W);
    arena_off = 0;
    float* te = alloc((size_t)N * mc);
    timestep_embedding(te, t_host, N, mc, s);
    float* emb_out = alloc((size_t)N * emb_total);
    embed_rows(te, N, emb_out, s);
    emb_gstride = emb_total;
    forward_core(x, N, emb_out, N, H, W, eps, s);
  }

  // One DDIM step of the on-device loop: everything step-dependent comes from device tables indexed by step_ctr,
  // so the launch sequence is identical for every step (capturable once, replayed S - 1 times).
  void ddim_step(int B, int N, int H, int W, long n, const float* cat, cudaStream_t s) {
    arena_off = 0;
    int* ctr = reinterpret_cast<int*>(step_ctr.p);
    select_row(emb_table.p, ctr, emb_cur.p, emb_total, s);
    emb_gstride = 0;
    if (out_w9c4.p) {
      forward_core(ddim_x.p, B, emb_cur.p, N, H, W, nullptr, s, cat);      // ... -> GN -> [out conv + CFG + x_prev update]
    } else {
      forward_core(ddim_x.p, B, emb_cur.p, N, H, W, ddim_eps.p, s, cat);
      ddim_update_tab(ddim_x.p, ddim_eps.p, N == B ? 1 : 0, coef_table.p, ctr, B, n, ddim_x.p, ddim_p0.p, s);
    }
    step_inc(ctr, s);
  }
};

Handle* unet_create(const agpt_unet_cfg* cfg, const float* const* W, int nW, int device) {
  DeviceGuard dg_(device);
  const int mc = cfg->model_channels, temb = 4 * mc, ctx = cfg->context_dim, depth = cfg->transformer_depth;
  AGPT_CHECK(mc % 32 == 0, "model_channels must be a multiple of 32 (GroupNorm32)");
  AGPT_CHECK(cfg->num_levels >= 1 && cfg->num_levels <= AGPT_MAX_LEVELS, "levels");
  std::unique_ptr<Unet> u(new Unet());
  u->magic = kMagicUnet; u->device = device; u->cfg = *cfg;
  u->mc = mc; u->temb = temb; u->ctx_dim = ctx;
  WeightCursor wc{W, nW};

  { auto w = wc.next(); auto b = wc.next(); pack_conv(u->time0, w, b, temb, mc, 1, false); }
  { auto w = wc.next(); auto b = wc.next(); pack_conv(u->time2, w, b, temb, temb, 1, false); }

  std::vector<float> embw, embb, kvw;   // batched projections, filled while walking the blocks
  int emb_off = 0, kv_off = 0;

  auto heads_for = [&](int ch, int& nh, int& dh) {
    if (cfg->num_head_channels == -1) { nh = cfg->num_heads; dh = ch / nh; }
    else { nh = ch / cfg->num_head_channels; dh = cfg->num_head_channels; }
  };

  auto make_res = [&](int cin, int cout, int updown = 0) -> int {
    u->res.emplace_back();
    ResW& r = u->res.back();
    r.cin = cin; r.cout = cout; r.updown = updown;
    AGPT_CHECK(cin % 32 == 0 && cout % 32 == 0, "ResBlock channels must be multiples of 32");
    { auto g = wc.next(); auto b = wc.next(); r.gn1_g.upload(g, cin); r.gn1_b.upload(b, cin); }
    { auto w = wc.next(); auto b = wc.next(); pack_conv(r.conv1, w, b, cout, cin, 9, true); }
    { auto w = wc.next(); auto b = wc.next();
      embw.insert(embw.end(), w, w + (size_t)cout * temb); embb.insert(embb.end(), b, b + cout);
      r.emb_off = emb_off; emb_off += cout; }
    { auto g = wc.next(); auto b = wc.next(); r.gn2_g.upload(g, cout); r.gn2_b.upload(b, cout); }
    { auto w = wc.next(); auto b = wc.next(); pack_conv(r.conv2, w, b, cout, cout, 9, true); }
    if (cin != cout) { auto w = wc.next(); auto b = wc.next(); pack_conv(r.skip, w, b, cout, cin, 1, false); r.has_skip = true; }
    return (int)u->res.size() - 1;
  };

  auto make_st = [&](int ch) -> int {
    u->st.emplace_back();
    StW& t = u->st.back();
    t.ch = ch; heads_for(ch, t.heads, t.dhead); t.inner = t.heads * t.dhead;
    const int C = t.inner;
    { auto g = wc.next(); auto b = wc.next(); t.gn_g.upload(g, ch); t.gn_b.upload(b, ch); }
    { auto w = wc.next(); auto b = wc.next(); pack_conv(t.proj_in, w, b, C, ch, 1, false); }
    t.blocks.resize(depth);
    for (int d = 0; d < depth; ++d) {
      XfBlockW& b = t.blocks[d];
      {  // attn1: to_q, to_k, to_v (no bias) -> one [3C][C] GEMM ; to_out.0 (bias)
        auto wq = wc.next(); auto wk = wc.next(); auto wv = wc.next();
        std::vector<float> cat((size_t)3 * C * C);
        memcpy(&cat[0], wq, sizeof(float) * C * C);
        memcpy(&cat[(size_t)C * C], wk, sizeof(float) * C * C);
        memcpy(&cat[(size_t)2 * C * C], wv, sizeof(float) * C * C);
        pack_conv(b.qkv1, cat.data(), nullptr, 3 * C, C, 1, false);
        auto wo = wc.next(); auto bo = wc.next(); pack_conv(b.out1, wo, bo, C, C, 1, false);
      }
      {  // attn2: to_q on x; to_k/to_v on the context -> hoisted, batched over all blocks
        auto wq = wc.next(); auto wk = wc.next(); auto wv = wc.next();
        pack_conv(b.q2, wq, nullptr, C, C, 1, false);
        kvw.insert(kvw.end(), wk, wk + (size_t)C * ctx);
        kvw.insert(kvw.end(), wv, wv + (size_t)C * ctx);
        b.kv_off = kv_off; kv_off += 2 * C;
        auto wo = wc.next(); auto bo = wc.next(); pack_conv(b.out2, wo, bo, C, C, 1, false);
      }
      { auto w = wc.next(); auto bb = wc.next(); pack_conv_pairs(b.ff1, w, bb, 8 * C, C, 1); }
      { auto w = wc.next(); auto bb = wc.next(); pack_conv(b.ff2, w, bb, C, 4 * C, 1, false); }
      { auto g = wc.next(); auto bb = wc.next(); b.ln1_g.upload(g, C); b.ln1_b.upload(bb, C); }
      { auto g = wc.next(); auto bb = wc.next(); b.ln2_g.upload(g, C); b.ln2_b.upload(bb, C); }
      { auto g = wc.next(); auto bb = wc.next(); b.ln3_g.upload(g, C); b.ln3_b.upload(bb, C); }
    }
    { auto w = wc.next(); auto b = wc.next(); pack_conv(t.proj_out, w, b, ch, C, 1, false); }
    return (int)u->st.size() - 1;
  };

  auto make_attn = [&](int ch) -> int {
    u->attn.emplace_back();
    AttnW& a = u->attn.back();
    a.ch = ch; heads_for(ch, a.heads, a.dhead);
    AGPT_CHECK(a.heads >= 1 && a.heads * a.dhead == ch, "AttentionBlock channels must split evenly into heads");
    { auto g = wc.next(); auto b = wc.next(); a.gn_g.upload(g, ch); a.gn_b.upload(b, ch); }
    {
      auto w = wc.next(); auto b = wc.next();   // qkv: Conv1d [3C][C][1] + bias
      if (cfg->attention_order == 1) {
        pack_conv(a.qkv, w, b, 3 * ch, ch, 1, false);   // QKVAttention: already [Q | K | V]
      } else {
        // QKVAttentionLegacy: rows per head h are [q_h ; k_h ; v_h] (d each) -> row j*C + h*d + i of [Q | K | V]
        const int d = a.dhead;
        std::vector<float> wp((size_t)3 * ch * ch), bp((size_t)3 * ch);
        for (int h = 0; h < a.heads; ++h)
          for (int j = 0; j < 3; ++j)
            for (int i = 0; i < d; ++i) {
              const size_t src = (size_t)h * 3 * d + j * d + i, dst = (size_t)j * ch + h * d + i;
              memcpy(&wp[dst * ch], &w[src * ch], sizeof(float) * ch);
              bp[dst] = b[src];
            }
        pack_conv(a.qkv, wp.data(), bp.data(), 3 * ch, ch, 1, false);
      }
    }
    { auto w = wc.next(); auto b = wc.next(); pack_conv(a.proj_out, w, b, ch, ch, 1, false); }
    return (int)u->attn.size() - 1;
  };
  auto attn_layer = [&](int ch) -> Layer {
    return cfg->use_spatial_transformer ? Layer{L_ST, make_st(ch), 0} : Layer{L_ATTN, make_attn(ch), 0};
  };
  AGPT_CHECK(cfg->attention_order == 0 || cfg->attention_order == 1, "attention_order must be 0 (legacy) or 1");

  // ---- walk the constructor rules (openaimodel.py:516-693) ----
  u->cin_pad = round_up(cfg->in_channels, 4);
  {
    auto w = wc.next(); auto b = wc.next();
    // input conv: pad Cin to a multiple of 4 so that activation rows stay float4-aligned
    std::vector<float> wp((size_t)mc * u->cin_pad * 9, 0.f);
    for (int co = 0; co < mc; ++co)
      for (int ci = 0; ci < cfg->in_channels; ++ci)
        memcpy(&wp[((size_t)co * u->cin_pad + ci) * 9], &w[((size_t)co * cfg->in_channels + ci) * 9], sizeof(float) * 9);
    pack_conv(u->conv_in, wp.data(), b, mc, u->cin_pad, 9, true);
    Block blk; blk.layers.push_back({L_CONV_IN, 0, mc});
    u->in_blocks.push_back(blk);
  }
  std::vector<int> chans{mc};
  int ch = mc;
  for (int level = 0; level < cfg->num_levels; ++level) {
    const int m = cfg->channel_mult[level];
    for (int i = 0; i < cfg->num_res_blocks; ++i) {
      Block blk;
      blk.layers.push_back({L_RES, make_res(ch, m * mc), 0});
      ch = m * mc;
      if (cfg->attn_at_level[level]) blk.layers.push_back(attn_layer(ch));
      u->in_blocks.push_back(blk);
      chans.push_back(ch);
    }
    if (level != cfg->num_levels - 1 && cfg->resblock_updown) {
      Block blk; blk.layers.push_back({L_RES, make_res(ch, ch, 1), 0});
      u->in_blocks.push_back(blk);
      chans.push_back(ch);
    } else if (level != cfg->num_levels - 1) {
      auto w = wc.next(); auto b = wc.next();
      // stride-2 conv as im2col + GEMM: weight [Cout][Cin][3][3] -> [Cout][(kh*3+kw)*Cin + ci]
      std::vector<float> wp((size_t)ch * 9 * ch);
      for (int co = 0; co < ch; ++co)
        for (int ci = 0; ci < ch; ++ci)
          for (int k = 0; k < 9; ++k) wp[((size_t)co * 9 + k) * ch + ci] = w[((size_t)co * ch + ci) * 9 + k];
      u->down_convs.emplace_back();
      pack_conv(u->down_convs.back(), wp.data(), b, ch, 9 * ch, 1, false);
      Block blk; blk.layers.push_back({L_DOWN, (int)u->down_convs.size() - 1, ch});
      u->in_blocks.push_back(blk);
      chans.push_back(ch);
    }
  }
  {
    const int r1 = make_res(ch, ch);
    const Layer a1 = attn_layer(ch);
    const int r2 = make_res(ch, ch);
    u->mid.layers = {{L_RES, r1, 0}, a1, {L_RES, r2, 0}};
  }
  for (int level = cfg->num_levels - 1; level >= 0; --level) {
    const int m = cfg->channel_mult[level];
    for (int i = 0; i <= cfg->num_res_blocks; ++i) {
      const int ich = chans.back(); chans.pop_back();
      Block blk;
      blk.layers.push_back({L_RES, make_res(ch + ich, mc * m), 0});
      ch = mc * m;
      if (cfg->attn_at_level[level]) blk.layers.push_back(attn_layer(ch));
      if (level && i == cfg->num_res_blocks && cfg->resblock_updown) {
        blk.layers.push_back({L_RES, make_res(ch, ch, 2), 0});
      } else if (level && i == cfg->num_res_blocks) {
        auto w = wc.next(); auto b = wc.next();
        u->up_convs.emplace_back();
        pack_conv(u->up_convs.back(), w, b, ch, ch, 9, true);
        blk.layers.push_back({L_UP, (int)u->up_convs.size() - 1, ch});
      }
      u->out_blocks.push_back(blk);
    }
  }
  u->final_ch = ch;
  { auto g = wc.next(); auto b = wc.next(); u->out_gn_g.upload(g, ch); u->out_gn_b.upload(b, ch); }
  { auto w = wc.next(); auto b = wc.next(); pack_conv(u->conv_out, w, b, cfg->out_channels, ch, 9, true);
    if (cfg->out_channels == 4) {   // the sampling loop's latent has 4 channels (any concat conditioning aside)
      std::vector<float> w9((size_t)9 * ch * 4), b4(4);
      for (int co = 0; co < 4; ++co) {
        b4[co] = b[co];
        for (int ci = 0; ci < ch; ++ci)
          for (int k = 0; k < 9; ++k) w9[((size_t)k * ch + ci) * 4 + co] = w[((size_t)co * ch + ci) * 9 + k];
      }
      u->out_w9c4.upload(w9); u->out_b4.upload(b4);
    } }
  wc.done();

  u->emb_total = emb_off; u->kv_total = kv_off;
  pack_conv(u->emb_all, embw.data(), embb.data(), emb_off, temb, 1, false);
  if (kv_off) pack_conv(u->ctx_kv_all, kvw.data(), nullptr, kv_off, ctx, 1, false);   // no cross-attention: no context
  return u.release();
}

void unet_set_context(Handle* hh, const float* ctx, int N, int S, cudaStream_t st) {
  auto* u = static_cast<Unet*>(hh);
  DeviceGuard dg_(u->device);
  AGPT_CHECK(N >= 1 && S >= 1, "empty context");
  u->set_context(ctx, N, S, st);
}

void unet_set_concat(Handle* hh, const float* c, int N, int C, int H, int W, cudaStream_t st) {
  auto* u = static_cast<Unet*>(hh);
  DeviceGuard dg_(u->device);
  u->set_concat(c, N, C, H, W, st);
}

void unet_forward(Handle* hh, const float* x, const int* t_host, int N, int H, int W, float* eps, cudaStream_t st) {
  auto* u = static_cast<Unet*>(hh);
  DeviceGuard dg_(u->device);
  u->forward(x, t_host, N, H, W, eps, st);
}

// Whole DDIM loop (ddim.py:143-164 + p_sample_ddim): the context holds [uncond ; cond] (2B rows) when
// cfg_scale != 1, else B rows.  Step-invariant work is hoisted: the time-embedding MLP and the 12 ResBlock
// embedding projections run ONCE for all S timesteps (one GEMM with S rows); step 0 runs eagerly (sizes every
// buffer), then one step is captured into a CUDA graph and replayed S - 1 times (plain launches while profiling).
void unet_ddim_sample(Handle* hh, const float* x_T, int B, int H, int W, int S, const int* t_steps,
                      const float* a_t, const float* a_prev, const float* sigma, const float* sqrt_om,
                      float cfg_scale, float* x_out, float* pred_x0_out, cudaStream_t st) {
  auto* u = static_cast<Unet*>(hh);
  DeviceGuard dg_(u->device);
  const bool cfg_on = cfg_scale != 1.0f;
  const int N = cfg_on ? 2 * B : B;
  if (u->kv_total)
    AGPT_CHECK(u->ctxN == N, "agpt_unet_set_context must hold [uncond;cond] (2B rows) for guided sampling, B rows otherwise");
  const bool concat = u->cfg.in_channels > u->cfg.out_channels;
  if (concat) {
    AGPT_CHECK(!cfg_on, "the on-device loop with concat conditioning samples without guidance (cfg_scale 1)");
    AGPT_CHECK(u->catN == B && u->catH == H && u->catW == W,
               "agpt_unet_set_concat must hold the conditioning of this call (B rows, the latent's H and W)");
  } else {
    AGPT_CHECK(u->cfg.in_channels == u->cfg.out_channels, "the on-device loop needs in_channels >= out_channels");
  }
  for (int i = 0; i < S; ++i) AGPT_CHECK(sigma[i] == 0.f, "the on-device loop is the eta = 0 sampler (noise is drawn by the step-wise path)");
  const long n = (long)u->cfg.out_channels * H * W;     // the loop state is the latent
  const float* cat = concat ? u->cat_cl.p : nullptr;
  u->prepare(N, H, W);
  u->ddim_eps.ensure((size_t)N * n);
  u->ddim_x.ensure((size_t)B * n);
  u->ddim_p0.ensure((size_t)B * n);
  u->emb_table.ensure((size_t)S * u->emb_total);
  u->emb_cur.ensure((size_t)u->emb_total);
  u->coef_table.ensure((size_t)S * 6);
  u->tsteps_dev.ensure((size_t)S);
  u->step_ctr.ensure(4);
  // ---- per-call tables (fp32 scalar algebra exactly as torch.full(...).sqrt() would do it, ddim.py:205-224)
  std::vector<float> coef((size_t)S * 6);
  for (int i = 0; i < S; ++i) {
    float* c = &coef[(size_t)i * 6];
    c[0] = sqrtf(a_t[i]); c[1] = sqrtf(a_prev[i]); c[2] = sqrtf(1.0f - a_prev[i] - sigma[i] * sigma[i]);
    c[3] = sigma[i]; c[4] = sqrt_om[i]; c[5] = cfg_scale;
  }
  AGPT_CUDA(cudaMemcpyAsync(u->coef_table.p, coef.data(), coef.size() * sizeof(float), cudaMemcpyHostToDevice, st));
  AGPT_CUDA(cudaMemcpyAsync(u->tsteps_dev.p, t_steps, (size_t)S * sizeof(int), cudaMemcpyHostToDevice, st));
  AGPT_CUDA(cudaMemsetAsync(u->step_ctr.p, 0, sizeof(int), st));
  AGPT_CUDA(cudaStreamSynchronize(st));     // coef / t_steps are caller-owned host memory
  u->arena_off = 0;
  {
    float* te = u->alloc((size_t)S * u->mc);
    timestep_embedding_dev(te, reinterpret_cast<const int*>(u->tsteps_dev.p), S, u->mc, st);
    u->embed_rows(te, S, u->emb_table.p, st);
  }
  AGPT_CUDA(cudaMemcpyAsync(u->ddim_x.p, x_T, (size_t)B * n * sizeof(float), cudaMemcpyDeviceToDevice, st));

  const long l0 = launch_count_now();
  u->ddim_step(B, N, H, W, n, cat, st);                              // step 0, eager
  u->launches_per_step = launch_count_now() - l0;
  int done = 1;
  if (S > 1 && !profile_enabled()) {
    Unet::GraphKey k;
    k.N = N; k.H = H; k.W = W; k.single = cfg_on ? 0 : 1; k.arena = u->arena.p; k.ctx = u->ctx_kv.p; k.x = u->ddim_x.p; k.ctxS = u->ctxS;
    k.cat = cat;
    const bool same = u->step_graph && k.N == u->gkey.N && k.H == u->gkey.H && k.W == u->gkey.W && k.single == u->gkey.single &&
                      k.arena == u->gkey.arena && k.ctx == u->gkey.ctx && k.x == u->gkey.x && k.ctxS == u->gkey.ctxS &&
                      k.cat == u->gkey.cat;
    if (!same) {
      if (u->step_graph) { cudaGraphExecDestroy(u->step_graph); u->step_graph = nullptr; }
      cudaGraph_t g = nullptr;
      // capture on a private stream (the caller's may be the legacy default stream, which cannot capture);
      // nothing executes during capture, so no ordering with `st` is needed
      if (!u->cap_stream) AGPT_CUDA(cudaStreamCreateWithFlags(&u->cap_stream, cudaStreamNonBlocking));
      AGPT_CUDA(cudaStreamBeginCapture(u->cap_stream, cudaStreamCaptureModeThreadLocal));
      try {
        u->ddim_step(B, N, H, W, n, cat, u->cap_stream);
      } catch (...) {
        cudaStreamEndCapture(u->cap_stream, &g);
        if (g) cudaGraphDestroy(g);
        throw;
      }
      AGPT_CUDA(cudaStreamEndCapture(u->cap_stream, &g));
      const cudaError_t ie = cudaGraphInstantiate(&u->step_graph, g, 0);
      cudaGraphDestroy(g);
      AGPT_CUDA(ie);
      u->gkey = k;
      count_launch(-u->launches_per_step);       // the captured pass launched nothing
    }
    for (; done < S; ++done) AGPT_CUDA(cudaGraphLaunch(u->step_graph, st));
    count_launch(u->launches_per_step * (S - 1));
  }
  for (; done < S; ++done) u->ddim_step(B, N, H, W, n, cat, st);
  AGPT_CUDA(cudaMemcpyAsync(x_out, u->ddim_x.p, (size_t)B * n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (pred_x0_out)
    AGPT_CUDA(cudaMemcpyAsync(pred_x0_out, u->ddim_p0.p, (size_t)B * n * sizeof(float), cudaMemcpyDeviceToDevice, st));
}

long unet_launches_per_step(Handle* hh) { return static_cast<Unet*>(hh)->launches_per_step; }

}  // namespace agpt
