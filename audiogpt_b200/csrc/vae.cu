// AutoencoderKL (Make-An-Audio first stage) on sm_90a.
//   decode: latent [B,4,10,78] -> mel image [B,1,80,624]
//   encode: mel image [B,1,80,848] -> moments [B,8,10,106] (mean and logvar of the posterior)
// Reference: ldm/models/autoencoder.py:345-354 (encode = quant_conv(encoder(x)), decode = decoder(post_quant_conv(z))),
//            ldm/modules/diffusionmodules/model.py:368-459 (Encoder), :462-568 (Decoder), :121-143 (ResnetBlock,
//            temb None), :150-203 (AttnBlock: single head of width C, scale C^-0.5), :43-49 (Upsample: nearest x2 then
//            conv), :60-79 (Downsample: F.pad (0,1,0,1) then a 3x3 stride-2 conv), :33-39 (swish, GroupNorm(32, eps 1e-6)).
// Activations are channels-last rows [B][H*W][C]; every 3x3 / 1x1 conv is a tap-GEMM on the tensor-core kernel
// (wide maps -- 156 to 848 columns -- in STRIP mode, TapConvParams::strips: the halo of a 128-row tile would
// otherwise span two 625-wide image rows); GroupNorm(+swish) is the fused single-kernel GroupNorm of nn_kernels.cu;
// the AttnBlocks (decoder: 780 tokens x 512 ch, 3 120 tokens x 256 ch; encoder: 1 060 x 512, 4 240 x 256) run as
// Q K^T / row softmax / P V with the activation as the GEMM's weight operand (fp32).  The encoder's stride-2
// Downsample conv is an im2col gather followed by a 1-tap GEMM over 9*C input channels.
// Both engines share the layer drivers and the buffer rotation of VaeBase; each is its own handle, built from its
// own half of the state dict.
// Parity: tests/test_vae_gpu.py and tests/test_vae_encoder_gpu.py against tests/golden/vae_{small,txt2audio}.npz
// and vae_enc_{small,txt2audio}.npz (made by the reference modules) and the CPU oracles oracle/vae_ref.py and
// oracle/vae_enc_ref.py.
#include "common.cuh"
#include "tapconv.cuh"
#include "nn_kernels.h"
#include "models.h"

namespace agpt {

struct VResW {
  int cin = 0, cout = 0;
  DevBuf g1, b1, g2, b2;
  PackedConv conv1, conv2, nin;
  bool has_nin = false;
};
struct VAttnW {
  int c = 0;
  DevBuf g, b;
  PackedConv qkv, proj;
};
struct VLevel {
  std::vector<VResW> res;
  std::vector<int> attn;      // index into VaeBase::attns or -1, one per res block
  bool up = false;            // decoder: ends in an Upsample (upconv)
  bool down = false;          // encoder: ends in a Downsample (downconv, im2col form [C][9*C])
  PackedConv upconv, downconv;
};

// What the decoder and the encoder have in common: the layer drivers, the attention scratch and the rotating
// activation buffers.
struct VaeBase : Handle {
  std::vector<VAttnW> attns;
  DevBuf buf[6], qkv, sc, kT, vpad;
  // rotating buffers: cur holds the block input, the others are scratch / output
  int ci = 0;
  float* cur = nullptr;

  // strips of at most 78 columns: virtual width 80, halo tile of 128 + 2*80 + 2 rows -- the largest operand tile
  // the one-tile-per-CTA kernel fits next to its staging buffer (the UNet's 78-column maps use the same budget)
  static int pick_strip(int W) {
    if (W <= 79) return 0;
    const int n = cdiv(W, 78);
    return cdiv(W, n);
  }
  void conv3x3(const PackedConv& pc, const float* in, float* out, int N, int H, int W, int epi, const float* res_,
               cudaStream_t s, long out_gstride = -1, int out_pitch = -1) {
    TapConvParams P = tapconv_params(pc, N, H * W, W, 1);
    const int sw = pick_strip(W);
    if (sw) tapconv_set_strips(P, sw);
    P.in = in; P.in_gstride = (long)H * W * pc.Cin; P.in_pitch = pc.Cin;
    P.out = out; P.out_gstride = out_gstride >= 0 ? out_gstride : (long)H * W * pc.Cout; P.out_pitch = out_pitch >= 0 ? out_pitch : pc.Cout;
    P.epi = epi;
    P.res = res_; P.res_gstride = (long)H * W * pc.Cout; P.res_pitch = pc.Cout;
    tapconv_launch(P, s);
  }
  void linear(const PackedConv& pc, const float* in, int in_pitch, float* out, int out_pitch, long rows, int epi,
              const float* res_, int res_pitch, cudaStream_t s) {
    TapConvParams P = tapconv_params(pc, 1, (int)rows, 0, 1);
    P.in = in; P.in_pitch = in_pitch;
    P.out = out; P.out_pitch = out_pitch;
    P.epi = epi;
    P.res = res_; P.res_pitch = res_pitch;
    tapconv_launch(P, s);
  }
  // out [rows][cout] = in [rows][cin] x wT, with the fp32 ACTIVATION matrix w [cin_pad][cout_pad] as the weight operand
  void act_gemm(const float* in, int in_pitch, int rows, int cin, const float* w, int cin_padv, int cout, int cout_padv,
                float* out, int out_pitch, cudaStream_t s) {
    TapConvParams P;
    memset(&P, 0, sizeof(P));
    P.w = w; P.G = 1; P.L = rows; P.Cin = cin; P.cin_pad = cin_padv; P.Cout = cout; P.cout_pad = cout_padv;
    P.ntaps = 1; P.scale = 1.f; P.flops_scale = 1.f;
    P.in = in; P.in_pitch = in_pitch;
    P.out = out; P.out_pitch = out_pitch;
    P.epi = EPI_BIAS;
    tapconv_launch(P, s);          // no tensor-core image (w_h == nullptr): the fp32-FMA tap-GEMM
  }

  // h = conv2(swish(norm2(conv1(swish(norm1(x)))))) + shortcut(x)      (model.py:121-143, temb is None)
  float* run_res(const VResW& r, const float* x, float* t1, float* t2, float* t3, float* out, int N, int H, int W, cudaStream_t s) {
    const int HW = H * W;
    groupnorm(x, t1, r.g1.p, r.b1.p, N, HW, r.cin, 32, 1e-6f, true, nullptr, s);
    conv3x3(r.conv1, t1, t2, N, H, W, EPI_BIAS, nullptr, s);
    groupnorm(t2, t1, r.g2.p, r.b2.p, N, HW, r.cout, 32, 1e-6f, true, nullptr, s);
    const float* sk = x;
    if (r.has_nin) {
      linear(r.nin, x, r.cin, t3, r.cout, (long)N * HW, EPI_BIAS, nullptr, 0, s);
      sk = t3;
    }
    conv3x3(r.conv2, t1, out, N, H, W, EPI_RES, sk, s);
    return out;
  }

  // x + proj_out(softmax(q k^T / sqrt(C)) v)     (model.py:177-203)
  float* run_attn(const VAttnW& a, const float* x, float* t1, float* t2, float* out, int N, int H, int W, cudaStream_t s) {
    const int HW = H * W, C = a.c;
    const long rows = (long)N * HW;
    groupnorm(x, t1, a.g.p, a.b.p, N, HW, C, 32, 1e-6f, false, nullptr, s);
    qkv.ensure((size_t)rows * 3 * C);
    linear(a.qkv, t1, C, qkv.p, 3 * C, rows, EPI_BIAS, nullptr, 0, s);
    const int Lp = round_up(HW, 32);
    sc.ensure((size_t)HW * Lp); kT.ensure((size_t)C * Lp); vpad.ensure((size_t)Lp * C);
    const float scale = 1.0f / sqrtf((float)C);          // int(c) ** (-0.5)
    for (int n = 0; n < N; ++n) {
      const float* q = qkv.p + (long)n * HW * 3 * C;
      transpose_pad(q + C, 3 * C, HW, C, kT.p, Lp, s);                       // K^T [C][Lp]
      act_gemm(q, 3 * C, HW, C, kT.p, round_up(C, TC_KC), HW, Lp, sc.p, Lp, s);   // scores [HW][HW]
      softmax_rows(sc.p, Lp, HW, HW, scale, s);
      copy_pad_rows(q + 2 * C, 3 * C, HW, C, vpad.p, Lp, s);                 // V [Lp][C], zero rows beyond HW
      act_gemm(sc.p, Lp, HW, HW, vpad.p, round_up(HW, TC_KC), C, C, t2 + (long)n * HW * C, C, s);
    }
    linear(a.proj, t2, C, out, C, rows, EPI_RES, x, C, s);
    return out;
  }

  void rot_reset() { ci = 0; cur = buf[0].p; }
  float* other(int k) { return buf[(ci + k) % 6].p; }
  void rot_advance(int k) { ci = (ci + k) % 6; cur = buf[ci].p; }
  void res_step(const VResW& r, int N, int h, int w, cudaStream_t s) {
    run_res(r, cur, other(1), other(2), other(3), other(4), N, h, w, s);
    rot_advance(4);
  }
  void attn_step(const VAttnW& a, int N, int h, int w, cudaStream_t s) {
    run_attn(a, cur, other(1), other(2), other(3), N, h, w, s);
    rot_advance(3);
  }
  void ensure_bufs(size_t floats) { for (auto& b : buf) b.ensure(floats); }

  void load_res(VResW& r, WeightCursor& wc, int cin, int cout) {
    r.cin = cin; r.cout = cout;
    AGPT_CHECK(cin % 32 == 0 && cout % 32 == 0, "ResnetBlock channels must be multiples of 32");
    { auto g = wc.next(); auto b = wc.next(); r.g1.upload(g, cin); r.b1.upload(b, cin); }
    { auto w = wc.next(); auto b = wc.next(); pack_conv(r.conv1, w, b, cout, cin, 9, true); }
    { auto g = wc.next(); auto b = wc.next(); r.g2.upload(g, cout); r.b2.upload(b, cout); }
    { auto w = wc.next(); auto b = wc.next(); pack_conv(r.conv2, w, b, cout, cout, 9, true); }
    if (cin != cout) { auto w = wc.next(); auto b = wc.next(); pack_conv(r.nin, w, b, cout, cin, 1, false); r.has_nin = true; }
  }
  int load_attn(WeightCursor& wc, int c) {
    attns.emplace_back();
    VAttnW& a = attns.back();
    a.c = c;
    { auto g = wc.next(); auto b = wc.next(); a.g.upload(g, c); a.b.upload(b, c); }
    auto wq = wc.next(); auto bq = wc.next(); auto wk = wc.next(); auto bk = wc.next(); auto wv = wc.next(); auto bv = wc.next();
    std::vector<float> cat((size_t)3 * c * c), cb((size_t)3 * c);
    memcpy(&cat[0], wq, sizeof(float) * c * c); memcpy(&cat[(size_t)c * c], wk, sizeof(float) * c * c);
    memcpy(&cat[(size_t)2 * c * c], wv, sizeof(float) * c * c);
    memcpy(&cb[0], bq, sizeof(float) * c); memcpy(&cb[c], bk, sizeof(float) * c); memcpy(&cb[2 * c], bv, sizeof(float) * c);
    pack_conv(a.qkv, cat.data(), cb.data(), 3 * c, c, 1, false);
    { auto w = wc.next(); auto b = wc.next(); pack_conv(a.proj, w, b, c, c, 1, false); }
    return (int)attns.size() - 1;
  }
};

struct Vae : VaeBase {
  agpt_vae_cfg cfg;
  int block_in = 0, last_ch = 0, cin_pad = 4;
  PackedConv post_quant, conv_in, conv_out;
  VResW mid1, mid2;            // attns[0] = mid.attn_1
  std::vector<VLevel> levels;
  DevBuf gno, bno, zcl;

  size_t max_elems(int H, int W) const {
    size_t mx = (size_t)H * W * block_in;
    int h = H, w = W;
    for (const VLevel& l : levels) {
      for (const VResW& r : l.res) mx = std::max(mx, (size_t)h * w * std::max(r.cin, r.cout));
      if (l.up) { h *= 2; w *= 2; mx = std::max(mx, (size_t)h * w * l.res.back().cout); }
    }
    return mx;
  }

  void forward(const float* z, int B, int H, int W, float* out, cudaStream_t s) {
    AGPT_CHECK(B >= 1 && H >= 1 && W >= 1, "empty latent");
    const size_t mx = max_elems(H, W) * (size_t)B;
    ensure_bufs(mx);
    zcl.ensure((size_t)B * H * W * 2 * cin_pad);
    float* z_cl = zcl.p;
    float* z_pq = zcl.p + (size_t)B * H * W * cin_pad;
    cf_to_cl_pad(z, z_cl, B, cfg.embed_dim, cin_pad, H * W, s);
    linear(post_quant, z_cl, cin_pad, z_pq, cin_pad, (long)B * H * W, EPI_BIAS, nullptr, 0, s);
    rot_reset();
    conv3x3(conv_in, z_pq, cur, B, H, W, EPI_BIAS, nullptr, s);
    int h = H, w = W;
    res_step(mid1, B, h, w, s);
    attn_step(attns[0], B, h, w, s);
    res_step(mid2, B, h, w, s);
    for (const VLevel& l : levels) {
      for (size_t j = 0; j < l.res.size(); ++j) {
        res_step(l.res[j], B, h, w, s);
        if (l.attn[j] >= 0) attn_step(attns[l.attn[j]], B, h, w, s);
      }
      if (l.up) {
        const int C = l.res.back().cout;
        upsample_nearest2(cur, other(1), B, h, w, C, s);
        h *= 2; w *= 2;
        conv3x3(l.upconv, other(1), other(2), B, h, w, EPI_BIAS, nullptr, s);
        rot_advance(2);
      }
    }
    groupnorm(cur, other(1), gno.p, bno.p, B, h * w, last_ch, 32, 1e-6f, true, nullptr, s);
    {
      TapConvParams P = tapconv_params(conv_out, B, h * w, w, 1);
      const int sw = pick_strip(w);
      if (sw) tapconv_set_strips(P, sw);
      P.in = other(1); P.in_gstride = (long)h * w * last_ch; P.in_pitch = last_ch;
      P.out = out; P.out_gstride = (long)cfg.out_ch * h * w; P.out_pitch = 0;
      P.epi = EPI_STORE_CF;
      tapconv_launch(P, s);
    }
  }
};

Handle* vae_create(const agpt_vae_cfg* cfg, const float* const* W, int nW, int device) {
  DeviceGuard dg_(device);
  const int nl = cfg->num_levels;
  AGPT_CHECK(nl >= 1 && nl <= AGPT_MAX_LEVELS && cfg->ch % 32 == 0, "bad VAE config (ch must be a multiple of 32: GroupNorm(32))");
  std::unique_ptr<Vae> v(new Vae());
  v->magic = kMagicVae; v->device = device; v->cfg = *cfg;
  WeightCursor wc{W, nW};
  const int zc = cfg->z_channels, ed = cfg->embed_dim;
  v->cin_pad = round_up(std::max(zc, ed), 4);
  {  // post_quant_conv: Conv2d(embed_dim -> z_channels, 1); channel counts padded to a multiple of 4 with zeros
    auto w = wc.next(); auto b = wc.next();
    std::vector<float> wp((size_t)v->cin_pad * v->cin_pad, 0.f), bp(v->cin_pad, 0.f);
    for (int co = 0; co < zc; ++co) {
      for (int ci = 0; ci < ed; ++ci) wp[(size_t)co * v->cin_pad + ci] = w[(size_t)co * ed + ci];
      bp[co] = b[co];
    }
    pack_conv(v->post_quant, wp.data(), bp.data(), v->cin_pad, v->cin_pad, 1, false);
  }
  const int block_in = cfg->ch * cfg->ch_mult[nl - 1];
  v->block_in = block_in;
  {
    auto w = wc.next(); auto b = wc.next();
    std::vector<float> wp((size_t)block_in * v->cin_pad * 9, 0.f);
    for (int co = 0; co < block_in; ++co)
      for (int ci = 0; ci < zc; ++ci)
        memcpy(&wp[((size_t)co * v->cin_pad + ci) * 9], &w[((size_t)co * zc + ci) * 9], sizeof(float) * 9);
    pack_conv(v->conv_in, wp.data(), b, block_in, v->cin_pad, 9, true);
  }
  v->load_res(v->mid1, wc, block_in, block_in);
  v->load_attn(wc, block_in);
  v->load_res(v->mid2, wc, block_in, block_in);
  int bi = block_in;
  for (int il = nl - 1; il >= 0; --il) {
    const int bo = cfg->ch * cfg->ch_mult[il];
    v->levels.emplace_back();
    VLevel& l = v->levels.back();
    for (int j = 0; j <= cfg->num_res_blocks; ++j) {
      l.res.emplace_back();
      v->load_res(l.res.back(), wc, bi, bo);
      bi = bo;
      l.attn.push_back(cfg->attn_at_level[il] ? v->load_attn(wc, bo) : -1);
    }
    l.up = il != 0;
    if (l.up) { auto w = wc.next(); auto b = wc.next(); pack_conv(l.upconv, w, b, bo, bo, 9, true); }
  }
  v->last_ch = bi;
  { auto g = wc.next(); auto b = wc.next(); v->gno.upload(g, bi); v->bno.upload(b, bi); }
  { auto w = wc.next(); auto b = wc.next(); pack_conv(v->conv_out, w, b, cfg->out_ch, bi, 9, true); }
  wc.done();
  return v.release();
}

void vae_decode(Handle* hh, const float* z, int B, int H, int W, float* out, cudaStream_t st) {
  auto* v = static_cast<Vae*>(hh);
  DeviceGuard dg_(v->device);
  v->forward(z, B, H, W, out, st);
}

// AutoencoderKL.encode's arithmetic: moments = quant_conv(Encoder(x))     (autoencoder.py:345-349, model.py:368-459)
struct VaeEnc : VaeBase {
  agpt_vae_cfg cfg;
  int in_ch = 1, cin_pad = 4, last_ch = 0, out_ch = 0;
  PackedConv conv_in, conv_out;   // conv_out carries quant_conv, folded in on the host
  VResW mid1, mid2;
  int mid_attn = -1;
  std::vector<VLevel> levels;
  DevBuf gno, bno, xcl, col;

  // largest activation (floats per sample) and largest Downsample im2col matrix
  std::pair<size_t, size_t> max_elems(int H, int W) const {
    size_t mx = (size_t)H * W * std::max(cfg.ch, cin_pad), mc = 0;
    int h = H, w = W;
    for (const VLevel& l : levels) {
      for (const VResW& r : l.res) mx = std::max(mx, (size_t)h * w * std::max(r.cin, r.cout));
      if (l.down) {
        const int C = l.res.back().cout;
        h /= 2; w /= 2;
        mc = std::max(mc, (size_t)h * w * 9 * C);
      }
    }
    return {mx, mc};
  }

  void forward(const float* x, int B, int H, int W, float* moments, cudaStream_t s) {
    const int f = 1 << (cfg.num_levels - 1);
    AGPT_CHECK(B >= 1, "empty batch");
    if (H < f || W < f)
      throw Error("VAE encoder: a " + std::to_string(H) + " x " + std::to_string(W) + " input shrinks to zero size after " +
                  std::to_string(cfg.num_levels - 1) + " Downsample steps (H and W must be at least " + std::to_string(f) + ")");
    AGPT_CHECK(x && moments, "null argument");   // after the size check: a zero-size moments tensor has no storage
    const auto need = max_elems(H, W);
    ensure_bufs(need.first * B);
    col.ensure(std::max<size_t>(need.second * B, 1));
    xcl.ensure((size_t)B * H * W * cin_pad);
    cf_to_cl_pad(x, xcl.p, B, in_ch, cin_pad, H * W, s);
    rot_reset();
    conv3x3(conv_in, xcl.p, cur, B, H, W, EPI_BIAS, nullptr, s);
    int h = H, w = W;
    for (const VLevel& l : levels) {
      for (size_t j = 0; j < l.res.size(); ++j) {
        res_step(l.res[j], B, h, w, s);
        if (l.attn[j] >= 0) attn_step(attns[l.attn[j]], B, h, w, s);
      }
      if (l.down) {   // F.pad(x, (0,1,0,1)) then Conv2d(k3, stride 2, padding 0): floor(h/2) x floor(w/2)
        const int C = l.res.back().cout, ho = h / 2, wo = w / 2;
        im2col_stride2(cur, col.p, B, h, w, C, ho, wo, 0, s);
        linear(l.downconv, col.p, 9 * C, other(1), C, (long)B * ho * wo, EPI_BIAS, nullptr, 0, s);
        rot_advance(1);
        h = ho; w = wo;
      }
    }
    res_step(mid1, B, h, w, s);
    attn_step(attns[mid_attn], B, h, w, s);
    res_step(mid2, B, h, w, s);
    groupnorm(cur, other(1), gno.p, bno.p, B, h * w, last_ch, 32, 1e-6f, true, nullptr, s);
    {  // conv_out with quant_conv folded in, stored channels-first: the moments [B][2*embed_dim][h][w]
      TapConvParams P = tapconv_params(conv_out, B, h * w, w, 1);
      const int sw = pick_strip(w);
      if (sw) tapconv_set_strips(P, sw);
      P.in = other(1); P.in_gstride = (long)h * w * last_ch; P.in_pitch = last_ch;
      P.out = moments; P.out_gstride = (long)out_ch * h * w; P.out_pitch = 0;
      P.epi = EPI_STORE_CF;
      tapconv_launch(P, s);
    }
  }
};

Handle* vae_encoder_create(const agpt_vae_cfg* cfg, int in_channels, const float* const* W, int nW, int device) {
  DeviceGuard dg_(device);
  const int nl = cfg->num_levels, ch = cfg->ch;
  AGPT_CHECK(nl >= 1 && nl <= AGPT_MAX_LEVELS && ch % 32 == 0, "bad VAE config (ch must be a multiple of 32: GroupNorm(32))");
  AGPT_CHECK(cfg->num_res_blocks >= 1, "the encoder needs num_res_blocks >= 1");
  AGPT_CHECK(in_channels >= 1 && in_channels <= 64, "in_channels must be in [1, 64]");
  std::unique_ptr<VaeEnc> v(new VaeEnc());
  v->magic = kMagicVaeEnc; v->device = device; v->cfg = *cfg;
  v->in_ch = in_channels;
  v->cin_pad = round_up(in_channels, 4);
  WeightCursor wc{W, nW};
  {  // conv_in: Conv2d(in_channels -> ch, 3, padding 1); input channels zero-padded to a multiple of 4
    auto w = wc.next(); auto b = wc.next();
    std::vector<float> wp((size_t)ch * v->cin_pad * 9, 0.f);
    for (int co = 0; co < ch; ++co)
      for (int ci = 0; ci < in_channels; ++ci)
        memcpy(&wp[((size_t)co * v->cin_pad + ci) * 9], &w[((size_t)co * in_channels + ci) * 9], sizeof(float) * 9);
    pack_conv(v->conv_in, wp.data(), b, ch, v->cin_pad, 9, true);
  }
  int bi = ch;   // in_ch_mult = (1,) + ch_mult
  for (int il = 0; il < nl; ++il) {
    const int bo = ch * cfg->ch_mult[il];
    v->levels.emplace_back();
    VLevel& l = v->levels.back();
    for (int j = 0; j < cfg->num_res_blocks; ++j) {
      l.res.emplace_back();
      v->load_res(l.res.back(), wc, bi, bo);
      bi = bo;
      l.attn.push_back(cfg->attn_at_level[il] ? v->load_attn(wc, bo) : -1);
    }
    l.down = il != nl - 1;
    if (l.down) {  // stride-2 conv as im2col + GEMM: weight [C][C][3][3] -> [C][(kh*3+kw)*C + ci]
      auto w = wc.next(); auto b = wc.next();
      std::vector<float> wp((size_t)bi * 9 * bi);
      for (int co = 0; co < bi; ++co)
        for (int ci = 0; ci < bi; ++ci)
          for (int k = 0; k < 9; ++k) wp[((size_t)co * 9 + k) * bi + ci] = w[((size_t)co * bi + ci) * 9 + k];
      pack_conv(l.downconv, wp.data(), b, bi, 9 * bi, 1, false);
    }
  }
  v->load_res(v->mid1, wc, bi, bi);
  v->mid_attn = v->load_attn(wc, bi);
  v->load_res(v->mid2, wc, bi, bi);
  v->last_ch = bi;
  { auto g = wc.next(); auto b = wc.next(); v->gno.upload(g, bi); v->bno.upload(b, bi); }
  {  // conv_out [2z][C][3][3] followed by quant_conv [2e][2z][1][1]: one 3x3 conv [2e][C][3][3], composed in fp64
    const int z2 = 2 * cfg->z_channels, e2 = 2 * cfg->embed_dim;
    auto w = wc.next(); auto b = wc.next(); auto qw = wc.next(); auto qb = wc.next();
    std::vector<float> wf((size_t)e2 * bi * 9), bf(e2);
    for (int o = 0; o < e2; ++o) {
      double acc = qb[o];
      for (int m = 0; m < z2; ++m) acc += (double)qw[(size_t)o * z2 + m] * b[m];
      bf[o] = (float)acc;
      for (size_t k = 0; k < (size_t)bi * 9; ++k) {
        double a = 0.0;
        for (int m = 0; m < z2; ++m) a += (double)qw[(size_t)o * z2 + m] * w[(size_t)m * bi * 9 + k];
        wf[(size_t)o * bi * 9 + k] = (float)a;
      }
    }
    v->out_ch = e2;
    pack_conv(v->conv_out, wf.data(), bf.data(), e2, bi, 9, true);
  }
  wc.done();
  return v.release();
}

void vae_encode(Handle* hh, const float* x, int B, int H, int W, float* moments, cudaStream_t st) {
  auto* v = static_cast<VaeEnc*>(hh);
  DeviceGuard dg_(v->device);
  v->forward(x, B, H, W, moments, st);
}

}  // namespace agpt
