// AutoencoderKL.decode (Make-An-Audio first stage) on sm_90a: latent [B,4,10,78] -> mel image [B,1,80,624].
// Reference: ldm/models/autoencoder.py:351-354 (decode = post_quant_conv -> decoder),
//            ldm/modules/diffusionmodules/model.py:462-568 (Decoder), :121-143 (ResnetBlock, temb None),
//            :150-203 (AttnBlock: single head of width C, scale C^-0.5), :43-49 (Upsample: nearest x2 then conv),
//            :33-39 (swish, GroupNorm(32, eps 1e-6)).
// Activations are channels-last rows [B][H*W][C]; every 3x3 / 1x1 conv is a tap-GEMM on the tensor-core kernel
// (wide maps -- 156, 312, 624 columns -- in STRIP mode, TapConvParams::strips: the halo of a 128-row tile would
// otherwise span two 625-wide image rows); GroupNorm(+swish) is the fused single-kernel GroupNorm of nn_kernels.cu;
// the seven AttnBlocks (780 tokens x 512 ch, 3 120 tokens x 256 ch) run as Q K^T / row softmax / P V with the
// activation as the GEMM's weight operand (fp32).
// Parity: tests/test_vae_gpu.py against tests/golden/vae_{small,txt2audio}.npz (made by the reference Decoder) and
// oracle/vae_ref.py.
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
  std::vector<int> attn;      // index into Vae::attns or -1, one per res block
  bool up = false;
  PackedConv upconv;
};

static void upload_vec_(DevBuf& d, const float* p, int n) { d.upload(std::vector<float>(p, p + n)); }

struct Vae : Handle {
  agpt_vae_cfg cfg;
  int block_in = 0, last_ch = 0, cin_pad = 4;
  PackedConv post_quant, conv_in, conv_out;
  VResW mid1, mid2;
  std::vector<VAttnW> attns;   // [0] = mid.attn_1
  std::vector<VLevel> levels;
  DevBuf gno, bno;
  DevBuf buf[6], qkv, sc, kT, vpad, zcl;

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
    for (auto& b : buf) b.ensure(mx);
    zcl.ensure((size_t)B * H * W * 2 * cin_pad);
    float* z_cl = zcl.p;
    float* z_pq = zcl.p + (size_t)B * H * W * cin_pad;
    cf_to_cl_pad(z, z_cl, B, cfg.embed_dim, cin_pad, H * W, s);
    linear(post_quant, z_cl, cin_pad, z_pq, cin_pad, (long)B * H * W, EPI_BIAS, nullptr, 0, s);
    // rotating buffers: cur holds the block input, the others are scratch / output
    int ci = 0;
    auto other = [&](int k) { return buf[(ci + k) % 6].p; };
    float* cur = buf[0].p;
    conv3x3(conv_in, z_pq, cur, B, H, W, EPI_BIAS, nullptr, s);
    auto res = [&](const VResW& r, int h, int w) {
      run_res(r, cur, other(1), other(2), other(3), other(4), B, h, w, s);
      ci = (ci + 4) % 6; cur = buf[ci].p;
    };
    auto attn = [&](const VAttnW& a, int h, int w) {
      run_attn(a, cur, other(1), other(2), other(3), B, h, w, s);
      ci = (ci + 3) % 6; cur = buf[ci].p;
    };
    int h = H, w = W;
    res(mid1, h, w);
    attn(attns[0], h, w);
    res(mid2, h, w);
    for (const VLevel& l : levels) {
      for (size_t j = 0; j < l.res.size(); ++j) {
        res(l.res[j], h, w);
        if (l.attn[j] >= 0) attn(attns[l.attn[j]], h, w);
      }
      if (l.up) {
        const int C = l.res.back().cout;
        upsample_nearest2(cur, other(1), B, h, w, C, s);
        h *= 2; w *= 2;
        conv3x3(l.upconv, other(1), other(2), B, h, w, EPI_BIAS, nullptr, s);
        ci = (ci + 2) % 6; cur = buf[ci].p;
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
  auto* v = new Vae();
  v->magic = kMagicVae; v->device = device; v->cfg = *cfg;
  const int nl = cfg->num_levels;
  AGPT_CHECK(nl >= 1 && nl <= AGPT_MAX_LEVELS && cfg->ch % 32 == 0, "bad VAE config (ch must be a multiple of 32: GroupNorm(32))");
  int idx = 0;
  auto next = [&]() -> const float* { AGPT_CHECK(idx < nW, "too few weight arrays"); return W[idx++]; };
  const int zc = cfg->z_channels, ed = cfg->embed_dim;
  v->cin_pad = round_up(std::max(zc, ed), 4);
  {  // post_quant_conv: Conv2d(embed_dim -> z_channels, 1); channel counts padded to a multiple of 4 with zeros
    auto w = next(); auto b = next();
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
    auto w = next(); auto b = next();
    std::vector<float> wp((size_t)block_in * v->cin_pad * 9, 0.f);
    for (int co = 0; co < block_in; ++co)
      for (int ci = 0; ci < zc; ++ci)
        memcpy(&wp[((size_t)co * v->cin_pad + ci) * 9], &w[((size_t)co * zc + ci) * 9], sizeof(float) * 9);
    pack_conv(v->conv_in, wp.data(), b, block_in, v->cin_pad, 9, true);
  }
  auto load_res = [&](VResW& r, int cin, int cout) {
    r.cin = cin; r.cout = cout;
    AGPT_CHECK(cin % 32 == 0 && cout % 32 == 0, "ResnetBlock channels must be multiples of 32");
    { auto g = next(); auto b = next(); upload_vec_(r.g1, g, cin); upload_vec_(r.b1, b, cin); }
    { auto w = next(); auto b = next(); pack_conv(r.conv1, w, b, cout, cin, 9, true); }
    { auto g = next(); auto b = next(); upload_vec_(r.g2, g, cout); upload_vec_(r.b2, b, cout); }
    { auto w = next(); auto b = next(); pack_conv(r.conv2, w, b, cout, cout, 9, true); }
    if (cin != cout) { auto w = next(); auto b = next(); pack_conv(r.nin, w, b, cout, cin, 1, false); r.has_nin = true; }
  };
  auto load_attn = [&](int c) -> int {
    v->attns.emplace_back();
    VAttnW& a = v->attns.back();
    a.c = c;
    { auto g = next(); auto b = next(); upload_vec_(a.g, g, c); upload_vec_(a.b, b, c); }
    auto wq = next(); auto bq = next(); auto wk = next(); auto bk = next(); auto wv = next(); auto bv = next();
    std::vector<float> cat((size_t)3 * c * c), cb((size_t)3 * c);
    memcpy(&cat[0], wq, sizeof(float) * c * c); memcpy(&cat[(size_t)c * c], wk, sizeof(float) * c * c);
    memcpy(&cat[(size_t)2 * c * c], wv, sizeof(float) * c * c);
    memcpy(&cb[0], bq, sizeof(float) * c); memcpy(&cb[c], bk, sizeof(float) * c); memcpy(&cb[2 * c], bv, sizeof(float) * c);
    pack_conv(a.qkv, cat.data(), cb.data(), 3 * c, c, 1, false);
    { auto w = next(); auto b = next(); pack_conv(a.proj, w, b, c, c, 1, false); }
    return (int)v->attns.size() - 1;
  };
  load_res(v->mid1, block_in, block_in);
  load_attn(block_in);
  load_res(v->mid2, block_in, block_in);
  int bi = block_in;
  for (int il = nl - 1; il >= 0; --il) {
    const int bo = cfg->ch * cfg->ch_mult[il];
    v->levels.emplace_back();
    VLevel& l = v->levels.back();
    for (int j = 0; j <= cfg->num_res_blocks; ++j) {
      l.res.emplace_back();
      load_res(l.res.back(), bi, bo);
      bi = bo;
      l.attn.push_back(cfg->attn_at_level[il] ? load_attn(bo) : -1);
    }
    l.up = il != 0;
    if (l.up) { auto w = next(); auto b = next(); pack_conv(l.upconv, w, b, bo, bo, 9, true); }
  }
  v->last_ch = bi;
  { auto g = next(); auto b = next(); upload_vec_(v->gno, g, bi); upload_vec_(v->bno, b, bi); }
  { auto w = next(); auto b = next(); pack_conv(v->conv_out, w, b, cfg->out_ch, bi, 9, true); }
  AGPT_CHECK(idx == nW, "weight array count does not match the config");
  return v;
}

void vae_decode(Handle* hh, const float* z, int B, int H, int W, float* out, cudaStream_t st) {
  auto* v = static_cast<Vae*>(hh);
  DeviceGuard dg_(v->device);
  v->forward(z, B, H, W, out, st);
}

}  // namespace agpt
