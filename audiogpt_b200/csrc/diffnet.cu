// DiffNet epsilon-predictor + GaussianDiffusion step arithmetic on sm_90a.
// Reference: NeuralSeq/modules/diff/net.py:58-130 (DiffNet, ResidualBlock, SinusoidalPosEmb),
//            NeuralSeq/modules/diff/shallow_diffusion_tts.py:134-204 (p_sample / PLMS algebra).
// Parity: tests/test_diffusion_gpu.py against oracle/diffusion_ref.py and tests/golden/diffusion_*.npz.
#include "common.cuh"
#include "tapconv.cuh"
#include "models.h"
#include "nn_kernels.h"
#include "voc_kernels.cuh"

namespace agpt {

constexpr int kMaxBatchParam = 256;
struct StepT { int t[kMaxBatchParam]; };

// SinusoidalPosEmb (net.py:37-44): sin || cos, exponent divisor (half-1)
__global__ void diff_step_embed_kernel(float* __restrict__ out, const __grid_constant__ StepT st, int B, int C, float neg_emb) {
  const int b = blockIdx.x;
  const int half = C / 2;
  for (int j = threadIdx.x; j < C; j += blockDim.x) {
    const int i = j < half ? j : j - half;
    const float f = expf((float)i * neg_emb);
    const float a = (float)st.t[b] * f;
    out[(long)b * C + j] = j < half ? sinf(a) : cosf(a);
  }
}

// x_out = c1*clamp(A*x - Bc*eps, -1, 1) + c2*x + s*noise      (shallow_diffusion_tts.py:134-166)
// coef[b] = {A, Bc, c1, c2, s}
__global__ void p_sample_kernel(const float* __restrict__ x, const float* __restrict__ eps, const float* __restrict__ noise,
                                const float* __restrict__ coef, int clip, long n, float* __restrict__ out) {
  const int b = blockIdx.y;
  const float A = coef[b * 5 + 0], Bc = coef[b * 5 + 1], c1 = coef[b * 5 + 2], c2 = coef[b * 5 + 3], s = coef[b * 5 + 4];
  const long base = (long)b * n;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const float xv = x[base + i];
    float x0 = A * xv - Bc * eps[base + i];
    if (clip) x0 = fminf(fmaxf(x0, -1.f), 1.f);
    float o = c1 * x0 + c2 * xv;
    if (noise) o += s * noise[base + i];
    out[base + i] = o;
  }
}

// table versions for the graph-replayed loop: step k = *ctr handles t = t_hi - 1 - k
__global__ void diff_step_embed_dev_kernel(float* __restrict__ out, const int* __restrict__ t, int C, float neg_emb) {
  const int b = blockIdx.x;
  const int half = C / 2;
  const float tv = (float)t[b];
  for (int j = threadIdx.x; j < C; j += blockDim.x) {
    const int i = j < half ? j : j - half;
    const float f = expf((float)i * neg_emb);
    const float a = tv * f;
    out[(long)b * C + j] = j < half ? sinf(a) : cosf(a);
  }
}
__global__ void p_sample_tab_kernel(float* __restrict__ x, const float* __restrict__ eps, const float* const* __restrict__ noises_pp,
                                    long noise_stride, const float* __restrict__ coef_tab, const int* __restrict__ ctr,
                                    int nsteps, int clip, long n) {
  const int k = *ctr;
  const float* coef = coef_tab + 5 * (long)k;
  const float A = coef[0], Bc = coef[1], c1 = coef[2], c2 = coef[3], s = coef[4];
  const float* noises = *noises_pp;      // per-call base pointer lives in device memory: the captured step stays valid
  const float* noise = noises ? noises + (long)(nsteps - 1 - k) * noise_stride : nullptr;
  const long base = (long)blockIdx.y * n;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const float xv = x[base + i];
    float x0 = A * xv - Bc * eps[base + i];
    if (clip) x0 = fminf(fmaxf(x0, -1.f), 1.f);
    float o = c1 * x0 + c2 * xv;
    if (noise) o += s * noise[base + i];
    x[base + i] = o;
  }
}

// net.py:41: emb = log(10000) / (half_dim - 1), rounded to fp32 once on the host
static float step_embed_neg_emb(int C) {
  AGPT_CHECK(C % 2 == 0 && C / 2 > 1, "step embedding: needs an even C with C / 2 > 1 (the exponent divides by C / 2 - 1)");
  return (float)(-(std::log(10000.0) / (double)(C / 2 - 1)));
}

void diff_step_embed(const int* t_host, float* out, int B, int C, cudaStream_t st) {
  AGPT_CHECK(B >= 1 && B <= kMaxBatchParam && t_host, "step embedding: needs 1 <= B <= 256 host timesteps");
  const float neg_emb = step_embed_neg_emb(C);
  StepT stp;
  for (int b = 0; b < B; ++b) stp.t[b] = t_host[b];
  diff_step_embed_kernel<<<B, 128, 0, st>>>(out, stp, B, C, neg_emb);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

void diff_step_embed_dev(const int* t_dev, float* out, int N, int C, cudaStream_t st) {
  AGPT_CHECK(N >= 1, "step embedding: needs N >= 1");
  const float neg_emb = step_embed_neg_emb(C);
  diff_step_embed_dev_kernel<<<N, 128, 0, st>>>(out, t_dev, C, neg_emb);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

void p_sample_tab(float* x, const float* eps, const float* const* noises_pp, long noise_stride, const float* coef_tab,
                  const int* ctr, int nsteps, int clip, int B, long n, cudaStream_t st) {
  AGPT_CHECK(B >= 1 && n >= 1 && nsteps >= 1, "p_sample_tab: needs B >= 1, n >= 1 and nsteps >= 1");
  dim3 grid((unsigned)std::min<long>(cdivl(n, 256), 1184), B);
  p_sample_tab_kernel<<<grid, dim3(256), 0, st>>>(x, eps, noises_pp, noise_stride, coef_tab, ctr, nsteps, clip, n);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

__global__ void axpby5_kernel(const float* __restrict__ x, const float* __restrict__ e0, const float* __restrict__ e1,
                              const float* __restrict__ e2, const float* __restrict__ e3,
                              const float* __restrict__ coef, long n, float* __restrict__ out) {
  const int b = blockIdx.y;
  const float a0 = coef[b * 5], a1 = coef[b * 5 + 1], a2 = coef[b * 5 + 2], a3 = coef[b * 5 + 3], a4 = coef[b * 5 + 4];
  const long base = (long)b * n;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    float o = a0 * x[base + i];
    if (e0) o += a1 * e0[base + i];
    if (e1) o += a2 * e1[base + i];
    if (e2) o += a3 * e2[base + i];
    if (e3) o += a4 * e3[base + i];
    out[base + i] = o;
  }
}

// staging for per-sample coefficient rows, one ring per device (stream-ordered reuse)
static DevBuf g_coef[16];
static int g_coef_slot[16] = {0};
constexpr int kCoefSlots = 8, kCoefMaxB = 1024;

static const float* upload_coef(const float* coef_host, int B, cudaStream_t st) {
  int dev = 0;
  AGPT_CUDA(cudaGetDevice(&dev));
  AGPT_CHECK(dev < 16 && B <= kCoefMaxB, "coefficient staging");
  float* base = g_coef[dev].ensure((size_t)kCoefSlots * kCoefMaxB * 5);
  float* slot = base + (size_t)(g_coef_slot[dev]++ % kCoefSlots) * kCoefMaxB * 5;
  AGPT_CUDA(cudaMemcpyAsync(slot, coef_host, (size_t)B * 5 * sizeof(float), cudaMemcpyHostToDevice, st));
  return slot;
}

void axpby5(const float* x, const float* e0, const float* e1, const float* e2, const float* e3,
            const float* coef_host, int B, long n, float* out, cudaStream_t st) {
  const float* coef = upload_coef(coef_host, B, st);
  dim3 grid((unsigned)std::min<long>(cdivl(n, 256), 1184), B);
  axpby5_kernel<<<grid, 256, 0, st>>>(x, e0, e1, e2, e3, coef, n, out);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

struct Diffnet : Handle {
  agpt_diffnet_cfg cfg;
  PackedConv in_proj, mlp0, mlp2, dproj_all, cond_all, skip_proj, out_proj;
  std::vector<PackedConv> dil, outp;
  // state
  int B = 0, T = 0;
  DevBuf condT, condp, xT, xcur, z, skip, hbuf, emb, e1, e2, dproj, eps_tmp;
  // sampling-loop state (one captured step replayed; see gd_sample_loop)
  DevBuf dproj_table, dproj_cur, coef_table, t_dev, step_ctr, loop_eps, loop_x;
  cudaGraphExec_t step_graph = nullptr;
  cudaStream_t cap_stream = nullptr;
  struct GraphKey { int B = 0, T = 0, nsteps = 0, clip = 0; const void *x = nullptr, *condp = nullptr, *xcur = nullptr, *z = nullptr; long stride = 0; } gkey;
  long launches_per_step = 0;

  ~Diffnet() override {
    if (step_graph) cudaGraphExecDestroy(step_graph);
    if (cap_stream) cudaStreamDestroy(cap_stream);
  }

  void set_cond(const float* cond, int B_, int T_, cudaStream_t st) {
    const int H = cfg.hidden_size, C = cfg.residual_channels, L = cfg.residual_layers;
    AGPT_CHECK(B_ >= 1 && B_ <= kMaxBatchParam && T_ >= 1, "batch size must be in [1,256]");
    B = B_; T = T_;
    condT.ensure((size_t)B * T * H);
    condp.ensure((size_t)B * T * L * 2 * C);
    launch_cf_to_cl(cond, condT.p, B, H, T, st);
    TapConvParams P = tapconv_params(cond_all, B, T, 0, 1);
    P.in = condT.p; P.in_gstride = (long)T * H; P.in_pitch = H;
    P.out = condp.p; P.out_gstride = (long)T * L * 2 * C; P.out_pitch = L * 2 * C;
    P.epi = EPI_BIAS;
    tapconv_launch(P, st);
  }

  void ensure_bufs() {
    const int C = cfg.residual_channels, L = cfg.residual_layers, M = cfg.in_dims;
    const size_t rows = (size_t)B * T;
    xT.ensure(rows * M); xcur.ensure(rows * C); z.ensure(rows * C); skip.ensure(rows * C); hbuf.ensure(rows * C);
    emb.ensure((size_t)B * C); e1.ensure((size_t)B * 4 * C); e2.ensure((size_t)B * C); dproj.ensure((size_t)B * L * C);
  }

  // diffusion-step embedding MLP and the per-layer diffusion projections for `rows` timestep embeddings
  // (net.py:118-119, 67): embv [rows][C] -> out [rows][L*C]; e1v / e2v are scratch of rows*4C / rows*C floats
  void step_mlp(const float* embv, int rows, float* e1v, float* e2v, float* out, cudaStream_t st) {
    const int C = cfg.residual_channels, L = cfg.residual_layers;
    auto lin = [&](const PackedConv& pc, const float* in, int cin, float* o, int cout, int epi) {
      TapConvParams P = tapconv_params(pc, 1, rows, 0, 1);
      P.in = in; P.in_gstride = 0; P.in_pitch = cin;
      P.out = o; P.out_gstride = 0; P.out_pitch = cout;
      P.epi = epi;
      tapconv_launch(P, st);
    };
    lin(mlp0, embv, C, e1v, 4 * C, EPI_MISH);
    lin(mlp2, e1v, 4 * C, e2v, C, EPI_BIAS);
    lin(dproj_all, e2v, C, out, L * C, EPI_BIAS);
  }

  void eps(const float* x, const int* t_host, float* out, cudaStream_t st) {
    AGPT_CHECK(B > 0, "agpt_diffnet_set_cond must be called first");
    const int C = cfg.residual_channels, L = cfg.residual_layers;
    ensure_bufs();
    diff_step_embed(t_host, emb.p, B, C, st);
    step_mlp(emb.p, B, e1.p, e2.p, dproj.p, st);
    eps_core(x, dproj.p, L * C, out, st);
  }

  // everything after the step embedding; dprojv [.][L*C] with per-sample row stride dproj_gs (0: shared row)
  void eps_core(const float* x, const float* dprojv, int dproj_gs, float* out, cudaStream_t st) {
    const int C = cfg.residual_channels, L = cfg.residual_layers, M = cfg.in_dims;
    launch_cf_to_cl(x, xT.p, B, M, T, st);
    {
      TapConvParams P = tapconv_params(in_proj, B, T, 0, 1);
      P.in = xT.p; P.in_gstride = (long)T * M; P.in_pitch = M;
      P.out = xcur.p; P.out_gstride = (long)T * C; P.out_pitch = C;
      P.epi = EPI_RELU;
      tapconv_launch(P, st);
    }
    const long gs = (long)T * C;
    for (int l = 0; l < L; ++l) {
      const int d = 1 << (l % cfg.dilation_cycle_length);
      {  // y = dilated_conv(x + dproj) + cond_proj ; z = sigmoid(gate)*tanh(filter)   (net.py:67-74)
        TapConvParams P = tapconv_params(dil[l], B, T, 0, d);
        P.in = xcur.p; P.in_gstride = gs; P.in_pitch = C;
        P.pro = PRO_ADDVEC; P.pvec = dprojv + (long)l * C; P.pvec_gstride = dproj_gs;
        P.epi = EPI_GATE;
        P.res = condp.p + (long)l * 2 * C; P.res_gstride = (long)T * L * 2 * C; P.res_pitch = L * 2 * C;
        P.out = z.p; P.out_gstride = gs; P.out_pitch = C;
        tapconv_launch(P, st);
      }
      {  // output_projection; x <- (x + residual)/sqrt2 ; skip += skip_l    (net.py:76-78)
        TapConvParams P = tapconv_params(outp[l], B, T, 0, 1);
        P.in = z.p; P.in_gstride = gs; P.in_pitch = C;
        P.epi = EPI_DIFFOUT; P.csplit = C; P.accumulate = (l > 0);
        P.out = xcur.p; P.out_gstride = gs; P.out_pitch = C;
        P.out2 = skip.p; P.out2_gstride = gs; P.out2_pitch = C;
        tapconv_launch(P, st);
      }
    }
    {  // relu(skip_projection(sum skip / sqrt(L)))   (1/sqrt(L) folded into the weights)
      TapConvParams P = tapconv_params(skip_proj, B, T, 0, 1);
      P.in = skip.p; P.in_gstride = gs; P.in_pitch = C;
      P.out = hbuf.p; P.out_gstride = gs; P.out_pitch = C;
      P.epi = EPI_RELU;
      tapconv_launch(P, st);
    }
    {
      TapConvParams P = tapconv_params(out_proj, B, T, 0, 1);
      P.in = hbuf.p; P.in_gstride = gs; P.in_pitch = C;
      P.out = out; P.out_gstride = (long)M * T; P.out_pitch = 0;
      P.epi = EPI_STORE_CF;
      tapconv_launch(P, st);
    }
  }
};

Handle* diffnet_create(const agpt_diffnet_cfg* cfg, const float* const* W, int nW, int device) {
  DeviceGuard dg_(device);
  const int C = cfg->residual_channels, H = cfg->hidden_size, M = cfg->in_dims, L = cfg->residual_layers;
  AGPT_CHECK(C % 8 == 0 && C >= 8 && L >= 1 && cfg->dilation_cycle_length >= 1, "bad DiffNet config");
  std::unique_ptr<Diffnet> h(new Diffnet());
  h->magic = kMagicDiffnet; h->device = device; h->cfg = *cfg;
  WeightCursor wc{W, nW};
  { auto w = wc.next(); auto b = wc.next(); pack_conv(h->in_proj, w, b, C, M, 1, false); }
  { auto w = wc.next(); auto b = wc.next(); pack_conv(h->mlp0, w, b, 4 * C, C, 1, false); }
  { auto w = wc.next(); auto b = wc.next(); pack_conv(h->mlp2, w, b, C, 4 * C, 1, false); }
  h->dil.resize(L); h->outp.resize(L);
  std::vector<float> dpw((size_t)L * C * C), dpb((size_t)L * C), cw((size_t)L * 2 * C * H), cb((size_t)L * 2 * C);
  for (int l = 0; l < L; ++l) {
    { auto w = wc.next(); auto b = wc.next(); pack_conv_pairs(h->dil[l], w, b, 2 * C, C, 3); }
    { auto w = wc.next(); auto b = wc.next();
      memcpy(&dpw[(size_t)l * C * C], w, sizeof(float) * C * C); memcpy(&dpb[(size_t)l * C], b, sizeof(float) * C); }
    { auto w = wc.next(); auto b = wc.next();   // conditioner: interleave (gate,filter) like the dilated conv
      for (int co = 0; co < 2 * C; ++co) {
        const int dst = 2 * (co % C) + co / C;
        memcpy(&cw[((size_t)l * 2 * C + dst) * H], w + (size_t)co * H, sizeof(float) * H);
        cb[(size_t)l * 2 * C + dst] = b[co];
      } }
    { auto w = wc.next(); auto b = wc.next(); pack_conv(h->outp[l], w, b, 2 * C, C, 1, false); }
  }
  pack_conv(h->dproj_all, dpw.data(), dpb.data(), L * C, C, 1, false);
  pack_conv(h->cond_all, cw.data(), cb.data(), L * 2 * C, H, 1, false);
  { auto w = wc.next(); auto b = wc.next(); pack_conv(h->skip_proj, w, b, C, C, 1, false, 1.f / std::sqrt((float)L)); }
  { auto w = wc.next(); auto b = wc.next(); pack_conv(h->out_proj, w, b, M, C, 1, false); }
  wc.done();
  return h.release();
}

void diffnet_set_cond(Handle* hh, const float* cond, int B, int T, cudaStream_t st) {
  auto* h = static_cast<Diffnet*>(hh);
  DeviceGuard dg_(h->device);
  h->set_cond(cond, B, T, st);
}

void diffnet_eps(Handle* hh, const float* x, const int* t_host, float* eps, cudaStream_t st) {
  auto* h = static_cast<Diffnet*>(hh);
  DeviceGuard dg_(h->device);
  h->eps(x, t_host, eps, st);
}

void gd_p_sample(Handle* hh, const float* x, const float* eps_or_null, const int* t_host, const float* coef_host,
                 const float* noise, int clip, int B, long n, float* x_out, cudaStream_t st) {
  const float* e = eps_or_null;
  int dev_cur = 0;
  AGPT_CUDA(cudaGetDevice(&dev_cur));
  DeviceGuard dg_(e ? dev_cur : static_cast<Diffnet*>(hh)->device);
  if (!e) {
    auto* h = static_cast<Diffnet*>(hh);
    AGPT_CHECK(B == h->B && n == (long)h->cfg.in_dims * h->T, "shape differs from the cond set by agpt_diffnet_set_cond");
    h->eps_tmp.ensure((size_t)B * n);
    h->eps(x, t_host, h->eps_tmp.p, st);
    e = h->eps_tmp.p;
  }
  const float* coef = upload_coef(coef_host, B, st);
  dim3 grid((unsigned)std::min<long>(cdivl(n, 256), 1184), B);
  p_sample_kernel<<<grid, 256, 0, st>>>(x, e, noise, coef, clip, n, x_out);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// Whole ancestral sampling loop (shallow_diffusion_tts.py:263-272): for t = t_hi-1 .. t_lo: x <- p_sample(x, t, noise_t),
// every sample at the same t (as the reference's loop does).  The step-embedding MLP and the 20 diffusion
// projections run ONCE for all steps (one GEMM of nsteps rows); step 0 runs eagerly, then ONE captured step
// (CUDA graph; device step counter, coefficient / projection tables) is replayed.  coef_host [nsteps][5] rows in
// sampling order (row k belongs to t = t_hi-1-k); noises: device [nsteps][B][n] indexed by t - t_lo, or NULL.
void gd_sample_loop(Handle* hh, float* x_io, int t_hi, int t_lo, const float* coef_host, const float* noises,
                    long noise_stride, int clip, cudaStream_t st) {
  auto* h = static_cast<Diffnet*>(hh);
  DeviceGuard dg_(h->device);
  AGPT_CHECK(h->B > 0, "agpt_diffnet_set_cond must be called first");
  const int nsteps = t_hi - t_lo;
  AGPT_CHECK(nsteps >= 1 && t_lo >= 0, "empty step range");
  const int C = h->cfg.residual_channels, L = h->cfg.residual_layers, M = h->cfg.in_dims, B = h->B;
  const long n = (long)M * h->T;
  h->ensure_bufs();
  h->dproj_table.ensure((size_t)nsteps * L * C);
  h->dproj_cur.ensure((size_t)L * C);
  h->coef_table.ensure((size_t)nsteps * 5);
  h->t_dev.ensure((size_t)nsteps);
  h->step_ctr.ensure(4);
  h->loop_eps.ensure((size_t)B * n);
  h->loop_x.ensure((size_t)B * n);
  std::vector<int> ts(nsteps);
  for (int k = 0; k < nsteps; ++k) ts[k] = t_hi - 1 - k;
  AGPT_CUDA(cudaMemcpyAsync(h->t_dev.p, ts.data(), (size_t)nsteps * sizeof(int), cudaMemcpyHostToDevice, st));
  AGPT_CUDA(cudaMemcpyAsync(h->coef_table.p, coef_host, (size_t)nsteps * 5 * sizeof(float), cudaMemcpyHostToDevice, st));
  AGPT_CUDA(cudaMemsetAsync(h->step_ctr.p, 0, sizeof(int), st));
  AGPT_CUDA(cudaMemcpyAsync(h->step_ctr.p + 2, &noises, sizeof(noises), cudaMemcpyHostToDevice, st));   // floats 2..3 = the pointer slot
  AGPT_CUDA(cudaMemcpyAsync(h->loop_x.p, x_io, (size_t)B * n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  AGPT_CUDA(cudaStreamSynchronize(st));        // ts / coef_host / &noises are host memory
  {
    DevBuf &te = h->z, &t1 = h->skip, &t2 = h->hbuf;      // scratch: free before the first step
    te.ensure((size_t)nsteps * C); t1.ensure((size_t)nsteps * 4 * C); t2.ensure((size_t)nsteps * C);
    diff_step_embed_dev(reinterpret_cast<const int*>(h->t_dev.p), te.p, nsteps, C, st);
    h->step_mlp(te.p, nsteps, t1.p, t2.p, h->dproj_table.p, st);
    h->ensure_bufs();                                        // (scratch may have grown the buffers: keep sizes valid)
  }
  int* ctr = reinterpret_cast<int*>(h->step_ctr.p);
  const float* const* noise_pp = reinterpret_cast<const float* const*>(h->step_ctr.p + 2);
  float* xl = h->loop_x.p;
  auto step = [&](cudaStream_t s) {
    select_row(h->dproj_table.p, ctr, h->dproj_cur.p, L * C, s);
    h->eps_core(xl, h->dproj_cur.p, 0, h->loop_eps.p, s);
    p_sample_tab(xl, h->loop_eps.p, noise_pp, noise_stride, h->coef_table.p, ctr, nsteps, clip, B, n, s);
    step_inc(ctr, s);
  };
  const long long l0 = launch_count_now();
  step(st);
  h->launches_per_step = (long)(launch_count_now() - l0);
  int done = 1;
  if (nsteps > 1 && !profile_enabled()) {
    Diffnet::GraphKey k;
    k.B = B; k.T = h->T; k.nsteps = nsteps; k.clip = clip; k.x = xl; k.condp = h->condp.p; k.xcur = h->xcur.p; k.z = h->z.p; k.stride = noise_stride;
    const Diffnet::GraphKey& o = h->gkey;
    const bool same = h->step_graph && k.B == o.B && k.T == o.T && k.nsteps == o.nsteps && k.clip == o.clip && k.x == o.x &&
                      k.condp == o.condp && k.xcur == o.xcur && k.z == o.z && k.stride == o.stride;
    if (!same) {
      if (h->step_graph) { cudaGraphExecDestroy(h->step_graph); h->step_graph = nullptr; }
      cudaGraph_t g = nullptr;
      if (!h->cap_stream) AGPT_CUDA(cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking));
      AGPT_CUDA(cudaStreamBeginCapture(h->cap_stream, cudaStreamCaptureModeThreadLocal));
      try {
        step(h->cap_stream);
      } catch (...) {
        cudaStreamEndCapture(h->cap_stream, &g);
        if (g) cudaGraphDestroy(g);
        throw;
      }
      AGPT_CUDA(cudaStreamEndCapture(h->cap_stream, &g));
      const cudaError_t ie = cudaGraphInstantiate(&h->step_graph, g, 0);
      cudaGraphDestroy(g);
      AGPT_CUDA(ie);
      h->gkey = k;
      count_launch(-h->launches_per_step);
    }
    for (; done < nsteps; ++done) AGPT_CUDA(cudaGraphLaunch(h->step_graph, st));
    count_launch(h->launches_per_step * (nsteps - 1));
  }
  for (; done < nsteps; ++done) step(st);
  AGPT_CUDA(cudaMemcpyAsync(x_io, xl, (size_t)B * n * sizeof(float), cudaMemcpyDeviceToDevice, st));
}

long diffnet_launches_per_step(Handle* hh) { return static_cast<Diffnet*>(hh)->launches_per_step; }

}  // namespace agpt
