// tapconv kernel (fp32 FMA) + launcher.  See tapconv.cuh for the contract.
#include "tapconv.cuh"
#include "tapconv_epi.cuh"
#include "models.h"

namespace agpt {

// ---- optional per-launch CUDA-event profiling (bench.py's roofline leg) ----
struct ProfRec { cudaEvent_t e0, e1; int variant; double flops, bytes; int G, L, Cin, Cout, ntaps, span, epi, Wreal; };
static bool g_prof = false;
constexpr int PROF_PAIR = 16;   // record epi code of a fused ResBlock pair: 16 + the epilogue of its second conv
static std::vector<ProfRec> g_recs;
static long long g_tall = 0;    // recorded launches that ran 256-row tiles (the dump line has no field for it)
static long long g_plane = 0;   // recorded launches that were plane-fed (likewise)
static long long g_dual = 0;    // recorded launches of narrow pairs with overlapped tiles (likewise)
static long long g_pipe = 0;    // recorded launches of the two-tiles-per-CTA pair kernel (likewise)
static long long g_narrow = 0;  // recorded launches of the narrow pair pipeline (likewise)
static long long g_cpipe = 0;   // recorded launches of the plane-fed single-conv pipeline (likewise)

bool profile_enabled() { return g_prof; }

void profile_enable(int on) {
  g_prof = on != 0;
  if (!on) {
    for (auto& r : g_recs) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
    g_recs.clear();
    g_tall = 0;
    g_plane = 0;
    g_dual = 0;
    g_pipe = 0;
    g_narrow = 0;
    g_cpipe = 0;
  }
}

static thread_local int g_ran[5] = {-1, -1, -1, -1, -1};
void tapconv_note_launch(int tc, int bn, int mt, int plane, int kern) {
  g_ran[0] = tc; g_ran[1] = bn; g_ran[2] = mt; g_ran[3] = plane; g_ran[4] = kern;
}
void tapconv_last_launch(int ran[5]) { for (int i = 0; i < 5; ++i) ran[i] = g_ran[i]; }

void profile_count_tall() { if (g_prof) ++g_tall; }
long long profile_tall_launches() { return g_tall; }
void profile_count_plane() { if (g_prof) ++g_plane; }
long long profile_plane_launches() { return g_plane; }
void profile_count_dual() { if (g_prof) ++g_dual; }
long long profile_dual_launches() { return g_dual; }
void profile_count_pipe() { if (g_prof) ++g_pipe; }
long long profile_pipe_launches() { return g_pipe; }
void profile_count_narrow_pipe() { if (g_prof) ++g_narrow; }
long long profile_narrow_pipe_launches() { return g_narrow; }
void profile_count_conv_pipe() { if (g_prof) ++g_cpipe; }
long long profile_conv_pipe_launches() { return g_cpipe; }

// Sums over the records since profile_enable(1): per variant (FMA BN = 128, 64, 32; 3 = wgmma)
void profile_collect(double* ms, double* flops, double* bytes, long long* launches) {
  for (int v = 0; v < 4; ++v) { ms[v] = 0; flops[v] = 0; bytes[v] = 0; launches[v] = 0; }
  AGPT_CUDA(cudaDeviceSynchronize());
  for (auto& r : g_recs) {
    float t = 0.f;
    AGPT_CUDA(cudaEventElapsedTime(&t, r.e0, r.e1));
    ms[r.variant] += t; flops[r.variant] += r.flops; bytes[r.variant] += r.bytes; launches[r.variant] += 1;
  }
}

// One text line per recorded launch: "variant G L Cin Cout ntaps span epi Wreal ms flops" (dev tooling).  A fused
// ResBlock pair is one line with epi = PROF_PAIR + c2's epi and the taps / spans of both convs summed.
long profile_dump(char* out, long cap) {
  AGPT_CUDA(cudaDeviceSynchronize());
  long n = 0;
  for (auto& r : g_recs) {
    float t = 0.f;
    AGPT_CUDA(cudaEventElapsedTime(&t, r.e0, r.e1));
    char line[160];
    const int len = snprintf(line, sizeof(line), "%d %d %d %d %d %d %d %d %d %.6f %.6e\n", r.variant, r.G, r.L, r.Cin, r.Cout,
                             r.ntaps, r.span, r.epi, r.Wreal, t, r.flops);
    if (n + len < cap) { memcpy(out + n, line, len); n += len; }
  }
  if (cap > 0) out[n < cap ? n : cap - 1] = 0;
  return n;
}

// ---- fp32 FMA saturation probe: the measured denominator of the compute roofline ----
__global__ void fma_peak_kernel(float* out, int iters) {
  float a[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = (float)(threadIdx.x + i) * 1e-3f;
  const float b = 1.000001f, c = 1e-6f;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = fmaf(a[i], b, c);
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += a[i];
  if (s == 12345.678f) out[0] = s;
}

double fma_peak_tflops() {
  float* d = nullptr;
  AGPT_CUDA(cudaMalloc(&d, 4));
  int dev = 0, sms = 0;
  AGPT_CUDA(cudaGetDevice(&dev));
  AGPT_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int iters = 1 << 15, blocks = sms * 8, threads = 256;
  cudaEvent_t e0, e1;
  AGPT_CUDA(cudaEventCreate(&e0)); AGPT_CUDA(cudaEventCreate(&e1));
  double best = 0.0;
  for (int rep = 0; rep < 5; ++rep) {
    AGPT_CUDA(cudaEventRecord(e0));
    fma_peak_kernel<<<blocks, threads>>>(d, iters);
    AGPT_CUDA(cudaEventRecord(e1));
    AGPT_CUDA(cudaEventSynchronize(e1));
    float ms = 0.f;
    AGPT_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    const double fl = 2.0 * 8.0 * iters * (double)blocks * threads;
    best = std::max(best, fl / (ms * 1e-3) / 1e12);
  }
  cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(d);
  return best;
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gsrc));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;\n" ::); }

template <int BN>
__global__ void __launch_bounds__((BN / 8) * 16, (BN == 128 ? 2 : (BN == 64 ? 4 : 6)))
tapconv_kernel(const __grid_constant__ TapConvParams P) {
  constexpr int NTX = BN / 8, NT = NTX * 16, KC = TC_KC, BM = TC_BM;
  extern __shared__ __align__(16) float smem[];
  const int R = P.R;
  int* rowaddr = reinterpret_cast<int*>(smem);
  float* Xs = smem + (R + 8);
  float* Ws = Xs + 4 * KC * R;

  const int tid = threadIdx.x, tx = tid % NTX, ty = tid / NTX;
  const int gz = blockIdx.z, g = tc_sample(P, gz), co0 = blockIdx.y * BN, q0 = blockIdx.x * BM;
  const int Wv = tc_wv(P);
  const int Lv = tc_lv(P);

  for (int i = tid; i < R + 8; i += NT) {
    const int r = tc_row_in(P, gz, q0 + P.lo_al + i, Wv, Lv);
    rowaddr[i] = r >= 0 ? r * P.in_pitch : -1;
  }

  const float* __restrict__ ing = P.in + g * P.in_gstride;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  const int nchunks = P.cin_pad / KC, total = nchunks * P.ntaps;

  auto issue_w = [&](int it) {
    const int chunk = it / P.ntaps, tap = it - chunk * P.ntaps;
    const int ci = tid / (BN / 4), c4 = (tid % (BN / 4)) * 4;
    float* dst = Ws + (it & 1) * KC * BN + ci * BN + c4;
    if (co0 + c4 < P.cout_pad) {
      const float* src = P.w + ((long)(tap * P.cin_pad + chunk * KC + ci)) * P.cout_pad + co0 + c4;
      cp_async16(dst, src);
    } else {
      *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    cp_async_commit();
  };

  issue_w(0);
  int it = 0;
  for (int chunk = 0; chunk < nchunks; ++chunk) {
    __syncthreads();  // rowaddr ready (first) / everyone done reading Xs of the previous chunk
    {
      const int nitems = (R >> 2) * KC;
      for (int item = tid; item < nitems; item += NT) {
        const int ci = item % KC, m = item / KC;
        const int c = chunk * KC + ci;
        const bool cok = c < P.Cin;
        const int4 a0 = *reinterpret_cast<const int4*>(rowaddr + 4 * m);
        const int4 a1 = *reinterpret_cast<const int4*>(rowaddr + 4 * m + 4);
        const int aa[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        float pv = 0.f;
        if (P.pro == PRO_ADDVEC && cok) pv = P.pvec[(long)g * P.pvec_gstride + c];
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float x = 0.f;
          if (cok && aa[i] >= 0) {
            x = __ldg(ing + aa[i] + c);
            if (P.pro == PRO_LRELU) x = lrelu(x, P.slope);
            else if (P.pro == PRO_ADDVEC) x += pv;
            else if (P.pro == PRO_SILU) x = siluf_(x);
          }
          v[i] = x;
        }
#pragma unroll
        for (int s = 0; s < 4; ++s)
          *reinterpret_cast<float4*>(Xs + (s * KC + ci) * R + 4 * m) = make_float4(v[s], v[s + 1], v[s + 2], v[s + 3]);
      }
    }
    for (int tap = 0; tap < P.ntaps; ++tap, ++it) {
      cp_async_wait_all();
      __syncthreads();  // W(it) + Xs visible; everyone finished compute(it-1)
      if (it + 1 < total) issue_w(it + 1);
      const int e = P.tap_off[tap] - P.lo_al;
      const float* xs = Xs + (e & 3) * KC * R + (e & ~3) + ty * 4;
      const float* ws = Ws + (it & 1) * KC * BN + tx * 4;
#pragma unroll
      for (int ci = 0; ci < KC; ++ci) {
        const float4 xa = *reinterpret_cast<const float4*>(xs + ci * R);
        const float4 xb = *reinterpret_cast<const float4*>(xs + ci * R + 64);
        const float4 wa = *reinterpret_cast<const float4*>(ws + ci * BN);
        const float4 wb = *reinterpret_cast<const float4*>(ws + ci * BN + BN / 2);
        const float xv[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
        const float wv[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(xv[i], wv[j], acc[i][j]);
      }
    }
  }

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = (i < 4) ? (ty * 4 + i) : (64 + ty * 4 + (i - 4));
    const int p = tc_row_out(P, gz, q0 + r, Wv, Lv);
    if (p < 0) continue;
    tc_epilogue(P, g, p, co0 + tx * 4, make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]));
    tc_epilogue(P, g, p, co0 + BN / 2 + tx * 4, make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]));
  }
}


// Fill geometry-dependent fields (offsets, halo, smem rows) and launch.
static void fma_launch(TapConvParams P, cudaStream_t st) {
  int lo = P.tap_off[0], hi = P.tap_off[0];
  for (int t = 1; t < P.ntaps; ++t) { lo = min(lo, P.tap_off[t]); hi = max(hi, P.tap_off[t]); }
  P.lo_al = (lo >= 0) ? (lo / 4) * 4 : -(((-lo) + 3) / 4) * 4;
  int R = round_up(TC_BM + (hi - P.lo_al), 4);
  while (R % 32 != 4) R += 4;
  P.R = R;
  const int Lv = tc_lv(P);
  const int bn = tc_pick_bn(P.Cout);
  const size_t smem = ((size_t)(R + 8) + 4 * TC_KC * (size_t)R + 2 * TC_KC * (size_t)bn) * sizeof(float);
  dim3 grid(cdiv(Lv, TC_BM), cdiv(P.Cout, bn), tc_groups(P));
  int dev = 0;
  AGPT_CUDA(cudaGetDevice(&dev));
  static bool attr_done_dev[64] = {false};
  bool& attr_done = attr_done_dev[dev & 63];
  if (!attr_done) {
    AGPT_CUDA(cudaFuncSetAttribute(tapconv_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    AGPT_CUDA(cudaFuncSetAttribute(tapconv_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    AGPT_CUDA(cudaFuncSetAttribute(tapconv_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    attr_done = true;
  }
  AGPT_CHECK(smem <= 100 * 1024, "tapconv smem too large (image too wide?)");
  tapconv_note_launch(0, bn, TC_BM, 0, AGPT_TC_KERN_TILE);
  if (bn == 128) tapconv_kernel<128><<<grid, 256, smem, st>>>(P);
  else if (bn == 64) tapconv_kernel<64><<<grid, 128, smem, st>>>(P);
  else tapconv_kernel<32><<<grid, 64, smem, st>>>(P);
}

// Per-launch profiling record (bench.py's roofline leg): algorithmic FLOPs and bytes of one tap-GEMM launch.
// bytes_override > 0 replaces the fp32-tensor byte model (the plane-fed kernel moves fp16 planes).
void* profile_begin(const TapConvParams& P, bool tc, double bytes_override, cudaStream_t st) {
  if (!g_prof) return nullptr;
  g_recs.emplace_back();
  ProfRec* rec = &g_recs.back();
  const int bn = tc_pick_bn(P.Cout);
  rec->variant = tc ? 3 : (bn == 128 ? 0 : (bn == 64 ? 1 : 2));
  const double rows = (double)P.G * P.L;
  rec->flops = 2.0 * rows * P.Cin * P.Cout * P.ntaps * (P.flops_scale > 0.f ? P.flops_scale : 1.f);
  const int out_c = (P.epi == EPI_GATE || P.epi == EPI_GEGLU) ? P.Cout / 2 : P.Cout;
  // an input plane (fp16 hi + lo) moves 4 bytes per element like the fp32 tensor; an output plane adds 4 more, and
  // a plane-only output (out == nullptr) writes no fp32 tensor
  const double out_b = (P.out || !P.po_hi ? 1.0 : 0.0) + (P.po_hi ? 1.0 : 0.0);
  rec->bytes = bytes_override > 0 ? bytes_override
                                  : 4.0 * (rows * P.Cin + out_b * rows * out_c + (P.res ? rows * P.Cout : 0.0) +
                                           (P.epi == EPI_ACC && P.accumulate ? rows * P.Cout : 0.0) +
                                           (double)P.ntaps * P.Cin * P.Cout);
  rec->G = P.G; rec->L = P.L; rec->Cin = P.Cin; rec->Cout = P.Cout; rec->ntaps = P.ntaps; rec->epi = P.epi; rec->Wreal = P.Wreal;
  { int lo = P.tap_off[0], hi = P.tap_off[0];
    for (int t = 1; t < P.ntaps; ++t) { lo = std::min(lo, P.tap_off[t]); hi = std::max(hi, P.tap_off[t]); }
    rec->span = hi - lo; }
  AGPT_CUDA(cudaEventCreate(&rec->e0));
  AGPT_CUDA(cudaEventCreate(&rec->e1));
  AGPT_CUDA(cudaEventRecord(rec->e0, st));
  return rec;
}
// A fused pair (tcpair_launch): the algorithmic FLOPs of both convs (not the recomputed halo rows); bytes of x in,
// the residual, the output (+ the old accumulator) and both weight sets -- the intermediate never reaches HBM.
void* profile_begin_pair(const TapConvParams& c1, const TapConvParams& c2, cudaStream_t st) {
  if (!g_prof) return nullptr;
  const double rows = (double)c1.G * c1.L;
  const double bytes = 4.0 * (rows * c1.Cin + (2.0 + (c2.po_hi ? 1.0 : 0.0)) * rows * c2.Cout +
                              (c2.epi == EPI_ACC && c2.accumulate ? rows * c2.Cout : 0.0) +
                              (double)c1.ntaps * c1.Cin * c1.Cout + (double)c2.ntaps * c2.Cin * c2.Cout);
  ProfRec* rec = static_cast<ProfRec*>(profile_begin(c2, true, bytes, st));
  rec->flops += 2.0 * rows * c1.Cin * c1.Cout * c1.ntaps * (c1.flops_scale > 0.f ? c1.flops_scale : 1.f);
  int lo = c1.tap_off[0], hi = c1.tap_off[0];
  for (int t = 1; t < c1.ntaps; ++t) { lo = std::min(lo, c1.tap_off[t]); hi = std::max(hi, c1.tap_off[t]); }
  rec->ntaps += c1.ntaps;
  rec->span += hi - lo;
  rec->epi += PROF_PAIR;
  return rec;
}
void profile_end(void* r, cudaStream_t st) {
  if (r) AGPT_CUDA(cudaEventRecord(static_cast<ProfRec*>(r)->e1, st));
}

// Dispatch: tensor-core version when the layer has a tensor-core weight image and the operands are
// 16-byte addressable, else the fp32-FMA version.  Both are sm_90a CUDA; there is no other path.
void tapconv_launch(TapConvParams P, cudaStream_t st) {
  AGPT_CHECK(P.ntaps >= 1 && P.ntaps <= kMaxTaps, "ntaps");
  AGPT_CHECK(P.cin_pad % TC_KC == 0 && P.cout_pad % 4 == 0, "padding");
  AGPT_CHECK(P.epi == EPI_STORE_CF || P.out_pitch % (P.epi == EPI_GATE || P.epi == EPI_GEGLU ? 2 : 4) == 0, "pitch");
  const bool tc = tcconv_supported(P);
  AGPT_CHECK(tc || (!P.pi_hi && !P.po_hi), "operand planes need the tensor-core tap-GEMM");
  void* rec = profile_begin(P, tc, 0.0, st);
  if (tc) tcconv_launch(P, st);
  else fma_launch(P, st);
  profile_end(rec, st);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

}  // namespace agpt
