// BinauralNetwork (mono2binaural/src/models.py, warping.py) for the Binaural tool (audio-chatgpt.py:713-773): a
// geometric and a neural time warp of a mono signal to the left and right ear.
//
// Three launches cover every row (batch item or tool chunk) of a call:
//   binaural_frames_kernel  per (row, frame tile): the fp32 frame field f[row][ear][k] = ((-d) / 343) * 48000 + n, d the
//                           mouth-to-ear distance (quaternion step in fp64) and n the warpnet's output.  Nearest
//                           interpolation commutes with the elementwise ops, so selecting f per sample is what the
//                           reference computes per sample.
//   binaural_tilemax_kernel per (row, ear, sample tile): the largest clamped position of the tile, and of its group of
//                           kGroup tiles (an atomic max).
//   binaural_apply_kernel   per (row, ear, sample tile): the running max carried in from the earlier tiles -- at most
//                           kGroup - 1 tile maxima of its own group and one maximum per earlier group, so the carry
//                           costs a bounded number of reads per tile --, a block max-scan, the lerp, and the kept tail
//                           written straight into the output, optionally clamped to [-1, 1].
// The per-sample arithmetic uses explicit round-to-nearest intrinsics, so FMA contraction cannot change a rounding:
// given the same frame field the output is bitwise what the reference's torch ops compute.
#include <cfloat>
#include "models.h"

namespace agpt {
namespace {

constexpr int kViewDim = 7;
constexpr int kFrameTile = 32;           // frames per frames-kernel CTA
constexpr int kFrameThreads = 256;
constexpr int kWarpThreads = 256;
constexpr int kPerThread = 8;
constexpr int kSampleTile = kWarpThreads * kPerThread;
constexpr long kMaxT = 1L << 24;         // the reference's fp32 arange is exact below this
constexpr int kGroup = 64;               // tiles per group of the two-level carry: <= 128 groups per row at kMaxT
constexpr int kMaxLayers = 4, kMaxC = 64;
constexpr int kMaxStaging = 64;          // row-table uploads in flight before a call waits for the oldest

// dynamic shared memory of binaural_frames_kernel: the weights, then two activation buffers [max(C, 7)][tile + halo]
constexpr size_t frames_smem(int layers, int C) {
  return sizeof(float) * ((size_t)kViewDim * C * 2 + (size_t)(layers - 1) * (C * C * 2) + (size_t)layers * C + 2 * C + 2 +
                          2 * (size_t)(C > kViewDim ? C : kViewDim) * (kFrameTile + layers));
}

// a row as the kernels read it: the caller's descriptor and where its frame field starts
struct RowDev {
  agpt_binaural_row r;
  long frame_off;                        // f[row] starts here: [2][K]
};

// F.interpolate(mode = 'nearest', size = T) source frame of sample i (UpSample.h nearest_idx, float scale)
__device__ __forceinline__ long nearest_frame(long i, long K, long T) {
  if (K == T) return i;
  if (T == 2 * K) return i >> 1;
  const float scale = __fdiv_rn((float)K, (float)T);
  const long s = (long)floorf(__fmul_rn((float)i, scale));
  return s < K - 1 ? s : K - 1;
}

// pos = clamp(min(f, 0) + i, 0, T - 1), as -relu(-w), + arange, clamp in the reference
__device__ __forceinline__ float clamped_pos(const float* f, long i, long K, long T) {
  float w = f[nearest_frame(i, K, T)];
  w = -fmaxf(-w, 0.f);
  return fminf(fmaxf(__fadd_rn(w, (float)i), 0.f), (float)(T - 1));
}

__device__ __forceinline__ float block_max(float v, float* red) {
  for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  v = lane < (int)(blockDim.x >> 5) ? red[lane] : -FLT_MAX;
  for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// weights in shared memory: per layer l, w[l] [C][cin][2] then b[l] [C]; then linear [2][C] and its bias [2]
__global__ void __launch_bounds__(kFrameThreads) binaural_frames_kernel(const float* __restrict__ wts, int n_w, int layers, int C,
                                                                        const float* __restrict__ view, const RowDev* __restrict__ rows,
                                                                        float* __restrict__ field) {
  extern __shared__ float sm[];
  const RowDev rd = rows[blockIdx.y];
  const long K = rd.r.K;
  const long k0 = (long)blockIdx.x * kFrameTile;
  if (k0 >= K) return;
  const int W = kFrameTile + layers;               // the tile and its causal halo of `layers` frames
  float* w = sm;
  float* a0 = w + n_w;                              // [max(C, 7)][W]
  float* a1 = a0 + C * W;
  for (int i = threadIdx.x; i < n_w; i += blockDim.x) w[i] = wts[i];
  const float* v = view + rd.r.view_off;
  const long vs = rd.r.view_stride;
  for (int i = threadIdx.x; i < kViewDim * W; i += blockDim.x) {
    const int c = i / W, j = i % W;
    const long k = k0 - layers + j;
    a0[c * W + j] = (k >= 0 && k < K) ? v[c * vs + k] : 0.f;
  }
  __syncthreads();
  // causal convs: out[t] = W0 in[t - 1] + W1 in[t] + b, in[-1] = 0 at every layer (F.pad([1, 0]) before each)
  float* in = a0;
  float* out = a1;
  const float* wl = w;
  int cin = kViewDim;
  for (int l = 0; l < layers; ++l) {
    const float* bl = wl + C * cin * 2;
    for (int i = threadIdx.x; i < C * W; i += blockDim.x) {
      const int c = i / W, j = i % W;
      const long k = k0 - layers + j;
      float acc = bl[c];
      const float* wc = wl + c * cin * 2;
      for (int ci = 0; ci < cin; ++ci) {
        const float prev = j > 0 ? in[ci * W + j - 1] : 0.f;
        acc = fmaf(wc[2 * ci], prev, acc);
        acc = fmaf(wc[2 * ci + 1], in[ci * W + j], acc);
      }
      out[c * W + j] = k >= 0 ? fmaxf(acc, 0.f) : 0.f;
    }
    __syncthreads();
    wl = bl + C;
    cin = C;
    float* t = in; in = out; out = t;
  }
  const float* lw = wl;            // [2][C]
  const float* lb = wl + 2 * C;    // [2]
  for (int jj = threadIdx.x; jj < kFrameTile; jj += blockDim.x) {
    const long k = k0 + jj;
    if (k >= K) continue;
    const int j = jj + layers;
    float n[2];
    for (int e = 0; e < 2; ++e) {
      float acc = lb[e];
      for (int c = 0; c < C; ++c) acc = fmaf(lw[e * C + c], in[c * W + j], acc);
      n[e] = acc;
    }
    // the transmitter's mouth: (0.09, 0, -0.2) rotated by the inverse of the view's quaternion (x, y, z, w), in fp64
    // as scipy's Rotation does, then rounded to fp32; an all-zero quaternion gets +1 on every component first
    float q[4];
    for (int c = 0; c < 4; ++c) q[c] = v[(3 + c) * vs + k];
    if (q[0] == 0.f && q[1] == 0.f && q[2] == 0.f && q[3] == 0.f) q[0] = q[1] = q[2] = q[3] = 1.f;
    double x = q[0], y = q[1], z = q[2], ww = q[3];
    const double nrm = sqrt(x * x + y * y + z * z + ww * ww);
    x /= nrm; y /= nrm; z /= nrm; ww /= nrm;
    const double x2 = x * x, y2 = y * y, z2 = z * z, w2 = ww * ww;
    const double xy = x * y, xz = x * z, xw = x * ww, yz = y * z, yw = y * ww, zw = z * ww;
    const double m[3][3] = {{x2 - y2 - z2 + w2, 2 * (xy - zw), 2 * (xz + yw)},
                            {2 * (xy + zw), -x2 + y2 - z2 + w2, 2 * (yz - xw)},
                            {2 * (xz - yw), 2 * (yz + xw), -x2 - y2 + z2 + w2}};
    const double mo[3] = {0.09, 0.0, -0.20};
    float mouth[3];
    for (int r = 0; r < 3; ++r) mouth[r] = (float)(m[0][r] * mo[0] + m[1][r] * mo[1] + m[2][r] * mo[2]);
    const float ear[2][3] = {{0.f, -0.08f, -0.22f}, {0.f, 0.08f, -0.22f}};
    float* fr = field + rd.frame_off;
    for (int e = 0; e < 2; ++e) {
      float d2 = 0.f;
      for (int c = 0; c < 3; ++c) {
        const float dc = __fsub_rn(__fadd_rn(v[c * vs + k], mouth[c]), ear[e][c]);
        d2 = __fadd_rn(d2, __fmul_rn(dc, dc));
      }
      const float geo = __fmul_rn(__fdiv_rn(-sqrtf(d2), 343.f), 48000.f);
      fr[e * K + k] = __fadd_rn(geo, n[e]);
    }
  }
}

// a group maximum: the call's epoch above the position's bits (positions are >= +0, so their bits order as unsigned).
// A slot left by an earlier call holds a smaller epoch, so the first atomicMax of this call replaces it: no reset pass.
__device__ __forceinline__ unsigned long long group_word(unsigned epoch, float pos) {
  return ((unsigned long long)epoch << 32) | __float_as_uint(__fadd_rn(pos, 0.f));   // -0 -> +0
}

__global__ void __launch_bounds__(kWarpThreads) binaural_tilemax_kernel(const float* __restrict__ field, const RowDev* __restrict__ rows,
                                                                        int max_tiles, int max_groups, unsigned epoch,
                                                                        float* __restrict__ tmax, unsigned long long* __restrict__ gmax) {
  __shared__ float red[32];
  const RowDev rd = rows[blockIdx.y];
  const long T = rd.r.T, K = rd.r.K;
  const long i0 = (long)blockIdx.x * kSampleTile;
  if (i0 >= T) return;
  const float* f = field + rd.frame_off + blockIdx.z * K;
  float m = -FLT_MAX;
  const long a = i0 + (long)threadIdx.x * kPerThread;
  for (int s = 0; s < kPerThread; ++s)
    if (a + s < T) m = fmaxf(m, clamped_pos(f, a + s, K, T));
  m = block_max(m, red);
  if (threadIdx.x == 0) {
    const long re = (long)blockIdx.y * 2 + blockIdx.z;
    tmax[re * max_tiles + blockIdx.x] = m;
    atomicMax(gmax + re * max_groups + blockIdx.x / kGroup, group_word(epoch, m));
  }
}

__global__ void __launch_bounds__(kWarpThreads, 4) binaural_apply_kernel(const float* __restrict__ field, const float* __restrict__ mono,
                                                                      const RowDev* __restrict__ rows, int max_tiles, int max_groups,
                                                                      const float* __restrict__ tmax,
                                                                      const unsigned long long* __restrict__ gmax, int clamp,
                                                                      float* __restrict__ out) {
  __shared__ float red[32];
  const RowDev rd = rows[blockIdx.y];
  const long T = rd.r.T, K = rd.r.K;
  const long i0 = (long)blockIdx.x * kSampleTile;
  if (i0 >= T) return;
  const int e = blockIdx.z;
  const float* f = field + rd.frame_off + e * K;
  // the running max carried in: the largest position of every earlier tile of this row and ear (positions are >= 0),
  // from the earlier tiles of this tile's group and the maxima of the earlier groups (all written by the tilemax launch,
  // which precedes this one in the stream)
  const long re = (long)blockIdx.y * 2 + e;
  const int g = blockIdx.x / kGroup, own = blockIdx.x - g * kGroup;
  const float* tm = tmax + re * max_tiles + (long)g * kGroup;
  const unsigned long long* gm = gmax + re * max_groups;
  float carry = 0.f;
  for (int i = threadIdx.x; i < own + g; i += blockDim.x)
    carry = fmaxf(carry, i < own ? tm[i] : __uint_as_float((unsigned)(gm[i - own] & 0xffffffffull)));
  carry = block_max(carry, red);
  // this thread's samples, their running max, then an exclusive max-scan over the threads of the tile
  const long a = i0 + (long)threadIdx.x * kPerThread;
  float p[kPerThread];
  float run = 0.f;
#pragma unroll
  for (int s = 0; s < kPerThread; ++s) {
    if (a + s < T) run = fmaxf(run, clamped_pos(f, a + s, K, T));
    p[s] = run;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float incl = run;
  for (int o = 1; o < 32; o <<= 1) {
    const float u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl = fmaxf(incl, u);
  }
  __syncthreads();                                   // red is reused after block_max
  if (lane == 31) red[warp] = incl;
  __syncthreads();
  float before = carry;
  for (int w = 0; w < warp; ++w) before = fmaxf(before, red[w]);
  const float ex = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane > 0) before = fmaxf(before, ex);
  const float* x = mono + rd.r.mono_off;
  float* o0 = out + rd.r.out_off + e * rd.r.out_stride - rd.r.keep;
#pragma unroll
  for (int s = 0; s < kPerThread; ++s) {
    const long i = a + s;
    if (i >= T || i < rd.r.keep) continue;
    const float pos = fmaxf(before, p[s]);
    const float fl = floorf(pos);
    const long il = (long)fl;
    long ir = (long)ceilf(pos);
    if (ir > T - 1) ir = T - 1;
    const float alpha = __fsub_rn(pos, fl);
    float y = __fadd_rn(__fmul_rn(__fsub_rn(1.f, alpha), x[il]), __fmul_rn(alpha, x[ir]));
    if (clamp) y = fminf(fmaxf(y, -1.f), 1.f);
    o0[i] = y;
  }
}

// a pinned host copy of one call's row table, reusable once the upload that read it has run
struct Staging {
  RowDev* host = nullptr;
  size_t cap = 0;                                    // RowDev entries
  cudaEvent_t done = nullptr;
};

struct BinauralNet : Handle {
  int layers = 0, C = 0, n_w = 0;
  size_t smem = 0;
  DevBuf w, field, tmax, gmax, rows_dev;
  unsigned epoch = 0;                                // the group maxima's call counter
  // grows to the number of uploads in flight, so a call waits on the GPU only with kMaxStaging of them queued
  std::vector<Staging> staging;
  size_t next_wait = 0;
  ~BinauralNet() override {
    for (Staging& s : staging) {
      if (s.done) cudaEventDestroy(s.done);
      if (s.host) cudaFreeHost(s.host);
    }
  }

  // a staging buffer whose upload has completed (a new one while every buffer is still being read)
  Staging& free_staging(int n) {
    Staging* pick = nullptr;
    for (Staging& s : staging) {
      const cudaError_t q = cudaEventQuery(s.done);
      if (q == cudaSuccess) { pick = &s; break; }
      if (q != cudaErrorNotReady) AGPT_CUDA(q);
      if (cudaPeekAtLastError() == cudaErrorNotReady) (void)cudaGetLastError();   // not an error: do not leave it behind
    }
    if (!pick && staging.size() < (size_t)kMaxStaging) {
      staging.emplace_back();
      pick = &staging.back();
      AGPT_CUDA(cudaEventCreateWithFlags(&pick->done, cudaEventDisableTiming));
    }
    if (!pick) {                                       // kMaxStaging uploads queued: wait for one of them
      pick = &staging[next_wait++ % staging.size()];
      AGPT_CUDA(cudaEventSynchronize(pick->done));
    }
    if (pick->cap < (size_t)n) {
      if (pick->host) AGPT_CUDA(cudaFreeHost(pick->host));
      pick->host = nullptr;
      AGPT_CUDA(cudaMallocHost(&pick->host, sizeof(RowDev) * n));
      pick->cap = n;
    }
    return *pick;
  }

  // validate the rows and stage them, with their frame offsets, on the device (through pinned memory, without waiting
  // on earlier work);
  // also returns the frame-field size and the largest sample- and frame-tile counts of a row, which size the grids
  const RowDev* upload(const agpt_binaural_row* rows, int n, long* total_frames, int* max_tiles, int* max_ftiles, cudaStream_t st) {
    AGPT_CHECK(rows && n >= 1, "no rows");
    AGPT_CHECK(n <= 65535, "at most 65535 rows per call");
    std::vector<RowDev> rd(n);
    long fo = 0, mt = 1, mf = 1;
    for (int i = 0; i < n; ++i) {
      const agpt_binaural_row& r = rows[i];
      AGPT_CHECK(r.T >= 1 && r.T <= kMaxT, "row length T must be in [1, 2^24]");
      AGPT_CHECK(r.K >= 1, "a row needs at least one view frame (F.interpolate refuses an empty input)");
      AGPT_CHECK(r.keep >= 0 && r.keep < r.T, "keep must be in [0, T)");
      AGPT_CHECK(r.mono_off >= 0 && r.view_off >= 0 && r.out_off >= 0 && r.view_stride >= r.K && r.out_stride >= 0,
                 "bad row offsets or strides");
      rd[i].r = r;
      rd[i].frame_off = fo;
      fo += 2 * r.K;
      mt = std::max(mt, cdivl(r.T, kSampleTile));
      mf = std::max(mf, cdivl(r.K, kFrameTile));
    }
    AGPT_CHECK(mt <= 65535 && mf <= (1L << 30), "row too long");
    const size_t words = sizeof(RowDev) * n / sizeof(float);
    Staging& sg = free_staging(n);
    memcpy(sg.host, rd.data(), sizeof(RowDev) * n);
    rows_dev.ensure(words);
    AGPT_CUDA(cudaMemcpyAsync(rows_dev.p, sg.host, sizeof(RowDev) * n, cudaMemcpyHostToDevice, st));
    AGPT_CUDA(cudaEventRecord(sg.done, st));
    *total_frames = fo;
    *max_tiles = (int)mt;
    *max_ftiles = (int)mf;
    return reinterpret_cast<const RowDev*>(rows_dev.p);
  }

  void frames(const float* view, const RowDev* rd, int n, int max_ftiles, float* fieldp, cudaStream_t st) {
    binaural_frames_kernel<<<dim3(max_ftiles, n), kFrameThreads, smem, st>>>(w.p, n_w, layers, C, view, rd, fieldp);
    count_launch(1);
    AGPT_CUDA(cudaGetLastError());
  }

  void warp(const float* fieldp, const float* mono, const RowDev* rd, int n, int max_tiles, int clamp, float* out, cudaStream_t st) {
    const int max_groups = cdiv(max_tiles, kGroup);
    tmax.ensure((size_t)n * 2 * max_tiles);
    const size_t gwords = (size_t)n * 2 * max_groups * 2;     // unsigned long long = two floats
    const size_t had = gmax.n;
    gmax.ensure(gwords);
    if (++epoch == 0) epoch = 1;
    if (gmax.n != had || epoch == 1)                          // fresh memory, or the epoch wrapped: no stale slot may win
      AGPT_CUDA(cudaMemsetAsync(gmax.p, 0, gmax.n * sizeof(float), st));
    auto* gm = reinterpret_cast<unsigned long long*>(gmax.p);
    const dim3 grid(max_tiles, n, 2);
    binaural_tilemax_kernel<<<grid, kWarpThreads, 0, st>>>(fieldp, rd, max_tiles, max_groups, epoch, tmax.p, gm);
    count_launch(1);
    binaural_apply_kernel<<<grid, kWarpThreads, 0, st>>>(fieldp, mono, rd, max_tiles, max_groups, tmax.p, gm, clamp ? 1 : 0, out);
    count_launch(1);
    AGPT_CUDA(cudaGetLastError());
  }
};

BinauralNet* as_binaural(Handle* h) { return static_cast<BinauralNet*>(h); }

}  // namespace

Handle* binaural_create(const agpt_binaural_cfg* cfg, const float* const* W, int nW, int device) {
  DeviceGuard dg_(device);
  AGPT_CHECK(cfg->layers >= 1 && cfg->layers <= kMaxLayers, "BinauralNetwork: warpnet_layers must be in [1, 4]");
  AGPT_CHECK(cfg->channels >= 8 && cfg->channels <= kMaxC && cfg->channels % 8 == 0,
             "BinauralNetwork: warpnet_channels must be a multiple of 8 in [8, 64]");
  std::unique_ptr<BinauralNet> h(new BinauralNet());
  h->magic = kMagicBinaural; h->device = device;
  h->layers = cfg->layers; h->C = cfg->channels;
  const int C = cfg->channels;
  WeightCursor wc{W, nW};
  std::vector<float> w;
  int cin = kViewDim;
  for (int l = 0; l < cfg->layers; ++l) {     // warper.layers.{l}.weight [C][cin][2], .bias [C]
    const float* lw = wc.next(); const float* lb = wc.next();
    w.insert(w.end(), lw, lw + C * cin * 2);
    w.insert(w.end(), lb, lb + C);
    cin = C;
  }
  const float* lw = wc.next(); const float* lb = wc.next();   // warper.linear.weight [2][C][1], .bias [2]
  w.insert(w.end(), lw, lw + 2 * C);
  w.insert(w.end(), lb, lb + 2);
  wc.done();
  h->n_w = (int)w.size();
  AGPT_CHECK(sizeof(float) * w.size() + 2 * sizeof(float) * std::max(C, kViewDim) * (kFrameTile + cfg->layers) ==
             frames_smem(cfg->layers, C), "binaural: weight layout and shared-memory size disagree");
  h->w.upload(w);
  h->smem = frames_smem(cfg->layers, C);
  // the attribute belongs to the kernel on this device, shared by every handle: set it to what the largest covered
  // config needs, never to this handle's own size
  AGPT_CUDA(cudaFuncSetAttribute(binaural_frames_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)frames_smem(kMaxLayers, kMaxC)));
  return h.release();
}

void binaural_forward(Handle* hh, const float* mono, const float* view, const agpt_binaural_row* rows, int n, float* out, int clamp,
                      cudaStream_t st) {
  BinauralNet* h = as_binaural(hh);
  DeviceGuard dg_(h->device);
  long frames;
  int mt, mf;
  const RowDev* rd = h->upload(rows, n, &frames, &mt, &mf, st);
  h->field.ensure((size_t)frames);
  h->frames(view, rd, n, mf, h->field.p, st);
  h->warp(h->field.p, mono, rd, n, mt, clamp, out, st);
}

void binaural_frames(Handle* hh, const float* view, const agpt_binaural_row* rows, int n, float* field, cudaStream_t st) {
  BinauralNet* h = as_binaural(hh);
  DeviceGuard dg_(h->device);
  long frames;
  int mt, mf;
  const RowDev* rd = h->upload(rows, n, &frames, &mt, &mf, st);
  h->frames(view, rd, n, mf, field, st);
}

void binaural_warp(Handle* hh, const float* field, const float* mono, const agpt_binaural_row* rows, int n, float* out, int clamp,
                   cudaStream_t st) {
  BinauralNet* h = as_binaural(hh);
  DeviceGuard dg_(h->device);
  long frames;
  int mt, mf;
  const RowDev* rd = h->upload(rows, n, &frames, &mt, &mf, st);
  h->warp(field, mono, rd, n, mt, clamp, out, st);
}

}  // namespace agpt
