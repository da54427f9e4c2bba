// tcconv v5: the tap-GEMM on the Hopper tensor cores (wgmma) with error-compensated FP16 hi/lo operands.
//
// x = hi + lo with hi = fp16(x), lo = fp16(x - hi): both parts carry an 11-bit significand, so the three
// products x_hi*w_hi + x_lo*w_hi + x_hi*w_lo accumulated in fp32 have a 2^-22 relative truncation error.
//
// Range: fp16 is finite up to 65504.  WEIGHTS are pre-scaled per layer by a power of two so that
// max|w| lands in [2^13, 2^14) (both parts stay normal numbers; the exact inverse scale is applied
// to the accumulator in the epilogue).  ACTIVATIONS are converted with saturation (|x| <= 65504;
// the networks on this path stay orders of magnitude below); below 2^-14 the lo part becomes a
// subnormal, i.e. the absolute representation error of an activation is max(2^-22 |x|, 2^-25).
//
// One CTA = one [MT rows x BN] output tile (MT = 128, or 256 for narrow tiles).  K-major SWIZZLE_128B operand tiles,
// a conv tap = a row-shifted descriptor start address.  Two worker warpgroups convert fp32 activations into the fp16
// hi/lo tiles, then each issues wgmma for its MT / 2 rows (MT / 128 blocks of 64) with the accumulators in registers
// (one wgmma group in flight while the next chunk is converted), then runs the fused epilogue; warp 8 streams the
// weights (cp.async.bulk, mbarrier full/empty ring).  The plane-fed variant (tcconv5_pl_kernel) takes the input as
// pre-split fp16 hi/lo planes: warp 8 also loads them by TMA, and the workers skip the transform.
// The fused-pair kernels and the warp-specialised pipelines further down reuse the phases defined once here (hi/lo
// split, raw staging, one wgmma group, the c1 -> c2 hand-off, accumulator staging, the fused epilogue, a weight-ring
// step), so that every kernel that must match another bit for bit runs the same code for them.
#include "tapconv.cuh"
#include "tapconv_epi.cuh"
#include "tc_common.cuh"
#include "tc_h16.cuh"
#include "tc_tma.cuh"
#include "models.h"

#include <set>

namespace agpt {

namespace {

constexpr int MAX_NA = 4, MAX_NW = 8;
constexpr int kMaxDyn = 227 * 1024 - 256;   // the kernel also has a small static __shared__ block
// per CTA of tcpair2_kernel: two CTAs, each with its static block and the 1 KB the hardware reserves per CTA, share
// the SM's 228 KB
constexpr int kDualDyn = 113 * 1024 - 256;

struct Tc5Smem {
  uint32_t a_hi[MAX_NA], a_lo[MAX_NA], w[MAX_NW], raw[2], rowinfo, rowp, bars, total;
};
// pl: a plane-fed tile (the operand buffers' RRA is pl_rows of the tile's rows), which also has the operand buffers'
// full / empty barriers.  raw_pitch: bytes per row of a raw staging buffer (64 fp32 channels; 32 in tcpair2_kernel).
__host__ __device__ inline void tc5_layout(Tc5Smem& s, int BN, int MT, int RRA, int NA, int NW, int NR, bool pl = false,
                                           int raw_pitch = 256) {
  uint32_t o = 0;
  for (int i = 0; i < MAX_NA; ++i) { s.a_hi[i] = o; if (i < NA) o += RRA * 128; }
  for (int i = 0; i < MAX_NA; ++i) { s.a_lo[i] = o; if (i < NA) o += RRA * 128; }
  for (int i = 0; i < MAX_NW; ++i) { s.w[i] = o; if (i < NW) o += 2 * BN * 128; }
  for (int i = 0; i < 2; ++i) { s.raw[i] = o; if (i < NR) o += RRA * raw_pitch; }
  s.rowinfo = o; o += RRA * 4;
  s.rowp = o; o += MT * 4;
  o = (o + 15) & ~15u;
  s.bars = o; o += 2 * MAX_NW * 8;
  if (pl) o += 2 * MAX_NA * 8;
  s.total = o;
}

// A plane-fed operand chunk arrives as TMA boxes of at most 256 rows (the box limit) and whole 8-row swizzle atoms:
// pl_box_rows(R) rows each, pl_rows(R) >= R in all; the operand buffers of a plane-fed tile hold pl_rows(R) rows.
__host__ __device__ inline int pl_boxes(int R) { return (R + 255) / 256; }
__host__ __device__ inline int pl_box_rows(int R) { const int n = pl_boxes(R); return ((R + n - 1) / n + 7) / 8 * 8; }
__host__ __device__ inline int pl_rows(int R) { return pl_boxes(R) * pl_box_rows(R); }

constexpr int V5_THREADS = 288;   // 8 worker warps = 2 warpgroups (transform, wgmma, epilogue) + warp 8 (weight producer)
constexpr int NWK = 256;          // worker threads

// wgmma width of a BN-column tile: 128 where it divides BN, else 64, else 32 (BN = 96)
__host__ __device__ constexpr int tc5_nb(int bn) { return bn % 128 == 0 ? 128 : (bn % 64 == 0 ? 64 : 32); }

template <int NB>
__device__ __forceinline__ void wgmma_nb(float* d, uint64_t a, uint64_t b) {
  if constexpr (NB == 128) wgmma_n128(d, a, b);
  else if constexpr (NB == 64) wgmma_n64(d, a, b);
  else wgmma_n32(d, a, b);
}

// compiler-only fence on the accumulator registers (no instruction): keeps other code from being moved across the
// asynchronous wgmma that reads and writes them
template <int N>
__device__ __forceinline__ void fence_acc(float* a) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(a[i])::"memory");
}

// tile row of epilogue item i of worker xt, (xt + i NWK) / 8, as base + immediate: the tall tiles read the row table
// with it, so ptxas recomputes each item's row-table address instead of keeping one 64-bit address per item alive from
// one column block to the next (which spills at 168 registers).  The 128-row tiles keep the form they were tuned with.
__device__ __forceinline__ int item_row(int xt, int i) { return (xt >> 3) + i * (NWK / 8); }

constexpr int TC_TALL = 256;                 // rows of a tall tile (BN <= 64 only: the doubled accumulator still fits)
constexpr uint64_t BLK_DESC = (64 * 128) >> 4;   // descriptor start-address step from one 64-row block to the next

// A worker warpgroup's accumulator acc[MB][NJ][NH]: row block b = 64 rows, column block j = NB = 2 NH columns (wgmma
// fragment layout), BN = NJ NB columns in all.
template <int MB, int NJ, int NH>
__device__ __forceinline__ void fence_tile(float (&acc)[MB][NJ][NH]) {
#pragma unroll
  for (int b = 0; b < MB; ++b)
#pragma unroll
    for (int j = 0; j < NJ; ++j) fence_acc<NH>(acc[b][j]);
}
template <int MB, int NJ, int NH>
__device__ __forceinline__ void zero_tile(float (&acc)[MB][NJ][NH]) {
#pragma unroll
  for (int b = 0; b < MB; ++b)
#pragma unroll
    for (int j = 0; j < NJ; ++j)
#pragma unroll
      for (int i = 0; i < NH; ++i) acc[b][j][i] = 0.f;
}

// hi / lo fp16 parts of 8 channels (x0: channels 0..3, x1: 4..7): one 16-byte unit of the hi and of the lo operand tile
__device__ __forceinline__ void split8(const float4 x0, const float4 x1, uint4& h, uint4& l) {
  h.x = split2(x0.x, x0.y, l.x);
  h.y = split2(x0.z, x0.w, l.y);
  h.z = split2(x1.x, x1.y, l.z);
  h.w = split2(x1.z, x1.w, l.w);
}

// Raw fp32 staging of chunk c (channels 64 c ..) of the RRA operand rows into dst, by the NWK worker threads (xt);
// rowinfo[r]: row r's offset in ing, or -1 outside the sample.  Row r = 256 bytes; 16-byte unit u (4 channels) sits at
// slot (u >> 1) + 8 * (u & 1), so that the two units of one 8-channel item are read conflict-free by the transform.
__device__ __forceinline__ void issue_raw(uint8_t* dst, const TapConvParams& P, const float* __restrict__ ing,
                                          const int* rowinfo, int RRA, int c, int xt) {
  const int kv = min(H_KCH, P.Cin - c * H_KCH);          // valid channels of this chunk
  const int nu = ((kv + 15) >> 4) << 2;                  // 16-byte units the MMA k-steps will touch
  for (int idx = xt; idx < RRA * 16; idx += NWK) {
    const int row = idx >> 4, u = idx & 15;
    if (u >= nu) continue;
    const int ch = c * H_KCH + 4 * u;
    const int a = rowinfo[row];
    const bool ok = (a >= 0) && (ch < P.Cin);
    cp_async16_zfill(dst + row * 256 + (((u >> 1) + ((u & 1) << 3)) << 4), ok ? (ing + a + ch) : P.in, ok ? 16u : 0u);
  }
  cp_async_commit_();
}

// One wgmma group of one tap over a resident K-major SWIZZLE_128B operand tile: per k-step, row block b (the operand
// descriptors dah / dal shifted by 64 b rows) and column block j, the products x_hi w_hi + x_lo w_hi + x_hi w_lo into
// acc[b][j]; ws: the weight stage, [hi | lo][BN rows x 128 B].  At most this group stays in flight; the older one has
// then completed, so its weight stage, ring slot rel (-1: none), is released on w_empty[rel].
template <int MB, int NJ, int NH>
__device__ __forceinline__ void mma_group(float (&acc)[MB][NJ][NH], uint64_t dah, uint64_t dal, uint32_t ws, int ksteps,
                                          uint64_t* w_empty, int rel) {
  constexpr int NB = 2 * NH, BN = NJ * NB;
  fence_tile(acc);
  wgmma_fence();
  for (int k = 0; k < ksteps; ++k) {
    const uint64_t ko = (uint64_t)((k * 32) >> 4);
#pragma unroll
    for (int b = 0; b < MB; ++b)
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const uint64_t dwh = make_desc(ws + j * NB * 128) + ko, dwl = make_desc(ws + (BN + j * NB) * 128) + ko;
        const uint64_t ab = ko + b * BLK_DESC;
        wgmma_nb<NB>(acc[b][j], dah + ab, dwh);
        wgmma_nb<NB>(acc[b][j], dal + ab, dwh);
        wgmma_nb<NB>(acc[b][j], dah + ab, dwl);
      }
  }
  wgmma_commit();
  wgmma_wait<1>();
  fence_tile(acc);
  if (rel >= 0 && (threadIdx.x & 31) == 0) mbar_arrive(&w_empty[rel]);
}
// the end of a conv's wgmmas: all completed, the last weight stage, ring slot rel (-1: none), released on w_empty[rel]
template <int MB, int NJ, int NH>
__device__ __forceinline__ void mma_drain(float (&acc)[MB][NJ][NH], uint64_t* w_empty, int rel) {
  wgmma_wait<0>();
  fence_tile(acc);
  if (rel >= 0 && (threadIdx.x & 31) == 0) mbar_arrive(&w_empty[rel]);
}

// Columns cb .. cb + 31 of the accumulator x descale -> the swizzled staging block stg [rows][32 fp32]; r0 / c0: this
// thread's first fragment row (of row block 0) and column.
template <int MB, int NJ, int NH>
__device__ __forceinline__ void stage_block(const float (&acc)[MB][NJ][NH], uint8_t* stg, int cb, int r0, int c0, float dsc) {
  constexpr int NB = 2 * NH;
#pragma unroll
  for (int b = 0; b < MB; ++b) {
    const float* a = &acc[b][cb / NB][4 * ((cb % NB) / 8)];
    const int r = r0 + 64 * b;
#pragma unroll
    for (int i8 = 0; i8 < 4; ++i8) {
      const int col = 8 * i8 + c0;
      *reinterpret_cast<float2*>(stg + sw128(r, col >> 2) + (col & 3) * 4) = make_float2(a[4 * i8] * dsc, a[4 * i8 + 1] * dsc);
      *reinterpret_cast<float2*>(stg + sw128(r + 8, col >> 2) + (col & 3) * 4) =
          make_float2(a[4 * i8 + 2] * dsc, a[4 * i8 + 3] * dsc);
    }
  }
}

// The fused epilogue of a worker-warpgroup tile [MT rows x BN] of P at output columns co0 .. (rowp: a tile row's output
// row, or -1): registers (x inverse weight scale) -> swizzled staging block [MT rows][32 cols] in shared memory (two of
// them, 2 x MT x 128 B inside the first operand buffers, which are free by then: tc5_plan) -> coalesced (row, 16-byte
// chunk) items through the fused epilogue.  wg: the worker warpgroup (rows MT/2 wg .. of the tile).  The
// global READS of the first LA items of a block (residual / old accumulator) are issued one block ahead -- on a 128-row
// tile with LA = 4 for block 0 before the accumulator is complete.  A tall tile, and LA < 4 (tcpair2_kernel, within
// the registers of two CTAs per SM), read block 0 once that block is staged, not next to the whole accumulator, and
// item i + LA once item i is stored.
template <int BN, int MT, int LA, bool PL, int MB, int NJ, int NH>
__device__ __forceinline__ void tile_epilogue(float (&acc)[MB][NJ][NH], const TapConvParams& P, int g, int co0,
                                              const int* rowp, uint8_t* smem, const Tc5Smem& S, int wg, int xt) {
  constexpr bool early = MT == TC_ROWS && LA == 4;
  EpiPre pre[8];
  int pp[8];
  constexpr int nitem = (MT * 8) / NWK;   // 4 items per worker and block (8 on a tall tile)
  const float dsc = P.tc_descale;
  auto load_block = [&](int cb) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = xt + i * NWK;
      pp[i] = (i < LA && i < nitem) ? rowp[early ? idx >> 3 : item_row(xt, i)] : -1;
      if (pp[i] >= 0) epi_load(P, g, pp[i], co0 + cb + 4 * (idx & 7), pre[i]);
    }
  };
  if (early) load_block(0);
  mma_drain(acc, nullptr, -1);
  named_bar_sync(1, NWK);                      // both warpgroups' wgmmas are done reading the operand buffers
  uint8_t* stg0 = smem + S.a_hi[0];
  const int lane = xt & 31, r0 = wg * (MT / 2) + ((xt >> 5) & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
  for (int blk = 0; blk < BN / 32; ++blk) {
    const int cb = blk * 32;
    uint8_t* stg = stg0 + (blk & 1) * (MT * 128);
    stage_block(acc, stg, cb, r0, c0, dsc);
    if (!early && blk == 0) load_block(0);
    named_bar_sync(1, NWK);
    const int jc = xt & 7;                       // all items of this thread share the 4-channel group
    const float4 cv = epi_colvec(P, g, co0 + cb + 4 * jc);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = xt + i * NWK;
      const int row = (idx >> 3) & (MT - 1);   // pp[i] < 0 for i >= LA until read below
      if (pp[i] >= 0)
        epi_store_cv<PL>(P, g, pp[i], co0 + cb + 4 * jc, *reinterpret_cast<const float4*>(stg + sw128(row, jc)), pre[i], cv);
      if (i + LA < nitem) {
        const int idxa = idx + LA * NWK;
        pp[i + LA] = rowp[item_row(xt, i + LA)];
        if (pp[i + LA] >= 0) epi_load(P, g, pp[i + LA], co0 + cb + 4 * (idxa & 7), pre[i + LA]);
      }
    }
    if (cb + 32 < BN) load_block(cb + 32);
    // staging halves alternate; a half is rewritten two blocks later, after the next named
    // barrier, so no extra barrier is needed here
  }
}

// c1 -> c2 hand-off of a fused pair: c1's accumulator becomes c2's operand tile a2 with the arithmetic of c1's EPI_BIAS
// store followed by c2's PRO_LRELU transform (acc * descale + bias, leaky ReLU, hi/lo split), so c2 multiplies the
// operands a separate launch would.  The tile [P2.R rows][C channels] (K-major SWIZZLE_128B: nch2 hi blocks of 64
// channels, then nch2 lo blocks) replaces c1's operand buffers: rows outside the sample are c2's zero padding, channels
// >= C are zero, rows MT .. RR2 - 1 (RR2 = P2.R) feed only the discarded outputs and are zero (written by the nthr
// threads xt).  Lv = P1.L; r0 / c0: this thread's first fragment row and column; qa: the sample row of tile row 0.
// Clears acc for c2.
template <int MT, int MB, int NJ, int NH>
__device__ __forceinline__ void pair_handoff(float (&acc)[MB][NJ][NH], const TapConvParams& P1, const TapConvParams& P2,
                                             uint8_t* a2, int nch2, int RR2, int Lv, int r0, int c0, int qa, int xt, int nthr) {
  constexpr int NB = 2 * NH;
  const int C2 = P2.Cin;
  const uint32_t lo_part = (uint32_t)nch2 * RR2 * 128;   // the hi blocks, then the lo blocks
  const float dsc1 = P1.tc_descale;
#pragma unroll
  for (int j = 0; j < NJ; ++j)
#pragma unroll
    for (int i = 0; i < NB / 8; ++i) {
      const int col = j * NB + 8 * i + c0;   // accumulator fragment layout: see wgmma_n16
      const bool cok = col < C2;
      float2 bv = make_float2(0.f, 0.f);
      if (cok && P1.bias) bv = __ldg(reinterpret_cast<const float2*>(P1.bias + col));
      uint8_t* hi = a2 + (uint32_t)(col >> 6) * RR2 * 128;
#pragma unroll
      for (int b = 0; b < MB; ++b)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = r0 + 64 * b + 8 * h;
          float v0 = 0.f, v1 = 0.f;
          if (cok && qa + r >= 0 && qa + r < Lv) {
            v0 = lrelu(__fadd_rn(__fmul_rn(acc[b][j][4 * i + 2 * h], dsc1), bv.x), P2.slope);
            v1 = lrelu(__fadd_rn(__fmul_rn(acc[b][j][4 * i + 2 * h + 1], dsc1), bv.y), P2.slope);
          }
          uint32_t l;
          const uint32_t hw = split2(v0, v1, l);
          const uint32_t o = sw128(r, (col & 63) >> 3) + (col & 7) * 2;
          *reinterpret_cast<uint32_t*>(hi + o) = hw;
          *reinterpret_cast<uint32_t*>(hi + lo_part + o) = l;
        }
    }
  const int zitems = (RR2 - MT) * 8;         // 16-byte units of rows MT .. RR2 - 1 per block
  for (int idx = xt; idx < zitems * 2 * nch2; idx += nthr) {
    const int blk = idx / zitems, u = idx - blk * zitems;
    *reinterpret_cast<uint4*>(a2 + (uint32_t)blk * RR2 * 128 + MT * 128 + u * 16) = make_uint4(0u, 0u, 0u, 0u);
  }
  zero_tile(acc);
  fence_proxy_async();                       // generic-proxy stores -> visible to c2's wgmma operand reads
}

// Weight stage `it` of a ring of NW slots (smem + w[s]): once the wgmma warps released the slot's previous stage, copy
// `bytes` from src into it, completing on w_full[s].
__device__ __forceinline__ void ring_put(uint8_t* smem, const uint32_t* w, uint64_t* w_full, uint64_t* w_empty, int NW,
                                         int it, const uint8_t* src, uint32_t bytes) {
  const int s = it % NW, n = it / NW;
  if (n >= 1) mbar_wait(&w_empty[s], (uint32_t)((n - 1) & 1));
  mbar_arrive_expect_tx(&w_full[s], bytes);
  bulk_g2s(smem + w[s], src, bytes, &w_full[s]);
}

// Plane-fed operand chunk c (channels 64 c ..) of rows r0 .. r0 + R - 1 of sample g into operand buffer c % NA, hi
// and lo planes, completing on a_full; the buffer's previous chunk must have been released on a_empty first.  Rows
// outside the sample and channels past C load as zeros, which is the conv's zero padding: split(lrelu(0)) = 0.
__device__ __forceinline__ void pl_load_chunk(uint8_t* smem, const Tc5Smem& S, const CUtensorMap* tmh, const CUtensorMap* tml,
                                              uint64_t* a_full, uint64_t* a_empty, int NA, int c, int r0, int g, int R) {
  const int buf = c % NA, nb = pl_boxes(R), br = pl_box_rows(R);
  if (c >= NA) mbar_wait(&a_empty[buf], (uint32_t)((c / NA - 1) & 1));
  mbar_arrive_expect_tx(&a_full[buf], 2u * nb * br * 128u);
  for (int b = 0; b < nb; ++b) {
    tma_load_3d(smem + S.a_hi[buf] + b * br * 128, tmh, c * H_KCH, r0 + b * br, g, &a_full[buf]);
    tma_load_3d(smem + S.a_lo[buf] + b * br * 128, tml, c * H_KCH, r0 + b * br, g, &a_full[buf]);
  }
}

// PL: plane-fed (TapConvParams::pi_hi): the weight producer also loads each 64-channel chunk of the operand planes
// straight into the operand buffers with TMA (tmh / tml), so the workers only issue wgmma and run the epilogue; the
// epilogue may write the output's plane too.  Else the workers convert the fp32 input.
template <int BN, int MT, bool PL>
__device__ __forceinline__ void tcconv5_body(const TapConvParams& P, const CUtensorMap* tmh, const CUtensorMap* tml) {
  constexpr int NB = tc5_nb(BN), NJ = BN / NB, MB = MT / 128;   // MB: 64-row blocks per worker warpgroup
  static_assert(MT == TC_ROWS || (MT == TC_TALL && BN <= 64), "tall tiles are for narrow BN");
  extern __shared__ uint8_t smem_raw_[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw_) + 1023) & ~(uintptr_t)1023);
  const int RRA = P.R, NA = P.tc_na, NW = P.tc_nw, NR = PL ? 0 : P.tc_nr;
  __shared__ Tc5Smem S;
  if (threadIdx.x == 0) {
    if constexpr (PL) tc5_layout(S, BN, MT, pl_rows(RRA), NA, NW, 0, true);
    else tc5_layout(S, BN, MT, RRA, NA, NW, NR);
  }
  __syncthreads();
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S.bars);
  uint64_t* w_full = bars;                // [MAX_NW]
  uint64_t* w_empty = bars + MAX_NW;      // [MAX_NW]
  uint64_t* a_full = bars + 2 * MAX_NW;   // [MAX_NA] plane-fed only: operand chunk landed / operand buffer free
  uint64_t* a_empty = a_full + MAX_NA;
  int* rowinfo = reinterpret_cast<int*>(smem + S.rowinfo);
  int* rowp = reinterpret_cast<int*>(smem + S.rowp);

  const int tid = threadIdx.x, lane = tid & 31;
  // warpgroup index broadcast from lane 0: ptxas then sees the role branches as warpgroup-uniform, which keeps the
  // wgmmas of the worker warpgroups asynchronous instead of serialized
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);   // workers: output rows MT/2 wg .. MT/2 (wg + 1) - 1 of the tile
  const bool is_worker = wg < 2;
  const int xt = tid;                             // worker thread index 0..NWK-1
  const int gz = blockIdx.z, g = tc_sample(P, gz), co0 = blockIdx.y * BN, q0 = blockIdx.x * MT;
  const int Wv = tc_wv(P);
  const int Lv = tc_lv(P);
  const int nchunks = P.tc_chunks_h, ntaps = P.ntaps, total = nchunks * ntaps;
  const int lo = P.lo_al;

  if (tid == 0) {
    for (int i = 0; i < NW; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], NWK / 32); }
    if constexpr (PL)
      for (int i = 0; i < NA; ++i) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], NWK / 32); }
    fence_barrier_init();
  }
  if (is_worker) {
    if constexpr (!PL)
      for (int i = xt; i < RRA; i += NWK) {
        const int r = tc_row_in(P, gz, q0 + lo + i, Wv, Lv);
        rowinfo[i] = r >= 0 ? r * P.in_pitch : -1;
      }
    if (xt < MT) rowp[xt] = tc_row_out(P, gz, q0 + xt, Wv, Lv);   // output row -> real position (or -1)
  }
  __syncthreads();

  if (is_worker) {
    // =========================== worker warps: transform ===========================
    const float* __restrict__ ing = P.in + g * P.in_gstride;
    const float* pvg = (P.pro == PRO_ADDVEC) ? (P.pvec + (long)g * P.pvec_gstride) : nullptr;
    if constexpr (!PL) {
      issue_raw(smem + S.raw[0], P, ing, rowinfo, RRA, 0, xt);
      if (NR == 2 && nchunks > 1) issue_raw(smem + S.raw[1], P, ing, rowinfo, RRA, 1, xt);
    }
    {  // pull the epilogue's global operands (residual / old accumulator) into L2 while the main loop runs
      const float* pf0 = nullptr; long gs0 = 0; int pitch0 = 0;
      const float* pf1 = nullptr; long gs1 = 0; int pitch1 = 0;
      if ((P.epi == EPI_RES || P.epi == EPI_ACC || P.epi == EPI_GATE || P.epi == EPI_GEGLU) && P.res) {
        pf0 = P.res; gs0 = P.res_gstride; pitch0 = P.res_pitch;
      }
      if (P.epi == EPI_ACC && P.accumulate) { pf1 = P.out; gs1 = P.out_gstride; pitch1 = P.out_pitch; }
      if (P.epi == EPI_DIFFOUT) { pf0 = P.out; gs0 = P.out_gstride; pitch0 = P.out_pitch; }
      const int lines = (BN * 4) / 128 > 0 ? (BN * 4) / 128 : 1;     // 128-byte lines per output row
      for (int idx = xt; idx < MT * lines; idx += NWK) {
        const int p = rowp[idx / lines];
        const int co = co0 + (idx % lines) * 32;
        if (p >= 0 && co < P.Cout) {
          if (pf0) asm volatile("prefetch.global.L2 [%0];" ::"l"(pf0 + g * gs0 + (long)p * pitch0 + co));
          if (pf1) asm volatile("prefetch.global.L2 [%0];" ::"l"(pf1 + g * gs1 + (long)p * pitch1 + co));
        }
      }
    }
    // this warpgroup's accumulator: row block b = rows MT/2 wg + 64 b .. + 63, BN columns in NJ blocks of NB (wgmma
    // fragment layout)
    float acc[MB][NJ][NB / 2];
    zero_tile(acc);
    const int items = RRA * 8;
    int it = 0, prev = -1;     // prev: weight stage of the newest wgmma group, released once that group has completed
    for (int c = 0; c < nchunks; ++c) {
      const int buf = c % NA;
      const int rb = (NR == 2) ? (c & 1) : 0;
      const int kv = min(H_KCH, P.Cin - c * H_KCH);
      const int nq = ((kv + 15) >> 4) << 1;                 // 16-byte fp16 chunks (8 channels) the k-steps touch
      const int ksteps = (kv + 15) >> 4;
      if constexpr (PL) {
        mbar_wait(&a_full[buf], (uint32_t)((c / NA) & 1));   // the producer's TMA of chunk c landed
      } else {
        // raw(c) landed?  (with NR == 2 one younger group -- raw(c+1) -- may still be in flight)
        if (NR == 2 && c + 1 < nchunks) asm volatile("cp.async.wait_group 1;" ::: "memory");
        else cp_async_wait_all_();
        // past this barrier raw(c) is visible to every worker, and the wgmmas that last read a_*[buf] (chunk c - NA)
        // have completed in both warpgroups: each warpgroup keeps at most one wgmma group in flight, and none across a
        // chunk boundary when NA == 1
        named_bar_sync(1, NWK);
      }
      uint8_t* ahi = smem + S.a_hi[buf];
      uint8_t* alo = smem + S.a_lo[buf];
      if constexpr (!PL) {
      const uint8_t* rawb = smem + S.raw[rb];
#pragma unroll 2
      for (int idx = xt; idx < items; idx += NWK) {
        const int row = idx >> 3, q = idx & 7;
        if (q >= nq) continue;
        const float4 v0 = *reinterpret_cast<const float4*>(rawb + row * 256 + q * 16);         // channels 8q .. 8q+3
        const float4 v1 = *reinterpret_cast<const float4*>(rawb + row * 256 + 128 + q * 16);   // channels 8q+4 .. 8q+7
        const int ch = c * H_KCH + 8 * q;
        const bool rowok = (P.pro == PRO_ADDVEC) ? (rowinfo[row] >= 0) : true;
        const float4 x0 = pro_apply5(P, v0, rowok && ch < P.Cin, pvg ? (pvg + ch) : nullptr);
        const float4 x1 = pro_apply5(P, v1, rowok && ch + 4 < P.Cin, pvg ? (pvg + ch + 4) : nullptr);
        uint4 h, l;
        split8(x0, x1, h, l);
        const uint32_t o = sw128(row, q);
        *reinterpret_cast<uint4*>(ahi + o) = h;
        *reinterpret_cast<uint4*>(alo + o) = l;
      }
      fence_proxy_async();               // generic-proxy stores -> visible to wgmma operand reads
      named_bar_sync(1, NWK);            // a_*[buf] complete; everyone finished reading raw[rb]
      const int cn = c + NR;
      if (cn < nchunks) issue_raw(smem + S.raw[rb], P, ing, rowinfo, RRA, cn, xt);
      }
      // =========================== worker warps: wgmma over the taps of chunk c ===========================
      // a tap is a start address shifted by rows, a row block one shifted by 64 rows more: every block reuses the
      // weight stage, which is released (one group later) when the group holding all blocks' wgmmas has completed
      const uint32_t ahi0 = smem_u32(ahi) + (uint32_t)(wg * (MT / 2) - lo) * 128u, alo0 = smem_u32(alo) + (uint32_t)(wg * (MT / 2) - lo) * 128u;
      for (int t = 0; t < ntaps; ++t, ++it) {
        const int s = it % NW;
        mbar_wait(&w_full[s], (uint32_t)((it / NW) & 1));
        const uint32_t shift = (uint32_t)P.tap_off[t] * 128u;
        mma_group(acc, make_desc(ahi0 + shift), make_desc(alo0 + shift), smem_u32(smem + S.w[s]), ksteps, w_empty, prev);
        // plane-fed: chunk c - 1's wgmmas have all completed now, so its operand buffer may be refilled
        if (PL && NA > 1 && t == 0 && c > 0 && lane == 0) mbar_arrive(&a_empty[(c - 1) % NA]);
        prev = s;
      }
      if (NA == 1) {
        mma_drain(acc, w_empty, prev);
        if (PL && lane == 0) mbar_arrive(&a_empty[0]);
        prev = -1;
      }
    }
    // =========================== worker warps: epilogue ===========================
    tile_epilogue<BN, MT, 4, PL>(acc, P, g, co0, rowp, smem, S, wg, xt);
  } else if (lane == 0) {
    // =========================== weight producer (warp 8) ===========================
    const uint32_t bytes = 2u * BN * 128u;
    const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(P.w_h) + (size_t)blockIdx.y * (size_t)total * bytes;
    for (int it = 0; it < total; ++it) {
      if constexpr (PL)   // a chunk's operand tile ahead of its first weight stage
        if (it % ntaps == 0) pl_load_chunk(smem, S, tmh, tml, a_full, a_empty, NA, it / ntaps, q0 + lo, gz, RRA);
      ring_put(smem, S.w, w_full, w_empty, NW, it, wsrc + (size_t)it * bytes, bytes);
    }
  }
}

template <int BN, int MT>
__global__ void __launch_bounds__(V5_THREADS, 1) tcconv5_kernel(const __grid_constant__ TapConvParams P) {
  tcconv5_body<BN, MT, false>(P, nullptr, nullptr);
}
// plane-fed: tmh / tml map the input planes P.pi_hi / P.pi_lo (pl_tensor_maps)
template <int BN, int MT>
__global__ void __launch_bounds__(V5_THREADS, 1) tcconv5_pl_kernel(const __grid_constant__ TapConvParams P,
                                                                  const __grid_constant__ CUtensorMap tmh,
                                                                  const __grid_constant__ CUtensorMap tml) {
  tcconv5_body<BN, MT, true>(P, &tmh, &tml);
}

// One ResBlock1 pair, out = x + c2(lrelu(c1(lrelu(x)))), in one CTA per tile (tcpair_launch): the tcconv5 pipeline
// runs c1 over the MT intermediate rows qa .. qa + MT - 1 (qa = q0 + lowest tap of c2), c1's accumulator becomes c2's
// operand tile in shared memory, and the tcconv5 pipeline runs c2 over it; a tile keeps the MT - span(c2) outputs
// that read only those rows.  P1 / P2: the two convs' launch parameters (leaky-ReLU prologue, 1-D rows, one co-tile,
// BN >= C, fp32 input and output); P2's epilogue (EPI_RES / EPI_ACC) writes the output.  The weight producer streams
// c1's stages, then c2's, through one mbarrier ring.
// HALF: c1's input (Cin <= 64: one chunk) is staged in 32-channel halves of 128-byte rows, P1.tc_nr of them in flight
// (tcpair2_kernel: two CTAs per SM, where 256-byte staging rows would not fit).
// c1's chunk loop stays apart from tcconv5_body's: sharing it would make the pair's transform evaluate the PRO_ADDVEC
// row and channel guards of a general prologue, work the pair does not do today.
template <int BN, int MT, bool HALF = false>
__device__ __forceinline__ void tcpair_body(const TapConvParams& P1, const TapConvParams& P2) {
  constexpr int NB = tc5_nb(BN), NJ = BN / NB, MB = MT / 128;
  static_assert(MT == TC_ROWS || (MT == TC_TALL && BN <= 64), "tall tiles are for narrow BN");
  static_assert(!HALF || (MT == TC_ROWS && BN <= 64), "half staging is for 128-row tiles");
  extern __shared__ uint8_t smem_raw_[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw_) + 1023) & ~(uintptr_t)1023);
  const int RRA = P1.R, NA = P1.tc_na, NW = P1.tc_nw, NR = P1.tc_nr;
  __shared__ Tc5Smem S;
  if (threadIdx.x == 0) tc5_layout(S, BN, MT, RRA, NA, NW, NR, false, HALF ? 128 : 256);
  __syncthreads();
  uint64_t* w_full = reinterpret_cast<uint64_t*>(smem + S.bars);
  uint64_t* w_empty = w_full + MAX_NW;
  int* rowinfo = reinterpret_cast<int*>(smem + S.rowinfo);
  int* rowp = reinterpret_cast<int*>(smem + S.rowp);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);   // warpgroup-uniform role branches (see tcconv5_kernel)
  const bool is_worker = wg < 2;
  const int xt = tid;
  int span2 = 0;
  for (int t = 0; t < P2.ntaps; ++t) span2 = max(span2, P2.tap_off[t] - P2.lo_al);
  const int g = blockIdx.z, Lv = P1.L, q0 = blockIdx.x * (MT - span2), qa = q0 + P2.lo_al;
  const int nchunks = P1.tc_chunks_h, total = nchunks * P1.ntaps;
  const int lo = P1.lo_al;

  if (tid == 0) {
    for (int i = 0; i < NW; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], NWK / 32); }
    fence_barrier_init();
  }
  if (is_worker) {
    for (int i = xt; i < RRA; i += NWK) {
      const int r = qa + lo + i;
      rowinfo[i] = (r >= 0 && r < Lv) ? r * P1.in_pitch : -1;
    }
    if (xt < MT) rowp[xt] = (xt < MT - span2 && q0 + xt < Lv) ? q0 + xt : -1;
  }
  __syncthreads();

  if (is_worker) {
    const float* __restrict__ ing = P1.in + g * P1.in_gstride;
    // issue_raw for c1's input, kept as a copy: with issue_raw called here tcpair_kernel<128, 128> compiles to 8 more
    // SASS instructions than with this lambda (ptxas, sm_90a)
    auto issue_raw1 = [&](int c, int rb) {
      uint8_t* dst = smem + S.raw[rb];
      const int kv = min(H_KCH, P1.Cin - c * H_KCH);
      const int nu = ((kv + 15) >> 4) << 2;
      for (int idx = xt; idx < RRA * 16; idx += NWK) {
        const int row = idx >> 4, u = idx & 15;
        if (u >= nu) continue;
        const int ch = c * H_KCH + 4 * u;
        const int a = rowinfo[row];
        const bool ok = (a >= 0) && (ch < P1.Cin);
        cp_async16_zfill(dst + row * 256 + (((u >> 1) + ((u & 1) << 3)) << 4), ok ? (ing + a + ch) : P1.in, ok ? 16u : 0u);
      }
      cp_async_commit_();
    };
    // HALF: 32-channel half h of the input rows into raw[rb], 128 bytes per row.  16-byte unit u (4 channels) of row r
    // sits at slot ((u >> 1) + 4 (u & 1)) ^ 4 ((r >> 2) & 1): the two units of an 8-channel item, and the rows r and
    // r + 4 that one quarter-warp of the transform reads, fall into different banks
    auto issue_half = [&](int h, int rb) {
      uint8_t* dst = smem + S.raw[rb];
      const int nu = (((P1.Cin + 15) >> 4) << 2) - 8 * h;   // units of this half the MMA k-steps touch
      for (int idx = xt; idx < RRA * 8; idx += NWK) {
        const int row = idx >> 3, u = idx & 7;
        if (u >= nu) continue;
        const int ch = h * 32 + 4 * u;
        const int a = rowinfo[row];
        const bool ok = (a >= 0) && (ch < P1.Cin);
        const int slot = ((u >> 1) + ((u & 1) << 2)) ^ (((row >> 2) & 1) << 2);
        cp_async16_zfill(dst + row * 128 + (slot << 4), ok ? (ing + a + ch) : P1.in, ok ? 16u : 0u);
      }
      cp_async_commit_();
    };
    if constexpr (HALF) {
      issue_half(0, 0);
      if (NR == 2) issue_half(1, 1);
    } else {
      issue_raw1(0, 0);
      if (NR == 2 && nchunks > 1) issue_raw1(1, 1);
    }
    {  // the epilogue's residual / old accumulator rows into L2 while the main loop runs
      const int lines = (BN * 4) / 128 > 0 ? (BN * 4) / 128 : 1;
      for (int idx = xt; idx < MT * lines; idx += NWK) {
        const int p = rowp[idx / lines];
        const int co = (idx % lines) * 32;
        if (p >= 0 && co < P2.Cout) {
          asm volatile("prefetch.global.L2 [%0];" ::"l"(P2.res + g * P2.res_gstride + (long)p * P2.res_pitch + co));
          if (P2.epi == EPI_ACC && P2.accumulate)
            asm volatile("prefetch.global.L2 [%0];" ::"l"(P2.out + g * P2.out_gstride + (long)p * P2.out_pitch + co));
        }
      }
    }
    float acc[MB][NJ][NB / 2];   // row block b: rows MT/2 wg + 64 b .. + 63 of the tile
    zero_tile(acc);
    int it = 0, prev = -1;     // prev: weight stage of the newest wgmma group, released once that group has completed
    // wgmma over the taps of one conv and one 64-channel chunk of its operand tile (ahi0 / alo0: this warpgroup's rows)
    auto mma_taps = [&](const TapConvParams& Q, uint32_t ahi0, uint32_t alo0, int ksteps) {
      for (int t = 0; t < Q.ntaps; ++t, ++it) {
        const int s = it % NW;
        mbar_wait(&w_full[s], (uint32_t)((it / NW) & 1));
        const uint32_t shift = (uint32_t)Q.tap_off[t] * 128u;
        mma_group(acc, make_desc(ahi0 + shift), make_desc(alo0 + shift), smem_u32(smem + S.w[s]), ksteps, w_empty, prev);
        prev = s;
      }
    };
    // =========================== c1: transform + wgmma, chunk by chunk ===========================
    for (int c = 0; c < nchunks; ++c) {
      const int buf = c % NA;
      const int rb = (NR == 2) ? (c & 1) : 0;
      const int kv = min(H_KCH, P1.Cin - c * H_KCH);
      const int nq = ((kv + 15) >> 4) << 1;
      if constexpr (!HALF) {
        if (NR == 2 && c + 1 < nchunks) asm volatile("cp.async.wait_group 1;" ::: "memory");
        else cp_async_wait_all_();
        named_bar_sync(1, NWK);
      }
      uint8_t* ahi = smem + S.a_hi[buf];
      uint8_t* alo = smem + S.a_lo[buf];
      if constexpr (HALF) {
      // the chunk's halves: both in flight (NR == 2), or staged one after the other in raw[0]
      const int nh = (kv + 31) >> 5;
      for (int h = 0; h < nh; ++h) {
        if (NR == 2 && h + 1 < nh) asm volatile("cp.async.wait_group 1;" ::: "memory");
        else cp_async_wait_all_();
        named_bar_sync(1, NWK);
        const uint8_t* rawb = smem + S.raw[NR == 2 ? h : 0];
#pragma unroll 2
        for (int idx = xt; idx < RRA * 4; idx += NWK) {
          // a quarter-warp converts items q = 0..3 of rows r and r + 4: its swizzled operand stores hit 8 distinct slots
          const int row = ((idx >> 5) << 3) + ((idx >> 3) & 3) + (((idx >> 2) & 1) << 2), q = idx & 3, qg = 4 * h + q;
          if (qg >= nq) continue;
          const int sw = ((row >> 2) & 1) << 6;
          const float4 x0 = pro_apply5(P1, *reinterpret_cast<const float4*>(rawb + row * 128 + ((q * 16) ^ sw)), true, nullptr);
          const float4 x1 = pro_apply5(P1, *reinterpret_cast<const float4*>(rawb + row * 128 + ((64 + q * 16) ^ sw)), true, nullptr);
          uint4 hv, lv;
          split8(x0, x1, hv, lv);
          const uint32_t o = sw128(row, qg);
          *reinterpret_cast<uint4*>(ahi + o) = hv;
          *reinterpret_cast<uint4*>(alo + o) = lv;
        }
        if (NR == 1 && h + 1 < nh) {
          named_bar_sync(1, NWK);          // everyone finished reading raw[0]
          issue_half(h + 1, 0);
        }
      }
      fence_proxy_async();
      named_bar_sync(1, NWK);
      } else {
      const uint8_t* rawb = smem + S.raw[rb];
#pragma unroll 2
      for (int idx = xt; idx < RRA * 8; idx += NWK) {
        const int row = idx >> 3, q = idx & 7;
        if (q >= nq) continue;
        const float4 x0 = pro_apply5(P1, *reinterpret_cast<const float4*>(rawb + row * 256 + q * 16), true, nullptr);
        const float4 x1 = pro_apply5(P1, *reinterpret_cast<const float4*>(rawb + row * 256 + 128 + q * 16), true, nullptr);
        uint4 h, l;
        split8(x0, x1, h, l);
        const uint32_t o = sw128(row, q);
        *reinterpret_cast<uint4*>(ahi + o) = h;
        *reinterpret_cast<uint4*>(alo + o) = l;
      }
      fence_proxy_async();
      named_bar_sync(1, NWK);
      if (c + NR < nchunks) issue_raw1(c + NR, rb);
      }
      mma_taps(P1, smem_u32(ahi) + (uint32_t)(wg * (MT / 2) - lo) * 128u, smem_u32(alo) + (uint32_t)(wg * (MT / 2) - lo) * 128u,
               (kv + 15) >> 4);
      if (NA == 1) {
        mma_drain(acc, w_empty, prev);
        prev = -1;
      }
    }
    // =========================== c1's epilogue -> c2's operand tile ===========================
    mma_drain(acc, w_empty, prev);
    prev = -1;
    named_bar_sync(1, NWK);                    // both warpgroups' c1 wgmmas are done reading the operand buffers
    const int nch2 = P2.tc_chunks_h;
    uint8_t* a2 = smem + S.a_hi[0];
    const uint32_t lo_part = (uint32_t)nch2 * P2.R * 128;
    const int r0 = wg * (MT / 2) + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
    pair_handoff<MT>(acc, P1, P2, a2, nch2, P2.R, Lv, r0, c0, qa, xt, NWK);
    named_bar_sync(1, NWK);
    // =========================== c2: wgmma over the resident tile ===========================
    for (int c = 0; c < nch2; ++c) {
      const uint32_t ahi0 = smem_u32(a2) + (uint32_t)c * P2.R * 128 + (uint32_t)(wg * (MT / 2) - P2.lo_al) * 128u;
      mma_taps(P2, ahi0, ahi0 + lo_part, (min(H_KCH, P2.Cin - c * H_KCH) + 15) >> 4);
    }
    // =========================== c2's epilogue ===========================
    tile_epilogue<BN, MT, HALF ? 1 : 4, false>(acc, P2, g, 0, rowp, smem, S, wg, xt);
  } else if (lane == 0) {
    // =========================== weight producer (warp 8): c1's stages, then c2's ===========================
    const uint32_t bytes = 2u * BN * 128u;
    const int total2 = P2.tc_chunks_h * P2.ntaps;
    for (int it = 0; it < total + total2; ++it) {
      const uint8_t* src = it < total ? reinterpret_cast<const uint8_t*>(P1.w_h) + (size_t)it * bytes
                                      : reinterpret_cast<const uint8_t*>(P2.w_h) + (size_t)(it - total) * bytes;
      ring_put(smem, S.w, w_full, w_empty, NW, it, src, bytes);
    }
  }
}

template <int BN, int MT>
__global__ void __launch_bounds__(V5_THREADS, 1) tcpair_kernel(const __grid_constant__ TapConvParams P1,
                                                               const __grid_constant__ TapConvParams P2) {
  tcpair_body<BN, MT>(P1, P2);
}
// The same 128-row pair tile with two CTAs per SM (tcpair_plan_dual): one tile's input load, transform, c1 -> c2
// hand-off and epilogue run beside the other tile's wgmmas.  Needs <= 112 registers per thread and <= kDualDyn bytes
// of shared memory.
template <int BN>
__global__ void __launch_bounds__(V5_THREADS, 2) tcpair2_kernel(const __grid_constant__ TapConvParams P1,
                                                                const __grid_constant__ TapConvParams P2) {
  tcpair_body<BN, TC_ROWS, true>(P1, P2);
}

// ---- C = 128 fused pairs with two tiles in flight per CTA (tcpair_pipe_kernel) ----
// tcpair_kernel<128, 128> runs load -> transform -> c1 -> hand-off -> c2 -> epilogue in order, and its 168 registers
// and 70+ KB operand tiles rule out a second CTA per SM.  This kernel splits the roles instead: warpgroups 0-1 only
// issue c1's wgmmas, hand c1's accumulator over to c2's operand tile, issue c2's and dump c2's accumulator (x descale)
// as fp32; warpgroup 2 converts the NEXT tile's input and runs the PREVIOUS tile's epilogue from its dump; warp 12
// streams the weights through one ring across c1, c2 and the tiles.  Each CTA walks a strided sequence of the pair's
// tiles with two operand sets used ping-pong; a set's life is input(t) -> c1 operand -> c2 operand -> fp32 dump(t) ->
// epilogue(t) -> input(t + 2).  Every output row sums the same wgmma products in the same order, and its epilogue
// runs the same float operations, as in tcpair_kernel<128, 128>: the results are bit-identical.
// 4 warpgroups: 2 wgmma, 1 data, 1 whose warp 12 streams the weights.  Launched at 128 registers per thread, the
// warpgroups then rebalance them (setmaxnreg): 2 x 168 (accumulator + hand-off) + 152 (input transform, epilogue) + 24.
// The weights stream in half-stages of 16 KB (P.w_hk: one tap's 32 input channels, k-steps 2 h and 2 h + 1, in
// SWIZZLE_64B rows), one wgmma group each.  A stage is released once the group after it has been issued and its own
// group has completed, so with 32 KB stages a 2-stage ring gave each stage's load one group of wgmmas to arrive in;
// the same 64 KB as 4 half-stages give it three half-groups (1.5 groups), and spare shared memory holds more.
// tcpair_pipe_kernel<true> (the staged form) splits the data warpgroup's work, which bounded the k = 3 pairs: 640
// threads, warpgroup 2 converts each tile's input in place from shared memory, warpgroup 3 runs the epilogue, and of
// the last warpgroup warp 16 streams the weights, warp 17 loads each tile's fp32 input rows by TMA straight into its
// operand set (32-channel boxes, zero outside the sample; box b of row r fills the bytes of row r of operand quarter
// b) and warp 18 loads the residual (the pair's input) by TMA in 32 x 32 boxes through a small ring.  A set's life
// gains one step: ... -> epilogue(t) -> set_free -> TMA input(t + 2).
constexpr int PIPE_THREADS = 512;
constexpr uint32_t PIPE_STAGE = 2u * 128u * 64u;   // bytes of a half-stage: hi and lo, 128 rows x 64 B
// wgmma descriptor of a K-major SWIZZLE_64B tile (8-row groups 512 B apart)
__device__ __forceinline__ uint64_t make_desc64(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(512 >> 4) << 32;
  d |= (uint64_t)2 << 62;
  return d;
}
constexpr int PIPE_MMA = 256, PIPE_DATA = 128;
template <int N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

// operand set s: [hi chunk 0][hi chunk 1][lo chunk 0][lo chunk 1] of R1 rows x 128 B (c1's input), then c2's tile in
// the same form with R2 <= R1 rows, then the dump: 4 column blocks of [128 rows][32 fp32] (64 KB <= 512 R1 B)
// STAGED (tc_pipe == 1): the residual arrives in boxes of 32 rows x 32 fp32 channels (4 KB) through a ring of
// NSP slots after the weight stages and (R1 - 128) / 8 slots in each set past its dump (free once c2 is done).
constexpr int PIPE_MAX_NW = 8, PIPE_MAX_RES = 8;
constexpr uint32_t PIPE_RES_BOX = 32u * 128u, PIPE_DUMP = 128u * 512u;
struct PipeSmem { uint32_t set[2], w[PIPE_MAX_NW], res[PIPE_MAX_RES], bars, total; };
__host__ __device__ inline void pipe_layout(PipeSmem& s, int R1, int NW, int NSP) {
  uint32_t o = 0;
  for (int i = 0; i < 2; ++i) { s.set[i] = o; o += (uint32_t)R1 * 512; }
  for (int i = 0; i < PIPE_MAX_NW; ++i) { s.w[i] = o; if (i < NW) o += PIPE_STAGE; }
  for (int i = 0; i < PIPE_MAX_RES; ++i) { s.res[i] = o; if (i < NSP) o += PIPE_RES_BOX; }
  s.bars = o; o += (2 * PIPE_MAX_NW + 8 + 2 * PIPE_MAX_RES) * 8;
  s.total = o;
}
// STAGED: 5 warpgroups, launched at 96 registers per thread: 2 x 168 (wgmma) + 48 (transform) + 72 (epilogue) + 24
constexpr int PIPE_STAGED_THREADS = 640, PIPE_XF_REGS = 48, PIPE_EPI_REGS = 72;

template <bool STAGED>
__global__ void __launch_bounds__(STAGED ? PIPE_STAGED_THREADS : PIPE_THREADS, 1)
    tcpair_pipe_kernel(const __grid_constant__ TapConvParams P1, const __grid_constant__ TapConvParams P2,
                       const __grid_constant__ CUtensorMap tmx, const __grid_constant__ CUtensorMap tmr) {
  constexpr int BN = 128, MT = TC_ROWS;
  extern __shared__ uint8_t smem_raw_[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw_) + 1023) & ~(uintptr_t)1023);
  const int R1 = P1.R, NW = P1.tc_nw, NSP = P1.tc_na;
  __shared__ PipeSmem S;
  if (threadIdx.x == 0) pipe_layout(S, R1, NW, NSP);
  __syncthreads();
  uint64_t* w_full = reinterpret_cast<uint64_t*>(smem + S.bars);
  uint64_t* w_empty = w_full + PIPE_MAX_NW;
  uint64_t* in_full = w_full + 2 * PIPE_MAX_NW;   // [2] the set holds its tile's c1 operand (data warpgroup -> wgmma)
  uint64_t* acc_full = in_full + 2;           // [2] the set holds its tile's c2 dump (wgmma -> data warpgroup)
  uint64_t* raw_full = acc_full + 2;          // [2] STAGED: the tile's fp32 input rows landed in the set (TMA -> transform)
  uint64_t* set_free = raw_full + 2;          // [2] STAGED: the epilogue is done with the set (epilogue -> TMA)
  uint64_t* res_full = set_free + 2;          // [PIPE_MAX_RES] STAGED: a residual box landed (TMA -> epilogue)
  uint64_t* res_empty = res_full + PIPE_MAX_RES;   // [PIPE_MAX_RES] STAGED: the epilogue is done with it

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);   // warpgroup-uniform role branches (see tcconv5_kernel)
  int span2 = 0;
  for (int t = 0; t < P2.ntaps; ++t) span2 = max(span2, P2.tap_off[t] - P2.lo_al);
  const int Lv = P1.L, MTO = MT - span2, ntx = (Lv + MTO - 1) / MTO, ntiles = ntx * P1.G;
  const int nloc = (int)blockIdx.x < ntiles ? (ntiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;   // this CTA's tiles
  const int lo = P1.lo_al, nch = P1.tc_chunks_h, total1 = 2 * nch * P1.ntaps;   // half-stages per tile
  const int RR2 = P2.R, nch2 = P2.tc_chunks_h, total2 = 2 * nch2 * P2.ntaps;
  auto tile_of = [&](int k, int& g, int& q0) {   // local tile k -> sample g, first output row q0
    const int T = (int)blockIdx.x + k * (int)gridDim.x;
    g = T / ntx;
    q0 = (T - g * ntx) * MTO;
  };

  // STAGED: residual ring of NRS slots; a tile's 4 column blocks x nj row boxes pass through it in order
  const int NSL = (R1 - 128) / 8, NRS = NSP + NSL, nj = (MTO + 31) / 32, NU = 4 * nj;
  auto res_slot = [&](int j, int s) -> uint8_t* {
    return j < NSP ? smem + S.res[j] : smem + S.set[s] + PIPE_DUMP + (uint32_t)(j - NSP) * PIPE_RES_BOX;
  };

  if (tid == 0) {
    for (int i = 0; i < NW; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], PIPE_MMA / 32); }
    for (int i = 0; i < 2; ++i) { mbar_init(&in_full[i], PIPE_DATA); mbar_init(&acc_full[i], PIPE_MMA); }
    if constexpr (STAGED) {
      for (int i = 0; i < 2; ++i) { mbar_init(&raw_full[i], 1); mbar_init(&set_free[i], PIPE_DATA); }
      for (int i = 0; i < NRS; ++i) { mbar_init(&res_full[i], 1); mbar_init(&res_empty[i], PIPE_DATA); }
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg < 2) {
    // =========================== wgmma warpgroups: rows 64 wg .. 64 wg + 63 of each tile ===========================
    setmaxnreg_inc<168>();
    float acc[1][1][BN / 2];
    int it = 0, prev = -1;   // prev: weight stage of the newest wgmma group, released once that group has completed
    // one 64-channel chunk (4 k-steps) in tcpair_body's product order, the k-steps of a tap in two SWIZZLE_64B
    // half-stages: a copy of mma_group's loop for that weight layout
    auto mma_taps = [&](const TapConvParams& Q, uint32_t ahi0, uint32_t alo0) {
      for (int t = 0; t < Q.ntaps; ++t)
        for (int hf = 0; hf < 2; ++hf, ++it) {
          const int s = it % NW;
          mbar_wait(&w_full[s], (uint32_t)((it / NW) & 1));
          const uint32_t shift = (uint32_t)Q.tap_off[t] * 128u;
          const uint64_t dah = make_desc(ahi0 + shift) + 4 * hf, dal = make_desc(alo0 + shift) + 4 * hf;
          const uint32_t ws = smem_u32(smem + S.w[s]);
          fence_tile(acc);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            const uint64_t ko = (uint64_t)((k * 32) >> 4);
            const uint64_t dwh = make_desc64(ws) + ko, dwl = make_desc64(ws + BN * 64) + ko;
            wgmma_n128(acc[0][0], dah + ko, dwh);
            wgmma_n128(acc[0][0], dal + ko, dwh);
            wgmma_n128(acc[0][0], dah + ko, dwl);
          }
          wgmma_commit();
          wgmma_wait<1>();
          fence_tile(acc);
          if (prev >= 0 && lane == 0) mbar_arrive(&w_empty[prev]);
          prev = s;
        }
    };
    const int r0 = wg * (MT / 2) + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
    for (int k = 0; k < nloc; ++k) {
      int g, q0;
      tile_of(k, g, q0);
      const int qa = q0 + P2.lo_al;
      uint8_t* set = smem + S.set[k & 1];
      zero_tile(acc);
      mbar_wait(&in_full[k & 1], (uint32_t)((k >> 1) & 1));
      // c1 over both resident chunks of the input
      for (int c = 0; c < nch; ++c) {
        const uint32_t ahi0 = smem_u32(set) + (uint32_t)c * R1 * 128 + (uint32_t)(wg * (MT / 2) - lo) * 128u;
        mma_taps(P1, ahi0, ahi0 + (uint32_t)nch * R1 * 128);
      }
      mma_drain(acc, w_empty, prev);
      prev = -1;
      named_bar_sync(1, PIPE_MMA);             // both warpgroups' c1 wgmmas are done reading the set
      pair_handoff<MT>(acc, P1, P2, set, nch2, RR2, Lv, r0, c0, qa, tid, PIPE_MMA);
      named_bar_sync(1, PIPE_MMA);
      // c2 over the resident tile
      const uint32_t lo_part = (uint32_t)nch2 * RR2 * 128;
      for (int c = 0; c < nch2; ++c) {
        const uint32_t ahi0 = smem_u32(set) + (uint32_t)c * RR2 * 128 + (uint32_t)(wg * (MT / 2) - P2.lo_al) * 128u;
        mma_taps(P2, ahi0, ahi0 + lo_part);
      }
      mma_drain(acc, w_empty, prev);
      prev = -1;
      named_bar_sync(1, PIPE_MMA);             // both warpgroups' c2 wgmmas are done reading the set
      // accumulator x descale -> the set's dump: one [128][32] staging block per 32 columns
#pragma unroll
      for (int blk = 0; blk < BN / 32; ++blk) stage_block(acc, set + blk * (MT * 128), blk * 32, r0, c0, P2.tc_descale);
      mbar_arrive(&acc_full[k & 1]);
    }
  } else if (STAGED && wg == 2) {
    // ================ transform: the set's fp32 input rows -> c1's hi / lo operand, in place ================
    // Box b (channels 32 b ..) of row r sits in the 128 B of row r of the set's quarter b, the same bytes that hold
    // row r of operand quarter b afterwards, so a half-warp reads all 16 items of its row before any is written.
    setmaxnreg_dec<PIPE_XF_REGS>();
    const int dt = tid - PIPE_MMA, i16 = dt & 15, c = i16 >> 3, q = i16 & 7, odd = q >> 2;
    const uint32_t qsz = (uint32_t)R1 * 128, src = (uint32_t)(2 * c + odd) * qsz;
    for (int k = 0; k < nloc; ++k) {
      const int s = k & 1;
      mbar_wait(&raw_full[s], (uint32_t)((k >> 1) & 1));
      uint8_t* set = smem + S.set[s];
      for (int row = dt >> 4; row < R1; row += PIPE_DATA / 16) {
        // channels 8 q' .. 8 q' + 7 (q' = 8 c + q): 16-byte units 2 (q & 3) and + 1 of box 2 c + q / 4 (TMA
        // SWIZZLE_128B); the upper half-quarter reads its pair odd unit first, off the lower one's banks
        const uint8_t* rr = set + src + row * 128;
        const int u0 = 2 * (q & 3), sw = row & 7;
        const float4 a = *reinterpret_cast<const float4*>(rr + (((u0 + odd) ^ sw) << 4));
        const float4 b = *reinterpret_cast<const float4*>(rr + (((u0 + 1 - odd) ^ sw) << 4));
        __syncwarp();
        const float4 x0 = pro_apply5(P1, odd ? b : a, true, nullptr), x1 = pro_apply5(P1, odd ? a : b, true, nullptr);
        uint4 h, l;
        split8(x0, x1, h, l);
        const uint32_t o = (uint32_t)c * qsz + sw128(row, q);
        *reinterpret_cast<uint4*>(set + o) = h;
        *reinterpret_cast<uint4*>(set + 2 * qsz + o) = l;
      }
      fence_proxy_async();                  // generic-proxy stores -> visible to the wgmma operand reads
      mbar_arrive(&in_full[s]);
    }
  } else if (STAGED && wg == 3) {
    // ================ epilogue: the dump + the residual boxes through c2's fused epilogue (epi_store_cv) ================
    setmaxnreg_dec<PIPE_EPI_REGS>();
    const int dt = tid - PIPE_MMA - PIPE_DATA, jc = dt & 7;
    int n = 0;   // residual boxes consumed so far
    for (int k = 0; k < nloc; ++k) {
      int g, q0;
      tile_of(k, g, q0);
      const int s = k & 1;
      const uint8_t* set = smem + S.set[s];
      mbar_wait(&acc_full[s], (uint32_t)((k >> 1) & 1));
      for (int b = 0; b < 4; ++b) {
        const int co = 32 * b + 4 * jc;
        const uint8_t* stg = set + b * (MT * 128);
        const float4 cv = epi_colvec(P2, g, co);
        for (int j = 0; j < nj; ++j, ++n) {
          float4 ob[2];   // the old MRF sum (EPI_ACC with accumulate), read before the residual box is waited for
          int pp[2];
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int row = 32 * j + (dt >> 3) + 16 * i;
            pp[i] = (row < MTO && q0 + row < Lv) ? q0 + row : -1;
            ob[i] = pp[i] >= 0 ? epi_load_b(P2, g, pp[i], co) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
          const int slot = n % NRS;
          mbar_wait(&res_full[slot], (uint32_t)((n / NRS) & 1));
          const uint8_t* rb = res_slot(slot, s);
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int rl = (dt >> 3) + 16 * i, row = 32 * j + rl;
            EpiPre pre;
            pre.a = *reinterpret_cast<const float4*>(rb + sw128(rl, jc));
            pre.b = ob[i];
            if (pp[i] >= 0) epi_store_cv(P2, g, pp[i], co, *reinterpret_cast<const float4*>(stg + sw128(row, jc)), pre, cv);
          }
          mbar_arrive(&res_empty[slot]);
        }
      }
      fence_proxy_async();                  // the dump's generic stores before the next TMA into the set
      mbar_arrive(&set_free[s]);
    }
  } else if (!STAGED && wg == 2) {
    // =========================== data warpgroup: next tile's input, previous tile's epilogue ===========================
    setmaxnreg_inc<152>();
    const int dt = tid - PIPE_MMA;
    auto transform = [&](int k) {   // fp32 rows -> leaky ReLU -> hi / lo operand chunks of set k & 1 (zeros outside)
      int g, q0;
      tile_of(k, g, q0);
      const int rin = q0 + P2.lo_al + lo;   // input row of operand row 0
      const float* __restrict__ ing = P1.in + g * P1.in_gstride;
      uint8_t* set = smem + S.set[k & 1];
      const int items = R1 * nch * 8;       // (row, chunk, 8-channel group)
#pragma unroll 4
      for (int idx = dt; idx < items; idx += PIPE_DATA) {
        const int row = idx / (nch * 8), c = (idx >> 3) % nch, q = idx & 7;
        const int r = rin + row, ch = c * H_KCH + 8 * q;
        float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0;
        if (r >= 0 && r < Lv && ch < P1.Cin) {
          v0 = ldg_stream(ing + (long)r * P1.in_pitch + ch);
          v1 = ldg_stream(ing + (long)r * P1.in_pitch + ch + 4);
        }
        const float4 x0 = pro_apply5(P1, v0, true, nullptr), x1 = pro_apply5(P1, v1, true, nullptr);
        uint4 h, l;
        split8(x0, x1, h, l);
        const uint32_t o = (uint32_t)c * R1 * 128 + sw128(row, q);
        *reinterpret_cast<uint4*>(set + o) = h;
        *reinterpret_cast<uint4*>(set + (uint32_t)nch * R1 * 128 + o) = l;
      }
      fence_proxy_async();                  // generic-proxy stores -> visible to the wgmma operand reads
      mbar_arrive(&in_full[k & 1]);
    };
    auto epilogue = [&](int k) {   // the set's dump through c2's fused epilogue (epi_store_cv)
      int g, q0;
      tile_of(k, g, q0);
      const uint8_t* set = smem + S.set[k & 1];
      const int jc = dt & 7;
      for (int blk = 0; blk < BN / 32; ++blk) {
        const int cb = blk * 32;
        const uint8_t* stg = set + blk * (MT * 128);
        const float4 cv = epi_colvec(P2, g, cb + 4 * jc);
        for (int h = 0; h < 2; ++h) {   // 8 items per block, the global reads of 4 in flight at a time
          EpiPre pre[4];
          int pp[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int row = (dt + (4 * h + i) * PIPE_DATA) >> 3;
            pp[i] = (row < MTO && q0 + row < Lv) ? q0 + row : -1;
            if (pp[i] >= 0) epi_load(P2, g, pp[i], cb + 4 * jc, pre[i]);
          }
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int row = (dt + (4 * h + i) * PIPE_DATA) >> 3;
            if (pp[i] >= 0)
              epi_store_cv(P2, g, pp[i], cb + 4 * jc, *reinterpret_cast<const float4*>(stg + sw128(row, jc)), pre[i], cv);
          }
        }
      }
    };
    if (nloc > 0) transform(0);
    for (int k = 0; k < nloc; ++k) {
      if (k + 1 < nloc) transform(k + 1);   // into the set tile k - 1 used; its epilogue is done
      mbar_wait(&acc_full[k & 1], (uint32_t)((k >> 1) & 1));
      epilogue(k);
      named_bar_sync(2, PIPE_DATA);         // every data thread is done reading the dump before transform(k + 2)
    }
  } else {
    setmaxnreg_dec<24>();
    constexpr int wwarp = STAGED ? 16 : 12;   // the first warp of the last warpgroup
    if (lane != 0) return;
    if (STAGED && warp == wwarp + 1) {
      // ================ input rows of each tile (TMA, 4 boxes of 32 channels, zero outside the sample) ================
      tma_prefetch_desc(&tmx);
      for (int k = 0; k < nloc; ++k) {
        int g, q0;
        tile_of(k, g, q0);
        const int s = k & 1;
        if (k >= 2) mbar_wait(&set_free[s], (uint32_t)(((k >> 1) - 1) & 1));
        mbar_arrive_expect_tx(&raw_full[s], 4u * R1 * 128u);
        for (int b = 0; b < 4; ++b)
          tma_load_3d(smem + S.set[s] + (uint32_t)b * R1 * 128, &tmx, 32 * b, q0 + P2.lo_al + lo, g, &raw_full[s]);
      }
      return;
    }
    if (STAGED && warp == wwarp + 2) {
      // ================ residual boxes of each tile's output rows (TMA), in the epilogue's order ================
      tma_prefetch_desc(&tmr);
      int n = 0;
      for (int k = 0; k < nloc; ++k) {
        int g, q0;
        tile_of(k, g, q0);
        const int s = k & 1;
        bool c2_done = false;
        for (int u = 0; u < NU; ++u, ++n) {
          const int slot = n % NRS;
          if (n >= NRS) mbar_wait(&res_empty[slot], (uint32_t)((n / NRS - 1) & 1));
          if (slot >= NSP && !c2_done) {   // a slot past the dump: c2's wgmmas are done with the set
            mbar_wait(&acc_full[s], (uint32_t)((k >> 1) & 1));
            c2_done = true;
          }
          mbar_arrive_expect_tx(&res_full[slot], PIPE_RES_BOX);
          tma_load_3d(res_slot(slot, s), &tmr, 32 * (u / nj), q0 + 32 * (u % nj), g, &res_full[slot]);
        }
      }
      return;
    }
    if (warp != wwarp) return;
    // ====================== weight producer: per tile c1's half-stages, then c2's ======================
    int n_it = 0;
    for (int k = 0; k < nloc; ++k)
      for (int it = 0; it < total1 + total2; ++it, ++n_it) {
        const uint8_t* src = it < total1 ? reinterpret_cast<const uint8_t*>(P1.w_hk) + (size_t)it * PIPE_STAGE
                                         : reinterpret_cast<const uint8_t*>(P2.w_hk) + (size_t)(it - total1) * PIPE_STAGE;
        ring_put(smem, S.w, w_full, w_empty, NW, n_it, src, PIPE_STAGE);
      }
  }
}

// ---- narrow fused pairs (BN = 64 / 32) on a persistent, warp-specialised tile pipeline (tcpair_narrow_kernel) ----
// At C <= 64 a pair tile's wgmmas are a small part of its time; the rest is per-row work (input load, hi/lo transform,
// hand-off, epilogue) and the latencies around it, and every tap's wgmmas accumulate in order into one accumulator, a
// dependent chain.  This kernel gives each kind of work its own warps and keeps NS tiles in flight per CTA:
//   warpgroups 0-1  each runs whole tiles (0: tiles 0, 2, ..; 1: tiles 1, 3, ..) in two 64-row accumulators, so four
//                   chains run per SM: c1's wgmmas, the c1 -> c2 hand-off, c2's wgmmas, c2's accumulator x descale ->
//                   fp32 dump
//   warpgroup 2     transform: the staged fp32 input rows -> leaky ReLU -> hi / lo operand tile
//   warpgroup 3     epilogue: the dump + bias + residual (read from the staged input rows: P2.res is P1.in) + the old
//                   MRF sum (EPI_ACC) -> stores; it loads the old sum before the dump is ready
//   warp 16         the input rows of each tile by TMA (32-channel fp32 boxes, zero outside the sample), NS tiles ahead
//   warp 17         the weight stages: all of c1's and c2's loaded once where they fit (NW == iterations per tile),
//                   else streamed through one ring, one pass per pair of tiles, read by both wgmma warpgroups
// Set s (tiles k = s mod NS) is an operand region of 256 R1 bytes (c1's hi / lo tile, then c2's, then the dump) and a
// staging region of R1 x 128 B per 32 input channels; its life is raw(k) -> operand(k) -> c2 operand(k) -> dump(k) ->
// epilogue(k) -> raw(k + NS).  Tile geometry, wgmma shapes and per-row order, operand bits, hand-off and epilogue
// arithmetic are those of tcpair_kernel<BN, 128>, so every output is bit-identical.  Launched at 96 registers per
// thread, the warpgroups rebalance them (setmaxnreg): 2 x 112 (wgmma) + 80 (transform) + 152 (epilogue) + 24.
constexpr int NARROW_THREADS = 640;
constexpr int NARROW_MMA = 256, NARROW_DATA = 128, NARROW_WG = 128;
constexpr int NARROW_MMA_REGS = 112, NARROW_XF_REGS = 80, NARROW_EPI_REGS = 152;   // + 24: 5 x 96 in all
constexpr int NARROW_MAX_NS = 4, NARROW_MAX_NW = 22;
struct NarrowSmem { uint32_t op[NARROW_MAX_NS], raw[NARROW_MAX_NS], w[NARROW_MAX_NW], bars, total; };
__host__ __device__ inline void narrow_layout(NarrowSmem& s, int BN, int R1, int nbox, int NS, int NW) {
  uint32_t o = 0;
  for (int i = 0; i < NARROW_MAX_NS; ++i) { s.op[i] = o; if (i < NS) o += (uint32_t)R1 * 256; }
  for (int i = 0; i < NARROW_MAX_NS; ++i) { s.raw[i] = o; if (i < NS) o += (uint32_t)R1 * 128 * nbox; }
  for (int i = 0; i < NARROW_MAX_NW; ++i) { s.w[i] = o; if (i < NW) o += 2u * BN * 128; }
  s.bars = o; o += (2 * NARROW_MAX_NW + 4 * NARROW_MAX_NS) * 8;
  s.total = o;
}

template <int BN>
__global__ void __launch_bounds__(NARROW_THREADS, 1) tcpair_narrow_kernel(const __grid_constant__ TapConvParams P1,
                                                                          const __grid_constant__ TapConvParams P2,
                                                                          const __grid_constant__ CUtensorMap tmx) {
  constexpr int NB = tc5_nb(BN), MT = TC_ROWS;
  static_assert(NB == BN && BN <= 64, "narrow pairs: one wgmma column block");
  extern __shared__ uint8_t smem_raw_[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw_) + 1023) & ~(uintptr_t)1023);
  const int R1 = P1.R, NS = P1.tc_na, NW = P1.tc_nw, nbox = (P1.Cin + 31) >> 5;
  __shared__ NarrowSmem S;
  if (threadIdx.x == 0) narrow_layout(S, BN, R1, nbox, NS, NW);
  __syncthreads();
  uint64_t* w_full = reinterpret_cast<uint64_t*>(smem + S.bars);
  uint64_t* w_empty = w_full + NARROW_MAX_NW;
  uint64_t* raw_full = w_empty + NARROW_MAX_NW;   // [NS] the tile's input rows landed (TMA -> transform)
  uint64_t* in_full = raw_full + NARROW_MAX_NS;   // [NS] the set holds the tile's c1 operand (transform -> wgmma)
  uint64_t* acc_full = in_full + NARROW_MAX_NS;   // [NS] the set holds the tile's c2 dump (wgmma -> epilogue)
  uint64_t* set_free = acc_full + NARROW_MAX_NS;  // [NS] the epilogue is done with the set (epilogue -> TMA)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);   // warpgroup-uniform role branches (see tcconv5_kernel)
  int span2 = 0;
  for (int t = 0; t < P2.ntaps; ++t) span2 = max(span2, P2.tap_off[t] - P2.lo_al);
  const int Lv = P1.L, MTO = MT - span2, ntx = (Lv + MTO - 1) / MTO, ntiles = ntx * P1.G;
  const int nloc = (int)blockIdx.x < ntiles ? (ntiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  const int lo = P1.lo_al, RR2 = P2.R;
  const int total1 = P1.ntaps, iters = total1 + P2.ntaps;   // one 64-channel chunk per conv
  const bool wres = NW == iters;                            // resident weights: stage it of every tile is stage it
  auto tile_of = [&](int k, int& g, int& q0) {
    const int T = (int)blockIdx.x + k * (int)gridDim.x;
    g = T / ntx;
    q0 = (T - g * ntx) * MTO;
  };

  if (tid == 0) {
    for (int i = 0; i < NW; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], NARROW_MMA / 32); }
    for (int i = 0; i < NS; ++i) {
      mbar_init(&raw_full[i], 1);
      mbar_init(&in_full[i], NARROW_DATA);
      mbar_init(&acc_full[i], NARROW_WG);
      mbar_init(&set_free[i], NARROW_DATA);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg < 2) {
    // ====================== wgmma warpgroups: warpgroup wg runs the whole of tiles wg, wg + 2, .. ======================
    // rows 64 b .. 64 b + 63 of the tile in accumulator b
    setmaxnreg_inc<NARROW_MMA_REGS>();
    float acc[2][1][BN / 2];
    int it = 0, prev = -1;   // prev: weight stage of the newest wgmma group, released once that group has completed
    auto mma_taps = [&](const TapConvParams& Q, uint32_t ahi0, uint32_t alo0, int ksteps) {
      for (int t = 0; t < Q.ntaps; ++t, ++it) {
        const int s = it % NW;
        mbar_wait(&w_full[s], wres ? 0u : (uint32_t)((it / NW) & 1));
        const uint32_t shift = (uint32_t)Q.tap_off[t] * 128u;
        mma_group(acc, make_desc(ahi0 + shift), make_desc(alo0 + shift), smem_u32(smem + S.w[s]), ksteps,
                  w_empty, wres ? -1 : prev);
        prev = s;
      }
    };
    const int bar = 1 + wg, wt = tid - wg * NARROW_WG;   // this warpgroup's named barrier and thread index
    const int r0 = (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
    const uint32_t lo_part = (uint32_t)RR2 * 128;
    int k = wg;
    for (; k < nloc; k += 2) {
      int g, q0;
      tile_of(k, g, q0);
      const int qa = q0 + P2.lo_al, s = k % NS;
      uint8_t* set = smem + S.op[s];
      zero_tile(acc);
      mbar_wait(&in_full[s], (uint32_t)((k / NS) & 1));
      {
        const uint32_t ahi0 = smem_u32(set) + (uint32_t)(-lo) * 128u;
        mma_taps(P1, ahi0, ahi0 + (uint32_t)R1 * 128, (P1.Cin + 15) >> 4);
      }
      mma_drain(acc, w_empty, wres ? -1 : prev);
      prev = -1;
      named_bar_sync(bar, NARROW_WG);          // all of the warpgroup's c1 wgmmas are done reading the set
      pair_handoff<MT>(acc, P1, P2, set, 1, RR2, Lv, r0, c0, qa, wt, NARROW_WG);
      named_bar_sync(bar, NARROW_WG);
      {
        const uint32_t ahi0 = smem_u32(set) + (uint32_t)(-P2.lo_al) * 128u;
        mma_taps(P2, ahi0, ahi0 + lo_part, (P2.Cin + 15) >> 4);
      }
      mma_drain(acc, w_empty, wres ? -1 : prev);
      prev = -1;
      named_bar_sync(bar, NARROW_WG);          // all of the warpgroup's c2 wgmmas are done reading the set
      // accumulator x descale -> the set's dump: one [128][32] staging block per 32 columns
#pragma unroll
      for (int blk = 0; blk < BN / 32; ++blk) stage_block(acc, set + blk * (MT * 128), blk * 32, r0, c0, P2.tc_descale);
      mbar_arrive(&acc_full[s]);
    }
    // The weight ring is shared: the producer streams one pass per pair of tiles and a stage is refilled once both
    // warpgroups released it.  With an odd tile count warpgroup 1 has no tile in the last pair and releases its stages
    // unused.
    if (!wres && k < 2 * ((nloc + 1) / 2))
      for (int t = 0; t < iters; ++t, ++it) {
        const int s = it % NW;
        mbar_wait(&w_full[s], (uint32_t)((it / NW) & 1));
        if (lane == 0) mbar_arrive(&w_empty[s]);
      }
  } else if (wg == 2) {
    // =========================== transform: staged fp32 rows -> c1's hi / lo operand tile ===========================
    setmaxnreg_dec<NARROW_XF_REGS>();
    const int dt = tid - NARROW_MMA;
    const int lq = P1.Cin > 32 ? 3 : (P1.Cin > 16 ? 2 : 1);   // log2 of the 8-channel groups the k-steps touch
    for (int k = 0; k < nloc; ++k) {
      const int s = k % NS;
      mbar_wait(&raw_full[s], (uint32_t)((k / NS) & 1));
      const uint8_t* raw = smem + S.raw[s];
      uint8_t* set = smem + S.op[s];
#pragma unroll 2
      for (int idx = dt; idx < (R1 << lq); idx += NARROW_DATA) {
        const int row = idx >> lq, q = idx & ((1 << lq) - 1);
        // channels 8q .. 8q + 7: 16-byte units 2q, 2q + 1 of box q / 4, in the TMA's SWIZZLE_128B order
        const uint8_t* rr = raw + (uint32_t)(q >> 2) * R1 * 128 + row * 128;
        const int j0 = (2 * q) & 7, sw = row & 7;
        const float4 x0 = pro_apply5(P1, *reinterpret_cast<const float4*>(rr + ((j0 ^ sw) << 4)), true, nullptr);
        const float4 x1 = pro_apply5(P1, *reinterpret_cast<const float4*>(rr + (((j0 + 1) ^ sw) << 4)), true, nullptr);
        uint4 h, l;
        split8(x0, x1, h, l);
        const uint32_t o = sw128(row, q);
        *reinterpret_cast<uint4*>(set + o) = h;
        *reinterpret_cast<uint4*>(set + (uint32_t)R1 * 128 + o) = l;
      }
      fence_proxy_async();                    // generic-proxy stores -> visible to the wgmma operand reads
      mbar_arrive(&in_full[s]);
    }
  } else if (wg == 3) {
    // =========================== epilogue: the dump through c2's fused epilogue ===========================
    setmaxnreg_inc<NARROW_EPI_REGS>();
    const int dt = tid - NARROW_MMA - NARROW_DATA, jc = dt & 7;
    const int roff = -(P1.lo_al + P2.lo_al);   // staged input row of output row 0
    const bool old_sum = P2.epi == EPI_ACC && P2.accumulate;
    for (int k = 0; k < nloc; ++k) {
      int g, q0;
      tile_of(k, g, q0);
      const int s = k % NS;
      const uint8_t* set = smem + S.op[s];
      const uint8_t* raw = smem + S.raw[s];
      // the old MRF sum of every item, read before the dump is ready
      float4 ob[BN / 32][8];
#pragma unroll
      for (int b = 0; b < BN / 32; ++b)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int row = (dt >> 3) + 16 * i;
          ob[b][i] = (old_sum && row < MTO && q0 + row < Lv) ? epi_load_b(P2, g, q0 + row, 32 * b + 4 * jc)
                                                             : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      mbar_wait(&acc_full[s], (uint32_t)((k / NS) & 1));
#pragma unroll
      for (int b = 0; b < BN / 32; ++b) {
        const int co = 32 * b + 4 * jc;
        const uint8_t* stg = set + b * (MT * 128);
        const float4 cv = epi_colvec(P2, g, co);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int row = (dt >> 3) + 16 * i;
          if (row < MTO && q0 + row < Lv) {
            const int rr = row + roff;
            EpiPre pre;
            pre.a = *reinterpret_cast<const float4*>(raw + (uint32_t)b * R1 * 128 + sw128(rr, jc));
            pre.b = ob[b][i];
            epi_store_cv(P2, g, q0 + row, co, *reinterpret_cast<const float4*>(stg + sw128(row, jc)), pre, cv);
          }
        }
      }
      mbar_arrive(&set_free[s]);
    }
  } else {
    setmaxnreg_dec<24>();
    if (lane != 0) return;
    if (warp == 16) {
      // =========================== input rows of each tile (TMA) ===========================
      tma_prefetch_desc(&tmx);
      for (int k = 0; k < nloc; ++k) {
        int g, q0;
        tile_of(k, g, q0);
        const int s = k % NS;
        if (k >= NS) mbar_wait(&set_free[s], (uint32_t)((k / NS - 1) & 1));
        mbar_arrive_expect_tx(&raw_full[s], (uint32_t)nbox * R1 * 128);
        for (int b = 0; b < nbox; ++b)
          tma_load_3d(smem + S.raw[s] + (uint32_t)b * R1 * 128, &tmx, 32 * b, q0 + P2.lo_al + lo, g, &raw_full[s]);
      }
    } else if (warp == 17) {
      // =========================== weight stages: c1's, then c2's ===========================
      const uint32_t bytes = 2u * BN * 128u;
      auto src = [&](int it) {
        return it < total1 ? reinterpret_cast<const uint8_t*>(P1.w_h) + (size_t)it * bytes
                           : reinterpret_cast<const uint8_t*>(P2.w_h) + (size_t)(it - total1) * bytes;
      };
      if (wres) {
        for (int it = 0; it < iters && nloc > 0; ++it) {
          mbar_arrive_expect_tx(&w_full[it], bytes);
          bulk_g2s(smem + S.w[it], src(it), bytes, &w_full[it]);
        }
      } else {
        int n_it = 0;
        for (int j = 0; j < (nloc + 1) / 2; ++j)   // one pass per pair of tiles, read by both wgmma warpgroups
          for (int it = 0; it < iters; ++it, ++n_it) ring_put(smem, S.w, w_full, w_empty, NW, n_it, src(it), bytes);
      }
    }
  }
}

// ---- plane-fed single tap-GEMMs at BN = 128 on a persistent, warp-specialised pipeline (tcconv_pipe_pl_kernel) ----
// tcconv5_pl_kernel<128, 128> runs one tile per CTA in phases: operand load, wgmmas, epilogue; the tensor cores idle
// while a CTA loads and stores, and all CTAs of a wave hit HBM at about the same time.  This kernel splits the roles:
//   warpgroups 0-1  each runs whole units (0: the CTA's units 0, 2, ..; 1: units 1, 3, ..) in two 64-row
//                   accumulators, then the unit's fused epilogue straight from its registers, while the other
//                   warpgroup issues the next unit's wgmmas
//   warp 8          loads each unit's 64-channel hi / lo plane chunks by TMA into a ring of NA operand buffers, and
//                   its weight stages into a ring of NW, in unit order
// Both warpgroups read the two rings, so they take turns: a warpgroup starts a unit's wgmmas once the other one has
// waited for every chunk and stage of the previous unit.  A ring slot's full barrier is then never more than one phase
// ahead of its waiter (a parity wait cannot tell phase m from m + 2), and the tensor cores pass from one unit to the
// next without a gap.
// A unit is one 128-row tile of one 128-wide output-channel tile.  CTA b walks units b, b + grid, .. with the
// output-channel tile varying fastest, so the co-tiles of one row tile run on neighbouring CTAs at the same time and
// all but the first read of those plane rows should hit L2.  When the last round has at most half as many units as CTAs,
// it runs as 64-row half-units (one accumulator block each) on twice as many CTAs.
// Chunk and tap order, the wgmma shapes, the hi.hi, lo.hi, hi.lo order per 64-row block, the descale and the
// epilogue's float operations are those of tcconv5_pl_kernel<128, 128>, so every output is bit-identical.
// Launched at 168 registers per thread, the warpgroups rebalance them (setmaxnreg): 2 x 232 (the 128-register
// accumulator and the epilogue) + 40.
constexpr int CPIPE_THREADS = 384;
constexpr int CPIPE_MMA_REGS = 232, CPIPE_LOAD_REGS = 40;
// operand buffer i: PR hi rows then PR lo rows of 128 B (PR = pl_rows(R)); weight stage i: 32 KB
struct CpipeSmem { uint32_t a[MAX_NA], w[MAX_NW], bars, total; };
__host__ __device__ inline void cpipe_layout(CpipeSmem& s, int PR, int NA, int NW) {
  uint32_t o = 0;
  for (int i = 0; i < MAX_NA; ++i) { s.a[i] = o; if (i < NA) o += (uint32_t)PR * 256; }
  for (int i = 0; i < MAX_NW; ++i) { s.w[i] = o; if (i < NW) o += 2 * 128 * 128; }
  s.bars = o; o += (2 * (MAX_NW + MAX_NA) + 2) * 8;
  s.total = o;
}
// CTAs of a launch of `units` units: every SM, or fewer units than SMs as half-units where twice their count fits
inline int cpipe_grid(int units, int sms) {
  return units >= sms ? sms : (2 * units <= sms ? 2 * units : units);
}

__global__ void __launch_bounds__(CPIPE_THREADS, 1) tcconv_pipe_pl_kernel(const __grid_constant__ TapConvParams P,
                                                                         const __grid_constant__ CUtensorMap tmh,
                                                                         const __grid_constant__ CUtensorMap tml) {
  constexpr int BN = 128, MT = TC_ROWS;
  extern __shared__ uint8_t smem_raw_[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw_) + 1023) & ~(uintptr_t)1023);
  const int NA = P.tc_na, NW = P.tc_nw, PR = pl_rows(P.R);
  __shared__ CpipeSmem S;
  if (threadIdx.x == 0) cpipe_layout(S, PR, NA, NW);
  __syncthreads();
  uint64_t* w_full = reinterpret_cast<uint64_t*>(smem + S.bars);
  uint64_t* w_empty = w_full + MAX_NW;
  uint64_t* a_full = w_empty + MAX_NW;   // [NA] the chunk landed (TMA -> wgmma)
  uint64_t* a_empty = a_full + MAX_NA;   // [NA] its unit's wgmmas are done with it (wgmma -> TMA)
  uint64_t* turn = a_empty + MAX_NA;      // [2] warpgroup wg may start its next unit (the other warpgroup -> wg)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);   // warpgroup-uniform role branches (see tcconv5_kernel)
  const int Lv = P.L, ntx = (Lv + MT - 1) / MT, nct = (P.Cout + BN - 1) / BN;
  const int grid = (int)gridDim.x, cta = (int)blockIdx.x;
  const int units = ntx * P.G * nct, nfull = units / grid, rem = units - nfull * grid;
  const bool split = rem > 0 && 2 * rem <= grid;   // the last round as half-units
  const int nloc = nfull + (cta < (split ? 2 * rem : rem) ? 1 : 0);
  const int nch = P.tc_chunks_h, ntaps = P.ntaps, total = nch * ntaps, lo = P.lo_al;
  // local item k -> sample g, first row q0, co-tile ct, half (-1: all 128 rows, else the 64-row block it runs)
  auto item = [&](int k, int& g, int& q0, int& ct, int& half) {
    int u;
    if (k < nfull) { u = cta + k * grid; half = -1; }
    else if (split) { u = nfull * grid + (cta >> 1); half = cta & 1; }
    else { u = nfull * grid + cta; half = -1; }
    const int rt = u / nct;
    ct = u - rt * nct;
    g = rt / ntx;
    q0 = (rt - g * ntx) * MT;
  };

  if (tid == 0) {
    for (int i = 0; i < NW; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], 4); }
    for (int i = 0; i < NA; ++i) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], 4); }
    for (int i = 0; i < 2; ++i) mbar_init(&turn[i], 4);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg < 2) {
    // =========================== wgmma warpgroups: warpgroup wg runs items wg, wg + 2, .. ===========================
    setmaxnreg_inc<CPIPE_MMA_REGS>();
    float acc[2][BN / 2];   // rows 64 b .. 64 b + 63 of the unit in acc[b]
    const int wt = tid - wg * 128, rw = (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
    const float dsc = P.tc_descale;
    const bool resacc = P.epi != EPI_BIAS, accum = P.epi == EPI_ACC && P.accumulate;
    for (int k = wg; k < nloc; k += 2) {
      int g, q0, ct, half;
      item(k, g, q0, ct, half);
      const int co0 = ct * BN;
      const bool b0 = half != 1, b1 = half != 0;
      {  // the epilogue's residual / old MRF sum rows into L2 while the wgmmas run
        const float* pf0 = (resacc && P.res) ? P.res + g * P.res_gstride : nullptr;
        const float* pf1 = accum ? P.out + g * P.out_gstride : nullptr;
        for (int idx = wt; idx < MT * 4; idx += 128) {
          const int row = idx >> 2, p = q0 + row, co = co0 + (idx & 3) * 32;
          if (p < Lv && co < P.Cout && (row < 64 ? b0 : b1)) {
            if (pf0) asm volatile("prefetch.global.L2 [%0];" ::"l"(pf0 + (long)p * P.res_pitch + co));
            if (pf1) asm volatile("prefetch.global.L2 [%0];" ::"l"(pf1 + (long)p * P.out_pitch + co));
          }
        }
      }
#pragma unroll
      for (int b = 0; b < 2; ++b)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[b][i] = 0.f;
      int prev = -1;   // weight stage of the newest wgmma group, released once that group has completed
      if (k > 0) mbar_wait(&turn[wg], (uint32_t)(((k - 1) >> 1) & 1));   // the other warpgroup's unit k - 1 is issued
      for (int c = 0; c < nch; ++c) {
        const int n = k * nch + c, buf = n % NA;   // n: the CTA's chunk sequence
        mbar_wait(&a_full[buf], (uint32_t)((n / NA) & 1));
        const uint32_t ahi0 = smem_u32(smem + S.a[buf]) - (uint32_t)lo * 128u, alo0 = ahi0 + (uint32_t)PR * 128u;
        const int ksteps = (min(H_KCH, P.Cin - c * H_KCH) + 15) >> 4;
        for (int t = 0; t < ntaps; ++t) {
          const int it = k * total + c * ntaps + t, s = it % NW;   // it: the CTA's weight-stage sequence
          mbar_wait(&w_full[s], (uint32_t)((it / NW) & 1));
          const uint32_t shift = (uint32_t)P.tap_off[t] * 128u;
          const uint64_t dah = make_desc(ahi0 + shift), dal = make_desc(alo0 + shift);
          const uint32_t ws = smem_u32(smem + S.w[s]);
          fence_acc<BN / 2>(acc[0]);
          fence_acc<BN / 2>(acc[1]);
          wgmma_fence();
          for (int kk = 0; kk < ksteps; ++kk) {
            const uint64_t ko = (uint64_t)((kk * 32) >> 4);
            const uint64_t dwh = make_desc(ws) + ko, dwl = make_desc(ws + BN * 128) + ko;
            if (b0) {
              wgmma_n128(acc[0], dah + ko, dwh);
              wgmma_n128(acc[0], dal + ko, dwh);
              wgmma_n128(acc[0], dah + ko, dwl);
            }
            if (b1) {
              wgmma_n128(acc[1], dah + ko + BLK_DESC, dwh);
              wgmma_n128(acc[1], dal + ko + BLK_DESC, dwh);
              wgmma_n128(acc[1], dah + ko + BLK_DESC, dwl);
            }
          }
          wgmma_commit();
          wgmma_wait<1>();
          fence_acc<BN / 2>(acc[0]);
          fence_acc<BN / 2>(acc[1]);
          if (prev >= 0 && lane == 0) mbar_arrive(&w_empty[prev]);
          // chunk n - 1's wgmmas have all completed now, so its operand buffer may be refilled
          if (t == 0 && c > 0 && lane == 0) mbar_arrive(&a_empty[(n - 1) % NA]);
          prev = s;
        }
      }
      if (lane == 0) mbar_arrive(&turn[wg ^ 1]);
      wgmma_wait<0>();
      fence_acc<BN / 2>(acc[0]);
      fence_acc<BN / 2>(acc[1]);
      if (lane == 0) {
        mbar_arrive(&w_empty[prev]);
        mbar_arrive(&a_empty[(k * nch + nch - 1) % NA]);
      }
      // =========================== epilogue, from the accumulator fragments ===========================
      // per element the float operations of tcconv5_body (acc x descale) and epi_store_cv<true> (+ bias,
      // + residual, EPI_ACC: x scale + old sum), explicitly rounded so that no multiply-add is contracted
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        if (!(b ? b1 : b0)) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int p = q0 + 64 * b + rw + 8 * h;
          if (p >= Lv) continue;
          const long ro = g * P.out_gstride + (long)p * P.out_pitch, rr = g * P.res_gstride + (long)p * P.res_pitch;
#pragma unroll
          for (int q = 0; q < 2; ++q) {   // 64 columns at a time: their global reads in flight together
            float2 ra[8], ob[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int co = co0 + 64 * q + 8 * i + c0;
              ra[i] = make_float2(0.f, 0.f);
              ob[i] = ra[i];
              if (co < P.Cout) {
                if (resacc && P.res) ra[i] = __ldg(reinterpret_cast<const float2*>(P.res + rr + co));
                if (accum) ob[i] = *reinterpret_cast<const float2*>(P.out + ro + co);
              }
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int co = co0 + 64 * q + 8 * i + c0;
              if (co >= P.Cout) continue;
              const float* a = &acc[b][4 * (8 * q + i) + 2 * h];
              float2 bv = make_float2(0.f, 0.f);
              if (P.bias) bv = __ldg(reinterpret_cast<const float2*>(P.bias + co));
              float v0 = __fadd_rn(__fmul_rn(a[0], dsc), bv.x), v1 = __fadd_rn(__fmul_rn(a[1], dsc), bv.y);
              if (resacc) { v0 = __fadd_rn(v0, ra[i].x); v1 = __fadd_rn(v1, ra[i].y); }
              if (P.epi == EPI_ACC) {
                v0 = __fadd_rn(__fmul_rn(v0, P.scale), ob[i].x);
                v1 = __fadd_rn(__fmul_rn(v1, P.scale), ob[i].y);
              }
              if (P.out) *reinterpret_cast<float2*>(P.out + ro + co) = make_float2(v0, v1);
              if (P.po_hi) {   // epi_store_plane
                uint32_t l;
                const uint32_t hw = split2(lrelu(v0, P.po_slope), lrelu(v1, P.po_slope), l);
                *reinterpret_cast<uint32_t*>(P.po_hi + ro + co) = hw;
                *reinterpret_cast<uint32_t*>(P.po_lo + ro + co) = l;
              }
            }
          }
        }
      }
    }
  } else {
    setmaxnreg_dec<CPIPE_LOAD_REGS>();
    if (warp != 8 || lane != 0) return;
    // =========================== warp 8: per item its plane chunks and weight stages ===========================
    tma_prefetch_desc(&tmh);
    tma_prefetch_desc(&tml);
    const uint32_t bytes = 2u * BN * 128u;
    const int nb = pl_boxes(P.R), br = pl_box_rows(P.R);
    for (int k = 0; k < nloc; ++k) {
      int g, q0, ct, half;
      item(k, g, q0, ct, half);
      const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(P.w_h) + (size_t)ct * (size_t)total * bytes;
      for (int i = 0; i < total; ++i) {
        if (i % ntaps == 0) {   // a chunk's operand rows ahead of its first weight stage, as pl_load_chunk
          const int c = i / ntaps, n = k * nch + c, buf = n % NA;
          if (n >= NA) mbar_wait(&a_empty[buf], (uint32_t)((n / NA - 1) & 1));
          mbar_arrive_expect_tx(&a_full[buf], 2u * nb * br * 128u);
          for (int bx = 0; bx < nb; ++bx) {
            tma_load_3d(smem + S.a[buf] + bx * br * 128, &tmh, c * H_KCH, q0 + lo + bx * br, g, &a_full[buf]);
            tma_load_3d(smem + S.a[buf] + (PR + bx * br) * 128, &tml, c * H_KCH, q0 + lo + bx * br, g, &a_full[buf]);
          }
        }
        ring_put(smem, S.w, w_full, w_empty, NW, k * total + i, wsrc + (size_t)i * bytes, bytes);
      }
    }
  }
}

// fp16 hi/lo weight image: [co-tile][chunk64][tap][hi | lo][BN rows x 128 B, SWIZZLE_128B], pre-scaled
void build_h_image(const PackedConv& pc, const std::vector<float>& h, int BN, float wscale, DevBuf& dst) {
  const int nct = cdiv(pc.Cout, BN), nch = cdiv(pc.Cin, H_KCH), nt = pc.ntaps;
  const size_t blk = (size_t)BN * 64;  // halves per hi (or lo) block
  std::vector<uint16_t> img((size_t)nct * nch * nt * 2 * blk, 0);
  for (int ct = 0; ct < nct; ++ct)
    for (int c = 0; c < nch; ++c)
      for (int t = 0; t < nt; ++t) {
        uint16_t* hi = &img[((((size_t)ct * nch + c) * nt + t) * 2) * blk];
        uint16_t* lo = hi + blk;
        for (int j = 0; j < BN; ++j) {
          const int co = ct * BN + j;
          if (co >= pc.Cout) continue;
          for (int k = 0; k < H_KCH; ++k) {
            const int ci = c * H_KCH + k;
            if (ci >= pc.Cin) continue;
            const float w = h[((size_t)t * pc.cin_pad + ci) * pc.cout_pad + co] * wscale;
            const __half wh = __float2half_rn(w);
            const __half wl = __float2half_rn(w - __half2float(wh));
            const size_t off = (size_t)j * 64 + (size_t)(((k >> 3) ^ (j & 7)) << 3) + (k & 7);
            memcpy(&hi[off], &wh, 2);
            memcpy(&lo[off], &wl, 2);
          }
        }
      }
  std::vector<float> packed((img.size() + 1) / 2, 0.f);
  memcpy(packed.data(), img.data(), img.size() * 2);
  dst.upload(packed);
}

// fp32 tensor -> operand plane (TapConvParams::pi_hi), for inputs of plane-fed launches that no tap-GEMM epilogue
// wrote: the same lrelu + split2 as the fp32 transform and epi_store_plane, 4 elements per thread
__global__ void plane_split_kernel(const float4* __restrict__ x, uint2* __restrict__ hi, uint2* __restrict__ lo, long n4,
                                  float slope) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
    float4 v = x[i];
    v.x = lrelu(v.x, slope); v.y = lrelu(v.y, slope); v.z = lrelu(v.z, slope); v.w = lrelu(v.w, slope);
    uint2 h, l;
    h.x = split2(v.x, v.y, l.x);
    h.y = split2(v.z, v.w, l.y);
    hi[i] = h;
    lo[i] = l;
  }
}

}  // namespace

void plane_split(const float* x, __half* hi, __half* lo, long n, float slope, cudaStream_t st) {
  AGPT_CHECK(n % 4 == 0, "plane_split: element count must be a multiple of 4");
  const long n4 = n / 4;
  const int blocks = (int)std::min<long>(cdivl(n4, 256), 132L * 16);
  plane_split_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<const float4*>(x), reinterpret_cast<uint2*>(hi),
                                             reinterpret_cast<uint2*>(lo), n4, slope);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
}

// The BN = 128 image of a 128 -> 128 conv in half-stages for tcpair_pipe_kernel: [chunk64][tap][half][hi | lo][128 rows
// x 64 B, SWIZZLE_64B], half h holding input channels 32 h .. 32 h + 31 of the chunk (the k-steps 2 h, 2 h + 1).  The
// same fp16 values as build_h_image's, in 16 KB stages.
static void build_hk_image(const PackedConv& pc, const std::vector<float>& h, float wscale, DevBuf& dst) {
  const int nch = cdiv(pc.Cin, H_KCH), nt = pc.ntaps;
  const size_t blk = (size_t)128 * 32;   // halves per hi (or lo) block
  std::vector<uint16_t> img((size_t)nch * nt * 2 * 2 * blk, 0);
  for (int c = 0; c < nch; ++c)
    for (int t = 0; t < nt; ++t)
      for (int hf = 0; hf < 2; ++hf) {
        uint16_t* hi = &img[((((size_t)c * nt + t) * 2 + hf) * 2) * blk];
        uint16_t* lo = hi + blk;
        for (int j = 0; j < 128; ++j)
          for (int k = 0; k < 32; ++k) {
            const int ci = c * H_KCH + hf * 32 + k;
            const float w = h[((size_t)t * pc.cin_pad + ci) * pc.cout_pad + j] * wscale;
            const __half wh = __float2half_rn(w);
            const __half wl = __float2half_rn(w - __half2float(wh));
            const size_t off = (size_t)j * 32 + (size_t)(((k >> 3) ^ ((j >> 1) & 3)) << 3) + (k & 7);
            memcpy(&hi[off], &wh, 2);
            memcpy(&lo[off], &wl, 2);
          }
      }
  std::vector<float> packed((img.size() + 1) / 2, 0.f);
  memcpy(packed.data(), img.data(), img.size() * 2);
  dst.upload(packed);
}

void pack_h_weights(PackedConv& pc, const std::vector<float>& h) {
  float mx = 0.f;
  for (float v : h) mx = std::max(mx, std::fabs(v));
  int e = 0;
  float wscale = 1.f;
  if (mx > 0.f && std::isfinite(mx)) {
    std::frexp(mx, &e);                       // mx = m * 2^e, m in [0.5, 1)  ->  mx * 2^(14 - e) in [2^13, 2^14)
    wscale = std::ldexp(1.f, std::max(-60, std::min(60, 14 - e)));
  }
  pc.h_descale = 1.f / wscale;
  pc.h_chunks = cdiv(pc.Cin, H_KCH);
  build_h_image(pc, h, pc.tc_bn, wscale, pc.w_h);
  if (pc.tc_bn == 128) build_h_image(pc, h, 64, wscale, pc.w_h64);   // narrower tiles for launches that would not fill the SMs
  if (pc.tc_bn == 128 && pc.Cout > 128) build_h_image(pc, h, 96, wscale, pc.w_h96);
  if (pc.tc_bn == 128 && pc.Cin == 128 && pc.Cout == 128 && !pc.is2d) build_hk_image(pc, h, wscale, pc.w_hk);
}

// lo_al = the lowest tap offset, R = operand-tile rows (MT + tap span, rounded to the 8-row swizzle atom); returns the span
static int tc5_rows(TapConvParams& P, int MT) {
  int lo = P.tap_off[0], hi = P.tap_off[0];
  for (int t = 1; t < P.ntaps; ++t) { lo = std::min(lo, P.tap_off[t]); hi = std::max(hi, P.tap_off[t]); }
  P.lo_al = lo;
  P.R = round_up(MT + (hi - lo), 8);
  return hi - lo;
}

// Shared-memory plan of a BN x MT tile (operand, raw-staging and weight-ring buffers) for P after tc5_rows; false when
// it does not fit.  a_min: bytes the operand buffers must span at least; iters: weight stages the kernel streams.
// A plane-fed tile (P.pi_hi) has no raw staging; its operand buffers hold pl_rows(R) rows, and it keeps up to every
// chunk of the operand resident (TMA loads run ahead of the wgmmas), as long as a 4-stage weight ring still fits.
static bool tc5_plan(TapConvParams& P, int BN, int MT, long a_min, int iters, size_t& smem) {
  const int RRA = P.R;
  const bool pl = P.pi_hi != nullptr;
  P.tc_bn = BN;
  const long avail = (long)kMaxDyn - 1024 /*align*/ - (RRA * 4 + MT * 4 + 512) /*row tables + barriers*/;
  const long abytes = 2L * (pl ? pl_rows(RRA) : RRA) * 128, wbytes = 2L * BN * 128;
  const long rbytes = (long)RRA * 256;
  const long stg = 2L * MT * 128;   // the epilogue stages 2 x [MT][32] fp32 through the operand buffers
  const int nch = P.tc_chunks_h;
  int NA = pl ? MAX_NA : ((P.ntaps == 1) ? 3 : 2);
  NA = std::max(1, std::min(NA, nch));
  if ((long)NA * abytes < stg) NA = (int)cdiv(stg, abytes);
  int NR = pl ? 0 : ((nch > 1) ? 2 : 1);
  auto fits4 = [&](int na) { return na * abytes + 4 * wbytes <= avail; };
  while (pl && NA > 2 && !fits4(NA) && (NA - 1) * abytes >= stg) --NA;
  auto fits = [&](int na, int nr, int nw) { return na * abytes + nr * rbytes + nw * wbytes <= avail; };
  if (!fits(NA, NR, 2) && NA == 3) NA = 2;
  if (!fits(NA, NR, 2) && NR == 2) NR = 1;
  if (!fits(NA, NR, 2) && NA == 2 && abytes >= stg) NA = 1;
  if (NA * abytes < a_min) {
    NA = (int)cdiv(a_min, abytes);
    if (!fits(NA, NR, 2) && NR == 2) NR = 1;
  }
  if (NA > MAX_NA || !fits(NA, NR, 2)) return false;
  int NW = (int)std::min<long>(MAX_NW, (avail - NA * abytes - NR * rbytes) / wbytes);
  NW = std::max(2, std::min(NW, std::max(2, iters)));
  P.tc_na = NA; P.tc_nw = NW; P.tc_nr = NR;
  Tc5Smem S;
  tc5_layout(S, BN, MT, pl ? pl_rows(RRA) : RRA, NA, NW, NR, pl);
  smem = (size_t)S.total + 1024;
  return smem <= (size_t)kMaxDyn;
}

// Shared-memory plan of tcpair2_kernel for P (c1 of a pair, after tc5_rows) within kDualDyn: operand buffers of at
// least a_min bytes (c2's resident tile) and the epilogue's staging, the raw input in 32-channel halves of 128-byte rows
// (both in flight where they fit, else one after the other), and as many weight stages as the rest holds, at least 2.
// False when it does not fit or c1 has more than one 64-channel chunk.
static bool tcpair_plan_dual(TapConvParams& P, int BN, long a_min, int iters, size_t& smem) {
  if (P.tc_chunks_h != 1) return false;
  const long abytes = 2L * P.R * 128, wbytes = 2L * BN * 128;
  const int NA = (int)cdiv(std::max(a_min, 2L * TC_ROWS * 128), abytes);
  if (NA > MAX_NA) return false;
  for (int NR = cdiv(P.Cin, 32); NR >= 1; --NR) {
    Tc5Smem S;
    tc5_layout(S, BN, TC_ROWS, P.R, NA, 2, NR, false, 128);
    const long spare = (long)kDualDyn - 1024 - S.total;
    if (spare < 0) continue;
    const int NW = (int)std::min<long>(std::min<long>(MAX_NW, std::max(2, iters)), 2 + spare / wbytes);
    tc5_layout(S, BN, TC_ROWS, P.R, NA, NW, NR, false, 128);
    P.tc_bn = BN; P.tc_na = NA; P.tc_nw = NW; P.tc_nr = NR;
    smem = (size_t)S.total + 1024;
    return smem <= (size_t)kDualDyn;
  }
  return false;
}

// Dynamic shared-memory limit of a tap-GEMM kernel, set once per kernel and device: kMaxDyn, or for tcpair2_kernel
// (dual) kDualDyn with the max-shared carveout, so that two CTAs fit an SM.  Occupancy queries depend on it too.
static void tc_func_attrs(const void* kern, bool dual) {
  int dev = 0;
  AGPT_CUDA(cudaGetDevice(&dev));
  static std::set<std::pair<const void*, int>> done;
  if (done.count({kern, dev})) return;
  AGPT_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, dual ? kDualDyn : kMaxDyn));
  if (dual) AGPT_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  done.insert({kern, dev});
}
template <typename... KArgs, typename... Args>
static void tc_launch(void (*kern)(KArgs...), bool dual, dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  tc_func_attrs(reinterpret_cast<const void*>(kern), dual);
  kern<<<grid, block, smem, st>>>(std::forward<Args>(args)...);
  AGPT_CUDA(cudaGetLastError());
}

// the instantiation of each tile-kernel family for a BN-column, MT-row tile (BN <= 64 for MT = TC_TALL)
static auto tcconv5_kern(int BN, int MT) {
  if (MT == TC_TALL) return BN == 64 ? tcconv5_kernel<64, TC_TALL> : tcconv5_kernel<32, TC_TALL>;
  return BN == 128 ? tcconv5_kernel<128, TC_ROWS>
                   : BN == 96 ? tcconv5_kernel<96, TC_ROWS> : BN == 64 ? tcconv5_kernel<64, TC_ROWS> : tcconv5_kernel<32, TC_ROWS>;
}
static auto tcconv5_pl_kern(int BN, int MT) {
  if (MT == TC_TALL) return BN == 64 ? tcconv5_pl_kernel<64, TC_TALL> : tcconv5_pl_kernel<32, TC_TALL>;
  return BN == 128 ? tcconv5_pl_kernel<128, TC_ROWS>
                   : BN == 96 ? tcconv5_pl_kernel<96, TC_ROWS>
                              : BN == 64 ? tcconv5_pl_kernel<64, TC_ROWS> : tcconv5_pl_kernel<32, TC_ROWS>;
}
static auto tcpair_kern(int BN, int MT) {
  if (MT == TC_TALL) return BN == 64 ? tcpair_kernel<64, TC_TALL> : tcpair_kernel<32, TC_TALL>;
  return BN == 128 ? tcpair_kernel<128, TC_ROWS> : BN == 64 ? tcpair_kernel<64, TC_ROWS> : tcpair_kernel<32, TC_ROWS>;
}

static int tc5_sms() {
  int dev = 0;
  AGPT_CUDA(cudaGetDevice(&dev));
  static int sms_dev[64] = {0};
  if (!sms_dev[dev & 63]) AGPT_CUDA(cudaDeviceGetAttribute(&sms_dev[dev & 63], cudaDevAttrMultiProcessorCount, dev));
  return sms_dev[dev & 63];
}

// 256-row tiles: the handle allows them (TapConvParams::tc_tall), the tile is narrow (a BN = 128 accumulator doubled
// would spill), the conv runs over plain 1-D rows, and the grid of tall tiles still fills every SM four times over.
// A tall tile pays the fixed per-tile latency (operand load, first weight stage, epilogue) once for twice the rows and
// reuses every weight stage across twice the rows.
static bool tc5_tall(const TapConvParams& P, int bn, long tall_tiles, int sms) {
  return P.tc_tall && bn <= 64 && !P.Wreal && !P.strips && tall_tiles >= 4L * sms;
}

// Tensor maps of P's input planes (P.pi_hi / pi_lo) for boxes of 64 channels x pl_box_rows(P.R) rows (after tc5_rows)
struct PlMaps { CUtensorMap hi, lo; };
static PlMaps pl_tensor_maps(const TapConvParams& P) {
  AGPT_CHECK(!P.Wreal && !P.strips, "plane-fed tap-GEMMs run over plain 1-D rows");
  PlMaps m;
  const int br = pl_box_rows(P.R);
  AGPT_CHECK(tma_encode_rows_h(&m.hi, P.pi_hi, P.Cin, P.L, P.G, P.in_pitch, P.in_gstride, br) &&
                 tma_encode_rows_h(&m.lo, P.pi_lo, P.Cin, P.L, P.G, P.in_pitch, P.in_gstride, br),
             "cannot encode the operand-plane tensor maps");
  return m;
}

// Try one tile shape; returns false when it does not fit the shared-memory budget.
static bool tcconv5_try(TapConvParams P, int BN, int MT, cudaStream_t st) {
  tc5_rows(P, MT);
  size_t smem = 0;
  if (!tc5_plan(P, BN, MT, 0, P.tc_chunks_h * P.ntaps, smem)) return false;
  const int Lv = tc_lv(P);
  dim3 grid(cdiv(Lv, MT), cdiv(P.Cout, BN), tc_groups(P));
  tapconv_note_launch(1, BN, MT, P.pi_hi ? 1 : 0, AGPT_TC_KERN_TILE);
  if (P.pi_hi) {
    const PlMaps m = pl_tensor_maps(P);
    tc_launch(tcconv5_pl_kern(BN, MT), false, grid, dim3(V5_THREADS), smem, st, P, m.hi, m.lo);
  } else {
    tc_launch(tcconv5_kern(BN, MT), false, grid, dim3(V5_THREADS), smem, st, P);
  }
  if (MT == TC_TALL) profile_count_tall();
  if (P.pi_hi) profile_count_plane();
  return true;
}

// Tile width: the candidate (native 128|64|32, or 96 and 64 for native-128 layers) with the smallest waves x per-tile
// cost, where waves = ceil(tiles / SMs): wider tiles amortise the activation operand, narrower ones fill the SMs.  No
// 256-wide tile: its accumulator (128 registers per thread of a warpgroup) spills next to the transform's registers.
// Tile height: 256 rows where tc5_tall allows it, else 128.
HTile pick_h_tile(const TapConvParams& P, int sms) {
  const int Lv = tc_lv(P);
  const long rt = (long)cdiv(Lv, TC_ROWS) * tc_groups(P);
  auto cost = [](int bn) { return bn == 128 ? 1.0 : (bn == 96 ? 0.82 : (bn == 64 ? 0.62 : 0.45)); };
  HTile best{P.tc_bn, P.w_h, rt * cdiv(P.Cout, P.tc_bn), TC_ROWS};
  double bs = (double)cdiv(best.ntiles, (long)sms) * cost(P.tc_bn);
  auto consider = [&](int bn, const float* w) {
    if (!w) return;
    const long nt = rt * cdiv(P.Cout, bn);
    const double sc = (double)cdiv(nt, (long)sms) * cost(bn);
    if (sc < bs - 1e-9) { bs = sc; best = HTile{bn, w, nt, TC_ROWS}; }
  };
  if (P.tc_bn == 128) consider(64, P.w_h64);
  if (P.tc_bn == 128) consider(96, P.w_h96);     // e.g. 640 channels on 16 row tiles: 112 tiles in one wave
  const long tall = (long)cdiv(Lv, TC_TALL) * tc_groups(P) * cdiv(P.Cout, best.bn);
  if (tc5_tall(P, best.bn, tall, sms)) { best.mt = TC_TALL; best.ntiles = tall; }
  return best;
}

// One launch of tcpair_kernel<BN, MT>, or with dual of tcpair2_kernel<BN> (MT = 128); false -- nothing launched -- when
// it does not fit shared memory, or (dual) the SM does not take two CTAs of it.
static bool tcpair_try(TapConvParams P1, TapConvParams P2, int MT, bool dual, cudaStream_t st) {
  const int BN = P1.tc_bn;
  tc5_rows(P1, MT);
  const int span2 = tc5_rows(P2, MT);
  P2.tc_bn = BN;
  size_t smem = 0;
  const long a2bytes = 2L * P2.tc_chunks_h * P2.R * 128;   // c2's hi / lo operand tile, in c1's operand buffers
  const int iters = P1.tc_chunks_h * P1.ntaps + P2.tc_chunks_h * P2.ntaps;
  if (dual ? !tcpair_plan_dual(P1, BN, a2bytes, iters, smem) : !tc5_plan(P1, BN, MT, a2bytes, iters, smem)) return false;
  dim3 grid(cdiv(tc_lv(P1), MT - span2), 1, tc_groups(P1));
  const auto dual_kern = BN == 64 ? tcpair2_kernel<64> : tcpair2_kernel<32>;
  if (dual) {
    tc_func_attrs(reinterpret_cast<const void*>(dual_kern), true);
    int per_sm = 0;
    AGPT_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, dual_kern, V5_THREADS, smem));
    if (per_sm != 2) return false;
  }
  void* rec = profile_begin_pair(P1, P2, st);
  tapconv_note_launch(1, BN, MT, 0, dual ? AGPT_TC_KERN_DUAL : AGPT_TC_KERN_TILE);
  if (dual) {
    tc_launch(dual_kern, true, grid, dim3(V5_THREADS), smem, st, P1, P2);
    profile_count_dual();
  } else {
    tc_launch(tcpair_kern(BN, MT), false, grid, dim3(V5_THREADS), smem, st, P1, P2);
    if (MT == TC_TALL) profile_count_tall();
  }
  profile_end(rec, st);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
  return true;
}

// One launch of tcpair_pipe_kernel: min(tiles, SMs) CTAs, each with two operand sets of 512 R1 bytes (R1: c1's operand
// rows) and as many 16 KB weight half-stages as the rest of kMaxDyn holds, at least 4.  False -- nothing launched --
// when the handle does not allow it (TapConvParams::tc_pipe), the pair is not 128 -> 128 channels converted from fp32
// with half-stage images, or the sets and four half-stages do not fit (c1 with a tap span of about 30 rows or more:
// k = 11 at dilation 5).
//
// tc_pipe == 1 runs the staged form (STAGED): the input rows arrive by TMA, a transform warpgroup and an epilogue
// warpgroup split the data work, and the residual (the pair's own input) arrives by TMA in 32 x 32 boxes through the
// shared memory left beside the weight ring plus each set's bytes past its dump: R1 = 136 / 144 / 152 / 160 get
// 2 + 1 / 0 + 2 / 2 + 3 / 0 + 4 slots at 5 / 5 / 4 / 4 half-stages, the same rings as without it.  tc_pipe == 2, a
// residual that is not the pair's input, or an input the tensor maps cannot describe keep one data warpgroup with
// plain global loads.
static bool tcpair_pipe_try(TapConvParams P1, TapConvParams P2, cudaStream_t st) {
  if (!P1.tc_pipe || P1.tc_bn != 128 || P1.Cin != 128 || P1.Cout != 128 || P2.Cout != 128 || !P1.w_hk || !P2.w_hk)
    return false;
  tc5_rows(P1, TC_ROWS);
  const int span2 = tc5_rows(P2, TC_ROWS);
  if (P2.R > P1.R) return false;   // c2's tile lives in c1's operand set
  const long wbytes = PIPE_STAGE;
  PipeSmem S;
  pipe_layout(S, P1.R, 0, 0);
  const long spare = (long)kMaxDyn - 1024 - (long)S.total;
  if (spare < 4 * wbytes) return false;
  const int iters = 2 * (P1.tc_chunks_h * P1.ntaps + P2.tc_chunks_h * P2.ntaps);
  P1.tc_nw = (int)std::min<long>(std::min<long>(PIPE_MAX_NW, iters), spare / wbytes);
  const int nsl = (P1.R - 128) / 8;
  const int nsp = (int)std::min<long>(PIPE_MAX_RES - nsl, (spare - P1.tc_nw * wbytes) / PIPE_RES_BOX);
  CUtensorMap tmx{}, tmr{};
  const bool staged = P1.tc_pipe == 1 && P2.res == P1.in && P2.res_pitch == P1.in_pitch &&
                      P2.res_gstride == P1.in_gstride && nsl + nsp >= 1 &&
                      tma_encode_rows(&tmx, P1.in, 128, P1.L, P1.G, P1.in_pitch, P1.in_gstride, P1.R) &&
                      tma_encode_rows(&tmr, P1.in, 128, P1.L, P1.G, P1.in_pitch, P1.in_gstride, 32);
  P1.tc_na = staged ? nsp : 0;
  P2.tc_bn = 128;
  pipe_layout(S, P1.R, P1.tc_nw, P1.tc_na);
  const size_t smem = (size_t)S.total + 1024;
  const long tiles = (long)cdiv(P1.L, TC_ROWS - span2) * P1.G;
  dim3 grid((unsigned)std::min<long>(tiles, tc5_sms()));
  void* rec = profile_begin_pair(P1, P2, st);
  tapconv_note_launch(1, 128, TC_ROWS, 0, AGPT_TC_KERN_PAIR_PIPE);
  if (staged)
    tc_launch(tcpair_pipe_kernel<true>, false, grid, dim3(PIPE_STAGED_THREADS), smem, st, P1, P2, tmx, tmr);
  else
    tc_launch(tcpair_pipe_kernel<false>, false, grid, dim3(PIPE_THREADS), smem, st, P1, P2, tmx, tmr);
  profile_count_pipe();
  profile_end(rec, st);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
  return true;
}

// Two 128-row CTAs per SM (tcpair2_kernel) instead of one 256- or 128-row CTA: the handle allows it
// (TapConvParams::tc_dual) and the pair is narrow (BN <= 64: one 64-channel chunk).
static bool tcpair_dual(const TapConvParams& P1) {
  return P1.tc_dual && P1.tc_bn <= 64;
}

// One launch of tcpair_narrow_kernel for a pair that tcpair_dual allows: min(tiles, SMs) CTAs.  Shared-memory plan:
// a set is 256 R1 bytes of operand tile and R1 x 128 B of staged input per 32 channels.  Where every weight stage of
// c1 and c2 fits beside two sets, the stages are loaded once per CTA and the rest holds as many sets as fit (at most
// 4); else two sets and as deep a ring as the rest holds.  At C = 64 the sets are large (68-94 KB), so a k = 11 pair
// keeps a ring of 2-4 of its 22 stages, which both wgmma warpgroups must release before it refills; those pairs are
// faster on tcpair2_kernel (measured on H100, DESIGN.md section 4) and are left to it: at BN = 64 the pipeline takes
// at most 14 weight stages per tile (k <= 7).  False -- nothing launched -- when the handle does not allow it
// (TapConvParams::tc_narrow_pipe), that limit is passed, the residual is not the pair's input, c2's tile or the
// residual rows do not lie inside c1's operand rows, or the plan does not fit.
static bool tcpair_narrow_try(TapConvParams P1, TapConvParams P2, cudaStream_t st) {
  const int BN = P1.tc_bn, iters = P1.ntaps + P2.ntaps;   // weight stages per tile: one 64-channel chunk per conv
  if (!P1.tc_narrow_pipe || (BN != 64 && BN != 32) || (BN == 64 && iters > 14) || P1.Cin > BN ||
      P2.res != P1.in || P2.res_pitch != P1.in_pitch || P2.res_gstride != P1.in_gstride)
    return false;
  const int span1 = tc5_rows(P1, TC_ROWS);
  const int span2 = tc5_rows(P2, TC_ROWS);
  // staged row of output row r is r - lo1 - lo2, for r < 128 - span2 it must lie in 0 .. R1 - 1
  if (P2.R > P1.R || P1.R > 256 || P1.lo_al > 0 || P2.lo_al > 0 || (P1.lo_al + span1) + (P2.lo_al + span2) < 0)
    return false;
  const int nbox = cdiv(P1.Cin, 32);
  const long wbytes = 2L * BN * 128, set = 256L * P1.R + 128L * nbox * P1.R;
  NarrowSmem S;
  narrow_layout(S, BN, P1.R, nbox, 0, 0);
  const long avail = (long)kMaxDyn - 1024 - (long)S.total;
  int NS = 2, NW;
  if (avail - iters * wbytes >= 2 * set) {
    NW = iters;
    NS = (int)std::min<long>(NARROW_MAX_NS, (avail - iters * wbytes) / set);
  } else {
    NW = (int)std::min<long>(iters, (avail - NS * set) / wbytes);
    if (NW < 2) return false;
  }
  CUtensorMap tmx;
  if (!tma_encode_rows(&tmx, P1.in, P1.Cin, P1.L, P1.G, P1.in_pitch, P1.in_gstride, P1.R)) return false;
  P1.tc_na = NS; P1.tc_nw = NW;
  P2.tc_bn = BN;
  narrow_layout(S, BN, P1.R, nbox, NS, NW);
  const size_t smem = (size_t)S.total + 1024;
  const long tiles = (long)cdiv(P1.L, TC_ROWS - span2) * P1.G;
  dim3 grid((unsigned)std::min<long>(tiles, tc5_sms()));
  void* rec = profile_begin_pair(P1, P2, st);
  tapconv_note_launch(1, BN, TC_ROWS, 0, AGPT_TC_KERN_NARROW_PIPE);
  tc_launch(BN == 64 ? tcpair_narrow_kernel<64> : tcpair_narrow_kernel<32>, false, grid, dim3(NARROW_THREADS), smem, st, P1,
            P2, tmx);
  profile_count_dual();
  profile_count_narrow_pipe();
  profile_end(rec, st);
  count_launch(1);
  AGPT_CUDA(cudaGetLastError());
  return true;
}

// One ResBlock1 pair, out = x + c2(lrelu(c1(lrelu(x)))) (c2's epilogue EPI_RES / EPI_ACC), as one launch of
// tcpair_kernel: c1's output tile stays in shared memory as c2's operand tile, so the intermediate tensor never
// reaches HBM.  A tile yields MT - span(c2) output rows (c1 is recomputed on the halo rows of neighbouring tiles);
// two 128-row tiles in flight per CTA where tcpair_pipe_try takes the pair (128 -> 128 channels); where tcpair_dual
// allows it, the narrow pipeline (tcpair_narrow_try), else two 128-row CTAs per SM where that plan fits; else MT = 256
// where tc5_tall allows it, else 128.
// Returns false -- nothing launched -- when the pair needs more than one co-tile, reads or writes an operand plane
// (TapConvParams::pi_hi / po_hi: the fused kernels convert fp32 and store fp32 only), or does not fit shared memory.
bool tcpair_launch(TapConvParams P1, TapConvParams P2, cudaStream_t st) {
  if (!tcconv_supported(P1) || !P2.w_h) return false;
  const int BN = P1.tc_bn;
  if (P1.pi_hi || P2.po_hi) return false;
  if (P2.tc_bn != BN || P1.Cout > BN || P2.Cin != P1.Cout || P2.Cout > BN || P1.Wreal || P2.Wreal || P1.strips ||
      P1.G != P2.G || P1.L != P2.L || P1.pro != PRO_LRELU || P2.pro != PRO_LRELU || (P2.epi != EPI_RES && P2.epi != EPI_ACC))
    return false;
  if (tcpair_pipe_try(P1, P2, st)) return true;
  if (tcpair_dual(P1) && (tcpair_narrow_try(P1, P2, st) || tcpair_try(P1, P2, TC_ROWS, true, st))) return true;
  const int span2 = tc5_rows(P2, TC_TALL);
  if (tc5_tall(P1, BN, (long)cdiv(tc_lv(P1), TC_TALL - span2) * tc_groups(P1), tc5_sms()) &&
      tcpair_try(P1, P2, TC_TALL, false, st))
    return true;
  return tcpair_try(P1, P2, TC_ROWS, false, st);
}

// One launch of tcconv_pipe_pl_kernel for tile c (pick_h_tile): cpipe_grid CTAs, each with NA operand buffers (2 to 4,
// at most one per chunk unless there are fewer than 2 chunks) and NW weight stages: as many buffers as leave room for
// 3 stages, then as many stages as the rest holds.  At k = 11, d = 5 (184 operand rows, 46 KB a buffer) that is 2
// buffers and 4 stages.  False -- nothing launched -- when the handle does not allow it (TapConvParams::tc_conv_pipe),
// the launch is not plane-fed over 1-D rows at BN = 128 with 128-row tiles and a BIAS / RES / ACC epilogue, or 2
// buffers and 2 stages do not fit.
static bool tcconv_pipe_try(TapConvParams P, const HTile& c, cudaStream_t st) {
  if (!P.tc_conv_pipe || !P.pi_hi || P.Wreal || P.strips || c.bn != 128 || c.mt != TC_ROWS ||
      (P.epi != EPI_BIAS && P.epi != EPI_RES && P.epi != EPI_ACC))
    return false;
  P.w_h = c.w;
  P.tc_bn = 128;
  tc5_rows(P, TC_ROWS);
  const int PR = pl_rows(P.R);
  const long abytes = 256L * PR, wbytes = 2L * 128 * 128;
  CpipeSmem S;
  cpipe_layout(S, PR, 0, 0);
  const long avail = (long)kMaxDyn - 1024 - (long)S.total;
  int NA = std::min(MAX_NA, std::max(2, P.tc_chunks_h));
  while (NA > 2 && NA * abytes + 3 * wbytes > avail) --NA;
  const int NW = (int)std::min<long>(MAX_NW, (avail - NA * abytes) / wbytes);
  if (NW < 2) return false;
  P.tc_na = NA; P.tc_nw = NW;
  cpipe_layout(S, PR, NA, NW);
  const size_t smem = (size_t)S.total + 1024;
  const int units = cdiv(P.L, TC_ROWS) * P.G * cdiv(P.Cout, 128);
  const PlMaps m = pl_tensor_maps(P);
  tapconv_note_launch(1, 128, TC_ROWS, 1, AGPT_TC_KERN_CONV_PIPE);
  tc_launch(tcconv_pipe_pl_kernel, false, dim3(cpipe_grid(units, tc5_sms())), dim3(CPIPE_THREADS), smem, st, P, m.hi, m.lo);
  profile_count_plane();
  profile_count_conv_pipe();
  return true;
}

// returns false when the layer has no fp16 image or does not fit the shared-memory budget
bool tcconv5_launch(TapConvParams P, cudaStream_t st) {
  if (!P.w_h) return false;
  const HTile c = pick_h_tile(P, tc5_sms());
  if (tcconv_pipe_try(P, c, st)) return true;
  if (c.bn != P.tc_bn || c.mt != TC_ROWS) {
    TapConvParams Q = P;
    Q.w_h = c.w;
    if (tcconv5_try(Q, c.bn, c.mt, st)) return true;
  }
  return tcconv5_try(P, P.tc_bn, TC_ROWS, st);
}

}  // namespace agpt
