// TMA (tensor-map) helpers: host-side descriptor encoding through the driver entry point (no -lcuda
// link dependency) and the device-side PTX for tiled bulk-tensor loads / stores / reduce-add stores.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include "common.cuh"
#include "tc_common.cuh"

namespace agpt {

typedef CUresult (*TmaEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                 const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                 CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline TmaEncodeFn tma_encode_fn() {
  static TmaEncodeFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess &&
        qr == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<TmaEncodeFn>(p);
  }
  return fn;
}

// activation tensor [G][L][C] of elem-byte elements (C contiguous, row pitch and sample stride in elements) seen as a
// 3-D tensor {C, L, G}; box = {box_c channels (128 B, SWIZZLE_128B), box_rows, 1}.  Out-of-bounds elements load as zero.
inline bool tma_encode_3d(CUtensorMap* map, CUtensorMapDataType dt, int elem, const void* base, int C, long L, int G,
                          long pitch, long gstride, int box_c, int box_rows) {
  const TmaEncodeFn fn = tma_encode_fn();
  if (!fn) return false;
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (pitch * elem) % 16 != 0 || (gstride * elem) % 16 != 0 || C <= 0 ||
      L <= 0)
    return false;
  const cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)L, (cuuint64_t)(G > 0 ? G : 1)};
  const cuuint64_t strides[2] = {(cuuint64_t)pitch * elem, (cuuint64_t)(G > 1 ? gstride : pitch * L) * elem};
  const cuuint32_t box[3] = {(cuuint32_t)box_c, (cuuint32_t)box_rows, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  const CUresult r = fn(map, dt, 3, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

// fp32 activation tensor: boxes of 32 channels
inline bool tma_encode_rows(CUtensorMap* map, const float* base, int C, long L, int G, long pitch, long gstride,
                            int box_rows) {
  return tma_encode_3d(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, base, C, L, G, pitch, gstride, 32, box_rows);
}
// fp16 operand plane (tcconv5.cu): boxes of 64 channels, one K chunk of the wgmma tap-GEMM
inline bool tma_encode_rows_h(CUtensorMap* map, const __half* base, int C, long L, int G, long pitch, long gstride,
                              int box_rows) {
  return tma_encode_3d(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, base, C, L, G, pitch, gstride, 64, box_rows);
}

namespace {

__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, int c0, int c1, int c2, const void* src) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(src)) : "memory");
}
__device__ __forceinline__ void tma_reduce_add_3d(const CUtensorMap* map, int c0, int c1, int c2, const void* src) {
  asm volatile("cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.tile.bulk_group [%0, {%1, %2, %3}], [%4];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(src)) : "memory");
}
__device__ __forceinline__ void tma_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_wait_group_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void tma_wait_group() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

}  // namespace
}  // namespace agpt
