// Common host/device helpers for libagpt_b200 (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include <stdexcept>
#include <cstdlib>
#include <memory>
#include <utility>

namespace agpt {

// ---- error plumbing: C-ABI functions return int, message kept thread-local ----
void set_last_error(const std::string& msg);

struct Error : public std::runtime_error {
  explicit Error(const std::string& m) : std::runtime_error(m) {}
};

#define AGPT_CUDA(expr)                                                              \
  do {                                                                               \
    cudaError_t _e = (expr);                                                         \
    if (_e != cudaSuccess) {                                                         \
      throw ::agpt::Error(std::string(#expr) + ": " + cudaGetErrorString(_e) +      \
                          " @" + __FILE__ + ":" + std::to_string(__LINE__));         \
    }                                                                                \
  } while (0)

#define AGPT_CHECK(cond, msg)                                                        \
  do {                                                                               \
    if (!(cond)) throw ::agpt::Error(std::string("check failed: ") + #cond + ": " + (msg)); \
  } while (0)

inline int cdiv(int a, int b) { return (a + b - 1) / b; }
inline long cdivl(long a, long b) { return (a + b - 1) / b; }
inline int round_up(int a, int b) { return cdiv(a, b) * b; }

// ---- device memory owned by a handle -----------------------------------------
struct DevBuf {
  float* p = nullptr;
  size_t n = 0;  // floats
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), n(o.n) { o.p = nullptr; o.n = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { if (p) cudaFree(p); p = o.p; n = o.n; o.p = nullptr; o.n = 0; }
    return *this;
  }
  ~DevBuf() { if (p) cudaFree(p); }
  // grow-only; contents are NOT preserved
  float* ensure(size_t floats) {
    if (floats > n) {
      if (p) { cudaDeviceSynchronize(); cudaFree(p); p = nullptr; }
      AGPT_CUDA(cudaMalloc(&p, floats * sizeof(float)));
      n = floats;
    }
    return p;
  }
  void upload(const float* h, size_t count) {
    ensure(count);
    AGPT_CUDA(cudaMemcpy(p, h, count * sizeof(float), cudaMemcpyHostToDevice));
  }
  void upload(const std::vector<float>& h) { upload(h.data(), h.size()); }
};

// The host weight arrays of a *_create call, consumed in the order of the model's parameter table.
struct WeightCursor {
  const float* const* W;
  int n, idx = 0;
  const float* next() { AGPT_CHECK(idx < n, "too few weight arrays"); return W[idx++]; }
  void done() const { AGPT_CHECK(idx == n, "weight array count does not match the config"); }
};

// RAII device scope for the C-ABI entry points: the reference deployment pins tools to different GPUs in ONE
// process (audio-chatgpt.py:1051-1073), so an entry point must leave the calling thread's current device as it
// found it (torch reads it back with cudaGetDevice).
struct DeviceGuard {
  int prev = -1;
  bool switched = false;
  explicit DeviceGuard(int dev) {
    AGPT_CUDA(cudaGetDevice(&prev));
    if (prev != dev) { AGPT_CUDA(cudaSetDevice(dev)); switched = true; }
  }
  ~DeviceGuard() { if (switched) cudaSetDevice(prev); }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
};

// Base of every opaque handle handed across the C ABI.
struct Handle {
  uint32_t magic = 0;
  int device = 0;
  virtual ~Handle() {}
};
constexpr uint32_t kMagicHifigan = 0x48494649;  // 'HIFI'
constexpr uint32_t kMagicDiffnet = 0x44494646;  // 'DIFF'
constexpr uint32_t kMagicUnet = 0x554e4554;     // 'UNET'
constexpr uint32_t kMagicVae = 0x56414544;      // 'VAED'
constexpr uint32_t kMagicVaeEnc = 0x56414545;   // 'VAEE'
constexpr uint32_t kMagicPe = 0x50495443;       // 'PITC'
constexpr uint32_t kMagicFs2 = 0x46533220;      // 'FS2 '
constexpr uint32_t kMagicClap = 0x434c4150;     // 'CLAP'
constexpr uint32_t kMagicCnn14 = 0x434e4e45;    // 'CNNE'
constexpr uint32_t kMagicGs = 0x47535053;       // 'GSPS'
constexpr uint32_t kMagicLass = 0x4c415353;     // 'LASS'
constexpr uint32_t kMagicStft = 0x53544654;     // 'STFT'
constexpr uint32_t kMagicPvt = 0x50565432;      // 'PVT2'
constexpr uint32_t kMagicTsd = 0x54534430;      // 'TSD0'
constexpr uint32_t kMagicBinaural = 0x42494e30; // 'BIN0'
constexpr uint32_t kMagicW2v = 0x57325643;      // 'W2VC'
constexpr uint32_t kMagicEmo = 0x454d4f30;      // 'EMO0'

// ---- small device functions --------------------------------------------------
__device__ __forceinline__ float lrelu(float x, float a) { return x > 0.f ? x : a * x; }
__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float siluf_(float x) { return x / (1.f + expf(-x)); }
__device__ __forceinline__ float mishf_(float x) {
  const float sp = x > 20.f ? x : log1pf(expf(x));  // F.softplus (beta=1, threshold=20)
  return x * tanhf(sp);
}
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }

}  // namespace agpt
