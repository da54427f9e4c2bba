// Host entry of the fp16 hi/lo tensor-core tap-GEMM (the kernels, their tile choice and their launches live in
// tcconv5.cu):
//
//   out[g, p, co] = epi( bias[co] + sum_tap sum_ci pro(in[g, p + off_tap, ci]) * W[tap][ci][co] )
//
// Same TapConvParams contract (and the same fused prologue / epilogue table) as the fp32-FMA kernel in tapconv.cu;
// the inner product runs as wgmma on error-compensated fp16 hi/lo operand parts with fp32 accumulation in registers
// (header of tcconv5.cu).  This file packs the weights, holds the AGPT_TENSOR_CORES switch, decides whether a layer
// can run on the tensor cores, and fails the launch of a layer that fits no tile.
#include "tapconv.cuh"
#include "models.h"

namespace agpt {

void pack_tc_weights(PackedConv& pc, const std::vector<float>& h) {
  pc.tc_bn = tc_pick_bn(pc.Cout);
  pack_h_weights(pc, h);   // fp16 hi/lo operand images (tcconv5.cu)
}

static int g_tc_enabled = -1;   // -1: read AGPT_TENSOR_CORES from the environment on first use
void tc_set_enabled(int on) { g_tc_enabled = on != 0 ? 1 : 0; }
bool tc_enabled() {
  if (g_tc_enabled < 0) {
    const char* e = getenv("AGPT_TENSOR_CORES");
    g_tc_enabled = (e && e[0] == '0') ? 0 : 1;   // default ON (tests/test_*_gpu.py)
  }
  return g_tc_enabled == 1;
}

bool tcconv_supported(const TapConvParams& P) {
  if (!tc_enabled() || !P.w_h || P.tc_bn == 0) return false;
  if (P.in_pitch % 4 != 0 || P.Cin % 4 != 0) return false;        // 16-byte load granularity of the transform warps
  if ((reinterpret_cast<uintptr_t>(P.in) & 15) != 0 || (P.in_gstride % 4) != 0) return false;
  return true;
}

void tcconv_launch(TapConvParams P, cudaStream_t st) {
  if (tcconv5_launch(P, st)) return;
  throw Error("tcconv: layer does not fit the shared-memory budget of the tensor-core kernel (image too wide for the halo tile?)");
}

}  // namespace agpt
