// Micro-benchmark / tuning entry: one tapconv layer of a given shape on random data, timed with
// CUDA events; optionally returns the per-CTA phase timestamps of the tensor-core kernel.
#include <random>
#include "tapconv.cuh"
#include "models.h"

namespace agpt {

// out[0] = ms per launch, out[1] = TFLOP/s (algorithmic), out[2] = max |tc - fma| (when check != 0)
// dbg_avg[8]: averaged phase deltas in cycles (setup, first-A, mainloop, tail, epilogue, total, waitA, waitW)
void bench_tapconv(int G, int L, int Cin, int Cout, int K, int dil, int Wreal, int epi_res, int use_tc, int reps,
                   int check, double* out, double* dbg_avg, double x_scale, double w_spread, double* rel2) {
  std::mt19937 rng(1234);
  std::normal_distribution<float> nd(0.f, 1.f);
  const bool is2d = Wreal > 0;
  const int taps = is2d ? 9 : K;
  std::vector<float> w((size_t)Cout * Cin * taps), b(Cout);
  for (auto& v : w) v = nd(rng) / std::sqrt((float)Cin * taps);
  if (w_spread > 1.0) {   // weight-norm-like gain spread: output channel co scaled by w_spread^u, u log-uniform in [-1/2, 1/2]
    std::uniform_real_distribution<float> ud(-0.5f, 0.5f);
    for (int co = 0; co < Cout; ++co) {
      const float gsc = std::pow((float)w_spread, ud(rng));
      for (size_t i = 0; i < (size_t)Cin * taps; ++i) w[(size_t)co * Cin * taps + i] *= gsc;
    }
  }
  for (auto& v : b) v = 0.05f * nd(rng);
  PackedConv pc;
  pack_conv(pc, w.data(), b.data(), Cout, Cin, taps, is2d);
  const size_t nin = (size_t)G * L * Cin, nout = (size_t)G * L * Cout;
  std::vector<float> hx(nin);
  for (auto& v : hx) v = nd(rng) * (float)x_scale;
  DevBuf x, y, y2, r;
  x.upload(hx);
  y.ensure(nout); y2.ensure(nout); r.ensure(nout);
  AGPT_CUDA(cudaMemset(r.p, 0, nout * 4));
  TapConvParams P = tapconv_params(pc, G, L, Wreal, dil);
  P.in = x.p; P.in_gstride = (long)L * Cin; P.in_pitch = Cin;
  P.out = y.p; P.out_gstride = (long)L * Cout; P.out_pitch = Cout;
  P.pro = PRO_LRELU; P.slope = 0.1f;
  P.epi = epi_res ? EPI_RES : EPI_BIAS;
  P.res = epi_res ? r.p : nullptr; P.res_gstride = (long)L * Cout; P.res_pitch = Cout;
  const bool tc_prev = tc_enabled();
  tc_set_enabled(use_tc);
  DevBuf dbgbuf;
  const int Wv = Wreal > 0 ? Wreal + 1 : 0;
  const int Lv = Wv ? (L / Wreal) * Wv : L;
  const long nctas = (long)cdiv(Lv, 128) * cdiv(Cout, pc.tc_bn ? pc.tc_bn : 128) * G;
  if (dbg_avg && use_tc) {
    dbgbuf.ensure((size_t)nctas * 16);
    AGPT_CUDA(cudaMemset(dbgbuf.p, 0, (size_t)nctas * 64));
    P.dbg = reinterpret_cast<long long*>(dbgbuf.p);
    P.tc_flags_user = 2;
  }
  cudaStream_t st = nullptr;
  auto launch = [&]() { tapconv_launch(P, st); };
  for (int i = 0; i < 2; ++i) launch();
  cudaEvent_t e0, e1;
  AGPT_CUDA(cudaEventCreate(&e0)); AGPT_CUDA(cudaEventCreate(&e1));
  AGPT_CUDA(cudaEventRecord(e0, st));
  for (int i = 0; i < reps; ++i) launch();
  AGPT_CUDA(cudaEventRecord(e1, st));
  AGPT_CUDA(cudaEventSynchronize(e1));
  float ms = 0.f;
  AGPT_CUDA(cudaEventElapsedTime(&ms, e0, e1));
  out[0] = ms / reps;
  out[1] = 2.0 * G * (double)L * Cin * Cout * taps / (out[0] * 1e-3) / 1e12;
  out[2] = -1.0;
  if (dbg_avg && use_tc) {
    std::vector<long long> h((size_t)nctas * 8);
    AGPT_CUDA(cudaMemcpy(h.data(), dbgbuf.p, h.size() * 8, cudaMemcpyDeviceToHost));
    double acc[8] = {0};
    long n = 0;
    for (long c = 0; c < nctas; ++c) {
      const long long* d = &h[c * 8];
      if (d[0] == 0) continue;
      if (d[5] == 0) continue;
      acc[0] += (double)(d[1] - d[0]);   // setup
      acc[1] += (double)(d[2] - d[1]);   // until first activation tile is ready
      acc[2] += (double)(d[3] - d[2]);   // MMA issue loop
      acc[3] += (double)(d[4] - d[3]);   // last issue -> accumulator complete
      acc[4] += (double)(d[5] - d[4]);   // epilogue
      acc[5] += (double)(d[5] - d[0]);   // total
      acc[6] += (double)d[6];            // MMA thread waiting on activations
      acc[7] += (double)d[7];            // MMA thread waiting on weights
      ++n;
    }
    for (int i = 0; i < 8; ++i) dbg_avg[i] = n ? acc[i] / n : 0.0;
  }
  if (check) {
    tc_set_enabled(0);
    TapConvParams Q = P;
    Q.out = y2.p; Q.dbg = nullptr; Q.tc_flags_user = 0;
    tapconv_launch(Q, st);
    AGPT_CUDA(cudaDeviceSynchronize());
    std::vector<float> a(nout), c(nout);
    AGPT_CUDA(cudaMemcpy(a.data(), y.p, nout * 4, cudaMemcpyDeviceToHost));
    AGPT_CUDA(cudaMemcpy(c.data(), y2.p, nout * 4, cudaMemcpyDeviceToHost));
    double mx = 0, se = 0, sr = 0;
    bool finite = true;
    for (size_t i = 0; i < nout; ++i) {
      const double d = (double)a[i] - (double)c[i];
      if (!std::isfinite(a[i])) finite = false;
      mx = std::max(mx, std::fabs(d)); se += d * d; sr += (double)c[i] * c[i];
    }
    out[2] = mx;
    if (rel2) {   // {max |diff| / rms(reference), rms(diff) / rms(reference)}; reference = the fp32-FMA kernel
      const double rms = std::sqrt(sr / (double)nout);
      rel2[0] = finite ? (rms > 0 ? mx / rms : mx) : 1e30;
      rel2[1] = finite ? (rms > 0 ? std::sqrt(se / (double)nout) / rms : std::sqrt(se / (double)nout)) : 1e30;
    }
  }
  tc_set_enabled(tc_prev ? 1 : 0);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
}

}  // namespace agpt
