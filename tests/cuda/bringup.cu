// Stand-alone bring-up check of the split-precision wgmma contraction core through the C ABI
// (no Python, no torch): random fp32 operands -> lb_split_planes -> lb_gemm_split, compared against a
// double-precision host product of the same fp32 operands.  Also prints a throughput figure.
// Build: see Makefile target `bringup`.  Run on the GPU box: build/bringup
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../include/loftr_b200.h"

#define CK(x)                                                                              \
  do {                                                                                     \
    cudaError_t e = (x);                                                                   \
    if (e != cudaSuccess) {                                                                \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__);       \
      exit(2);                                                                             \
    }                                                                                      \
  } while (0)

static unsigned long long rng = 0x9E3779B97F4A7C15ull;
static float frand() {
  rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17;
  return static_cast<float>((rng >> 11) * (1.0 / 9007199254740992.0)) * 2.f - 1.f;
}

static int run_case(int batches, int M, int N, int K, bool b_batched, float amp, bool check) {
  const long a_elems = static_cast<long>(batches) * M * K;
  const long b_elems = static_cast<long>(b_batched ? batches : 1) * N * K;
  const long o_elems = static_cast<long>(batches) * M * N;
  std::vector<float> hA(a_elems), hB(b_elems), hO(o_elems);
  for (auto& v : hA) v = frand() * amp + 0.25f * amp;   // common-mode offset like the real features
  for (auto& v : hB) v = frand() * amp + 0.25f * amp;
  float *dA, *dB, *dO;
  void *ah, *al, *bh, *bl;
  CK(cudaMalloc(&dA, a_elems * 4)); CK(cudaMalloc(&dB, b_elems * 4)); CK(cudaMalloc(&dO, o_elems * 4));
  CK(cudaMalloc(&ah, a_elems * 2)); CK(cudaMalloc(&al, a_elems * 2));
  CK(cudaMalloc(&bh, b_elems * 2)); CK(cudaMalloc(&bl, b_elems * 2));
  CK(cudaMemcpy(dA, hA.data(), a_elems * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dB, hB.data(), b_elems * 4, cudaMemcpyHostToDevice));
  CK(cudaMemset(dO, 0xFF, o_elems * 4));
  if (lb_split_planes(dA, static_cast<long>(batches) * M, K, K, ah, al, K, 0, nullptr) ||
      lb_split_planes(dB, static_cast<long>(b_batched ? batches : 1) * N, K, K, bh, bl, K, 0, nullptr)) {
    printf("split failed: %s\n", lb_last_error());
    return 1;
  }
  auto call = [&]() {
    return lb_gemm_split(ah, al, K, static_cast<long>(M) * K, bh, bl, K, b_batched ? static_cast<long>(N) * K : 0, dO, N,
                         static_cast<long>(M) * N, batches, M, N, K, nullptr);
  };
  if (call()) {
    printf("gemm failed: %s\n", lb_last_error());
    return 1;
  }
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    printf("case b=%d M=%d N=%d K=%d: kernel error %s\n", batches, M, N, K, cudaGetErrorString(e));
    return 1;
  }
  int rc = 0;
  if (check) {
    CK(cudaMemcpy(hO.data(), dO, o_elems * 4, cudaMemcpyDeviceToHost));
    double max_err = 0, max_ref = 0;
    long bad = 0;
    for (int b = 0; b < batches; ++b)
      for (int m = 0; m < M; ++m)
        for (int n = 0; n < N; ++n) {
          const float* a = &hA[(static_cast<long>(b) * M + m) * K];
          const float* w = &hB[(static_cast<long>(b_batched ? b : 0) * N + n) * K];
          double acc = 0;
          for (int k = 0; k < K; ++k) acc += static_cast<double>(a[k]) * w[k];
          const double got = hO[(static_cast<long>(b) * M + m) * N + n];
          const double err = std::fabs(got - acc);
          if (!(err <= 1e30)) ++bad;
          if (err > max_err) max_err = err;
          if (std::fabs(acc) > max_ref) max_ref = std::fabs(acc);
        }
    const double rel = max_err / (max_ref + 1e-30);
    const bool ok = bad == 0 && rel < 5e-6;
    printf("case b=%d M=%d N=%d K=%d b_batched=%d: max_abs_err=%.3e max_ref=%.3e rel=%.3e nan=%ld %s\n", batches, M, N,
           K, (int)b_batched, max_err, max_ref, rel, bad, ok ? "OK" : "FAIL");
    if (!ok) {
      rc = 1;
      // print a small corner to help diagnose layout bugs
      for (int m = 0; m < 2 && m < M; ++m) {
        for (int n = 0; n < 8 && n < N; ++n) printf(" %10.4f", hO[static_cast<long>(m) * N + n]);
        printf("\n");
      }
    }
  } else {
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    for (int i = 0; i < 3; ++i) call();
    CK(cudaEventRecord(e0));
    const int iters = 10;
    for (int i = 0; i < iters; ++i) call();
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    ms /= iters;
    const double flops = 2.0 * batches * M * static_cast<double>(N) * K;
    printf("perf b=%d M=%d N=%d K=%d: %.3f ms  %.1f TFLOP/s algorithmic (x3 issued)\n", batches, M, N, K, ms,
           flops / ms * 1e-9);
  }
  cudaFree(dA); cudaFree(dB); cudaFree(dO); cudaFree(ah); cudaFree(al); cudaFree(bh); cudaFree(bl);
  return rc;
}

int main() {
  int rc = 0;
  printf("lb_version=%d\n", lb_version());
  rc |= run_case(1, 128, 256, 64, false, 1.f, true);     // one tile, one k-block
  rc |= run_case(1, 128, 256, 256, false, 1.f, true);    // k loop, ring wrap
  rc |= run_case(1, 300, 768, 256, false, 4.f, true);    // partial m tile, 3 n tiles
  rc |= run_case(1, 1000, 128, 128, false, 4.f, true);   // BLOCK_N = 128 instantiation
  rc |= run_case(1, 200, 384, 128, false, 4.f, true);    // N=384 -> BN 256 path with partial n tile
  rc |= run_case(3, 200, 512, 256, true, 8.f, true);     // batched B (score-matrix form)
  rc |= run_case(1, 3000, 512, 512, false, 2.f, true);   // K = 512, many tiles per CTA
  if (rc == 0) {
    run_case(1, 76800, 768, 256, false, 1.f, false);     // coarse qkv projection at batch 8
    run_case(1, 76800, 512, 512, false, 1.f, false);     // mlp[0]
    run_case(8, 4800, 4800, 256, true, 1.f, false);      // score matrix (fp32 store epilogue: HBM bound)
  }
  printf(rc == 0 ? "BRINGUP PASS\n" : "BRINGUP FAIL\n");
  return rc;
}
