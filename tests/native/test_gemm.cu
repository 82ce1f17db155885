// Stand-alone bring-up / regression test for vj_gemm on a real H100 (no torch involved).
// Compares every output element against a double-precision CPU reference and prints PASS/FAIL lines.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "vjepa_b200.h"

#define CK(x)                                                                     \
  do {                                                                            \
    cudaError_t e = (x);                                                          \
    if (e != cudaSuccess) {                                                       \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); \
      exit(2);                                                                    \
    }                                                                             \
  } while (0)

static uint32_t rng_state = 12345;
static float frand() {
  rng_state = rng_state * 1664525u + 1013904223u;
  return ((rng_state >> 8) & 0xFFFF) / 32768.0f - 1.0f;
}
static float bf(float x) { return __bfloat162float(__float2bfloat16(x)); }
static double gelu_ref(double x) { return 0.5 * x * (1.0 + erf(x / sqrt(2.0))); }
static double dgelu_ref(double x) {
  return 0.5 * (1.0 + erf(x / sqrt(2.0))) + x * exp(-0.5 * x * x) / sqrt(2.0 * M_PI);
}

struct Case {
  const char* name;
  int M, N, K, a_mn, b_mn, d_f32, epi, aux_f32, use_rowmap, aux_period, auxout, split_k, accumulate, bias;
};

static int run_case(const Case& c, bool verbose) {
  const int M = c.M, N = c.N, K = c.K;
  std::vector<float> A((size_t)M * K), B((size_t)N * K), bias(N), aux, D0;
  for (auto& v : A) v = bf(frand());
  for (auto& v : B) v = bf(frand() * 0.25f);
  for (auto& v : bias) v = c.bias ? frand() : 0.f;
  // storage: logical A[m][k]; if a_mn stored as [K][M]
  std::vector<__nv_bfloat16> hA((size_t)M * K), hB((size_t)N * K);
  for (int m = 0; m < M; ++m)
    for (int k = 0; k < K; ++k) {
      size_t idx = c.a_mn ? (size_t)k * M + m : (size_t)m * K + k;
      hA[idx] = __float2bfloat16(A[(size_t)m * K + k]);
    }
  for (int n = 0; n < N; ++n)
    for (int k = 0; k < K; ++k) {
      size_t idx = c.b_mn ? (size_t)k * N + n : (size_t)n * K + k;
      hB[idx] = __float2bfloat16(B[(size_t)n * K + k]);
    }
  int aux_rows = M;
  if (c.aux_period > 0) aux_rows = c.aux_period;
  if (c.use_rowmap) aux_rows = 97;
  std::vector<int> rowmap(M);
  for (int m = 0; m < M; ++m) rowmap[m] = (m * 7 + 3) % 97;
  const bool need_aux = c.epi == VJ_EPI_ADD || c.epi == VJ_EPI_DGELU || c.epi == VJ_EPI_MUL;
  aux.resize((size_t)aux_rows * N);
  for (auto& v : aux) v = c.aux_f32 ? frand() : bf(frand());
  D0.resize((size_t)M * N);
  for (auto& v : D0) v = c.accumulate ? frand() : 0.f;

  void *dA, *dB, *dD, *dAux = nullptr, *dX = nullptr;
  float* dBias;
  int* dMap = nullptr;
  CK(cudaMalloc(&dA, hA.size() * 2));
  CK(cudaMalloc(&dB, hB.size() * 2));
  CK(cudaMalloc(&dD, (size_t)M * N * 4));
  CK(cudaMalloc(&dBias, N * 4));
  CK(cudaMemcpy(dA, hA.data(), hA.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dB, hB.data(), hB.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dBias, bias.data(), N * 4, cudaMemcpyHostToDevice));
  // reduce-adding GEMMs start from D0 (zero for a split-K that does not accumulate); a plain store must overwrite NaNs
  if (c.d_f32 && (c.accumulate || c.split_k != 1)) CK(cudaMemcpy(dD, D0.data(), (size_t)M * N * 4, cudaMemcpyHostToDevice));
  else CK(cudaMemset(dD, 0xFF, (size_t)M * N * 4));
  if (need_aux) {
    if (c.aux_f32) {
      CK(cudaMalloc(&dAux, aux.size() * 4));
      CK(cudaMemcpy(dAux, aux.data(), aux.size() * 4, cudaMemcpyHostToDevice));
    } else {
      std::vector<__nv_bfloat16> h(aux.size());
      for (size_t i = 0; i < aux.size(); ++i) h[i] = __float2bfloat16(aux[i]);
      CK(cudaMalloc(&dAux, aux.size() * 2));
      CK(cudaMemcpy(dAux, h.data(), aux.size() * 2, cudaMemcpyHostToDevice));
    }
  }
  if (c.use_rowmap) {
    CK(cudaMalloc(&dMap, M * 4));
    CK(cudaMemcpy(dMap, rowmap.data(), M * 4, cudaMemcpyHostToDevice));
  }
  if (c.auxout) CK(cudaMalloc(&dX, (size_t)M * N * 2));

  const float alpha = 0.5f;
  int rc = vj_gemm(dA, c.a_mn ? M : K, c.a_mn, dB, c.b_mn ? N : K, c.b_mn, dD, N, c.d_f32, M, N, K,
                   c.bias ? dBias : nullptr, alpha, c.epi, dAux, N, c.aux_f32, dMap, c.aux_period, dX, N,
                   c.split_k, c.accumulate, nullptr);
  if (rc != 0) {
    printf("FAIL %-28s vj_gemm rc=%d: %s\n", c.name, rc, vj_last_error_string());
    return 1;
  }
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    printf("FAIL %-28s kernel error: %s\n", c.name, cudaGetErrorString(e));
    exit(3);  // context is dead
  }
  std::vector<float> out((size_t)M * N);
  if (c.d_f32) CK(cudaMemcpy(out.data(), dD, (size_t)M * N * 4, cudaMemcpyDeviceToHost));
  else {
    std::vector<__nv_bfloat16> h((size_t)M * N);
    CK(cudaMemcpy(h.data(), dD, (size_t)M * N * 2, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < h.size(); ++i) out[i] = __bfloat162float(h[i]);
  }
  std::vector<float> xout;
  if (c.auxout) {
    std::vector<__nv_bfloat16> h((size_t)M * N);
    CK(cudaMemcpy(h.data(), dX, (size_t)M * N * 2, cudaMemcpyDeviceToHost));
    xout.resize(h.size());
    for (size_t i = 0; i < h.size(); ++i) xout[i] = __bfloat162float(h[i]);
  }
  double max_err = 0, max_ref = 0, max_err_x = 0;
  int bad = 0;
  for (int m = 0; m < M; ++m) {
    for (int n = 0; n < N; ++n) {
      double acc = 0;
      const float* a = &A[(size_t)m * K];
      const float* b = &B[(size_t)n * K];
      for (int k = 0; k < K; ++k) acc += (double)a[k] * b[k];
      double v = acc * alpha + bias[n];
      double pre = v;
      int arow = c.use_rowmap ? rowmap[m] : (c.aux_period > 0 ? m % c.aux_period : m);
      if (c.epi == VJ_EPI_GELU) v = gelu_ref(v);
      else if (c.epi == VJ_EPI_GELU_GRAD) { v = gelu_ref(v); pre = dgelu_ref(pre); }
      else if (c.epi == VJ_EPI_MUL) v *= aux[(size_t)arow * N + n];
      else if (c.epi == VJ_EPI_ADD) v += aux[(size_t)arow * N + n];
      else if (c.epi == VJ_EPI_DGELU) v *= dgelu_ref(aux[(size_t)arow * N + n]);
      if (c.accumulate) v += D0[(size_t)m * N + n];
      double got = out[(size_t)m * N + n];
      double err = fabs(got - v);
      double tol = c.d_f32 ? 2e-3 + 1e-4 * fabs(v) : 2e-2 + 8e-3 * fabs(v);
      if (!(err <= tol)) {
        if (bad < 5 && verbose) printf("   mismatch m=%d n=%d got=%g ref=%g\n", m, n, got, v);
        ++bad;
      }
      if (err > max_err) max_err = err;
      if (fabs(v) > max_ref) max_ref = fabs(v);
      if (c.auxout) {
        double ex = fabs(xout[(size_t)m * N + n] - pre);
        if (ex > max_err_x) max_err_x = ex;
        if (!(ex <= 2e-2 + 8e-3 * fabs(pre))) ++bad;
      }
    }
  }
  printf("%s %-28s M=%d N=%d K=%d max_err=%.4g (max_ref=%.3g) auxout_err=%.3g bad=%d\n", bad ? "FAIL" : "PASS",
         c.name, M, N, K, max_err, max_ref, max_err_x, bad);
  cudaFree(dA); cudaFree(dB); cudaFree(dD); cudaFree(dBias);
  if (dAux) cudaFree(dAux);
  if (dMap) cudaFree(dMap);
  if (dX) cudaFree(dX);
  return bad ? 1 : 0;
}

static void perf(int M, int N, int K, int a_mn, int b_mn, int d_f32, int epi, int split_k, const char* name) {
  void *dA, *dB, *dD, *dAux;
  float* dBias;
  CK(cudaMalloc(&dA, (size_t)M * K * 2));
  CK(cudaMalloc(&dB, (size_t)N * K * 2));
  CK(cudaMalloc(&dD, (size_t)M * N * 4));
  CK(cudaMalloc(&dAux, (size_t)M * N * 4));
  CK(cudaMalloc(&dBias, N * 4));
  CK(cudaMemset(dA, 0x3C, (size_t)M * K * 2));
  CK(cudaMemset(dB, 0x3C, (size_t)N * K * 2));
  CK(cudaMemset(dAux, 0, (size_t)M * N * 4));
  CK(cudaMemset(dBias, 0, N * 4));
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  const int iters = 10;
  for (int i = 0; i < 3; ++i)
    vj_gemm(dA, a_mn ? M : K, a_mn, dB, b_mn ? N : K, b_mn, dD, N, d_f32, M, N, K, dBias, 1.f, epi, dAux, N, 0,
            nullptr, 0, epi == VJ_EPI_GELU_GRAD ? dAux : nullptr, N, split_k, split_k != 1, nullptr);
  CK(cudaDeviceSynchronize());
  cudaEventRecord(e0);
  for (int i = 0; i < iters; ++i)
    vj_gemm(dA, a_mn ? M : K, a_mn, dB, b_mn ? N : K, b_mn, dD, N, d_f32, M, N, K, dBias, 1.f, epi, dAux, N, 0,
            nullptr, 0, epi == VJ_EPI_GELU_GRAD ? dAux : nullptr, N, split_k, split_k != 1, nullptr);
  cudaEventRecord(e1);
  CK(cudaDeviceSynchronize());
  float ms;
  cudaEventElapsedTime(&ms, e0, e1);
  ms /= iters;
  printf("PERF %-28s M=%d N=%d K=%d  %.3f ms  %.1f TFLOP/s\n", name, M, N, K, ms, 2.0 * M * N * K / ms * 1e-9);
  cudaFree(dA); cudaFree(dB); cudaFree(dD); cudaFree(dAux); cudaFree(dBias);
}

int main(int argc, char** argv) {
  const bool verbose = true;
  int fails = 0;
  // name, M,N,K, a_mn,b_mn, d_f32, epi, aux_f32, rowmap, period, auxout, split, accum, bias
  Case base[] = {
      {"kk_bn64_none", 300, 192, 192, 0, 0, 0, VJ_EPI_NONE, 0, 0, 0, 0, 1, 0, 1},
      {"kk_bn128_none", 300, 384, 320, 0, 0, 0, VJ_EPI_NONE, 0, 0, 0, 0, 1, 0, 1},
      {"kk_bn256_none", 520, 512, 256, 0, 0, 0, VJ_EPI_NONE, 0, 0, 0, 0, 1, 0, 1},
      {"kk_bn256_f32", 520, 512, 256, 0, 0, 1, VJ_EPI_NONE, 0, 0, 0, 0, 1, 0, 1},
      {"kmn_bn128_dgrad", 300, 384, 320, 0, 1, 0, VJ_EPI_NONE, 0, 0, 0, 0, 1, 0, 0},
      {"kmn_bn256_dgrad", 300, 512, 192, 0, 1, 0, VJ_EPI_NONE, 0, 0, 0, 0, 1, 0, 0},
      {"mnmn_bn128_wgrad", 256, 384, 1000, 1, 1, 1, VJ_EPI_NONE, 0, 0, 0, 0, 1, 0, 0},
      {"mnmn_bn256_wgrad_split", 384, 256, 1000, 1, 1, 1, VJ_EPI_NONE, 0, 0, 0, 0, 3, 1, 0},
      {"mnmn_bn64_wgrad", 192, 192, 520, 1, 1, 1, VJ_EPI_NONE, 0, 0, 0, 0, 2, 1, 0},
      {"mnmn_bn128_wgrad_bf16out", 256, 384, 1000, 1, 1, 0, VJ_EPI_NONE, 0, 0, 0, 0, 1, 0, 0},
      {"mnmn_bn64_wgrad_store_bias", 136, 192, 333, 1, 1, 1, VJ_EPI_NONE, 0, 0, 0, 0, 1, 0, 1},
      {"mnmn_bn128_wgrad_m64_k174", 64, 1024, 174, 1, 1, 1, VJ_EPI_NONE, 0, 0, 0, 0, 1, 0, 0},
      {"mnmn_bn256_wgrad_streamk", 640, 512, 3000, 1, 1, 1, VJ_EPI_NONE, 0, 0, 0, 0, -1, 1, 0},
      {"mnmn_bn128_wgrad_streamk", 256, 384, 20000, 1, 1, 1, VJ_EPI_NONE, 0, 0, 0, 0, -1, 1, 0},
      {"kk_bn256_f32_streamk_bias", 520, 512, 1104, 0, 0, 1, VJ_EPI_NONE, 0, 0, 0, 0, -1, 1, 1},
      {"gelu_auxout", 300, 768, 192, 0, 0, 0, VJ_EPI_GELU, 0, 0, 0, 1, 1, 0, 1},
      {"gelu_noaux", 300, 256, 192, 0, 0, 0, VJ_EPI_GELU, 0, 0, 0, 0, 1, 0, 1},
      {"add_bf16_res", 300, 256, 192, 0, 0, 0, VJ_EPI_ADD, 0, 0, 0, 0, 1, 0, 1},
      {"add_f32_res_f32out", 300, 384, 192, 0, 0, 1, VJ_EPI_ADD, 1, 0, 0, 0, 1, 0, 1},
      {"add_f32_period", 300, 256, 192, 0, 0, 0, VJ_EPI_ADD, 1, 0, 100, 0, 1, 0, 1},
      {"add_f32_rowmap", 300, 256, 192, 0, 0, 0, VJ_EPI_ADD, 1, 1, 0, 0, 1, 0, 1},
      {"dgelu_dgrad", 300, 512, 256, 0, 1, 0, VJ_EPI_DGELU, 0, 0, 0, 0, 1, 0, 0},
      {"mul_dgrad", 300, 512, 256, 0, 1, 0, VJ_EPI_MUL, 0, 0, 0, 0, 1, 0, 0},
      {"mul_dgrad_bn128", 300, 384, 256, 0, 1, 0, VJ_EPI_MUL, 0, 0, 0, 0, 1, 0, 0},
      {"gelu_grad_auxout", 300, 768, 192, 0, 0, 0, VJ_EPI_GELU_GRAD, 0, 0, 0, 1, 1, 0, 1},
      {"gelu_grad_auxout_bn128", 300, 384, 192, 0, 0, 0, VJ_EPI_GELU_GRAD, 0, 0, 0, 1, 1, 0, 1},
      {"kk_big", 4000, 1024, 1024, 0, 0, 0, VJ_EPI_NONE, 0, 0, 0, 0, 1, 0, 1},
  };
  const char* only = argc > 1 ? argv[1] : nullptr;
  for (auto& c : base) {
    if (only && !strstr(c.name, only)) continue;
    fails += run_case(c, verbose);
  }
  if (!only || !strncmp(only, "perf", 4)) {
    const char* sub = (only && only[4] == ':') ? only + 5 : nullptr;   // "perf:<substring>" runs matching cases only
    struct P { int M, N, K, a, b, f32, epi, split; const char* name; };
    const P cases[] = {
        {50176, 4096, 1024, 0, 0, 0, VJ_EPI_GELU, 1, "fc1_gelu_target"},
        {50176, 1024, 4096, 0, 0, 0, VJ_EPI_ADD, 1, "fc2_add_target"},
        {50176, 3072, 1024, 0, 0, 0, VJ_EPI_NONE, 1, "qkv_target"},
        {13056, 4096, 1024, 0, 1, 0, VJ_EPI_NONE, 1, "dgrad_ctx"},
        {4096, 1024, 13056, 1, 1, 1, VJ_EPI_NONE, 1, "wgrad_ctx_fc1"},
        {1024, 1024, 13056, 1, 1, 1, VJ_EPI_NONE, 4, "wgrad_ctx_proj_split4"},
        {4096, 1024, 13056, 1, 1, 1, VJ_EPI_NONE, 2, "wgrad_ctx_fc1_split2"},
        {4096, 1024, 13056, 1, 1, 1, VJ_EPI_NONE, -1, "wgrad_ctx_fc1_streamk"},
        {3072, 1024, 13056, 1, 1, 1, VJ_EPI_NONE, 2, "wgrad_ctx_qkv_split2"},
        {3072, 1024, 13056, 1, 1, 1, VJ_EPI_NONE, -1, "wgrad_ctx_qkv_streamk"},
        {1024, 1024, 13056, 1, 1, 1, VJ_EPI_NONE, -1, "wgrad_ctx_proj_streamk"},
        {1536, 384, 76032, 1, 1, 1, VJ_EPI_NONE, -1, "fc1_wgrad_pred_streamk"},
        {384, 1536, 76032, 1, 1, 1, VJ_EPI_NONE, -1, "fc2_wgrad_pred_streamk"},
        {76032, 1536, 384, 0, 0, 0, VJ_EPI_GELU, 1, "fc1_pred"},
        {76032, 1536, 384, 0, 0, 0, VJ_EPI_NONE, 1, "qkv_pred"},
        {76032, 384, 512, 0, 0, 0, VJ_EPI_ADD, 1, "proj_pred"},
        {76032, 384, 1536, 0, 0, 0, VJ_EPI_ADD, 1, "fc2_pred"},
        {76032, 1536, 384, 0, 1, 0, VJ_EPI_DGELU, 1, "fc2_dgrad_pred"},
        {76032, 1536, 384, 0, 1, 0, VJ_EPI_MUL, 1, "fc2_dgrad_pred_mul"},
        {13056, 4096, 1024, 0, 1, 0, VJ_EPI_MUL, 1, "fc2_dgrad_ctx_mul"},
        {76032, 1536, 384, 0, 0, 0, VJ_EPI_GELU_GRAD, 1, "fc1_pred_gelugrad"},
        {13056, 4096, 1024, 0, 0, 0, VJ_EPI_GELU_GRAD, 1, "fc1_ctx_gelugrad"},
        {76032, 384, 1536, 0, 1, 0, VJ_EPI_NONE, 1, "fc1_dgrad_pred"},
        {76032, 1536, 384, 0, 1, 0, VJ_EPI_NONE, 1, "kmn_none_pred_1536x384"},
        {76032, 1536, 384, 0, 0, 0, VJ_EPI_DGELU, 1, "kk_dgelu_pred_1536x384"},
        {13056, 4096, 1024, 0, 1, 0, VJ_EPI_DGELU, 1, "fc2_dgrad_ctx"},
        {1536, 384, 76032, 1, 1, 1, VJ_EPI_NONE, 4, "fc1_wgrad_pred_split4"},
        {384, 1536, 76032, 1, 1, 1, VJ_EPI_NONE, 8, "fc2_wgrad_pred_split8"},
        {13056, 1024, 1024, 0, 0, 0, VJ_EPI_ADD, 1, "proj_ctx"},
        {13056, 4096, 1024, 0, 0, 0, VJ_EPI_GELU, 1, "fc1_ctx"},
    };
    for (const P& c : cases)
      if (!sub || strstr(c.name, sub)) perf(c.M, c.N, c.K, c.a, c.b, c.f32, c.epi, c.split, c.name);
  }
  printf("%s: %d failing case(s)\n", fails ? "FAILED" : "ALL PASSED", fails);
  return fails ? 1 : 0;
}
