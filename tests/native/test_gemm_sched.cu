// Tile-schedule coverage for vj_gemm on an H100 (no torch): shapes that give a CTA many tiles (odd and even counts, so
// both consumer warpgroups and the hand-over between them run), ragged M down to a last tile of fewer than 64 rows,
// N = 64 .. 512, every epilogue, K-major and MN-major B, the cooperative long-K schedule, and persistent grids of 1, 7
// and 131 CTAs.  Every output element is checked against a double-precision host reference, and the rows below M in
// D / aux_out must stay untouched.
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

static uint32_t rng_state = 777;
static float frand() {
  rng_state = rng_state * 1664525u + 1013904223u;
  return ((rng_state >> 8) & 0xFFFF) / 32768.0f - 1.0f;
}
static float bf(float x) { return __bfloat162float(__float2bfloat16(x)); }
static float bf16_bits(uint16_t b) {
  const uint32_t u = uint32_t(b) << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
static double gelu_ref(double x) { return 0.5 * x * (1.0 + erf(x / sqrt(2.0))); }
static double dgelu_ref(double x) {
  return 0.5 * (1.0 + erf(x / sqrt(2.0))) + x * exp(-0.5 * x * x) / sqrt(2.0 * M_PI);
}

struct Case {
  int M, N, K, b_mn, d_f32, epi, aux_f32, use_rowmap, aux_period, auxout, bias, sm_limit;
};

static const char* epi_name(int e) {
  switch (e) {
    case VJ_EPI_NONE: return "none";
    case VJ_EPI_GELU: return "gelu";
    case VJ_EPI_ADD: return "add";
    case VJ_EPI_DGELU: return "dgelu";
    case VJ_EPI_MUL: return "mul";
    default: return "gelu_grad";
  }
}

static int run_case(const Case& c) {
  const int M = c.M, N = c.N, K = c.K;
  const int guard = 64;   // rows past M that must not be written
  std::vector<float> A((size_t)M * K), B((size_t)N * K), bias(N), aux;
  for (auto& v : A) v = bf(frand());
  for (auto& v : B) v = bf(frand() * 0.25f);
  for (auto& v : bias) v = c.bias ? frand() : 0.f;
  std::vector<__nv_bfloat16> hA((size_t)M * K), hB((size_t)N * K);
  for (size_t i = 0; i < hA.size(); ++i) hA[i] = __float2bfloat16(A[i]);
  for (int n = 0; n < N; ++n)
    for (int k = 0; k < K; ++k) hB[c.b_mn ? (size_t)k * N + n : (size_t)n * K + k] = __float2bfloat16(B[(size_t)n * K + k]);
  int aux_rows = M;
  if (c.aux_period > 0) aux_rows = c.aux_period;
  if (c.use_rowmap) aux_rows = 97;
  std::vector<int> rowmap(M);
  for (int m = 0; m < M; ++m) rowmap[m] = (m * 7 + 3) % 97;
  const bool need_aux = c.epi == VJ_EPI_ADD || c.epi == VJ_EPI_DGELU || c.epi == VJ_EPI_MUL;
  aux.resize((size_t)aux_rows * N);
  for (auto& v : aux) v = c.aux_f32 ? frand() : bf(frand());

  const size_t esz = c.d_f32 ? 4 : 2;
  void *dA, *dB, *dD, *dAux = nullptr, *dX = nullptr;
  float* dBias;
  int* dMap = nullptr;
  CK(cudaMalloc(&dA, hA.size() * 2));
  CK(cudaMalloc(&dB, hB.size() * 2));
  CK(cudaMalloc(&dD, (size_t)(M + guard) * N * esz));
  CK(cudaMalloc(&dBias, N * 4));
  CK(cudaMemcpy(dA, hA.data(), hA.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dB, hB.data(), hB.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dBias, bias.data(), N * 4, cudaMemcpyHostToDevice));
  CK(cudaMemset(dD, 0xFF, (size_t)(M + guard) * N * esz));
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
  if (c.auxout) {
    CK(cudaMalloc(&dX, (size_t)(M + guard) * N * 2));
    CK(cudaMemset(dX, 0xFF, (size_t)(M + guard) * N * 2));
  }

  const float alpha = 0.5f;
  vj_set_sm_limit(c.sm_limit);
  int rc = vj_gemm(dA, K, 0, dB, c.b_mn ? N : K, c.b_mn, dD, N, c.d_f32, M, N, K, c.bias ? dBias : nullptr, alpha,
                   c.epi, dAux, N, c.aux_f32, dMap, c.aux_period, dX, N, 1, 0, nullptr);
  vj_set_sm_limit(0);
  char name[128];
  snprintf(name, sizeof(name), "%s%s%s%s B=%s d=%s sm=%d", epi_name(c.epi), c.bias ? "+bias" : "",
           c.aux_f32 ? (c.use_rowmap ? " aux32-rowmap" : (c.aux_period ? " aux32-period" : " aux32")) : "",
           c.auxout ? " aux_out" : "", c.b_mn ? "MN" : "K", c.d_f32 ? "f32" : "bf16", c.sm_limit);
  if (rc != 0) {
    printf("FAIL %-52s vj_gemm rc=%d: %s\n", name, rc, vj_last_error_string());
    return 1;
  }
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    printf("FAIL %-52s kernel error: %s\n", name, cudaGetErrorString(e));
    exit(3);  // context is dead
  }
  const size_t total = (size_t)(M + guard) * N;
  std::vector<float> out(total);
  int bad_guard = 0;
  if (c.d_f32) {
    std::vector<uint32_t> h(total);
    CK(cudaMemcpy(h.data(), dD, total * 4, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < total; ++i) {
      memcpy(&out[i], &h[i], 4);
      if (i >= (size_t)M * N && h[i] != 0xFFFFFFFFu) ++bad_guard;
    }
  } else {
    std::vector<uint16_t> h(total);
    CK(cudaMemcpy(h.data(), dD, total * 2, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < total; ++i) {
      out[i] = bf16_bits(h[i]);
      if (i >= (size_t)M * N && h[i] != 0xFFFF) ++bad_guard;
    }
  }
  std::vector<float> xout;
  if (c.auxout) {
    std::vector<uint16_t> h(total);
    CK(cudaMemcpy(h.data(), dX, total * 2, cudaMemcpyDeviceToHost));
    xout.resize(total);
    for (size_t i = 0; i < total; ++i) {
      xout[i] = bf16_bits(h[i]);
      if (i >= (size_t)M * N && h[i] != 0xFFFF) ++bad_guard;
    }
  }
  double max_err = 0, max_err_x = 0;
  int bad = 0;
  for (int m = 0; m < M; ++m) {
    for (int n = 0; n < N; ++n) {
      double acc = 0;
      const float* a = &A[(size_t)m * K];
      const float* b = &B[(size_t)n * K];
      for (int k = 0; k < K; ++k) acc += (double)a[k] * b[k];
      double v = acc * alpha + bias[n];
      double pre = v;
      const int arow = c.use_rowmap ? rowmap[m] : (c.aux_period > 0 ? m % c.aux_period : m);
      if (c.epi == VJ_EPI_GELU) v = gelu_ref(v);
      else if (c.epi == VJ_EPI_GELU_GRAD) { v = gelu_ref(v); pre = dgelu_ref(pre); }
      else if (c.epi == VJ_EPI_MUL) v *= aux[(size_t)arow * N + n];
      else if (c.epi == VJ_EPI_ADD) v += aux[(size_t)arow * N + n];
      else if (c.epi == VJ_EPI_DGELU) v *= dgelu_ref(aux[(size_t)arow * N + n]);
      const double err = fabs(out[(size_t)m * N + n] - v);
      const double tol = c.d_f32 ? 2e-3 + 1e-4 * fabs(v) : 2e-2 + 8e-3 * fabs(v);
      if (!(err <= tol)) {
        if (bad < 3) printf("   mismatch m=%d n=%d got=%g ref=%g\n", m, n, out[(size_t)m * N + n], v);
        ++bad;
      }
      if (err > max_err) max_err = err;
      if (c.auxout) {
        const double ex = fabs(xout[(size_t)m * N + n] - pre);
        if (ex > max_err_x) max_err_x = ex;
        if (!(ex <= 2e-2 + 8e-3 * fabs(pre))) ++bad;
      }
    }
  }
  const bool coop = N % 256 == 0 && (K + 63) / 64 >= 48;
  const int tiles = ((M + 127) / 128) * (N / (coop ? 256 : (N % 128 == 0 ? 128 : 64)));
  printf("%s %-52s M=%d N=%d K=%d tiles=%d max_err=%.3g auxout_err=%.3g bad=%d guard_written=%d\n",
         (bad || bad_guard) ? "FAIL" : "PASS", name, M, N, K, tiles, max_err, max_err_x, bad, bad_guard);
  cudaFree(dA); cudaFree(dB); cudaFree(dD); cudaFree(dBias);
  if (dAux) cudaFree(dAux);
  if (dMap) cudaFree(dMap);
  if (dX) cudaFree(dX);
  return (bad || bad_guard) ? 1 : 0;
}

int main() {
  int fails = 0;
  std::vector<Case> cases;
  // M, N, K, b_mn, d_f32, epi, aux_f32, rowmap, period, auxout, bias, sm_limit
  // 7 CTAs x 3 tiles (odd count per CTA: warpgroup 0 takes two, warpgroup 1 one), last tile 40 rows
  const int Ms[] = {808, 1000};
  const int Ns[] = {64, 128, 256, 384, 512};
  for (int N : Ns)
    for (int b_mn = 0; b_mn < 2; ++b_mn) {
      cases.push_back({808, N, 320, b_mn, 0, VJ_EPI_NONE, 0, 0, 0, 0, 0, 7});
      cases.push_back({1000, N, 192, b_mn, 0, VJ_EPI_NONE, 0, 0, 0, 0, 1, 1});
    }
  for (int M : Ms)
    for (int sm : {1, 7, 131}) {
      const int N = M == 808 ? 384 : 256;
      cases.push_back({M, N, 256, 0, 0, VJ_EPI_NONE, 0, 0, 0, 0, 1, sm});
      cases.push_back({M, N, 256, 0, 0, VJ_EPI_GELU, 0, 0, 0, 1, 1, sm});
      cases.push_back({M, N, 256, 0, 0, VJ_EPI_GELU, 0, 0, 0, 0, 1, sm});
      cases.push_back({M, N, 256, 0, 0, VJ_EPI_GELU_GRAD, 0, 0, 0, 1, 1, sm});
      cases.push_back({M, N, 256, 0, 0, VJ_EPI_ADD, 0, 0, 0, 0, 1, sm});
      cases.push_back({M, N, 256, 0, 0, VJ_EPI_ADD, 1, 1, 0, 0, 1, sm});
      cases.push_back({M, N, 256, 0, 0, VJ_EPI_ADD, 1, 0, 100, 0, 1, sm});
      cases.push_back({M, N, 256, 0, 1, VJ_EPI_ADD, 1, 0, 0, 0, 1, sm});
      cases.push_back({M, N, 256, 0, 0, VJ_EPI_DGELU, 0, 0, 0, 0, 0, sm});
      cases.push_back({M, N, 256, 1, 0, VJ_EPI_DGELU, 0, 0, 0, 0, 0, sm});
      cases.push_back({M, N, 256, 1, 0, VJ_EPI_MUL, 0, 0, 0, 0, 0, sm});
      cases.push_back({M, N, 256, 1, 1, VJ_EPI_NONE, 0, 0, 0, 0, 0, sm});
    }
  // 132 tiles (66 x 2): with the budget at 131 CTAs one CTA takes two tiles, the others one
  cases.push_back({8448, 256, 192, 0, 0, VJ_EPI_ADD, 0, 0, 0, 0, 1, 131});
  cases.push_back({8448, 256, 192, 1, 0, VJ_EPI_MUL, 0, 0, 0, 0, 0, 131});
  // long K (>= 48 k-blocks) with N % 256 == 0: the cooperative 128 x 256 schedule.  M = 1050: the last tile has 26
  // rows, so the second warpgroup's half of it lies wholly past M
  for (int sm : {1, 7, 0}) {
    cases.push_back({1050, 512, 3072, 0, 0, VJ_EPI_ADD, 0, 0, 0, 0, 1, sm});
    cases.push_back({1050, 512, 3072, 1, 0, VJ_EPI_NONE, 0, 0, 0, 0, 0, sm});
  }
  cases.push_back({1050, 256, 3072, 0, 0, VJ_EPI_GELU_GRAD, 0, 0, 0, 1, 1, 7});
  cases.push_back({1050, 256, 3072, 0, 0, VJ_EPI_GELU, 0, 0, 0, 1, 1, 7});
  cases.push_back({1050, 256, 3072, 0, 0, VJ_EPI_GELU, 0, 0, 0, 0, 1, 7});
  cases.push_back({1050, 256, 3072, 1, 0, VJ_EPI_DGELU, 0, 0, 0, 0, 0, 7});
  cases.push_back({1050, 256, 3072, 1, 0, VJ_EPI_MUL, 0, 0, 0, 0, 0, 7});
  cases.push_back({1050, 256, 3072, 0, 0, VJ_EPI_ADD, 1, 1, 0, 0, 1, 7});
  cases.push_back({1050, 256, 3072, 0, 1, VJ_EPI_ADD, 1, 0, 100, 0, 1, 7});
  cases.push_back({1050, 256, 3072, 1, 1, VJ_EPI_NONE, 0, 0, 0, 0, 0, 7});
  // N = 64 (one 64-wide tile column) with aux epilogues; a single-tile problem of 1 row and of a full tile
  cases.push_back({808, 64, 192, 1, 0, VJ_EPI_MUL, 0, 0, 0, 0, 0, 7});
  cases.push_back({808, 192, 192, 0, 0, VJ_EPI_GELU_GRAD, 0, 0, 0, 1, 1, 7});
  cases.push_back({808, 192, 192, 0, 0, VJ_EPI_ADD, 0, 0, 0, 0, 1, 7});
  cases.push_back({1, 128, 64, 0, 0, VJ_EPI_GELU, 0, 0, 0, 1, 1, 0});
  cases.push_back({128, 128, 1000, 0, 0, VJ_EPI_ADD, 0, 0, 0, 0, 1, 0});
  cases.push_back({50, 64, 64, 1, 0, VJ_EPI_DGELU, 0, 0, 0, 0, 0, 0});
  for (const Case& c : cases) fails += run_case(c);
  printf("%s: %d failing case(s)\n", fails ? "FAILED" : "ALL PASSED", fails);
  return fails ? 1 : 0;
}
