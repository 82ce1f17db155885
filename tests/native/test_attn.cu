// Stand-alone bring-up test for vj_attn_fwd / vj_attn_bwd on an H100 (no torch).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "vjepa_b200.h"

#define CK(x)                                                                        \
  do {                                                                               \
    cudaError_t e = (x);                                                             \
    if (e != cudaSuccess) {                                                          \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); \
      exit(2);                                                                       \
    }                                                                                \
  } while (0)

static uint32_t rng_state = 777;
static float frand() {
  rng_state = rng_state * 1664525u + 1013904223u;
  return ((rng_state >> 8) & 0xFFFF) / 32768.0f - 1.0f;
}
static float bf(float x) { return __bfloat162float(__float2bfloat16(x)); }

// hd_real < HD emulates the zero-padded predictor heads (24 -> 32)
static int run(int H, int HD, int hd_real, const std::vector<int>& lens, bool do_bwd) {
  const int nseq = (int)lens.size();
  std::vector<int> cu(nseq + 1, 0);
  int max_len = 0;
  for (int i = 0; i < nseq; ++i) { cu[i + 1] = cu[i] + lens[i]; if (lens[i] > max_len) max_len = lens[i]; }
  const int T = cu[nseq];
  const int W = 3 * H * HD, D = H * HD;
  const float scale = 1.0f / sqrtf((float)hd_real);
  std::vector<float> qkv((size_t)T * W), dO((size_t)T * D);
  for (int t = 0; t < T; ++t)
    for (int c = 0; c < W; ++c) {
      const int d = c % HD;
      qkv[(size_t)t * W + c] = d < hd_real ? bf(frand() * 2.0f) : 0.f;
    }
  for (int t = 0; t < T; ++t)
    for (int c = 0; c < D; ++c) dO[(size_t)t * D + c] = (c % HD) < hd_real ? bf(frand()) : 0.f;
  std::vector<__nv_bfloat16> hq(qkv.size()), hdo(dO.size());
  for (size_t i = 0; i < qkv.size(); ++i) hq[i] = __float2bfloat16(qkv[i]);
  for (size_t i = 0; i < dO.size(); ++i) hdo[i] = __float2bfloat16(dO[i]);
  void *dq, *dout, *ddo, *ddqkv;
  float *dlse, *ddelta, *ddqacc;
  int* dcu;
  CK(cudaMalloc(&dq, hq.size() * 2));
  CK(cudaMalloc(&dout, (size_t)T * D * 2));
  CK(cudaMalloc(&ddo, (size_t)T * D * 2));
  CK(cudaMalloc(&ddqkv, hq.size() * 2));
  CK(cudaMalloc(&dlse, (size_t)H * T * 4));
  CK(cudaMalloc(&ddelta, (size_t)H * T * 4));
  CK(cudaMalloc(&ddqacc, (size_t)T * D * 4));
  CK(cudaMalloc(&dcu, (nseq + 1) * 4));
  CK(cudaMemcpy(dq, hq.data(), hq.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(ddo, hdo.data(), hdo.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dcu, cu.data(), (nseq + 1) * 4, cudaMemcpyHostToDevice));
  CK(cudaMemset(dout, 0xFF, (size_t)T * D * 2));
  CK(cudaMemset(ddqkv, 0xFF, hq.size() * 2));
  int rc = vj_attn_fwd(dq, dout, dlse, dcu, nseq, max_len, H, HD, T, scale, nullptr);
  if (rc) { printf("FAIL attn_fwd rc=%d %s\n", rc, vj_last_error_string()); return 1; }
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("FAIL attn_fwd kernel error %s\n", cudaGetErrorString(e)); exit(3); }
  if (do_bwd) {
    rc = vj_attn_bwd(dq, dout, ddo, dlse, ddelta, ddqkv, ddqacc, dcu, nseq, max_len, H, HD, T, scale, nullptr);
    if (rc) { printf("FAIL attn_bwd rc=%d %s\n", rc, vj_last_error_string()); return 1; }
    e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { printf("FAIL attn_bwd kernel error %s\n", cudaGetErrorString(e)); exit(3); }
  }
  std::vector<__nv_bfloat16> ho((size_t)T * D), hdq(hq.size());
  std::vector<float> hl((size_t)H * T);
  CK(cudaMemcpy(ho.data(), dout, ho.size() * 2, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(hl.data(), dlse, hl.size() * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(hdq.data(), ddqkv, hdq.size() * 2, cudaMemcpyDeviceToHost));

  double max_err_o = 0, max_err_l = 0, max_err_g = 0, max_g = 0;
  int bad = 0;
  // reference per (seq, head); check a subset of heads for speed
  for (int s = 0; s < nseq; ++s) {
    const int L = lens[s], r0 = cu[s];
    for (int h = 0; h < H; h += (H > 4 ? H / 2 : 1)) {
      std::vector<double> P((size_t)L * L), O((size_t)L * HD), lse(L);
      for (int i = 0; i < L; ++i) {
        const float* q = &qkv[(size_t)(r0 + i) * W + h * HD];
        double mx = -1e30;
        for (int j = 0; j < L; ++j) {
          const float* k = &qkv[(size_t)(r0 + j) * W + D + h * HD];
          double sdot = 0;
          for (int d = 0; d < HD; ++d) sdot += (double)q[d] * k[d];
          P[(size_t)i * L + j] = sdot * scale;
          if (sdot * scale > mx) mx = sdot * scale;
        }
        double sum = 0;
        for (int j = 0; j < L; ++j) { P[(size_t)i * L + j] = exp(P[(size_t)i * L + j] - mx); sum += P[(size_t)i * L + j]; }
        for (int j = 0; j < L; ++j) P[(size_t)i * L + j] /= sum;
        lse[i] = (mx + log(sum)) * 1.4426950408889634;
        for (int d = 0; d < HD; ++d) {
          double acc = 0;
          for (int j = 0; j < L; ++j) acc += P[(size_t)i * L + j] * qkv[(size_t)(r0 + j) * W + 2 * D + h * HD + d];
          O[(size_t)i * HD + d] = acc;
          const double got = __bfloat162float(ho[(size_t)(r0 + i) * D + h * HD + d]);
          const double err = fabs(got - acc);
          if (err > max_err_o) max_err_o = err;
          if (!(err <= 2e-2 + 1e-2 * fabs(acc))) { if (bad < 5) printf("   O mismatch s=%d h=%d i=%d d=%d got=%g ref=%g\n", s, h, i, d, got, acc); ++bad; }
        }
        const double el = fabs(hl[(size_t)h * T + r0 + i] - lse[i]);
        if (el > max_err_l) max_err_l = el;
        if (!(el <= 2e-2)) { if (bad < 5) printf("   LSE mismatch s=%d h=%d i=%d got=%g ref=%g\n", s, h, i, hl[(size_t)h * T + r0 + i], lse[i]); ++bad; }
      }
      if (do_bwd) {
        // dV = P^T dO ; dP = dO V^T ; dS = P * (dP - rowsum(dO*O)) ; dQ = scale dS K ; dK = scale dS^T Q
        std::vector<double> dS((size_t)L * L);
        static unsigned badmap[3][512];
        memset(badmap, 0, sizeof(badmap));
        for (int i = 0; i < L; ++i) {
          double delta = 0;
          for (int d = 0; d < HD; ++d) delta += (double)dO[(size_t)(r0 + i) * D + h * HD + d] * O[(size_t)i * HD + d];
          for (int j = 0; j < L; ++j) {
            double dp = 0;
            for (int d = 0; d < HD; ++d)
              dp += (double)dO[(size_t)(r0 + i) * D + h * HD + d] * qkv[(size_t)(r0 + j) * W + 2 * D + h * HD + d];
            dS[(size_t)i * L + j] = P[(size_t)i * L + j] * (dp - delta);
          }
        }
        for (int i = 0; i < L; ++i)
          for (int d = 0; d < HD; ++d) {
            double gq = 0, gk = 0, gv = 0;
            for (int j = 0; j < L; ++j) {
              gq += dS[(size_t)i * L + j] * qkv[(size_t)(r0 + j) * W + D + h * HD + d];
              gk += dS[(size_t)j * L + i] * qkv[(size_t)(r0 + j) * W + h * HD + d];
              gv += P[(size_t)j * L + i] * dO[(size_t)(r0 + j) * D + h * HD + d];
            }
            gq *= scale; gk *= scale;
            const double ref[3] = {gq, gk, gv};
            for (int w = 0; w < 3; ++w) {
              const double got = __bfloat162float(hdq[(size_t)(r0 + i) * W + w * D + h * HD + d]);
              const double err = fabs(got - ref[w]);
              if (err > max_err_g) max_err_g = err;
              if (fabs(ref[w]) > max_g) max_g = fabs(ref[w]);
              if (!(err <= 3e-2 + 2e-2 * fabs(ref[w]))) {
                if (bad < 8) printf("   grad mismatch which=%d s=%d h=%d i=%d d=%d got=%g ref=%g\n", w, s, h, i, d, got, ref[w]);
                ++bad;
                if (getenv("VJ_TEST_BADMAP") && i < 512) { badmap[w][i] |= 1u << (d & 31); }
              }
            }
          }
        if (getenv("VJ_TEST_BADMAP")) {
          for (int w = 0; w < 3; ++w) {
            int nb = 0;
            for (int i = 0; i < L && i < 512; ++i) nb += badmap[w][i] != 0;
            if (!nb) continue;
            printf("   badmap which=%d s=%d h=%d: %d bad rows; row:mask(d) =", w, s, h, nb);
            for (int i = 0, k = 0; i < L && i < 512 && k < 24; ++i) if (badmap[w][i]) { printf(" %d:%08x", i, badmap[w][i]); ++k; }
            printf("\n");
          }
        }
      }
    }
  }
  printf("%s attn H=%d HD=%d(real %d) nseq=%d T=%d max_len=%d bwd=%d: max_err_O=%.4g lse=%.4g grad=%.4g (max grad %.3g) bad=%d\n",
         bad ? "FAIL" : "PASS", H, HD, hd_real, nseq, T, max_len, (int)do_bwd, max_err_o, max_err_l, max_err_g, max_g, bad);
  cudaFree(dq); cudaFree(dout); cudaFree(ddo); cudaFree(ddqkv); cudaFree(dlse); cudaFree(ddelta); cudaFree(dcu);
  return bad ? 1 : 0;
}

static void perf(int H, int HD, int nseq, int L, bool bwd) {
  const int T = nseq * L, W = 3 * H * HD, D = H * HD;
  std::vector<int> cu(nseq + 1);
  for (int i = 0; i <= nseq; ++i) cu[i] = i * L;
  void *dq, *dout, *ddo, *ddqkv; float *dlse, *ddelta, *ddqacc; int* dcu;
  CK(cudaMalloc(&dq, (size_t)T * W * 2)); CK(cudaMalloc(&dout, (size_t)T * D * 2));
  CK(cudaMalloc(&ddo, (size_t)T * D * 2)); CK(cudaMalloc(&ddqkv, (size_t)T * W * 2));
  CK(cudaMalloc(&dlse, (size_t)H * T * 4)); CK(cudaMalloc(&ddelta, (size_t)H * T * 4));
  CK(cudaMalloc(&ddqacc, (size_t)T * D * 4));
  CK(cudaMalloc(&dcu, (nseq + 1) * 4));
  CK(cudaMemset(dq, 0x3C, (size_t)T * W * 2)); CK(cudaMemset(ddo, 0x3C, (size_t)T * D * 2));
  CK(cudaMemcpy(dcu, cu.data(), (nseq + 1) * 4, cudaMemcpyHostToDevice));
  const float scale = 1.0f / sqrtf((float)HD);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int i = 0; i < 2; ++i) {
    vj_attn_fwd(dq, dout, dlse, dcu, nseq, L, H, HD, T, scale, nullptr);
    if (bwd) vj_attn_bwd(dq, dout, ddo, dlse, ddelta, ddqkv, ddqacc, dcu, nseq, L, H, HD, T, scale, nullptr);
  }
  CK(cudaDeviceSynchronize());
  const int iters = 5;
  cudaEventRecord(e0);
  for (int i = 0; i < iters; ++i) {
    if (!bwd) vj_attn_fwd(dq, dout, dlse, dcu, nseq, L, H, HD, T, scale, nullptr);
    else vj_attn_bwd(dq, dout, ddo, dlse, ddelta, ddqkv, ddqacc, dcu, nseq, L, H, HD, T, scale, nullptr);
  }
  cudaEventRecord(e1);
  CK(cudaDeviceSynchronize());
  float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= iters;
  const double flops = 4.0 * nseq * H * (double)L * L * HD * (bwd ? 2.5 : 1.0);
  printf("PERF attn %s H=%d HD=%d nseq=%d L=%d: %.3f ms  %.1f TFLOP/s (algorithmic)\n", bwd ? "bwd" : "fwd", H, HD, nseq, L, ms, flops / ms * 1e-9);
  cudaFree(dq); cudaFree(dout); cudaFree(ddo); cudaFree(ddqkv); cudaFree(dlse); cudaFree(ddelta); cudaFree(dcu);
}

int main(int argc, char** argv) {
  const bool bwd = !(argc > 1 && !strcmp(argv[1], "fwd"));
  int fails = 0;
  if (argc > 1 && !strcmp(argv[1], "perf")) {   // timing only (ablation experiments)
    perf(16, 64, 32, 1568, false);
    perf(16, 32, 32, 1184, false);
    perf(16, 64, 32, 360, true);
    perf(16, 32, 32, 1184, true);
    return 0;
  }
  if (argc > 1 && !strcmp(argv[1], "fwdbig")) {   // forward only: BASELINE sequence lengths, tails, persistence (> 132 work items)
    fails += run(2, 64, 64, {128}, false);
    fails += run(2, 64, 64, {1}, false);
    fails += run(2, 64, 64, {129, 127, 256, 257, 17}, false);
    fails += run(2, 64, 64, {1568}, false);
    fails += run(2, 32, 24, {1184, 1192}, false);
    fails += run(2, 64, 64, {360, 48, 360}, false);
    fails += run(1, 128, 80, {1568, 200}, false);
    fails += run(16, 64, 64, {300, 300, 300, 300, 300, 300, 300, 300, 40, 513}, false);   // 480 items: persistent CTAs, mixed 1- / 2-tile items
    fails += run(16, 32, 24, {520, 300, 300, 300, 300, 300, 300, 300}, false);
    fails += run(8, 128, 128, {300, 300, 300, 300, 300, 300, 300, 300, 300, 300, 300, 700}, false);
    perf(16, 64, 32, 1568, false);
    perf(16, 32, 32, 1184, false);
    perf(16, 64, 32, 360, false);
    perf(16, 128, 24, 1568, false);
    printf("%s: %d failing case(s)\n", fails ? "FAILED" : "ALL PASSED", fails);
    return fails ? 1 : 0;
  }
  if (argc > 2 && !strcmp(argv[1], "bwdone")) {   // one backward case: sequence length from the command line
    fails += run(2, 32, 24, {atoi(argv[2])}, true);
    return fails ? 1 : 0;
  }
  if (argc > 1 && !strcmp(argv[1], "bwdbig")) {   // backward at BASELINE predictor lengths, tails, persistence
    fails += run(2, 32, 24, {128}, true);
    fails += run(2, 32, 24, {1}, true);
    fails += run(2, 32, 24, {129, 127, 256, 257, 17, 300}, true);
    fails += run(2, 32, 24, {1184, 1192}, true);
    fails += run(1, 32, 32, {3680}, true);
    fails += run(16, 32, 24, {520, 300, 300, 300, 300, 300, 300, 300}, true);   // 384 items: persistent, mixed 1- / 2-tile items
    fails += run(2, 64, 64, {360, 48}, true);
    perf(16, 32, 32, 1184, true);
    perf(16, 32, 32, 1192, true);
    perf(16, 64, 32, 360, true);
    printf("%s: %d failing case(s)\n", fails ? "FAILED" : "ALL PASSED", fails);
    return fails ? 1 : 0;
  }
  fails += run(2, 64, 64, {128}, bwd);
  fails += run(2, 64, 64, {200, 48, 136}, bwd);
  fails += run(3, 32, 24, {296, 40}, bwd);
  fails += run(2, 128, 128, {160, 72}, bwd);
  fails += run(16, 64, 64, {392, 392, 56}, bwd);
  printf("%s: %d failing case(s)\n", fails ? "FAILED" : "ALL PASSED", fails);
  return fails ? 1 : 0;
}
