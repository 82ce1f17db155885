// Stand-alone test for the attentive probe's cross-attention (vj_cross_attn_fwd / _fwd_lse / _bwd) on an H100 (no torch):
// forward, softmax statistics and gradients against a double-precision host reference.
//   test_xattn        correctness cases, then "ALL PASSED" / "FAILED"
//   test_xattn perf   forward and backward timings at the ViT-L / ViT-H K400 probe shapes
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

static uint32_t rng_state = 4242;
static float frand() {
  rng_state = rng_state * 1664525u + 1013904223u;
  return ((rng_state >> 8) & 0xFFFF) / 32768.0f - 1.0f;
}
static float bf(float x) { return __bfloat162float(__float2bfloat16(x)); }
static float tof(__nv_bfloat16 x) { return __bfloat162float(x); }

static std::vector<__nv_bfloat16> to_bf16(const std::vector<float>& v) {
  std::vector<__nv_bfloat16> o(v.size());
  for (size_t i = 0; i < v.size(); ++i) o[i] = __float2bfloat16(v[i]);
  return o;
}

struct Tol {
  double max_abs = 0, max_ref = 0;
  int bad = 0;
  // |got - ref| <= rel * |ref| + floor_rel * max|ref| of the tensor (checked after the scan, see finish())
  std::vector<double> got, ref;
  void add(double g, double r) { got.push_back(g); ref.push_back(r); if (fabs(r) > max_ref) max_ref = fabs(r); }
  int finish(const char* what, double rel, double floor_rel) {
    for (size_t i = 0; i < got.size(); ++i) {
      const double e = fabs(got[i] - ref[i]);
      if (e > max_abs) max_abs = e;
      if (!(e <= rel * fabs(ref[i]) + floor_rel * max_ref)) {
        if (bad < 4) printf("   %s mismatch at %zu: got %.6g ref %.6g\n", what, i, got[i], ref[i]);
        ++bad;
      }
    }
    return bad;
  }
};

static int run(int B, int nq, int S, int H, int HD) {
  const int D = H * HD;
  const float scale = 1.0f / sqrtf((float)HD);
  std::vector<float> q((size_t)B * nq * D), kv((size_t)B * S * 2 * D), dO((size_t)B * nq * D);
  for (auto& x : q) x = bf(frand() * 2.0f);
  for (auto& x : kv) x = bf(frand() * 2.0f);
  for (auto& x : dO) x = bf(frand());
  // plant large keys late in the sequence for query 0 of every clip: the running max moves after most keys were seen
  for (int b = 0; b < B; ++b)
    for (int h = 0; h < H; ++h)
      for (int j : {S - 1, S - 1 - S / 3}) {
        if (j < 0 || S < 3) continue;
        for (int d = 0; d < HD; ++d) {
          const float qd = q[((size_t)b * nq) * D + h * HD + d];
          kv[((size_t)b * S + j) * 2 * D + h * HD + d] = bf(qd >= 0 ? 2.0f : -2.0f) * (j == S - 1 ? 1.0f : 0.75f);
        }
      }
  auto hq = to_bf16(q), hkv = to_bf16(kv), hdo = to_bf16(dO);
  void *dq_in, *dkv_in, *dout1, *dout2, *ddo, *ddkv;
  float *dlse, *ddq;
  const size_t ws_bytes = vj_cross_attn_bwd_workspace(B, nq, S, H, HD);
  void* dws;
  CK(cudaMalloc(&dq_in, hq.size() * 2)); CK(cudaMalloc(&dkv_in, hkv.size() * 2));
  CK(cudaMalloc(&dout1, hq.size() * 2)); CK(cudaMalloc(&dout2, hq.size() * 2)); CK(cudaMalloc(&ddo, hq.size() * 2));
  CK(cudaMalloc(&ddkv, hkv.size() * 2)); CK(cudaMalloc(&dlse, (size_t)B * nq * H * 4)); CK(cudaMalloc(&ddq, q.size() * 4));
  CK(cudaMalloc(&dws, ws_bytes));
  CK(cudaMemcpy(dq_in, hq.data(), hq.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dkv_in, hkv.data(), hkv.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(ddo, hdo.data(), hdo.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemset(dout1, 0xFF, hq.size() * 2)); CK(cudaMemset(dout2, 0xFF, hq.size() * 2));
  CK(cudaMemset(ddkv, 0xFF, hkv.size() * 2)); CK(cudaMemset(ddq, 0xFF, q.size() * 4));
  int rc = vj_cross_attn_fwd(dq_in, dkv_in, dout1, B, nq, S, H, HD, scale, nullptr);
  rc |= vj_cross_attn_fwd_lse(dq_in, dkv_in, dout2, dlse, B, nq, S, H, HD, scale, nullptr);
  if (rc) { printf("FAIL fwd rc=%d %s\n", rc, vj_last_error_string()); return 1; }
  rc = vj_cross_attn_bwd(dq_in, dkv_in, dout2, ddo, dlse, ddq, ddkv, dws, ws_bytes, B, nq, S, H, HD, scale, nullptr);
  if (rc) { printf("FAIL bwd rc=%d %s\n", rc, vj_last_error_string()); return 1; }
  CK(cudaDeviceSynchronize());
  std::vector<__nv_bfloat16> o1(hq.size()), o2(hq.size()), gkv(hkv.size()), gkv2(hkv.size());
  std::vector<float> lse((size_t)B * nq * H), gq(q.size()), gq2(q.size());
  CK(cudaMemcpy(o1.data(), dout1, o1.size() * 2, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(o2.data(), dout2, o2.size() * 2, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(lse.data(), dlse, lse.size() * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(gq.data(), ddq, gq.size() * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(gkv.data(), ddkv, gkv.size() * 2, cudaMemcpyDeviceToHost));
  // a second backward on the same inputs must be bitwise identical (no atomics)
  CK(cudaMemset(ddkv, 0, hkv.size() * 2)); CK(cudaMemset(ddq, 0, q.size() * 4));
  rc = vj_cross_attn_bwd(dq_in, dkv_in, dout2, ddo, dlse, ddq, ddkv, dws, ws_bytes, B, nq, S, H, HD, scale, nullptr);
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(gq2.data(), ddq, gq2.size() * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(gkv2.data(), ddkv, gkv2.size() * 2, cudaMemcpyDeviceToHost));
  int bad = 0;
  if (memcmp(o1.data(), o2.data(), o1.size() * 2)) { printf("   O differs between vj_cross_attn_fwd and _fwd_lse\n"); ++bad; }
  if (rc || memcmp(gq.data(), gq2.data(), gq.size() * 4) || memcmp(gkv.data(), gkv2.data(), gkv.size() * 2)) {
    printf("   backward is not bitwise reproducible\n");
    ++bad;
  }

  Tol to, tl, tq, tk, tv;
  std::vector<double> P(S), dp(S);
  for (int b = 0; b < B; ++b)
    for (int h = 0; h < H; ++h) {
      std::vector<double> dk((size_t)S * HD, 0.0), dv((size_t)S * HD, 0.0);
      for (int i = 0; i < nq; ++i) {
        const size_t r = (size_t)b * nq + i;
        const float* qi = &q[r * D + h * HD];
        const float* gi = &dO[r * D + h * HD];
        double mx = -1e300;
        for (int j = 0; j < S; ++j) {
          const float* kj = &kv[((size_t)b * S + j) * 2 * D + h * HD];
          double s = 0;
          for (int d = 0; d < HD; ++d) s += (double)qi[d] * kj[d];
          P[j] = s * scale;
          if (P[j] > mx) mx = P[j];
        }
        double sum = 0;
        for (int j = 0; j < S; ++j) { P[j] = exp(P[j] - mx); sum += P[j]; }
        for (int j = 0; j < S; ++j) P[j] /= sum;
        tl.add(lse[r * H + h], (mx + log(sum)) * 1.4426950408889634);
        std::vector<double> O(HD, 0.0);
        for (int j = 0; j < S; ++j)
          for (int d = 0; d < HD; ++d) O[d] += P[j] * kv[((size_t)b * S + j) * 2 * D + D + h * HD + d];
        // the backward sees the bf16 O the forward stored
        double delta = 0;
        for (int d = 0; d < HD; ++d) {
          to.add(tof(o2[r * D + h * HD + d]), O[d]);
          delta += (double)gi[d] * tof(o2[r * D + h * HD + d]);
        }
        std::vector<double> gq_ref(HD, 0.0);
        for (int j = 0; j < S; ++j) {
          const float* kj = &kv[((size_t)b * S + j) * 2 * D + h * HD];
          const float* vj = kj + D;
          double d_p = 0;
          for (int d = 0; d < HD; ++d) d_p += (double)gi[d] * vj[d];
          const double ds = P[j] * (d_p - delta);
          for (int d = 0; d < HD; ++d) {
            gq_ref[d] += ds * kj[d];
            dk[(size_t)j * HD + d] += scale * ds * qi[d];
            dv[(size_t)j * HD + d] += P[j] * gi[d];
          }
        }
        for (int d = 0; d < HD; ++d) tq.add(gq[r * D + h * HD + d], scale * gq_ref[d]);
      }
      for (int j = 0; j < S; ++j)
        for (int d = 0; d < HD; ++d) {
          tk.add(tof(gkv[((size_t)b * S + j) * 2 * D + h * HD + d]), dk[(size_t)j * HD + d]);
          tv.add(tof(gkv[((size_t)b * S + j) * 2 * D + D + h * HD + d]), dv[(size_t)j * HD + d]);
        }
    }
  bad += to.finish("O", 1e-2, 5e-3);
  bad += tl.finish("lse2", 1e-4, 1e-5);
  bad += tq.finish("dq", 1e-2, 5e-3);
  bad += tk.finish("dk", 1e-2, 5e-3);
  bad += tv.finish("dv", 1e-2, 5e-3);
  printf("%s xattn B=%d nq=%d S=%d H=%d HD=%d: max err O=%.3g lse2=%.3g dq=%.3g (max %.3g) dk=%.3g (max %.3g) dv=%.3g (max %.3g)\n",
         bad ? "FAIL" : "PASS", B, nq, S, H, HD, to.max_abs, tl.max_abs, tq.max_abs, tq.max_ref, tk.max_abs, tk.max_ref,
         tv.max_abs, tv.max_ref);
  cudaFree(dq_in); cudaFree(dkv_in); cudaFree(dout1); cudaFree(dout2); cudaFree(ddo); cudaFree(ddkv); cudaFree(dlse);
  cudaFree(ddq); cudaFree(dws);
  return bad ? 1 : 0;
}

// Timings at the frozen-evaluation shape: B clips of S tokens, nq = 1.  Bytes: the forward reads kv (B S 2D 2 bytes),
// the backward reads kv and writes dkv (2 x that); q, out, dout, lse2 and dq are negligible.
static void perf(const char* name, int B, int S, int H, int HD) {
  const int D = H * HD, nq = 1;
  const float scale = 1.0f / sqrtf((float)HD);
  const size_t nkv = (size_t)B * S * 2 * D;
  void *dq_in, *dkv_in, *dout, *ddo, *ddkv, *dws;
  float *dlse, *ddq;
  const size_t ws_bytes = vj_cross_attn_bwd_workspace(B, nq, S, H, HD);
  CK(cudaMalloc(&dq_in, (size_t)B * D * 2)); CK(cudaMalloc(&dkv_in, nkv * 2)); CK(cudaMalloc(&dout, (size_t)B * D * 2));
  CK(cudaMalloc(&ddo, (size_t)B * D * 2)); CK(cudaMalloc(&ddkv, nkv * 2)); CK(cudaMalloc(&dlse, (size_t)B * H * 4));
  CK(cudaMalloc(&ddq, (size_t)B * D * 4)); CK(cudaMalloc(&dws, ws_bytes));
  CK(cudaMemset(dq_in, 0x3C, (size_t)B * D * 2)); CK(cudaMemset(dkv_in, 0x3C, nkv * 2));
  CK(cudaMemset(ddo, 0x3C, (size_t)B * D * 2));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  const int iters = 20;
  float ms_f = 0, ms_b = 0;
  for (int rep = 0; rep < 2; ++rep) {   // first round warms up
    CK(cudaEventRecord(e0));
    for (int i = 0; i < iters; ++i) vj_cross_attn_fwd_lse(dq_in, dkv_in, dout, dlse, B, nq, S, H, HD, scale, nullptr);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    CK(cudaEventElapsedTime(&ms_f, e0, e1));
    CK(cudaEventRecord(e0));
    for (int i = 0; i < iters; ++i)
      vj_cross_attn_bwd(dq_in, dkv_in, dout, ddo, dlse, ddq, ddkv, dws, ws_bytes, B, nq, S, H, HD, scale, nullptr);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    CK(cudaEventElapsedTime(&ms_b, e0, e1));
  }
  CK(cudaGetLastError());
  ms_f /= iters; ms_b /= iters;
  const double gb = nkv * 2 * 1e-9;
  printf("PERF xattn %s B=%d S=%d H=%d HD=%d: fwd %.3f ms (%.0f GB/s of %.3f GB), bwd %.3f ms (%.0f GB/s of %.3f GB)\n",
         name, B, S, H, HD, ms_f, gb / ms_f * 1e3, gb, ms_b, 2 * gb / ms_b * 1e3, 2 * gb);
  cudaFree(dq_in); cudaFree(dkv_in); cudaFree(dout); cudaFree(ddo); cudaFree(ddkv); cudaFree(dlse); cudaFree(ddq);
  cudaFree(dws);
}

int main(int argc, char** argv) {
  if (argc > 1 && !strcmp(argv[1], "perf")) {
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    printf("device: %s\n", prop.name);
    perf("ViT-L", 4, 12544, 16, 64);
    perf("ViT-H", 4, 12544, 16, 80);
    return 0;
  }
  int fails = 0;
  for (int HD : {32, 64, 80, 128})
    for (int nq : {1, 3})
      for (int S : {1, 7, 33, 1568, 1571, 12544}) fails += run(2, nq, S, 2, HD);
  fails += run(4, 1, 1568, 16, 64);   // many heads: every (head, clip, key chunk) CTA of a probe-sized problem
  printf("%s: %d failing case(s)\n", fails ? "FAILED" : "ALL PASSED", fails);
  return fails ? 1 : 0;
}
