// Self-attention among the query tokens of the attentive probe: the `depth - 1` transformer Blocks that
// AttentivePooler(depth > 1) runs after its cross-attention block (src/models/attentive_pooler.py:52-102,
// Attention.forward of src/models/utils/modules.py:61-78).
//
//   qkv  [B*nq, 3*H*hd]   the Block's qkv Linear output: q | k | v thirds, head-major inside a third (the reference's
//                          reshape(B, N, 3, H, hd)); row b*nq + i = token i of clip b
//   out  [B*nq, H*hd]     = softmax(q k^T * scale) v within each clip's nq tokens, per head
//   lse2 fp32 [B*nq, H]   log2-domain softmax statistics for the backward (like vj_cross_attn_fwd_lse); optional
//   dqkv [B*nq, 3*H*hd]   backward, in the qkv layout, so the qkv dgrad / wgrad GEMMs read it directly
//
// nq <= 128 tokens per clip and hd in {32, 64, 80, 88, 104, 128}: a whole (clip, head) problem fits in shared memory,
// so one CTA takes one (head, clip).  The tokens are copied to shared memory as 16-bit rows of hd + 2 elements (an odd
// number of 32-bit words, so a warp whose lanes read 32 different rows hits 32 different banks); the probabilities live
// in an fp32 [nq][nq + 1] matrix.  Scores: one warp per query row, one lane per key.  Products with the probability
// matrix: one thread per (row, pair of columns), looping over the other token index in order.  Every output element is
// written once by one thread, with a fixed summation order: no atomics, the backward is deterministic.
//
// With nq = 1 the softmax over one key is exactly 1 (p / l with l = p), so out is bitwise v; in the backward delta_i
// and dO_i . v_j are the same dot product in the same order, so ds = 0 and dq = dk = 0 exactly.
#include "common.cuh"
#include "vjepa_b200.h"

namespace vj {

constexpr int kQattnThreads = 256;
constexpr int kQattnMaxTokens = 128;

// dot product of two 16-bit rows of HD elements read as 32-bit pairs, one fma chain in element order
template <typename T, int HD>
VJ_DEVINL float qattn_dot(const uint32_t* a, const uint32_t* b) {
  using E = Elt<T>;
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < HD / 2; ++w) {
    const uint32_t x = a[w], y = b[w];
    s = fmaf(E::lo(x), E::lo(y), s);
    s = fmaf(E::hi(x), E::hi(y), s);
  }
  return s;
}

template <int HD>
__host__ __device__ constexpr int qattn_row_words() { return HD / 2 + 1; }

// bytes of dynamic shared memory: `rows` 16-bit token matrices, the fp32 probability matrix and (backward) delta
template <int HD>
__host__ __device__ constexpr size_t qattn_smem(int nq, int rows, bool bwd) {
  return ((size_t)rows * nq * qattn_row_words<HD>() + (size_t)nq * (nq + 1) + (bwd ? nq : 0)) * 4;
}

// copy row r of `src` (16-bit, row stride ld elements, HD elements from column 0) into shared row r of dst
template <int HD, typename T>
VJ_DEVINL void qattn_load(uint32_t* dst, const T* src, long long ld, int nq) {
  constexpr int W = HD / 2, RS = qattn_row_words<HD>();
  for (int t = threadIdx.x; t < nq * W; t += kQattnThreads) {
    const int r = t / W, w = t % W;
    dst[r * RS + w] = reinterpret_cast<const uint32_t*>(src + r * ld)[w];
  }
}

// grid (H, B)
template <typename T, int HD>
__global__ void __launch_bounds__(kQattnThreads) qattn_fwd_kernel(const T* __restrict__ qkv, T* __restrict__ out,
                                                                  float* __restrict__ lse2, int nq, int H,
                                                                  float scale_log2) {
  using E = Elt<T>;
  constexpr int W = HD / 2, RS = qattn_row_words<HD>();
  extern __shared__ __align__(16) uint32_t qattn_sm[];
  uint32_t* sq = qattn_sm;
  uint32_t* sk = sq + nq * RS;
  uint32_t* sv = sk + nq * RS;
  float* sp = reinterpret_cast<float*>(sv + nq * RS);
  const int head = blockIdx.x, b = blockIdx.y;
  const long long D = (long long)H * HD;
  const T* base = qkv + (long long)b * nq * 3 * D + head * HD;
  qattn_load<HD>(sq, base, 3 * D, nq);
  qattn_load<HD>(sk, base + D, 3 * D, nq);
  qattn_load<HD>(sv, base + 2 * D, 3 * D, nq);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = warp; i < nq; i += kQattnThreads / 32) {
    float s[kQattnMaxTokens / 32], m = -INFINITY;
#pragma unroll
    for (int c = 0; c < kQattnMaxTokens / 32; ++c) {
      const int j = lane + 32 * c;
      s[c] = j < nq ? qattn_dot<T, HD>(sq + i * RS, sk + j * RS) * scale_log2 : -INFINITY;
      m = fmaxf(m, s[c]);
    }
    m = warp_max(m);
    float l = 0.f;
#pragma unroll
    for (int c = 0; c < kQattnMaxTokens / 32; ++c) {
      s[c] = lane + 32 * c < nq ? ex2_approx(s[c] - m) : 0.f;
      l += s[c];
    }
    l = warp_sum(l);
#pragma unroll
    for (int c = 0; c < kQattnMaxTokens / 32; ++c)
      if (lane + 32 * c < nq) sp[i * (nq + 1) + lane + 32 * c] = __fdiv_rn(s[c], l);
    if (lse2 != nullptr && lane == 0) lse2[((long long)b * nq + i) * H + head] = m + log2f(l);
  }
  __syncthreads();
  for (int t = threadIdx.x; t < nq * W; t += kQattnThreads) {
    const int r = t / W, w = t % W;
    float a0 = 0.f, a1 = 0.f;
    for (int j = 0; j < nq; ++j) {
      const float p = sp[r * (nq + 1) + j];
      const uint32_t v = sv[j * RS + w];
      a0 = fmaf(p, E::lo(v), a0);
      a1 = fmaf(p, E::hi(v), a1);
    }
    reinterpret_cast<uint32_t*>(out + ((long long)b * nq + r) * D + head * HD)[w] = E::pack(a0, a1);
  }
}

// grid (H, B).  p is recomputed from lse2; delta_i = dO_i . O_i; ds_ij = p_ij (dO_i . v_j - delta_i);
// dv_j = sum_i p_ij dO_i, dq_i = scale sum_j ds_ij k_j, dk_j = scale sum_i ds_ij q_i.
template <typename T, int HD>
__global__ void __launch_bounds__(kQattnThreads) qattn_bwd_kernel(const T* __restrict__ qkv, const T* __restrict__ out,
                                                                  const T* __restrict__ dout,
                                                                  const float* __restrict__ lse2, T* __restrict__ dqkv,
                                                                  int nq, int H, float scale_log2, float scale) {
  using E = Elt<T>;
  constexpr int W = HD / 2, RS = qattn_row_words<HD>();
  extern __shared__ __align__(16) uint32_t qattn_sm[];
  uint32_t* sq = qattn_sm;
  uint32_t* sk = sq + nq * RS;
  uint32_t* sv = sk + nq * RS;
  uint32_t* sdo = sv + nq * RS;
  float* sp = reinterpret_cast<float*>(sdo + nq * RS);
  float* sdelta = sp + nq * (nq + 1);
  const int head = blockIdx.x, b = blockIdx.y;
  const long long D = (long long)H * HD;
  const T* base = qkv + (long long)b * nq * 3 * D + head * HD;
  const long long obase = (long long)b * nq * D + head * HD;
  qattn_load<HD>(sq, base, 3 * D, nq);
  qattn_load<HD>(sk, base + D, 3 * D, nq);
  qattn_load<HD>(sv, base + 2 * D, 3 * D, nq);
  qattn_load<HD>(sdo, dout + obase, D, nq);
  __syncthreads();
  if (threadIdx.x < nq) {
    const int r = threadIdx.x;
    sdelta[r] = qattn_dot<T, HD>(sdo + r * RS, reinterpret_cast<const uint32_t*>(out + obase + r * D));
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = warp; i < nq; i += kQattnThreads / 32) {
    const float lse = lse2[((long long)b * nq + i) * H + head];
#pragma unroll
    for (int c = 0; c < kQattnMaxTokens / 32; ++c) {
      const int j = lane + 32 * c;
      if (j < nq) sp[i * (nq + 1) + j] = ex2_approx(qattn_dot<T, HD>(sq + i * RS, sk + j * RS) * scale_log2 - lse);
    }
  }
  __syncthreads();
  T* drow = dqkv + (long long)b * nq * 3 * D + head * HD;
  for (int t = threadIdx.x; t < nq * W; t += kQattnThreads) {          // dv
    const int r = t / W, w = t % W;
    float a0 = 0.f, a1 = 0.f;
    for (int i = 0; i < nq; ++i) {
      const float p = sp[i * (nq + 1) + r];
      const uint32_t d = sdo[i * RS + w];
      a0 = fmaf(p, E::lo(d), a0);
      a1 = fmaf(p, E::hi(d), a1);
    }
    reinterpret_cast<uint32_t*>(drow + r * 3 * D + 2 * D)[w] = E::pack(a0, a1);
  }
  __syncthreads();
  for (int i = warp; i < nq; i += kQattnThreads / 32) {                  // p -> ds in place
#pragma unroll
    for (int c = 0; c < kQattnMaxTokens / 32; ++c) {
      const int j = lane + 32 * c;
      if (j < nq) {
        const float dp = qattn_dot<T, HD>(sdo + i * RS, sv + j * RS);
        sp[i * (nq + 1) + j] *= dp - sdelta[i];
      }
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < nq * W; t += kQattnThreads) {          // dq (row r = query) and dk (row r = key)
    const int r = t / W, w = t % W;
    float q0 = 0.f, q1 = 0.f, k0 = 0.f, k1 = 0.f;
    for (int j = 0; j < nq; ++j) {
      const float dsq = sp[r * (nq + 1) + j], dsk = sp[j * (nq + 1) + r];
      const uint32_t kw = sk[j * RS + w], qw = sq[j * RS + w];
      q0 = fmaf(dsq, E::lo(kw), q0);
      q1 = fmaf(dsq, E::hi(kw), q1);
      k0 = fmaf(dsk, E::lo(qw), k0);
      k1 = fmaf(dsk, E::hi(qw), k1);
    }
    reinterpret_cast<uint32_t*>(drow + r * 3 * D)[w] = E::pack(q0 * scale, q1 * scale);
    reinterpret_cast<uint32_t*>(drow + r * 3 * D + D)[w] = E::pack(k0 * scale, k1 * scale);
  }
}

}  // namespace vj

using namespace vj;

template <typename T, int HD>
static int query_attn_launch(bool bwd, const void* qkv, const void* out, const void* dout, const float* lse2_in,
                             float* lse2_out, void* dst, int B, int nq, int H, float scale, cudaStream_t s) {
  const float sl2 = scale * 1.4426950408889634f;
  const size_t smem = qattn_smem<HD>(nq, bwd ? 4 : 3, bwd);
  static bool configured = false;  // per instantiation: the largest nq either kernel takes
  if (!configured) {
    VJ_CUDA(cudaFuncSetAttribute(qattn_fwd_kernel<T, HD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)qattn_smem<HD>(kQattnMaxTokens, 3, false)));
    VJ_CUDA(cudaFuncSetAttribute(qattn_bwd_kernel<T, HD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)qattn_smem<HD>(kQattnMaxTokens, 4, true)));
    configured = true;
  }
  dim3 grid(H, B);
  if (bwd)
    qattn_bwd_kernel<T, HD><<<grid, kQattnThreads, smem, s>>>(
        reinterpret_cast<const T*>(qkv), reinterpret_cast<const T*>(out), reinterpret_cast<const T*>(dout), lse2_in,
        reinterpret_cast<T*>(dst), nq, H, sl2, scale);
  else
    qattn_fwd_kernel<T, HD><<<grid, kQattnThreads, smem, s>>>(reinterpret_cast<const T*>(qkv), reinterpret_cast<T*>(dst),
                                                              lse2_out, nq, H, sl2);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

template <typename T>
static int query_attn(const char* name, bool bwd, const void* qkv, const void* out, const void* dout, const float* lse2_in,
                      float* lse2_out, void* dst, int B, int nq, int H, int HD, float scale, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(qkv && dst && (!bwd || (out && dout && lse2_in)), "%s: null pointer", name);
  VJ_CHECK_ARG(B > 0 && nq > 0 && H > 0, "%s: empty problem", name);
  VJ_CHECK_ARG(nq <= kQattnMaxTokens, "%s: nq = %d query tokens per clip; at most %d are supported", name, nq,
               kQattnMaxTokens);
  VJ_CHECK_ARG(B <= 65535, "%s: B = %d clips is too many", name, B);
  VJ_CHECK_ARG(((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(out) |
                 reinterpret_cast<uintptr_t>(dout)) & 3) == 0,
               "%s: pointers must be 4-byte aligned", name);
#define VJ_QATTN(HDV) \
  return query_attn_launch<T, HDV>(bwd, qkv, out, dout, lse2_in, lse2_out, dst, B, nq, H, scale, s)
  switch (HD) {
    case 32: VJ_QATTN(32);
    case 64: VJ_QATTN(64);
    case 80: VJ_QATTN(80);
    case 88: VJ_QATTN(88);
    case 104: VJ_QATTN(104);
    case 128: VJ_QATTN(128);
    default: set_error("%s: head dim %d unsupported (32 / 64 / 80 / 88 / 104 / 128)", name, HD); return -1;
  }
#undef VJ_QATTN
}

extern "C" int vj_query_attn_fwd(const void* qkv, void* out, float* lse2, int B, int nq, int H, int HD, float scale,
                                 void* stream) {
  return query_attn<__nv_bfloat16>("vj_query_attn_fwd", false, qkv, nullptr, nullptr, nullptr, lse2, out, B, nq, H, HD,
                                   scale, stream);
}

extern "C" int vj_query_attn_fwd_f16(const void* qkv, void* out, float* lse2, int B, int nq, int H, int HD, float scale,
                                     void* stream) {
  return query_attn<__half>("vj_query_attn_fwd_f16", false, qkv, nullptr, nullptr, nullptr, lse2, out, B, nq, H, HD,
                            scale, stream);
}

extern "C" int vj_query_attn_bwd(const void* qkv, const void* out, const void* dout, const float* lse2, void* dqkv, int B,
                                 int nq, int H, int HD, float scale, void* stream) {
  return query_attn<__nv_bfloat16>("vj_query_attn_bwd", true, qkv, out, dout, lse2, nullptr, dqkv, B, nq, H, HD, scale,
                                   stream);
}

extern "C" int vj_query_attn_bwd_f16(const void* qkv, const void* out, const void* dout, const float* lse2, void* dqkv,
                                     int B, int nq, int H, int HD, float scale, void* stream) {
  return query_attn<__half>("vj_query_attn_bwd_f16", true, qkv, out, dout, lse2, nullptr, dqkv, B, nq, H, HD, scale,
                            stream);
}
