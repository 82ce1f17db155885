// Cross-attention of a few learned query tokens over a long key / value sequence: the attentive probe of the frozen-
// encoder evaluations (src/models/utils/modules.py:122-153 CrossAttention.forward, used by AttentivePooler,
// src/models/attentive_pooler.py:96-102).  SURVEY section 8 row f4 (inference side).
//
//   q   bf16 [B*nq, H*hd]          (the q Linear's output; row b*nq + j = query j of clip b)
//   kv  bf16 [B*S, 2*H*hd]         (the kv Linear's output: k | v halves, head-major inside a half)
//   out bf16 [B*nq, H*hd] = softmax(q k^T * scale) v      per (clip, head, query)
// The _f16 entry points run the same kernels on fp16 q / kv / out / dout / dkv (the probe under the evals'
// autocast(float16)); lse2, dq and the dq partials stay fp32 either way.
//
// nq is 1 for the probe, S is 1568 .. 9216 encoder tokens: the work is a GEMV-shaped streaming pass over K and V
// (2 * S * hd * 2 bytes per (clip, head)), i.e. HBM / L2 bound, so there is nothing for the tensor cores to do: one CTA per
// (head, clip*query), eight warps split the keys, a group of hd/8 lanes owns one key at a time (16-byte loads), online
// softmax per group, groups and warps are merged through shared memory at the end.
//
// Training the probe needs the backward of the same attention.  The forward can also leave the softmax statistics
// lse2 fp32 [B*nq, H] (log2 domain, like vj_attn_fwd); the backward recomputes p from them:
//   p_ij = exp2(scale*log2e * q_i.k_j - lse2_i),  delta_i = dO_i.O_i,  ds_ij = p_ij (dO_i.v_j - delta_i)
//   dk_j = scale sum_i ds_ij q_i,  dv_j = sum_i p_ij dO_i,  dq_i = scale sum_j ds_ij k_j
// It is the same streaming pass (read kv, write dkv), so it keeps the forward's layout: one lane group per key, 16-byte
// loads and stores.  The key range is cut into chunks of kXattnBwdKeys keys per lane group so that an evaluation batch
// (B = 4 clips x 16 heads) still fills the GPU; every dkv element is written exactly once, and dq is summed over the
// per-chunk partials in chunk order by a second kernel: no atomics, the result is deterministic.
#include "common.cuh"
#include "vjepa_b200.h"

#include <type_traits>

namespace vj {

constexpr int kXattnThreads = 256;

// one 16-bit element of T from fp32, rounded to nearest (fp16: a value past 65504 becomes +-inf, never saturates)
template <typename T>
VJ_DEVINL T to_elt(float v) {
  if constexpr (std::is_same<T, __half>::value) return __float2half_rn(v);
  else return __float2bfloat16(v);
}

template <typename T, int LPK>   // T: bf16 or fp16 element type of q / kv / out; lanes per key = hd / 8
__global__ void __launch_bounds__(kXattnThreads) xattn_fwd_kernel(const T* __restrict__ q, const T* __restrict__ kv,
                                                                  T* __restrict__ out, float* __restrict__ lse2, int nq,
                                                                  int S, int H, float scale_log2) {
  using E = Elt<T>;
  constexpr int HD = LPK * 8;
  constexpr int KPW = 32 / LPK;                 // keys handled per warp iteration
  constexpr int NGROUPS = (kXattnThreads / 32) * KPW;
  const int head = blockIdx.x, bq = blockIdx.y;
  const int b = bq / nq;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int grp = lane / LPK, gl = lane % LPK;   // key slot inside the warp, 8-element slice of the head dim
  const bool active = grp < KPW;
  const long long D = (long long)H * HD;

  float qf[8];
  {
    const uint4 u = *reinterpret_cast<const uint4*>(q + (long long)bq * D + head * HD + (active ? gl : 0) * 8);
    qf[0] = E::lo(u.x); qf[1] = E::hi(u.x); qf[2] = E::lo(u.y); qf[3] = E::hi(u.y);
    qf[4] = E::lo(u.z); qf[5] = E::hi(u.z); qf[6] = E::lo(u.w); qf[7] = E::hi(u.w);
  }
  float m = -INFINITY, l = 0.f, o[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] = 0.f;
  const T* kbase = kv + (long long)b * S * 2 * D + head * HD + gl * 8;
  for (int j0 = warp * KPW; j0 < S; j0 += (kXattnThreads / 32) * KPW) {
    const int j = j0 + grp;
    const bool ok = active && j < S;
    float part = 0.f;
    uint4 vv = make_uint4(0, 0, 0, 0);
    if (ok) {
      const uint4 ku = *reinterpret_cast<const uint4*>(kbase + (long long)j * 2 * D);
      vv = *reinterpret_cast<const uint4*>(kbase + (long long)j * 2 * D + D);
      part = qf[0] * E::lo(ku.x) + qf[1] * E::hi(ku.x) + qf[2] * E::lo(ku.y) + qf[3] * E::hi(ku.y) +
             qf[4] * E::lo(ku.z) + qf[5] * E::hi(ku.z) + qf[6] * E::lo(ku.w) + qf[7] * E::hi(ku.w);
    }
    // score of key j = sum of the LPK partial dot products of its lane group (rotation inside the group)
    float s = part;
#pragma unroll
    for (int i = 1; i < LPK; ++i) s += __shfl_sync(0xffffffffu, part, grp * LPK + (gl + i) % LPK);
    if (ok) {
      s *= scale_log2;
      const float mn = fmaxf(m, s);
      const float corr = ex2_approx(m - mn);      // 0 on the first key (m = -inf)
      const float p = ex2_approx(s - mn);
      l = l * corr + p;
      o[0] = o[0] * corr + p * E::lo(vv.x); o[1] = o[1] * corr + p * E::hi(vv.x);
      o[2] = o[2] * corr + p * E::lo(vv.y); o[3] = o[3] * corr + p * E::hi(vv.y);
      o[4] = o[4] * corr + p * E::lo(vv.z); o[5] = o[5] * corr + p * E::hi(vv.z);
      o[6] = o[6] * corr + p * E::lo(vv.w); o[7] = o[7] * corr + p * E::hi(vv.w);
      m = mn;
    }
  }
  // merge the NGROUPS partial softmaxes: every group publishes (m, l, o[HD]); thread (gl) of group 0 / warp 0 combines
  __shared__ float sm_m[NGROUPS], sm_l[NGROUPS], sm_o[NGROUPS][HD];
  if (active) {
    const int g = warp * KPW + grp;
    if (gl == 0) { sm_m[g] = m; sm_l[g] = l; }
#pragma unroll
    for (int i = 0; i < 8; ++i) sm_o[g][gl * 8 + i] = o[i];
  }
  __syncthreads();
  if (threadIdx.x < HD) {
    const int d = threadIdx.x;
    float M = -INFINITY;
    for (int g = 0; g < NGROUPS; ++g) M = fmaxf(M, sm_m[g]);
    float L = 0.f, acc = 0.f;
    for (int g = 0; g < NGROUPS; ++g) {
      const float w = sm_m[g] == -INFINITY ? 0.f : ex2_approx(sm_m[g] - M);
      L += w * sm_l[g];
      acc += w * sm_o[g][d];
    }
    out[(long long)bq * D + head * HD + d] = to_elt<T>(acc / L);
    if (lse2 != nullptr && d == 0) lse2[(long long)bq * H + head] = M + log2f(L);
  }
}

// sum over the LPK lanes of a key's lane group; every lane of the group gets the same value (butterfly when LPK is a
// power of two, rotation otherwise - hd 80 has 10 lanes per key)
template <int LPK>
VJ_DEVINL float group_sum(float v) {
  if constexpr ((LPK & (LPK - 1)) == 0) {
#pragma unroll
    for (int o = 1; o < LPK; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
  } else {
    const int lane = threadIdx.x & 31, base = lane / LPK * LPK, gl = lane % LPK;
    float s = v;
#pragma unroll
    for (int i = 1; i < LPK; ++i) s += __shfl_sync(0xffffffffu, v, base + (gl + i) % LPK);
    return s;
  }
}

template <typename T>
VJ_DEVINL void unpack8(const uint4& u, float* f) {
  using E = Elt<T>;
  f[0] = E::lo(u.x); f[1] = E::hi(u.x); f[2] = E::lo(u.y); f[3] = E::hi(u.y);
  f[4] = E::lo(u.z); f[5] = E::hi(u.z); f[6] = E::lo(u.w); f[7] = E::hi(u.w);
}

template <typename T>
VJ_DEVINL float dot8(const float* a, const uint4& u) {
  using E = Elt<T>;
  return a[0] * E::lo(u.x) + a[1] * E::hi(u.x) + a[2] * E::lo(u.y) + a[3] * E::hi(u.y) +
         a[4] * E::lo(u.z) + a[5] * E::hi(u.z) + a[6] * E::lo(u.w) + a[7] * E::hi(u.w);
}

constexpr int kXattnBwdKeys = 2;   // keys per lane group per CTA, held in registers from the first load to the store

template <int LPK>
__host__ __device__ constexpr int xattn_bwd_chunk() { return (kXattnThreads / 32) * (32 / LPK) * kXattnBwdKeys; }

// grid (H, B, key chunks).  Lane group g of the CTA owns keys chunk*KPC + kk*NGROUPS + g, kk < kXattnBwdKeys, so
// consecutive groups read consecutive kv rows.  All nq queries of the clip are applied to those keys one after the other;
// the per-query dq partial of the chunk is reduced over the groups through shared memory in group order.
template <typename T, int LPK>
__global__ void __launch_bounds__(kXattnThreads, 2) xattn_bwd_kernel(
    const T* __restrict__ q, const T* __restrict__ kv, const T* __restrict__ out, const T* __restrict__ dout,
    const float* __restrict__ lse2, T* __restrict__ dkv, float* __restrict__ dq_part, int nq, int S, int H,
    float scale_log2, float scale) {
  using E = Elt<T>;
  constexpr int HD = LPK * 8;
  constexpr int KPW = 32 / LPK;
  constexpr int NGROUPS = (kXattnThreads / 32) * KPW;
  constexpr int KPC = xattn_bwd_chunk<LPK>();
  constexpr int NK = kXattnBwdKeys;
  const int head = blockIdx.x, b = blockIdx.y, chunk = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int grp = lane / LPK, gl = lane % LPK;
  const bool active = grp < KPW;
  const int g = warp * KPW + grp;
  const long long D = (long long)H * HD;
  const long long kvoff = (long long)b * S * 2 * D + head * HD + (active ? gl : 0) * 8;

  uint4 ku[NK], vu[NK];
  bool ok[NK];
#pragma unroll
  for (int kk = 0; kk < NK; ++kk) {
    const int j = chunk * KPC + kk * NGROUPS + g;
    ok[kk] = active && j < S;
    ku[kk] = vu[kk] = make_uint4(0, 0, 0, 0);
    if (ok[kk]) {
      ku[kk] = *reinterpret_cast<const uint4*>(kv + kvoff + (long long)j * 2 * D);
      vu[kk] = *reinterpret_cast<const uint4*>(kv + kvoff + (long long)j * 2 * D + D);
    }
  }
  float dk[NK][8], dv[NK][8];
#pragma unroll
  for (int kk = 0; kk < NK; ++kk)
#pragma unroll
    for (int e = 0; e < 8; ++e) dk[kk][e] = dv[kk][e] = 0.f;

  __shared__ float sm_dq[NGROUPS][HD];
  for (int i = 0; i < nq; ++i) {
    const long long row = (long long)b * nq + i;
    const long long c = row * D + head * HD + (active ? gl : 0) * 8;
    float qf[8], df[8], of[8];
    unpack8<T>(*reinterpret_cast<const uint4*>(q + c), qf);
    unpack8<T>(*reinterpret_cast<const uint4*>(dout + c), df);
    unpack8<T>(*reinterpret_cast<const uint4*>(out + c), of);
    float dpart = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) dpart += df[e] * of[e];
    const float delta = group_sum<LPK>(dpart);
    const float lse = lse2[row * H + head];
    float dqa[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) dqa[e] = 0.f;
#pragma unroll
    for (int kk = 0; kk < NK; ++kk) {
      const float s = group_sum<LPK>(dot8<T>(qf, ku[kk]));
      const float dp = group_sum<LPK>(dot8<T>(df, vu[kk]));
      if (ok[kk]) {
        const float p = ex2_approx(s * scale_log2 - lse);
        const float ds = p * (dp - delta);
        float kf[8];
        unpack8<T>(ku[kk], kf);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          dk[kk][e] += ds * qf[e];
          dv[kk][e] += p * df[e];
          dqa[e] += ds * kf[e];
        }
      }
    }
    if (active) {
#pragma unroll
      for (int e = 0; e < 8; ++e) sm_dq[g][gl * 8 + e] = dqa[e];
    }
    __syncthreads();
    if (threadIdx.x < HD) {
      float acc = 0.f;
      for (int gg = 0; gg < NGROUPS; ++gg) acc += sm_dq[gg][threadIdx.x];
      dq_part[((long long)chunk * gridDim.y * nq + row) * D + head * HD + threadIdx.x] = acc;
    }
    __syncthreads();
  }
#pragma unroll
  for (int kk = 0; kk < NK; ++kk) {
    if (!ok[kk]) continue;
    const int j = chunk * KPC + kk * NGROUPS + g;
    uint4 a, v;
    a.x = E::pack(dk[kk][0] * scale, dk[kk][1] * scale); a.y = E::pack(dk[kk][2] * scale, dk[kk][3] * scale);
    a.z = E::pack(dk[kk][4] * scale, dk[kk][5] * scale); a.w = E::pack(dk[kk][6] * scale, dk[kk][7] * scale);
    v.x = E::pack(dv[kk][0], dv[kk][1]); v.y = E::pack(dv[kk][2], dv[kk][3]);
    v.z = E::pack(dv[kk][4], dv[kk][5]); v.w = E::pack(dv[kk][6], dv[kk][7]);
    *reinterpret_cast<uint4*>(dkv + kvoff + (long long)j * 2 * D) = a;
    *reinterpret_cast<uint4*>(dkv + kvoff + (long long)j * 2 * D + D) = v;
  }
}

// dq[r] = scale * sum over chunks (in chunk order) of dq_part[chunk][r]
__global__ void xattn_dq_reduce_kernel(const float* __restrict__ dq_part, float* __restrict__ dq, long long n, int nchunk,
                                       float scale) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int c = 0; c < nchunk; ++c) acc += dq_part[c * n + i];
    dq[i] = acc * scale;
  }
}

static int xattn_bwd_chunks(int S, int HD) {
  int kpc = 0;
  switch (HD) {
    case 32: kpc = xattn_bwd_chunk<4>(); break;
    case 64: kpc = xattn_bwd_chunk<8>(); break;
    case 80: kpc = xattn_bwd_chunk<10>(); break;
    case 128: kpc = xattn_bwd_chunk<16>(); break;
    default: return -1;
  }
  return (S + kpc - 1) / kpc;
}

}  // namespace vj

using namespace vj;

template <typename T>
static int cross_attn_fwd(const char* name, const void* q, const void* kv, void* out, float* lse2, int B, int nq, int S,
                          int H, int HD, float scale, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(q && kv && out, "%s: null pointer", name);
  VJ_CHECK_ARG(B > 0 && nq > 0 && S > 0 && H > 0, "%s: empty problem", name);
  VJ_CHECK_ARG((reinterpret_cast<uintptr_t>(q) & 15) == 0 && (reinterpret_cast<uintptr_t>(kv) & 15) == 0,
               "%s: pointers must be 16-byte aligned", name);
  dim3 grid(H, B * nq);
  const float sl2 = scale * 1.4426950408889634f;
#define VJ_XATTN(LPK)                                                                                                    \
  xattn_fwd_kernel<T, LPK><<<grid, kXattnThreads, 0, s>>>(reinterpret_cast<const T*>(q), reinterpret_cast<const T*>(kv), \
                                                          reinterpret_cast<T*>(out), lse2, nq, S, H, sl2)
  switch (HD) {
    case 32: VJ_XATTN(4); break;
    case 64: VJ_XATTN(8); break;
    case 80: VJ_XATTN(10); break;
    case 128: VJ_XATTN(16); break;
    default: set_error("%s: head dim %d unsupported (32 / 64 / 80 / 128)", name, HD); return -1;
  }
#undef VJ_XATTN
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_cross_attn_fwd(const void* q, const void* kv, void* out, int B, int nq, int S, int H, int HD, float scale,
                                 void* stream) {
  return cross_attn_fwd<__nv_bfloat16>("vj_cross_attn_fwd", q, kv, out, nullptr, B, nq, S, H, HD, scale, stream);
}

extern "C" int vj_cross_attn_fwd_lse(const void* q, const void* kv, void* out, float* lse2, int B, int nq, int S, int H,
                                     int HD, float scale, void* stream) {
  VJ_CHECK_ARG(lse2, "vj_cross_attn_fwd_lse: null lse2");
  return cross_attn_fwd<__nv_bfloat16>("vj_cross_attn_fwd_lse", q, kv, out, lse2, B, nq, S, H, HD, scale, stream);
}

extern "C" int vj_cross_attn_fwd_f16(const void* q, const void* kv, void* out, int B, int nq, int S, int H, int HD,
                                     float scale, void* stream) {
  return cross_attn_fwd<__half>("vj_cross_attn_fwd_f16", q, kv, out, nullptr, B, nq, S, H, HD, scale, stream);
}

extern "C" int vj_cross_attn_fwd_lse_f16(const void* q, const void* kv, void* out, float* lse2, int B, int nq, int S,
                                         int H, int HD, float scale, void* stream) {
  VJ_CHECK_ARG(lse2, "vj_cross_attn_fwd_lse_f16: null lse2");
  return cross_attn_fwd<__half>("vj_cross_attn_fwd_lse_f16", q, kv, out, lse2, B, nq, S, H, HD, scale, stream);
}

extern "C" size_t vj_cross_attn_bwd_workspace(int B, int nq, int S, int H, int HD) {
  const int nchunk = xattn_bwd_chunks(S, HD);
  if (nchunk <= 0 || B <= 0 || nq <= 0 || H <= 0) return 0;
  return (size_t)nchunk * B * nq * H * HD * sizeof(float);
}

template <typename T>
static int cross_attn_bwd(const char* name, const void* q, const void* kv, const void* out, const void* dout,
                          const float* lse2, float* dq, void* dkv, void* workspace, size_t ws_bytes, int B, int nq, int S,
                          int H, int HD, float scale, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(q && kv && out && dout && lse2 && dq && dkv && workspace, "%s: null pointer", name);
  VJ_CHECK_ARG(B > 0 && nq > 0 && S > 0 && H > 0, "%s: empty problem", name);
  const int nchunk = xattn_bwd_chunks(S, HD);
  VJ_CHECK_ARG(nchunk > 0, "%s: head dim %d unsupported (32 / 64 / 80 / 128)", name, HD);
  VJ_CHECK_ARG(nchunk <= 65535, "%s: S = %d keys is too long", name, S);
  VJ_CHECK_ARG(ws_bytes >= vj_cross_attn_bwd_workspace(B, nq, S, H, HD), "%s: workspace too small", name);
  VJ_CHECK_ARG(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(kv) | reinterpret_cast<uintptr_t>(out) |
                 reinterpret_cast<uintptr_t>(dout) | reinterpret_cast<uintptr_t>(dkv)) & 15) == 0,
               "%s: pointers must be 16-byte aligned", name);
  dim3 grid(H, B, nchunk);
  const float sl2 = scale * 1.4426950408889634f;
  float* part = reinterpret_cast<float*>(workspace);
#define VJ_XATTN_BWD(LPK)                                                                                              \
  xattn_bwd_kernel<T, LPK><<<grid, kXattnThreads, 0, s>>>(                                                             \
      reinterpret_cast<const T*>(q), reinterpret_cast<const T*>(kv), reinterpret_cast<const T*>(out),                  \
      reinterpret_cast<const T*>(dout), lse2, reinterpret_cast<T*>(dkv), part, nq, S, H, sl2, scale)
  switch (HD) {
    case 32: VJ_XATTN_BWD(4); break;
    case 64: VJ_XATTN_BWD(8); break;
    case 80: VJ_XATTN_BWD(10); break;
    case 128: VJ_XATTN_BWD(16); break;
  }
#undef VJ_XATTN_BWD
  VJ_CUDA(cudaGetLastError());
  const long long n = (long long)B * nq * H * HD;
  const int blocks = (int)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024);
  xattn_dq_reduce_kernel<<<blocks, 256, 0, s>>>(part, dq, n, nchunk, scale);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(2);
  return 0;
}

extern "C" int vj_cross_attn_bwd(const void* q, const void* kv, const void* out, const void* dout, const float* lse2,
                                 float* dq, void* dkv, void* workspace, size_t ws_bytes, int B, int nq, int S, int H, int HD,
                                 float scale, void* stream) {
  return cross_attn_bwd<__nv_bfloat16>("vj_cross_attn_bwd", q, kv, out, dout, lse2, dq, dkv, workspace, ws_bytes, B, nq,
                                       S, H, HD, scale, stream);
}

extern "C" int vj_cross_attn_bwd_f16(const void* q, const void* kv, const void* out, const void* dout, const float* lse2,
                                     float* dq, void* dkv, void* workspace, size_t ws_bytes, int B, int nq, int S, int H,
                                     int HD, float scale, void* stream) {
  return cross_attn_bwd<__half>("vj_cross_attn_bwd_f16", q, kv, out, dout, lse2, dq, dkv, workspace, ws_bytes, B, nq, S,
                                H, HD, scale, stream);
}
