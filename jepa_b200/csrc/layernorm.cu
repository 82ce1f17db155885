// LayerNorm forward / backward (nn.LayerNorm(eps=1e-6) at src/models/utils/modules.py:115,119,
// src/models/vision_transformer.py:192-193, src/models/predictor.py:233).  HBM-bound: one warp per row,
// 16-byte vector accesses, the row lives in registers between the two passes.  Kernels are templated on
// NV = ceil(D / 256) (8-element chunks per lane) so no dead registers are carried and >= 4 CTAs of 8
// warps stay resident per SM; the grid is a multiple of the SM count.
#include "common.cuh"
#include "vjepa_b200.h"

#include <type_traits>

namespace vj {

// Storage type codes of the row kernels, the values of the ABI's x_f32 / y_f32 flags: 0 bf16, 1 fp32, 2 fp16
// (frozen evaluation under autocast(float16)).  `true` / `false` template arguments read as fp32 / bf16.
template <int DT>
using Half16 = typename std::conditional<DT == 2, __half, __nv_bfloat16>::type;

template <int DT>
VJ_DEVINL void ld8(const void* base, long long off, float (&v)[8]) {
  if (DT == 1) {
    const float4* p = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + off);
    const float4 a = p[0], b = p[1];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
    using E = Elt<Half16<DT>>;
    const uint4 u = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(base) + off);
    v[0] = E::lo(u.x); v[1] = E::hi(u.x); v[2] = E::lo(u.y); v[3] = E::hi(u.y);
    v[4] = E::lo(u.z); v[5] = E::hi(u.z); v[6] = E::lo(u.w); v[7] = E::hi(u.w);
  }
}
template <int DT>
VJ_DEVINL void st8(void* base, long long off, const float (&v)[8]) {
  if (DT == 1) {
    float4* p = reinterpret_cast<float4*>(reinterpret_cast<float*>(base) + off);
    p[0] = make_float4(v[0], v[1], v[2], v[3]);
    p[1] = make_float4(v[4], v[5], v[6], v[7]);
  } else {
    using E = Elt<Half16<DT>>;
    uint4 u;
    u.x = E::pack(v[0], v[1]); u.y = E::pack(v[2], v[3]);
    u.z = E::pack(v[4], v[5]); u.w = E::pack(v[6], v[7]);
    *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(base) + off) = u;
  }
}

template <int NV, int IN_F32, int OUT_F32>
__global__ void __launch_bounds__(256, NV <= 2 ? 4 : (NV <= 4 ? 3 : 1))
ln_fwd_kernel(const void* __restrict__ x, void* __restrict__ y, const float* __restrict__ gamma,
              const float* __restrict__ beta, float* __restrict__ mean_out, float* __restrict__ rstd_out, int T, int D,
              float eps) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const int nvec = D >> 3;
  const float invD = 1.0f / D;
  for (long long row = (long long)blockIdx.x * wpb + (threadIdx.x >> 5); row < T; row += (long long)gridDim.x * wpb) {
    float v[NV][8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) {
        ld8<IN_F32>(x, row * D + c * 8, v[i]);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += v[i][j];
      }
    }
    const float mean = warp_sum(s) * invD;
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[i][j] - mean;
          ss += d * d;
        }
      }
    }
    const float rstd = rsqrtf(warp_sum(ss) * invD + eps);
    if (lane == 0) {
      if (mean_out) mean_out[row] = mean;
      if (rstd_out) rstd_out[row] = rstd;
    }
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) {
        float o[8], g[8], b[8];   // gamma / beta come from L1 (same 4 KB for every row)
        ld8<true>(gamma, c * 8, g);
        ld8<true>(beta, c * 8, b);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = (v[i][j] - mean) * rstd * g[j] + b[j];
        st8<OUT_F32>(y, row * D + c * 8, o);
      }
    }
  }
}

// bf16 -> bf16 forward (the residual stream of both networks): two rows per warp iteration, rows kept packed.
template <int NV>
__global__ void __launch_bounds__(256, NV <= 2 ? 3 : (NV <= 4 ? 2 : 1))
ln_fwd2_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, const float* __restrict__ gamma,
               const float* __restrict__ beta, float* __restrict__ mean_out, float* __restrict__ rstd_out, int T, int D,
               float eps) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const int nvec = D >> 3;
  const float invD = 1.0f / D;
  auto unpack = [](const uint4& u, float (&f)[8]) {
    f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
    f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
  };
  for (long long row0 = 2 * ((long long)blockIdx.x * wpb + (threadIdx.x >> 5)); row0 < T;
       row0 += 2LL * gridDim.x * wpb) {
    uint4 xp[2][NV];
    bool ok[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      ok[r] = row0 + r < T;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = lane + 32 * i;
        xp[r][i] = (ok[r] && c < nvec) ? *reinterpret_cast<const uint4*>(x + (row0 + r) * D + c * 8) : make_uint4(0, 0, 0, 0);
      }
    }
    float mean[2], rstd[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        float f[8];
        unpack(xp[r][i], f);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += f[j];
      }
      mean[r] = warp_sum(s) * invD;
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float ss = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        if (lane + 32 * i < nvec) {
          float f[8];
          unpack(xp[r][i], f);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float d = f[j] - mean[r];
            ss = fmaf(d, d, ss);
          }
        }
      }
      rstd[r] = rsqrtf(warp_sum(ss) * invD + eps);
      if (lane == 0 && ok[r]) {
        if (mean_out) mean_out[row0 + r] = mean[r];
        if (rstd_out) rstd_out[row0 + r] = rstd[r];
      }
    }
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) {
        float g[8], b[8];   // gamma / beta come from L1 (same few KB for every row)
        ld8<true>(gamma, c * 8, g);
        ld8<true>(beta, c * 8, b);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float f[8], o[8];
          unpack(xp[r][i], f);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = fmaf((f[j] - mean[r]) * rstd[r], g[j], b[j]);
          if (ok[r]) st8<false>(y, (row0 + r) * D + c * 8, o);
        }
      }
    }
  }
}

// dx = dres + rstd * (g*dy - mean(g*dy) - xhat * mean(g*dy*xhat)).  The row (x, dy) stays in registers in
// its storage format between the two passes; dgamma/dbeta partial sums live in per-warp shared-memory
// slices (no atomics, no persistent registers), reduced per block into [gridDim.x, D] partials.
// DY: the 16-bit type of dy - bf16, or fp16 with an fp32 x (the attentive probe's LayerNorms under the evals'
// autocast(float16): fp32 inputs, fp16 gradients from the following fp16 Linear's dgrad).
template <int NV, bool X_F32, typename DY = __nv_bfloat16>
// (register caps chosen so nothing spills: with ~220 KB of the SM given to shared memory L1 is tiny and every
// local-memory access is an L2 round trip)
__global__ void __launch_bounds__(256, NV <= 2 ? 2 : 1)
ln_bwd_kernel(const DY* __restrict__ dy, const void* __restrict__ x, const float* __restrict__ gamma,
              const float* __restrict__ mean, const float* __restrict__ rstd, const void* __restrict__ dres,
              void* __restrict__ dx, float* __restrict__ part_dgamma, float* __restrict__ part_dbeta, int T, int D) {
  static_assert(std::is_same<DY, __nv_bfloat16>::value || X_F32, "an fp16 dy pairs with an fp32 x only");
  using E = Elt<DY>;
  extern __shared__ float sm[];  // [warps][2][D]
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int wpb = blockDim.x >> 5;
  const int nvec = D >> 3;
  const float invD = 1.0f / D;
  float* my_dg = sm + (size_t)wib * 2 * D;
  float* my_db = my_dg + D;
  // a lane owns the same 8*NV columns for every row it visits: dgamma / dbeta partials live in registers and reach
  // shared memory once, at the end
  float ag[NV][8], ab[NV][8];
#pragma unroll
  for (int i = 0; i < NV; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) ag[i][j] = ab[i][j] = 0.f;
  for (long long row = (long long)blockIdx.x * wpb + wib; row < T; row += (long long)gridDim.x * wpb) {
    const float mu = mean[row], rs = rstd[row];
    float xv[NV][X_F32 ? 8 : 1];
    uint4 xp[NV], dyp[NV];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) {
        float xf[8], dyf[8], g[8];
        if (X_F32) {
          ld8<true>(x, row * D + c * 8, xf);
#pragma unroll
          for (int j = 0; j < (X_F32 ? 8 : 1); ++j) xv[i][j] = xf[j];
        } else {
          xp[i] = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(x) + row * D + c * 8);
          xf[0] = bf16_lo(xp[i].x); xf[1] = bf16_hi(xp[i].x); xf[2] = bf16_lo(xp[i].y); xf[3] = bf16_hi(xp[i].y);
          xf[4] = bf16_lo(xp[i].z); xf[5] = bf16_hi(xp[i].z); xf[6] = bf16_lo(xp[i].w); xf[7] = bf16_hi(xp[i].w);
        }
        dyp[i] = *reinterpret_cast<const uint4*>(dy + row * D + c * 8);
        dyf[0] = E::lo(dyp[i].x); dyf[1] = E::hi(dyp[i].x); dyf[2] = E::lo(dyp[i].y); dyf[3] = E::hi(dyp[i].y);
        dyf[4] = E::lo(dyp[i].z); dyf[5] = E::hi(dyp[i].z); dyf[6] = E::lo(dyp[i].w); dyf[7] = E::hi(dyp[i].w);
        ld8<true>(gamma, c * 8, g);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float gy = g[j] * dyf[j];
          s1 += gy;
          s2 += gy * ((xf[j] - mu) * rs);
        }
      }
    }
    s1 = warp_sum(s1) * invD;
    s2 = warp_sum(s2) * invD;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) {
        float xf[8], dyf[8], g[8], o[8];
        if (X_F32) {
#pragma unroll
          for (int j = 0; j < (X_F32 ? 8 : 1); ++j) xf[j] = xv[i][j];
        } else {
          xf[0] = bf16_lo(xp[i].x); xf[1] = bf16_hi(xp[i].x); xf[2] = bf16_lo(xp[i].y); xf[3] = bf16_hi(xp[i].y);
          xf[4] = bf16_lo(xp[i].z); xf[5] = bf16_hi(xp[i].z); xf[6] = bf16_lo(xp[i].w); xf[7] = bf16_hi(xp[i].w);
        }
        dyf[0] = E::lo(dyp[i].x); dyf[1] = E::hi(dyp[i].x); dyf[2] = E::lo(dyp[i].y); dyf[3] = E::hi(dyp[i].y);
        dyf[4] = E::lo(dyp[i].z); dyf[5] = E::hi(dyp[i].z); dyf[6] = E::lo(dyp[i].w); dyf[7] = E::hi(dyp[i].w);
        ld8<true>(gamma, c * 8, g);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float xh = (xf[j] - mu) * rs;
          o[j] = rs * (g[j] * dyf[j] - s1 - xh * s2);
          ag[i][j] = fmaf(dyf[j], xh, ag[i][j]);
          ab[i][j] += dyf[j];
        }
        if (dres) {
          float r[8];
          ld8<X_F32>(dres, row * D + c * 8, r);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += r[j];
        }
        st8<X_F32>(dx, row * D + c * 8, o);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = lane + 32 * i;
    if (c < nvec) {
      float4* pg = reinterpret_cast<float4*>(my_dg + c * 8);
      float4* pb = reinterpret_cast<float4*>(my_db + c * 8);
      pg[0] = make_float4(ag[i][0], ag[i][1], ag[i][2], ag[i][3]);
      pg[1] = make_float4(ag[i][4], ag[i][5], ag[i][6], ag[i][7]);
      pb[0] = make_float4(ab[i][0], ab[i][1], ab[i][2], ab[i][3]);
      pb[1] = make_float4(ab[i][4], ab[i][5], ab[i][6], ab[i][7]);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    float a = 0.f, b = 0.f;
    for (int w = 0; w < wpb; ++w) {
      a += sm[(size_t)w * 2 * D + i];
      b += sm[(size_t)w * 2 * D + D + i];
    }
    part_dgamma[(long long)blockIdx.x * D + i] = a;
    part_dbeta[(long long)blockIdx.x * D + i] = b;
  }
}

// out_a[c] += sum_r a[r,c]; out_b[c] += sum_r b[r,c].  grid = (C/32, row chunks): 32 columns x 8 row groups per
// block, coalesced 128-byte row segments, one atomicAdd per (column, row chunk).
__global__ void __launch_bounds__(256) partial_reduce_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                             float* __restrict__ out_a, float* __restrict__ out_b,
                                                             int R, int C, int rows_per_block) {
  __shared__ float sm[2][8][33];
  const int col = blockIdx.x * 32 + (threadIdx.x & 31);
  const int rg = threadIdx.x >> 5;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(R, r0 + rows_per_block);
  float sa = 0.f, sb = 0.f;
  if (col < C) {
    for (int r = r0 + rg; r < r1; r += 8) {
      sa += a[(long long)r * C + col];
      sb += b[(long long)r * C + col];
    }
  }
  sm[0][rg][threadIdx.x & 31] = sa;
  sm[1][rg][threadIdx.x & 31] = sb;
  __syncthreads();
  if (threadIdx.x < 64) {
    const int which = threadIdx.x >> 5, cc = threadIdx.x & 31;
    const int c = blockIdx.x * 32 + cc;
    if (c < C) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) s += sm[which][i][cc];
      atomicAdd(&(which ? out_b : out_a)[c], s);
    }
  }
}

// bf16 residual-stream variant (what the training step uses): a warp walks TWO rows per iteration so that twice the
// bytes are in flight per SM (the kernel is latency-bound otherwise: one row's loads, then two dependent warp
// reductions, then the stores), dgamma / dbeta partials stay in registers (a lane owns the same 8*NV columns for
// every row) and reach shared memory once at the end.
template <int NV>
__global__ void __launch_bounds__(256, NV <= 2 ? 2 : 1)
ln_bwd2_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma,
               const float* __restrict__ mean, const float* __restrict__ rstd, const __nv_bfloat16* __restrict__ dres,
               __nv_bfloat16* __restrict__ dx, float* __restrict__ part_dgamma, float* __restrict__ part_dbeta, int T,
               int D) {
  extern __shared__ float sm[];  // [warps][2][D]
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int wpb = blockDim.x >> 5;
  const int nvec = D >> 3;
  const float invD = 1.0f / D;
  float ag[NV][8], ab[NV][8];
#pragma unroll
  for (int i = 0; i < NV; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) ag[i][j] = ab[i][j] = 0.f;
  auto unpack = [](const uint4& u, float (&f)[8]) {
    f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
    f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
  };
  for (long long row0 = 2 * ((long long)blockIdx.x * wpb + wib); row0 < T; row0 += 2LL * gridDim.x * wpb) {
    uint4 xp[2][NV], dyp[2][NV], rp[2][NV];
    float mu[2], rs[2];
    bool ok[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const long long row = row0 + r;
      ok[r] = row < T;
      mu[r] = ok[r] ? mean[row] : 0.f;
      rs[r] = ok[r] ? rstd[row] : 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = lane + 32 * i;
        const bool in = ok[r] && c < nvec;
        xp[r][i] = in ? *reinterpret_cast<const uint4*>(x + row * D + c * 8) : make_uint4(0, 0, 0, 0);
        dyp[r][i] = in ? *reinterpret_cast<const uint4*>(dy + row * D + c * 8) : make_uint4(0, 0, 0, 0);
        rp[r][i] = (in && dres) ? *reinterpret_cast<const uint4*>(dres + row * D + c * 8) : make_uint4(0, 0, 0, 0);
      }
    }
    float s1[2] = {0.f, 0.f}, s2[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) {
        float g[8];
        ld8<true>(gamma, c * 8, g);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float xf[8], dyf[8];
          unpack(xp[r][i], xf);
          unpack(dyp[r][i], dyf);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float gy = g[j] * dyf[j];
            s1[r] += gy;
            s2[r] = fmaf(gy, (xf[j] - mu[r]) * rs[r], s2[r]);
          }
        }
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      s1[r] = warp_sum(s1[r]) * invD;
      s2[r] = warp_sum(s2[r]) * invD;
    }
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) {
        float g[8];
        ld8<true>(gamma, c * 8, g);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float xf[8], dyf[8], rf[8], o[8];
          unpack(xp[r][i], xf);
          unpack(dyp[r][i], dyf);
          unpack(rp[r][i], rf);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float xh = (xf[j] - mu[r]) * rs[r];
            o[j] = fmaf(rs[r], g[j] * dyf[j] - s1[r] - xh * s2[r], rf[j]);
            ag[i][j] = fmaf(dyf[j], xh, ag[i][j]);   // rows past T carry dy = 0
            ab[i][j] += dyf[j];
          }
          if (ok[r]) st8<false>(dx, (row0 + r) * D + c * 8, o);
        }
      }
    }
  }
  float* my_dg = sm + (size_t)wib * 2 * D;
  float* my_db = my_dg + D;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = lane + 32 * i;
    if (c < nvec) {
      float4* pg = reinterpret_cast<float4*>(my_dg + c * 8);
      float4* pb = reinterpret_cast<float4*>(my_db + c * 8);
      pg[0] = make_float4(ag[i][0], ag[i][1], ag[i][2], ag[i][3]);
      pg[1] = make_float4(ag[i][4], ag[i][5], ag[i][6], ag[i][7]);
      pb[0] = make_float4(ab[i][0], ab[i][1], ab[i][2], ab[i][3]);
      pb[1] = make_float4(ab[i][4], ab[i][5], ab[i][6], ab[i][7]);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    float a = 0.f, b = 0.f;
    for (int w = 0; w < wpb; ++w) {
      a += sm[(size_t)w * 2 * D + i];
      b += sm[(size_t)w * 2 * D + D + i];
    }
    part_dgamma[(long long)blockIdx.x * D + i] = a;
    part_dbeta[(long long)blockIdx.x * D + i] = b;
  }
}

static int ln_grid(int T) {
  long long g = (T + 7) / 8;
  const long long cap = (long long)num_sms() * 8;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return int(g);
}
// upper bound on the number of blocks any ln_bwd launch uses (sizes the partials workspace); the launchers pick
// a whole number of resident waves below it
static int ln_bwd_grid(int T) {
  long long g = (T + 7) / 8;
  const long long cap = (long long)num_sms() * 4;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return int(g);
}

template <int NV>
static void launch_ln_fwd(const void* x, int x_f32, void* y, int y_f32, const float* gamma, const float* beta, float* mean,
                          float* rstd, int T, int D, float eps, cudaStream_t s) {
  const int grid = ln_grid(T);
  if (x_f32 == 2 || y_f32 == 2) {   // fp16 (evaluation under autocast(float16)): fp16 -> fp16 / fp32, fp32 -> fp16
    if (x_f32 == 2 && y_f32 == 2) ln_fwd_kernel<NV, 2, 2><<<grid, 256, 0, s>>>(x, y, gamma, beta, mean, rstd, T, D, eps);
    else if (x_f32 == 2) ln_fwd_kernel<NV, 2, 1><<<grid, 256, 0, s>>>(x, y, gamma, beta, mean, rstd, T, D, eps);
    else ln_fwd_kernel<NV, 1, 2><<<grid, 256, 0, s>>>(x, y, gamma, beta, mean, rstd, T, D, eps);
  } else if (x_f32 && y_f32) ln_fwd_kernel<NV, true, true><<<grid, 256, 0, s>>>(x, y, gamma, beta, mean, rstd, T, D, eps);
  else if (x_f32) ln_fwd_kernel<NV, true, false><<<grid, 256, 0, s>>>(x, y, gamma, beta, mean, rstd, T, D, eps);
  else if (y_f32) ln_fwd_kernel<NV, false, true><<<grid, 256, 0, s>>>(x, y, gamma, beta, mean, rstd, T, D, eps);
  else {
    // one resident wave of two-row warps
    long long g2 = (long long)num_sms() * (NV <= 2 ? 3 : (NV <= 4 ? 2 : 1));
    if (g2 > (T + 15) / 16) g2 = (T + 15) / 16;
    ln_fwd2_kernel<NV><<<int(g2), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<__nv_bfloat16*>(y),
                                               gamma, beta, mean, rstd, T, D, eps);
  }
}

template <int NV>
static int launch_ln_bwd(const void* dy, const void* x, int x_f32, const float* gamma, const float* mean,
                          const float* rstd, const void* dres, void* dx, float* pg, float* pb, int grid, int T, int D,
                          cudaStream_t s) {
  const size_t smem = (size_t)8 * 2 * D * sizeof(float);
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(ln_bwd_kernel<NV, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 2 * 2048 * 4);
    cudaFuncSetAttribute(ln_bwd_kernel<NV, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 2 * 2048 * 4);
    configured = true;
  }
  if (x_f32) {
    ln_bwd_kernel<NV, true><<<grid, 256, smem, s>>>(reinterpret_cast<const __nv_bfloat16*>(dy), x, gamma, mean, rstd,
                                                    dres, dx, pg, pb, T, D);
  } else if constexpr (NV > 5) {   // D > 1280: the two-row kernel would spill; one row per iteration
    ln_bwd_kernel<NV, false><<<grid, 256, smem, s>>>(reinterpret_cast<const __nv_bfloat16*>(dy), x, gamma, mean, rstd,
                                                     dres, dx, pg, pb, T, D);
  } else {
    static bool configured2 = false;
    if (!configured2) {
      cudaFuncSetAttribute(ln_bwd2_kernel<NV>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 2 * 2048 * 4);
      configured2 = true;
    }
    // exactly one resident wave (the grid-stride loop balances rows; a partial second wave would double the time)
    long long g2 = (long long)num_sms() * (NV <= 2 ? 2 : 1);
    if (g2 > (T + 15) / 16) g2 = (T + 15) / 16;
    if (g2 > grid) g2 = grid;
    grid = int(g2);
    ln_bwd2_kernel<NV><<<grid, 256, smem, s>>>(reinterpret_cast<const __nv_bfloat16*>(dy),
                                               reinterpret_cast<const __nv_bfloat16*>(x), gamma, mean, rstd,
                                               reinterpret_cast<const __nv_bfloat16*>(dres),
                                               reinterpret_cast<__nv_bfloat16*>(dx), pg, pb, T, D);
  }
  return grid;
}

template <int NV>
static int launch_ln_bwd_f16(const __half* dy, const float* x, const float* gamma, const float* mean, const float* rstd,
                             const float* dres, float* dx, float* pg, float* pb, int grid, int T, int D, cudaStream_t s) {
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(ln_bwd_kernel<NV, true, __half>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 2 * 2048 * 4);
    configured = true;
  }
  ln_bwd_kernel<NV, true, __half><<<grid, 256, (size_t)8 * 2 * D * sizeof(float), s>>>(dy, x, gamma, mean, rstd, dres, dx,
                                                                                       pg, pb, T, D);
  return grid;
}

}  // namespace vj

using namespace vj;

#define VJ_LN_DISPATCH(D, CALL)                   \
  do {                                            \
    const int nv_ = ((D) + 255) / 256;            \
    if (nv_ <= 1) { CALL(1); }                    \
    else if (nv_ == 2) { CALL(2); }               \
    else if (nv_ <= 4) { CALL(4); }               \
    else if (nv_ == 5) { CALL(5); }               \
    else { CALL(8); }                             \
  } while (0)

extern "C" int vj_layernorm_fwd(const void* x, int x_f32, void* y, int y_f32, const float* gamma, const float* beta,
                                float* mean, float* rstd, int T, int D, float eps, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  if (T <= 0) return 0;
  VJ_CHECK_ARG(x && y && gamma && beta, "vj_layernorm_fwd: null pointer");
  VJ_CHECK_ARG(D % 8 == 0 && D <= 2048, "vj_layernorm_fwd: D=%d unsupported (multiple of 8, <= 2048)", D);
  VJ_CHECK_ARG(x_f32 >= 0 && x_f32 <= 2 && y_f32 >= 0 && y_f32 <= 2 && !((x_f32 == 2) != (y_f32 == 2) && x_f32 + y_f32 != 3),
               "vj_layernorm_fwd: x_f32=%d y_f32=%d (0 bf16, 1 fp32, 2 fp16; fp16 pairs with fp16 or fp32)", x_f32, y_f32);
#define VJ_CALL(NV) launch_ln_fwd<NV>(x, x_f32, y, y_f32, gamma, beta, mean, rstd, T, D, eps, s)
  VJ_LN_DISPATCH(D, VJ_CALL);
#undef VJ_CALL
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" size_t vj_layernorm_bwd_workspace(int T, int D) {
  (void)T;
  return (size_t)4 * num_sms() * 2 * D * sizeof(float);
}

extern "C" int vj_layernorm_bwd(const void* dy, const void* x, int x_f32, const float* gamma, const float* mean,
                                const float* rstd, const void* dres, void* dx, float* dgamma, float* dbeta,
                                void* workspace, size_t ws_bytes, int T, int D, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  if (T <= 0) return 0;
  VJ_CHECK_ARG(dy && x && gamma && mean && rstd && dx && dgamma && dbeta && workspace, "vj_layernorm_bwd: null pointer");
  VJ_CHECK_ARG(D % 8 == 0 && D <= 2048, "vj_layernorm_bwd: D=%d unsupported (multiple of 8, <= 2048)", D);
  int grid = ln_bwd_grid(T);
  VJ_CHECK_ARG(ws_bytes >= (size_t)grid * 2 * D * sizeof(float), "vj_layernorm_bwd: workspace too small");
  float* pg = reinterpret_cast<float*>(workspace);
  float* pb = pg + (size_t)grid * D;
#define VJ_CALL(NV) grid = launch_ln_bwd<NV>(dy, x, x_f32, gamma, mean, rstd, dres, dx, pg, pb, grid, T, D, s)
  VJ_LN_DISPATCH(D, VJ_CALL);
#undef VJ_CALL
  VJ_CUDA(cudaGetLastError());
  {
    const int rows_per_block = 64;
    dim3 rgrid((D + 31) / 32, (grid + rows_per_block - 1) / rows_per_block);
    partial_reduce_kernel<<<rgrid, 256, 0, s>>>(pg, pb, dgamma, dbeta, grid, D, rows_per_block);
  }
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(2);
  return 0;
}

extern "C" int vj_layernorm_bwd_f16(const void* dy, const float* x, const float* gamma, const float* mean,
                                    const float* rstd, const float* dres, float* dx, float* dgamma, float* dbeta,
                                    void* workspace, size_t ws_bytes, int T, int D, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  if (T <= 0) return 0;
  VJ_CHECK_ARG(dy && x && gamma && mean && rstd && dx && dgamma && dbeta && workspace,
               "vj_layernorm_bwd_f16: null pointer");
  VJ_CHECK_ARG(D % 8 == 0 && D <= 2048, "vj_layernorm_bwd_f16: D=%d unsupported (multiple of 8, <= 2048)", D);
  int grid = ln_bwd_grid(T);
  VJ_CHECK_ARG(ws_bytes >= (size_t)grid * 2 * D * sizeof(float), "vj_layernorm_bwd_f16: workspace too small");
  float* pg = reinterpret_cast<float*>(workspace);
  float* pb = pg + (size_t)grid * D;
  const __half* dyh = reinterpret_cast<const __half*>(dy);
#define VJ_CALL(NV) grid = launch_ln_bwd_f16<NV>(dyh, x, gamma, mean, rstd, dres, dx, pg, pb, grid, T, D, s)
  VJ_LN_DISPATCH(D, VJ_CALL);
#undef VJ_CALL
  VJ_CUDA(cudaGetLastError());
  {
    const int rows_per_block = 64;
    dim3 rgrid((D + 31) / 32, (grid + rows_per_block - 1) / rows_per_block);
    partial_reduce_kernel<<<rgrid, 256, 0, s>>>(pg, pb, dgamma, dbeta, grid, D, rows_per_block);
  }
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(2);
  return 0;
}
