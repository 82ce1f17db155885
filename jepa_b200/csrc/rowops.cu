// HBM-bound row-wise kernels of the V-JEPA step: LayerNorm fwd/bwd, tubelet im2col, index
// gathers (apply_masks), predictor input assembly, target LN+gather, L1 loss, column sums.
// All are one-pass, 16-byte vectorised, one warp per row (D <= 2048), grid sized in multiples
// of the SM count.  Reference call sites are cited on each entry point in include/vjepa_b200.h.
#include "common.cuh"
#include "vjepa_b200.h"

#include <type_traits>

namespace vj {

constexpr int kMaxVec = 8;  // 8 chunks of 8 elements per lane -> D <= 2048

// ---- 8-element (16 B bf16 / 2x16 B fp32) row access helpers --------------------------------
template <bool F32>
VJ_DEVINL void load8(const void* base, long long elem_off, float (&v)[8]) {
  if (F32) {
    const float4* p = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + elem_off);
    const float4 a = p[0], b = p[1];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
    const uint4 u = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(base) + elem_off);
    v[0] = bf16_lo(u.x); v[1] = bf16_hi(u.x); v[2] = bf16_lo(u.y); v[3] = bf16_hi(u.y);
    v[4] = bf16_lo(u.z); v[5] = bf16_hi(u.z); v[6] = bf16_lo(u.w); v[7] = bf16_hi(u.w);
  }
}
template <bool F32>
VJ_DEVINL void store8(void* base, long long elem_off, const float (&v)[8]) {
  if (F32) {
    float4* p = reinterpret_cast<float4*>(reinterpret_cast<float*>(base) + elem_off);
    p[0] = make_float4(v[0], v[1], v[2], v[3]);
    p[1] = make_float4(v[4], v[5], v[6], v[7]);
  } else {
    uint4 u;
    u.x = pack_bf16x2(v[0], v[1]); u.y = pack_bf16x2(v[2], v[3]);
    u.z = pack_bf16x2(v[4], v[5]); u.w = pack_bf16x2(v[6], v[7]);
    *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(base) + elem_off) = u;
  }
}

// =============================================================================================
// Column sum of a bf16 [T, N] matrix into fp32 out[N] (+=): bias gradients; with a periodic row
// filter (rows r with lo <= r % period < hi) it is also the mask-token gradient.  T16 is the 16-bit row
// type when IN_F32 is false: bf16, or fp16 (the attentive probe's bias gradients under autocast(float16)).
// =============================================================================================
template <bool IN_F32, typename T16 = __nv_bfloat16>
__global__ void __launch_bounds__(256) colsum_kernel(const void* __restrict__ in, float* __restrict__ out, long long T,
                                                     int N, long long ld, int rows_per_block, int period, int lo,
                                                     int hi) {
  __shared__ float sm[8][256];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int col = blockIdx.x * 256 + lane * 8;
  const long long r0 = (long long)blockIdx.y * rows_per_block;
  const long long r1 = min(T, r0 + rows_per_block);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (col < N) {
    for (long long r = r0 + wib; r < r1; r += 8) {
      if (period > 0) {
        const int ph = int(r % period);
        if (ph < lo || ph >= hi) continue;
      }
      float v[8];
      if constexpr (IN_F32 || std::is_same<T16, __nv_bfloat16>::value) {
        load8<IN_F32>(in, r * ld + col, v);
      } else {
        using E = Elt<T16>;
        const uint4 u = *reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(in) + r * ld + col);
        v[0] = E::lo(u.x); v[1] = E::hi(u.x); v[2] = E::lo(u.y); v[3] = E::hi(u.y);
        v[4] = E::lo(u.z); v[5] = E::hi(u.z); v[6] = E::lo(u.w); v[7] = E::hi(u.w);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) sm[wib][lane * 8 + j] = acc[j];
  __syncthreads();
  const int c = threadIdx.x;
  if (blockIdx.x * 256 + c < N) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += sm[w][c];
    atomicAdd(&out[blockIdx.x * 256 + c], s);
  }
}

// =============================================================================================
// Tubelet im2col: clips fp32 [B,3,T,H,W] -> patches bf16 [rows, ld], P = 3*tub*ps*ps, column order
// (c, dt, dh, dw) = Conv3d weight flattening; row = (b, token) with token = (t', h', w') row-major
// or the gathered token idx[b, k].  One warp per (row, c, dt) slab of ps*ps contiguous outputs; V floats per load
// (4 when ps % 4 == 0, else 2: ps 14 is 7 pairs per patch row).  PAD: rows are ld = round_up(P, 64) long and the warp
// of the last slab also zeroes the ld - P pad columns; without PAD (P % 64 == 0, every ps-16 model) ld = P.
// =============================================================================================
template <typename TO, int V, bool PAD>
__global__ void __launch_bounds__(256) im2col_kernel(const float* __restrict__ clips, TO* __restrict__ out,
                                                     const long long* __restrict__ idx, int B, int C, int T, int H,
                                                     int W, int tub, int ps, int tokens_per_clip_out, int n_tokens) {
  const int gh = H / ps, gw = W / ps;
  const int P = C * tub * ps * ps;
  const int ld = PAD ? (P + 63) / 64 * 64 : P;
  const int slabs = C * tub;  // slabs of ps*ps per row
  const long long total = (long long)B * tokens_per_clip_out * slabs;
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  for (long long wi = (long long)blockIdx.x * warps_per_block + (threadIdx.x >> 5); wi < total;
       wi += (long long)gridDim.x * warps_per_block) {
    const int slab = int(wi % slabs);
    const long long row = wi / slabs;
    const int b = int(row / tokens_per_clip_out);
    const int kk = int(row % tokens_per_clip_out);
    const long long tok = idx ? idx[(long long)b * tokens_per_clip_out + kk] : kk;
    if (tok < 0 || tok >= n_tokens) continue;
    const int c = slab / tub, dt = slab % tub;
    const int tw = int(tok % gw), th = int((tok / gw) % gh), tt = int(tok / ((long long)gw * gh));
    const float* src = clips + ((((long long)b * C + c) * T + (tt * tub + dt)) * H + (long long)th * ps) * W + tw * ps;
    TO* dst = out + row * ld + (long long)slab * ps * ps;
    // ps*ps elements: dh rows of ps contiguous floats (ps % V == 0, so a load never crosses a row)
    for (int e = lane * V; e < ps * ps; e += 32 * V) {
      const int dh = e / ps, dw = e % ps;
      if constexpr (V == 4) {
        const float4 f = *reinterpret_cast<const float4*>(src + (long long)dh * W + dw);
        uint2 o;
        o.x = Elt<TO>::pack(f.x, f.y);
        o.y = Elt<TO>::pack(f.z, f.w);
        *reinterpret_cast<uint2*>(dst + e) = o;
      } else {
        const float2 f = *reinterpret_cast<const float2*>(src + (long long)dh * W + dw);
        *reinterpret_cast<uint32_t*>(dst + e) = Elt<TO>::pack(f.x, f.y);
      }
    }
    if constexpr (PAD) {
      if (slab == slabs - 1) {
        TO* const pad = dst - (long long)slab * ps * ps + P;
        for (int e = lane * 2; e < ld - P; e += 64) *reinterpret_cast<uint32_t*>(pad + e) = 0u;
      }
    }
  }
}

// =============================================================================================
// Row gather (apply_masks): out[b,k,:] = x[b, idx[b,k], :].  Bit-exact copy, 16 B granules.
// =============================================================================================
__global__ void __launch_bounds__(256) gather_rows_kernel(const uint4* __restrict__ x, uint4* __restrict__ out,
                                                          const long long* __restrict__ idx, int B, int N, int K,
                                                          int vec_per_row) {
  const long long total = (long long)B * K * vec_per_row;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = int(i % vec_per_row);
    const long long row = i / vec_per_row;
    const int b = int(row / K);
    const long long tok = idx[row];
    out[i] = x[((long long)b * N + tok) * vec_per_row + v];
  }
}

// Scatter-add backward of the gather: dx[b, idx[b,k], :] += dy[b,k,:]  (indices unique per row).
template <bool F32>
__global__ void __launch_bounds__(256) scatter_rows_add_kernel(const void* __restrict__ dy, void* __restrict__ dx,
                                                               const long long* __restrict__ idx, int B, int N, int K,
                                                               int D) {
  const int vec = D >> 3;
  const long long total = (long long)B * K * vec;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = int(i % vec);
    const long long row = i / vec;
    const int b = int(row / K);
    const long long tok = idx[row];
    float a[8], c[8];
    load8<F32>(dy, row * D + v * 8, a);
    load8<F32>(dx, ((long long)b * N + tok) * D + v * 8, c);
#pragma unroll
    for (int j = 0; j < 8; ++j) c[j] += a[j];
    store8<F32>(dx, ((long long)b * N + tok) * D + v * 8, c);
  }
}

// =============================================================================================
// Target path: out[b,k,:] = LN_noaffine(LN_affine(x[b, idx[b,k], :]; gamma, beta, eps1); eps2) fp32
// (final encoder norm + F.layer_norm + apply_masks fused; only the gathered rows are touched).
// =============================================================================================
__global__ void __launch_bounds__(256) target_ln_gather_kernel(const __nv_bfloat16* __restrict__ x,
                                                               float* __restrict__ out,
                                                               const long long* __restrict__ idx,
                                                               const float* __restrict__ gamma,
                                                               const float* __restrict__ beta, int B, int N, int K,
                                                               int D, float eps1, float eps2) {
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int nvec = D >> 3;
  const long long rows = (long long)B * K;
  for (long long row = (long long)blockIdx.x * warps_per_block + (threadIdx.x >> 5); row < rows;
       row += (long long)gridDim.x * warps_per_block) {
    const int b = int(row / K);
    const long long src = (long long)b * N + idx[row];
    float v[kMaxVec][8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) {
        load8<false>(x, src * D + c * 8, v[i]);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += v[i][j];
      }
    }
    float mean = warp_sum(s) / D;
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[i][j] - mean;
          ss += d * d;
        }
      }
    }
    float rstd = rsqrtf(warp_sum(ss) / D + eps1);
    s = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) {
        float g[8], bb[8];
        load8<true>(gamma, c * 8, g);
        load8<true>(beta, c * 8, bb);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          v[i][j] = (v[i][j] - mean) * rstd * g[j] + bb[j];
          s += v[i][j];
        }
      }
    }
    mean = warp_sum(s) / D;
    ss = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[i][j] - mean;
          ss += d * d;
        }
      }
    }
    rstd = rsqrtf(warp_sum(ss) / D + eps2);
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = (v[i][j] - mean) * rstd;
        store8<true>(out, row * D + c * 8, o);
      }
    }
  }
}

// =============================================================================================
// Predictor input assembly (predictor.py:194-221) for one mask:
//   x[b, k, :]      = emb[b*Ke + k, :] + pos[idx_ctx[b,k], :]            k <  Ke
//   x[b, Ke + k, :] = mask_token[:]    + pos[idx_tgt[b,k], :]            k <  Kp
// x is the predictor residual stream [B, Ke+Kp, Dp] (bf16 or fp32).
// =============================================================================================
template <bool OUT_F32>
__global__ void __launch_bounds__(256) pred_assemble_kernel(const __nv_bfloat16* __restrict__ emb,
                                                            const float* __restrict__ pos,
                                                            const float* __restrict__ mask_token,
                                                            const long long* __restrict__ idx_ctx,
                                                            const long long* __restrict__ idx_tgt,
                                                            void* __restrict__ x, int B, int Ke, int Kp, int Dp) {
  const int vec = Dp >> 3;
  const int S = Ke + Kp;
  const long long total = (long long)B * S * vec;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = int(i % vec);
    const long long row = i / vec;
    const int b = int(row / S), k = int(row % S);
    float a[8], p[8];
    if (k < Ke) {
      load8<false>(emb, ((long long)b * Ke + k) * Dp + v * 8, a);
      load8<true>(pos, idx_ctx[(long long)b * Ke + k] * Dp + v * 8, p);
    } else {
      load8<true>(mask_token, v * 8, a);
      load8<true>(pos, idx_tgt[(long long)b * Kp + (k - Ke)] * Dp + v * 8, p);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += p[j];
    store8<OUT_F32>(x, row * Dp + v * 8, a);
  }
}

// dEmb[b*Ke + k, :] = bf16(dx[b, k, :]) for k < Ke   (context part of the assembly backward)
template <bool IN_F32>
__global__ void __launch_bounds__(256) pred_split_ctx_kernel(const void* __restrict__ dx,
                                                             __nv_bfloat16* __restrict__ demb, int B, int Ke, int Kp,
                                                             int Dp) {
  const int vec = Dp >> 3;
  const int S = Ke + Kp;
  const long long total = (long long)B * Ke * vec;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = int(i % vec);
    const long long row = i / vec;
    const int b = int(row / Ke), k = int(row % Ke);
    float a[8];
    load8<IN_F32>(dx, ((long long)b * S + k) * Dp + v * 8, a);
    store8<false>(demb, row * Dp + v * 8, a);
  }
}

// Slice rows k >= Ke of each [Ke+Kp] sequence into a dense [B*Kp, D] matrix (and the reverse).
template <bool F32>
__global__ void __launch_bounds__(256) seq_slice_kernel(const void* __restrict__ src, void* __restrict__ dst, int B,
                                                        int Ke, int Kp, int D, int scatter, int zero_ctx) {
  const int vec = D >> 3;
  const int S = Ke + Kp;
  if (!scatter) {
    const long long total = (long long)B * Kp * vec;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
      const int v = int(i % vec);
      const long long row = i / vec;
      const int b = int(row / Kp), k = int(row % Kp);
      float a[8];
      load8<F32>(src, ((long long)b * S + Ke + k) * D + v * 8, a);
      store8<F32>(dst, row * D + v * 8, a);
    }
  } else {
    const long long total = (long long)B * S * vec;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
      const int v = int(i % vec);
      const long long row = i / vec;
      const int b = int(row / S), k = int(row % S);
      float a[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (k >= Ke) load8<F32>(src, ((long long)b * Kp + (k - Ke)) * D + v * 8, a);
      else if (!zero_ctx) continue;
      store8<F32>(dst, row * D + v * 8, a);
    }
  }
}

// =============================================================================================
// L1 latent loss (train.py:440-446): sum |z - h| -> loss_sum (fp32 atomics, fp32 block partials);
// backward: dz = sign(z - h) * scale (bf16).
// =============================================================================================
__global__ void __launch_bounds__(256) l1_loss_fwd_kernel(const __nv_bfloat16* __restrict__ z,
                                                          const float* __restrict__ h, float* __restrict__ loss_sum,
                                                          long long n8, float weight) {
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8;
       i += (long long)gridDim.x * blockDim.x) {
    float a[8], b[8];
    load8<false>(z, i * 8, a);
    load8<true>(h, i * 8, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc += fabsf(a[j] - b[j]);
  }
  __shared__ float sm[8];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += sm[w];
    atomicAdd(loss_sum, s * weight);
  }
}
__global__ void __launch_bounds__(256) l1_loss_bwd_kernel(const __nv_bfloat16* __restrict__ z,
                                                          const float* __restrict__ h,
                                                          const float* __restrict__ gscale, float scale,
                                                          __nv_bfloat16* __restrict__ dz, long long n8) {
  const float sc = scale * (gscale ? *gscale : 1.0f);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8;
       i += (long long)gridDim.x * blockDim.x) {
    float a[8], b[8], o[8];
    load8<false>(z, i * 8, a);
    load8<true>(h, i * 8, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float d = a[j] - b[j];
      o[j] = d > 0.f ? sc : (d < 0.f ? -sc : 0.f);
    }
    store8<false>(dz, i * 8, o);
  }
}

// General exponent p of loss_fn (train.py:440-446): sum |z - h|^p * weight (weight carries 1 / (M n p)); p = 1 has its own
// kernels above.
__global__ void __launch_bounds__(256) lp_loss_fwd_kernel(const __nv_bfloat16* __restrict__ z, const float* __restrict__ h,
                                                          float* __restrict__ loss_sum, long long n8, float weight, float p) {
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    float a[8], b[8];
    load8<false>(z, i * 8, a);
    load8<true>(h, i * 8, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float d = fabsf(a[j] - b[j]);
      acc += d > 0.f ? powf(d, p) : 0.f;
    }
  }
  __shared__ float sm[8];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += sm[w];
    atomicAdd(loss_sum, s * weight);
  }
}
// dz = sign(d) |d|^(p-1) * scale * (*gscale)   (the 1/p of the loss cancels the p of the derivative)
__global__ void __launch_bounds__(256) lp_loss_bwd_kernel(const __nv_bfloat16* __restrict__ z, const float* __restrict__ h,
                                                          const float* __restrict__ gscale, float scale,
                                                          __nv_bfloat16* __restrict__ dz, long long n8, float p) {
  const float sc = scale * (gscale ? *gscale : 1.0f);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    float a[8], b[8], o[8];
    load8<false>(z, i * 8, a);
    load8<true>(h, i * 8, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float d = a[j] - b[j];
      const float m = fabsf(d);
      o[j] = m > 0.f ? copysignf(sc * powf(m, p - 1.0f), d) : 0.f;
    }
    store8<false>(dz, i * 8, o);
  }
}

// Mean and unbiased variance of one (b, d) column of z over its K tokens (stride D), in two passes: the one-pass
// (sum v^2 - K mean^2) form cancels when |mean| >> std, which are exactly the channels where relu(1 - pstd) is active.
// The squared deviations are summed in double: an fp32 running sum over a few thousand tokens drifts by ~1e-5.
VJ_DEVINL void token_mean_var(const __nv_bfloat16* __restrict__ p, int K, int D, float& mean, float& var) {
  float s = 0.f;
  for (int k = 0; k < K; ++k) s += __bfloat162float(p[(long long)k * D]);
  mean = s / K;
  double ss = 0.0;
  for (int k = 0; k < K; ++k) {
    const double dv = __bfloat162float(p[(long long)k * D]) - mean;
    ss += dv * dv;
  }
  var = float(ss / (K - 1));
}

// Backward of the variance regulariser (train.py:448-449,458-459) for one mask:
//   loss_reg = mean_{b,d} relu(1 - pstd[b,d]),  pstd = sum_i w * sqrt(var_unbiased_k(z_i[b,k,d]) + eps)
//   d loss_reg / d z_i[b,k,d] = -[pstd < 1] / (B D) * w * (z - mean_k z) / ((K - 1) * sqrt(var + eps))
__global__ void __launch_bounds__(128) token_std_bwd_kernel(const __nv_bfloat16* __restrict__ z,
                                                            const float* __restrict__ pstd_total,
                                                            const float* __restrict__ gscale, float scale,
                                                            __nv_bfloat16* __restrict__ dz, int B, int K, int D, float eps,
                                                            float weight) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (d >= D) return;
  const __nv_bfloat16* p = z + (long long)b * K * D + d;
  __nv_bfloat16* q = dz + (long long)b * K * D + d;
  float mean, var;
  token_mean_var(p, K, D, mean, var);
  const float g = scale * (gscale ? *gscale : 1.0f);
  const float c = pstd_total[(long long)b * D + d] < 1.0f ? -g * weight / ((float)B * D * (K - 1) * sqrtf(var + eps)) : 0.f;
  for (int k = 0; k < K; ++k) q[(long long)k * D] = __float2bfloat16(c * (__bfloat162float(p[(long long)k * D]) - mean));
}

// Per-(b, d) unbiased variance of z over the token dim -> pstd = sqrt(var + 1e-4)  (train.py:448-449)
__global__ void __launch_bounds__(256) token_std_kernel(const __nv_bfloat16* __restrict__ z, float* __restrict__ pstd,
                                                        int B, int K, int D, float eps, float weight) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (d >= D) return;
  float mean, var;
  token_mean_var(z + (long long)b * K * D + d, K, D, mean, var);
  pstd[(long long)b * D + d] += weight * sqrtf(var + eps);
}

static int grid_for(long long work_items, int per_block) {
  long long g = (work_items + per_block - 1) / per_block;
  const long long cap = (long long)num_sms() * 8;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return int(g);
}

}  // namespace vj

using namespace vj;


// in_f32: 0 bf16, 1 fp32 (any non-zero value, as the ABI has always read it), 2 fp16 (vj_colsum_f16 only)
static int colsum(const char* name, const void* in, int in_f32, float* out, long long T, int N, long long ld, int period,
                  int lo, int hi, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(in && out, "%s: null pointer", name);
  VJ_CHECK_ARG(N % 8 == 0 && ld % 8 == 0, "%s: N/ld must be multiples of 8", name);
  if (T <= 0) return 0;
  const int gx = (N + 255) / 256;
  long long want = (long long)num_sms() * 4 / gx;
  if (want < 1) want = 1;
  long long rpb = (T + want - 1) / want;
  if (rpb < 64) rpb = 64;
  const int gy = int((T + rpb - 1) / rpb);
  dim3 grid(gx, gy);
  if (in_f32 == 2) colsum_kernel<false, __half><<<grid, 256, 0, s>>>(in, out, T, N, ld, int(rpb), period, lo, hi);
  else if (in_f32) colsum_kernel<true><<<grid, 256, 0, s>>>(in, out, T, N, ld, int(rpb), period, lo, hi);
  else colsum_kernel<false><<<grid, 256, 0, s>>>(in, out, T, N, ld, int(rpb), period, lo, hi);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_colsum(const void* in, int in_f32, float* out, long long T, int N, long long ld, int period, int lo,
                         int hi, void* stream) {
  return colsum("vj_colsum", in, in_f32 ? 1 : 0, out, T, N, ld, period, lo, hi, stream);
}

extern "C" int vj_colsum_f16(const void* in, float* out, long long T, int N, long long ld, int period, int lo, int hi,
                             void* stream) {
  return colsum("vj_colsum_f16", in, 2, out, T, N, ld, period, lo, hi, stream);
}

template <typename TO>
static int im2col_tubelets(const float* clips, void* patches, const long long* idx, int B, int C, int T, int H, int W,
                           int tubelet, int patch, int K, cudaStream_t s) {
  VJ_CHECK_ARG(clips && patches, "vj_im2col_tubelets: null pointer");
  // W % patch == 0 and an even patch keep every 8-byte (ps % 4 != 0) or 16-byte (ps % 4 == 0) load aligned
  VJ_CHECK_ARG(T % tubelet == 0 && H % patch == 0 && W % patch == 0 && patch % 2 == 0,
               "vj_im2col_tubelets: bad geometry (T %% tubelet, H %% patch, W %% patch must be 0 and patch even)");
  const int n_tokens = (T / tubelet) * (H / patch) * (W / patch);
  const int kout = idx ? K : n_tokens;
  if (B <= 0 || kout <= 0) return 0;
  const int P = C * tubelet * patch * patch;
  const long long warps = (long long)B * kout * C * tubelet;
  TO* out = reinterpret_cast<TO*>(patches);
  if (patch % 4 == 0 && P % 64 == 0)   // every ps-16 model: rows exactly P long
    im2col_kernel<TO, 4, false><<<grid_for(warps, 8), 256, 0, s>>>(clips, out, idx, B, C, T, H, W, tubelet, patch, kout,
                                                                   n_tokens);
  else if (patch % 4 == 0)
    im2col_kernel<TO, 4, true><<<grid_for(warps, 8), 256, 0, s>>>(clips, out, idx, B, C, T, H, W, tubelet, patch, kout,
                                                                  n_tokens);
  else
    im2col_kernel<TO, 2, true><<<grid_for(warps, 8), 256, 0, s>>>(clips, out, idx, B, C, T, H, W, tubelet, patch, kout,
                                                                  n_tokens);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_im2col_tubelets(const float* clips, void* patches, const long long* idx, int B, int C, int T, int H,
                                  int W, int tubelet, int patch, int K, void* stream) {
  return im2col_tubelets<__nv_bfloat16>(clips, patches, idx, B, C, T, H, W, tubelet, patch, K,
                                        reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vj_im2col_tubelets_f16(const float* clips, void* patches, const long long* idx, int B, int C, int T,
                                      int H, int W, int tubelet, int patch, int K, void* stream) {
  return im2col_tubelets<__half>(clips, patches, idx, B, C, T, H, W, tubelet, patch, K,
                                 reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vj_gather_rows(const void* x, void* out, const long long* idx, int B, int N, int K, int row_bytes,
                              void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0 || K <= 0) return 0;  // empty selection: nothing to do (empty tensors carry null pointers)
  VJ_CHECK_ARG(x && out && idx, "vj_gather_rows: null pointer");
  VJ_CHECK_ARG(row_bytes % 16 == 0, "vj_gather_rows: row_bytes must be a multiple of 16");
  const int vpr = row_bytes / 16;
  gather_rows_kernel<<<grid_for((long long)B * K * vpr, 256), 256, 0, s>>>(
      reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(out), idx, B, N, K, vpr);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_scatter_rows_add(const void* dy, void* dx, const long long* idx, int B, int N, int K, int D, int f32,
                                   void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(dy && dx && idx, "vj_scatter_rows_add: null pointer");
  VJ_CHECK_ARG(D % 8 == 0, "vj_scatter_rows_add: D must be a multiple of 8");
  if (B <= 0 || K <= 0) return 0;
  const int g = grid_for((long long)B * K * (D / 8), 256);
  if (f32) scatter_rows_add_kernel<true><<<g, 256, 0, s>>>(dy, dx, idx, B, N, K, D);
  else scatter_rows_add_kernel<false><<<g, 256, 0, s>>>(dy, dx, idx, B, N, K, D);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_target_ln_gather(const void* x, float* out, const long long* idx, const float* gamma,
                                   const float* beta, int B, int N, int K, int D, float eps_norm, float eps_target,
                                   void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(x && out && idx && gamma && beta, "vj_target_ln_gather: null pointer");
  VJ_CHECK_ARG(D % 8 == 0 && D <= 8 * 32 * kMaxVec, "vj_target_ln_gather: D=%d unsupported", D);
  if (B <= 0 || K <= 0) return 0;
  target_ln_gather_kernel<<<grid_for((long long)B * K, 8), 256, 0, s>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), out, idx, gamma, beta, B, N, K, D, eps_norm, eps_target);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_pred_assemble_fwd(const void* emb, const float* pos, const float* mask_token,
                                    const long long* idx_ctx, const long long* idx_tgt, void* x, int x_f32, int B,
                                    int Ke, int Kp, int Dp, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(emb && pos && mask_token && idx_ctx && idx_tgt && x, "vj_pred_assemble_fwd: null pointer");
  VJ_CHECK_ARG(Dp % 8 == 0, "vj_pred_assemble_fwd: Dp must be a multiple of 8");
  if (B <= 0) return 0;
  const int g = grid_for((long long)B * (Ke + Kp) * (Dp / 8), 256);
  if (x_f32)
    pred_assemble_kernel<true><<<g, 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(emb), pos, mask_token, idx_ctx,
                                                 idx_tgt, x, B, Ke, Kp, Dp);
  else
    pred_assemble_kernel<false><<<g, 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(emb), pos, mask_token, idx_ctx,
                                                  idx_tgt, x, B, Ke, Kp, Dp);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_pred_assemble_bwd(const void* dx, int dx_f32, void* demb, float* dmask_token, int B, int Ke, int Kp,
                                    int Dp, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(dx && demb && dmask_token, "vj_pred_assemble_bwd: null pointer");
  VJ_CHECK_ARG(Dp % 8 == 0, "vj_pred_assemble_bwd: Dp must be a multiple of 8");
  if (B <= 0) return 0;
  const int g = grid_for((long long)B * Ke * (Dp / 8), 256);
  if (dx_f32)
    pred_split_ctx_kernel<true><<<g, 256, 0, s>>>(dx, reinterpret_cast<__nv_bfloat16*>(demb), B, Ke, Kp, Dp);
  else
    pred_split_ctx_kernel<false><<<g, 256, 0, s>>>(dx, reinterpret_cast<__nv_bfloat16*>(demb), B, Ke, Kp, Dp);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  // mask-token gradient = column sum over the target rows of every sequence
  return vj_colsum(dx, dx_f32, dmask_token, (long long)B * (Ke + Kp), Dp, Dp, Ke + Kp, Ke, Ke + Kp, stream_);
}

extern "C" int vj_seq_slice(const void* src, void* dst, int f32, int B, int Ke, int Kp, int D, int scatter,
                            int zero_ctx, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(src && dst, "vj_seq_slice: null pointer");
  VJ_CHECK_ARG(D % 8 == 0, "vj_seq_slice: D must be a multiple of 8");
  if (B <= 0) return 0;
  const long long rows = scatter ? (long long)B * (Ke + Kp) : (long long)B * Kp;
  const int g = grid_for(rows * (D / 8), 256);
  if (f32) seq_slice_kernel<true><<<g, 256, 0, s>>>(src, dst, B, Ke, Kp, D, scatter, zero_ctx);
  else seq_slice_kernel<false><<<g, 256, 0, s>>>(src, dst, B, Ke, Kp, D, scatter, zero_ctx);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_l1_loss_fwd(const void* z, const float* h, float* loss_sum, long long n, float weight,
                              void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(z && h && loss_sum, "vj_l1_loss_fwd: null pointer");
  VJ_CHECK_ARG(n % 8 == 0, "vj_l1_loss_fwd: n must be a multiple of 8");
  if (n <= 0) return 0;
  l1_loss_fwd_kernel<<<grid_for(n / 8, 256 * 4), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(z), h, loss_sum,
                                                              n / 8, weight);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_l1_loss_bwd(const void* z, const float* h, const float* grad_scale_dev, float scale, void* dz,
                              long long n, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(z && h && dz, "vj_l1_loss_bwd: null pointer");
  VJ_CHECK_ARG(n % 8 == 0, "vj_l1_loss_bwd: n must be a multiple of 8");
  if (n <= 0) return 0;
  l1_loss_bwd_kernel<<<grid_for(n / 8, 256 * 4), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(z), h,
                                                              grad_scale_dev, scale,
                                                              reinterpret_cast<__nv_bfloat16*>(dz), n / 8);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_lp_loss_fwd(const void* z, const float* h, float* loss_sum, long long n, float weight, float p,
                              void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(z && h && loss_sum, "vj_lp_loss_fwd: null pointer");
  VJ_CHECK_ARG(n % 8 == 0 && p > 0.f, "vj_lp_loss_fwd: n must be a multiple of 8 and the exponent positive");
  if (n <= 0) return 0;
  lp_loss_fwd_kernel<<<grid_for(n / 8, 256 * 4), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(z), h, loss_sum,
                                                              n / 8, weight, p);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_lp_loss_bwd(const void* z, const float* h, const float* grad_scale_dev, float scale, void* dz,
                              long long n, float p, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(z && h && dz, "vj_lp_loss_bwd: null pointer");
  VJ_CHECK_ARG(n % 8 == 0 && p >= 1.f, "vj_lp_loss_bwd: n must be a multiple of 8 and the exponent >= 1");
  if (n <= 0) return 0;
  lp_loss_bwd_kernel<<<grid_for(n / 8, 256 * 4), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(z), h,
                                                              grad_scale_dev, scale,
                                                              reinterpret_cast<__nv_bfloat16*>(dz), n / 8, p);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_token_std_bwd(const void* z, const float* pstd_total, const float* grad_scale_dev, float scale, void* dz,
                                int B, int K, int D, float eps, float weight, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(z && pstd_total && dz, "vj_token_std_bwd: null pointer");
  VJ_CHECK_ARG(K > 1, "vj_token_std_bwd: needs K > 1");
  if (B <= 0) return 0;
  dim3 grid((D + 127) / 128, B);
  token_std_bwd_kernel<<<grid, 128, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(z), pstd_total, grad_scale_dev, scale,
                                            reinterpret_cast<__nv_bfloat16*>(dz), B, K, D, eps, weight);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_token_std_accum(const void* z, float* pstd, int B, int K, int D, float eps, float weight,
                                  void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(z && pstd, "vj_token_std_accum: null pointer");
  VJ_CHECK_ARG(K > 1, "vj_token_std_accum: needs K > 1");
  if (B <= 0) return 0;
  dim3 grid((D + 127) / 128, B);
  token_std_kernel<<<grid, 128, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(z), pstd, B, K, D, eps, weight);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}
