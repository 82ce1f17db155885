// Flash-attention backward on wgmma (sm_90a), dense var-len, deterministic (no atomics).
//
// Backward of F.scaled_dot_product_attention (src/models/utils/modules.py:66-69):
//   P = softmax(scale Q K^T), dV = P^T dO, dP = dO V^T, dS = P o (dP - rowsum(dO o O)),
//   dQ = scale dS K, dK = scale dS^T Q.
// Three kernels:
//   attn_delta_kernel  : delta[h,t] = sum_d dO[t,h,d] O[t,h,d]                      (HBM-bound)
//   attn_bwd_dkv_kernel: one CTA per 128-key tile (two warpgroups of 64 keys), loops over 64-query tiles; computes
//                        S^T = K Q^T and dP^T = V dO^T directly in the transposed orientation so P^T / dS^T are register
//                        A operands of dV += P^T dO and dK += dS^T Q, both accumulated in registers across the loop.
//   attn_bwd_dq_kernel : one CTA per 128-query tile, loops over 64-key tiles; dQ += dS K in registers.
// P is recomputed from the forward's log2-domain LSE.  Same qkv / O layouts as attn_fwd.cu; the
// gradient dqkv has the qkv layout [T, 3*H*HD] so the qkv wgrad/dgrad GEMMs consume it directly.
#include <stdlib.h>

#include "attn_common.cuh"
#include "vjepa_b200.h"

namespace vj {

constexpr int kBwdThreads = 256;
constexpr int kBwdStream = 64;   // rows of the streamed (query or key) tiles

struct AttnBwdParams {
  const int* cu_seqlens;
  const float* lse2;
  const float* delta;
  __nv_bfloat16* dqkv;
  int H, T;
  float scale, scale_log2;
};

template <int HD>
struct BwdCfg {
  using A = AttnCfg<HD>;
  // two resident [128 x HD] tiles (T0, T1) and two stages of the two streamed [64 x HD] tiles
  static constexpr int RES = A::template tile_bytes<128>();
  static constexpr int STR = A::template tile_bytes<kBwdStream>();
  static constexpr int T0 = 0, T1 = RES;
  static constexpr int S_OFF = 2 * RES;                 // stage st: tile a at S_OFF + st * 2 * STR, tile b at + STR
  static constexpr int BAR_OFF = S_OFF + 4 * STR;
  static constexpr int SMEM_BYTES = BAR_OFF + 64 + 1024;
};

// ---------------------------------------------------------------------------------------------
// delta[h, t] = sum_d dO[t, h*HD + d] * O[t, h*HD + d]
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) attn_delta_kernel(const __nv_bfloat16* __restrict__ o,
                                                         const __nv_bfloat16* __restrict__ dout,
                                                         float* __restrict__ delta, int T, int H, int HD) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const int D = H * HD;
  const int nvec = D >> 3;
  const int lanes_per_head = HD >> 3;
  for (long long t = (long long)blockIdx.x * wpb + (threadIdx.x >> 5); t < T; t += (long long)gridDim.x * wpb) {
    for (int c = lane; c < ((nvec + 31) / 32) * 32; c += 32) {
      float s = 0.f;
      if (c < nvec) {
        const uint4 a = *reinterpret_cast<const uint4*>(o + t * D + c * 8);
        const uint4 b = *reinterpret_cast<const uint4*>(dout + t * D + c * 8);
        s = bf16_lo(a.x) * bf16_lo(b.x) + bf16_hi(a.x) * bf16_hi(b.x) + bf16_lo(a.y) * bf16_lo(b.y) +
            bf16_hi(a.y) * bf16_hi(b.y) + bf16_lo(a.z) * bf16_lo(b.z) + bf16_hi(a.z) * bf16_hi(b.z) +
            bf16_lo(a.w) * bf16_lo(b.w) + bf16_hi(a.w) * bf16_hi(b.w);
      }
      for (int o2 = lanes_per_head >> 1; o2 > 0; o2 >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o2);
      if (c < nvec && (lane % lanes_per_head) == 0) delta[(long long)((c * 8) / HD) * T + t] = s;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// DKV = true : CTA = (128-key tile, sequence, head); resident K, V; streamed Q_i, dO_i.  Writes dK, dV.
// DKV = false: CTA = (128-query tile, sequence, head); resident Q, dO; streamed K_j, V_j.  Writes dQ.
// The two share the pipeline and the P / dS algebra; only the orientation of the score fragment differs: in the dK/dV
// kernel the fragment's rows are keys and its columns queries (lse2 / delta are per column), in the dQ kernel the
// reverse (lse2 / delta per row).
// ---------------------------------------------------------------------------------------------
template <int HD, bool DKV>
__global__ void __launch_bounds__(kBwdThreads, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmRes, const __grid_constant__ CUtensorMap tmStr,
                const __grid_constant__ CUtensorMap tmDO, const AttnBwdParams p) {
  using B = BwdCfg<HD>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  const int seq = blockIdx.y, head = blockIdx.z;
  const int row_begin = p.cu_seqlens[seq];
  const int len = p.cu_seqlens[seq + 1] - row_begin;
  const int t0 = blockIdx.x * 128;   // first resident row (key for DKV, query otherwise)
  if (t0 >= len) return;
  const int n_it = (len + kBwdStream - 1) / kBwdStream;
  const int HHD = p.H * HD;

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + B::BAR_OFF);
  const uint32_t bar_res = smem_u32(bars + 0);
  const uint32_t bar_s0 = smem_u32(bars + 1);   // 2 stages
  const uint32_t sT0 = smem_u32(smem + B::T0), sT1 = smem_u32(smem + B::T1), sS = smem_u32(smem + B::S_OFF);

  // resident: DKV -> T0 = K, T1 = V;  dQ -> T0 = Q, T1 = dO.   streamed: DKV -> a = Q_i, b = dO_i;  dQ -> a = K_j, b = V_j
  auto load_stream = [&](int i) {   // thread 0 only
    const int st = i & 1;
    const uint32_t a = sS + st * 2 * B::STR, b = a + B::STR, bar = bar_s0 + 8 * st;
    const int r0 = row_begin + i * kBwdStream;
    mbar_expect_tx(bar, 2 * B::STR);
    if (DKV) {
      attn_load_tile<HD, kBwdStream>(a, &tmStr, bar, head * HD, r0);
      attn_load_tile<HD, kBwdStream>(b, &tmDO, bar, head * HD, r0);
    } else {
      attn_load_tile<HD, kBwdStream>(a, &tmStr, bar, HHD + head * HD, r0);
      attn_load_tile<HD, kBwdStream>(b, &tmStr, bar, 2 * HHD + head * HD, r0);
    }
  };
  if (threadIdx.x == 0) {
    mbar_init(bar_res, 1);
    mbar_init(bar_s0, 1);
    mbar_init(bar_s0 + 8, 1);
    fence_mbar_init();
    mbar_expect_tx(bar_res, 2 * B::RES);
    if (DKV) {
      attn_load_tile<HD, 128>(sT0, &tmRes, bar_res, HHD + head * HD, row_begin + t0);
      attn_load_tile<HD, 128>(sT1, &tmRes, bar_res, 2 * HHD + head * HD, row_begin + t0);
    } else {
      attn_load_tile<HD, 128>(sT0, &tmRes, bar_res, head * HD, row_begin + t0);
      attn_load_tile<HD, 128>(sT1, &tmDO, bar_res, head * HD, row_begin + t0);
    }
    load_stream(0);
    if (n_it > 1) load_stream(1);
  }
  __syncthreads();

  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;
  const int r = wg * 64 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);   // first fragment row in the resident tile
  const float* lse_h = p.lse2 + (long long)head * p.T + row_begin;
  const float* del_h = p.delta + (long long)head * p.T + row_begin;
  float acc0[HD / 2], acc1[HD / 2];   // DKV: dV, dK;  dQ: dQ (acc1 unused)
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
  float row_lse[2], row_del[2];   // dQ kernel: per-row statistics of the resident queries
  if (!DKV) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int q = t0 + r + 8 * h;
      row_lse[h] = q < len ? lse_h[q] : 0.f;
      row_del[h] = q < len ? del_h[q] : 0.f;
    }
  }

  mbar_wait(bar_res, 0);
  for (int i = 0; i < n_it; ++i) {
    const int st = i & 1;
    const uint32_t sa = sS + st * 2 * B::STR, sb = sa + B::STR;
    const int c0 = i * kBwdStream;   // first streamed row (relative to the sequence)
    mbar_wait(bar_s0 + 8 * st, (i >> 1) & 1);
    // DKV: x = S^T = K Q_i^T, y = dP^T = V dO_i^T;   dQ: x = S = Q K_j^T, y = dP = dO V_j^T
    float x[kBwdStream / 2], y[kBwdStream / 2];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk)
      wgmma_ss<kBwdStream, 0, 0>(x, attn_kmajor_desc<HD, 128>(sT0, wg * 64, kk), attn_kmajor_desc<HD, kBwdStream>(sa, 0, kk),
                                 kk > 0);
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk)
      wgmma_ss<kBwdStream, 0, 0>(y, attn_kmajor_desc<HD, 128>(sT1, wg * 64, kk), attn_kmajor_desc<HD, kBwdStream>(sb, 0, kk),
                                 kk > 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(x);
    wgmma_fence_regs(y);

    // x <- P (or P^T), y <- dS (or dS^T);  fragment element [4c + 2h + e]: row r + 8h, column 8c + 2(lane % 4) + e
#pragma unroll
    for (int c = 0; c < kBwdStream / 8; ++c)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = c0 + 8 * c + 2 * (lane & 3) + e;
        const bool col_ok = col < len;
        float cl = 0.f, cd = 0.f;
        if (DKV && col_ok) { cl = lse_h[col]; cd = del_h[col]; }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float l2 = DKV ? cl : row_lse[h], dl = DKV ? cd : row_del[h];
          float& pv = x[4 * c + 2 * h + e];
          float& dv = y[4 * c + 2 * h + e];
          pv = col_ok ? ex2_approx(fmaf(pv, p.scale_log2, -l2)) : 0.f;
          dv = pv * (dv - dl);
        }
      }

    // DKV: dV += P^T dO_i, dK += dS^T Q_i;   dQ: dQ += dS K_j   (streamed operand read MN-major)
    wgmma_fence_regs(acc0);
    wgmma_fence_regs(acc1);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kBwdStream / 16; ++kk) {
      uint32_t a[4];
      if (DKV) {
        acc_to_afrag(x, kk, a);
        wgmma_rs<HD, 1>(acc0, a, attn_mnmajor_desc<HD, kBwdStream>(sb, kk), 1);
        acc_to_afrag(y, kk, a);
        wgmma_rs<HD, 1>(acc1, a, attn_mnmajor_desc<HD, kBwdStream>(sa, kk), 1);
      } else {
        acc_to_afrag(y, kk, a);
        wgmma_rs<HD, 1>(acc0, a, attn_mnmajor_desc<HD, kBwdStream>(sa, kk), 1);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(acc0);
    wgmma_fence_regs(acc1);
    __syncthreads();   // both warpgroups are done with stage st
    if (threadIdx.x == 0 && i + 2 < n_it) load_stream(i + 2);
  }

  __nv_bfloat16* rows = p.dqkv + (long long)(row_begin + t0) * 3 * HHD + head * HD;
  if (DKV) {
    store_frag_bf16<HD>(acc1, p.scale, rows + HHD, 3LL * HHD, r, len - t0);       // dK
    store_frag_bf16<HD>(acc0, 1.0f, rows + 2 * HHD, 3LL * HHD, r, len - t0);      // dV
  } else {
    store_frag_bf16<HD>(acc0, p.scale, rows, 3LL * HHD, r, len - t0);             // dQ
  }
}

template <int HD>
static int launch_attn_bwd(const void* qkv, const void* out, const void* dout, const float* lse2, float* delta,
                           void* dqkv, const int* cu, int nseq, int max_len, int H, int T, float scale, cudaStream_t s) {
  using C = AttnCfg<HD>;
  using B = BwdCfg<HD>;
  CUtensorMap tq128, tq64, tdo128, tdo64;
  const uint64_t W = (uint64_t)3 * H * HD;
  int rc = make_tmap_2d(&tq128, qkv, 0, W, T, W * 2, C::BOX_INNER, 128, C::TMAP_SWIZZLE);
  if (!rc) rc = make_tmap_2d(&tq64, qkv, 0, W, T, W * 2, C::BOX_INNER, kBwdStream, C::TMAP_SWIZZLE);
  if (!rc) rc = make_tmap_2d(&tdo128, dout, 0, (uint64_t)H * HD, T, (uint64_t)H * HD * 2, C::BOX_INNER, 128, C::TMAP_SWIZZLE);
  if (!rc) rc = make_tmap_2d(&tdo64, dout, 0, (uint64_t)H * HD, T, (uint64_t)H * HD * 2, C::BOX_INNER, kBwdStream,
                             C::TMAP_SWIZZLE);
  if (rc) return rc;
  auto kdkv = attn_bwd_kernel<HD, true>;
  auto kdq = attn_bwd_kernel<HD, false>;
  static bool configured = false;
  if (!configured) {
    VJ_CUDA(cudaFuncSetAttribute(kdkv, cudaFuncAttributeMaxDynamicSharedMemorySize, B::SMEM_BYTES));
    VJ_CUDA(cudaFuncSetAttribute(kdq, cudaFuncAttributeMaxDynamicSharedMemorySize, B::SMEM_BYTES));
    configured = true;
  }
  {
    int g = (T + 7) / 8;
    const int cap = num_sms() * 8;
    if (g > cap) g = cap;
    attn_delta_kernel<<<g, 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(out),
                                        reinterpret_cast<const __nv_bfloat16*>(dout), delta, T, H, HD);
    VJ_CUDA(cudaGetLastError());
    vj::count_launch(1);
  }
  AttnBwdParams p;
  p.cu_seqlens = cu; p.lse2 = lse2; p.delta = delta; p.dqkv = reinterpret_cast<__nv_bfloat16*>(dqkv);
  p.H = H; p.T = T; p.scale = scale; p.scale_log2 = scale * 1.4426950408889634f;
  dim3 grid((max_len + 127) / 128, nseq, H);
  kdkv<<<grid, kBwdThreads, B::SMEM_BYTES, s>>>(tq128, tq64, tdo64, p);
  VJ_CUDA(cudaGetLastError());
  kdq<<<grid, kBwdThreads, B::SMEM_BYTES, s>>>(tq128, tq64, tdo128, p);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(2);
  return 0;
}

}  // namespace vj

extern "C" int vj_attn_bwd(const void* qkv, const void* out, const void* dout, const float* lse2, float* delta_ws,
                           void* dqkv, float* dq_acc_ws, const int* cu_seqlens, int nseq, int max_len, int H, int HD,
                           int T, float scale, void* stream_) {
  using namespace vj;
  (void)dq_acc_ws;   // unused: dQ always comes from its own kernel (see the header)
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(qkv && out && dout && lse2 && delta_ws && dqkv && cu_seqlens, "vj_attn_bwd: null pointer");
  VJ_CHECK_ARG(nseq > 0 && max_len > 0 && H > 0 && T > 0, "vj_attn_bwd: empty problem");
  switch (HD) {
    case 32: return launch_attn_bwd<32>(qkv, out, dout, lse2, delta_ws, dqkv, cu_seqlens, nseq, max_len, H, T, scale, s);
    case 64: return launch_attn_bwd<64>(qkv, out, dout, lse2, delta_ws, dqkv, cu_seqlens, nseq, max_len, H, T, scale, s);
    case 128: return launch_attn_bwd<128>(qkv, out, dout, lse2, delta_ws, dqkv, cu_seqlens, nseq, max_len, H, T, scale, s);
    default: set_error("vj_attn_bwd: head dim %d unsupported (32/64/128)", HD); return -1;
  }
}
