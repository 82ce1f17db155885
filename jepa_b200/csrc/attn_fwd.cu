// Dense (non-causal) variable-length flash attention forward on wgmma (sm_90a).
//
// Replaces F.scaled_dot_product_attention at src/models/utils/modules.py:66-69 (the `mask`
// argument there is ignored - "masked attention" is attention over the gathered token subset,
// so every sequence is dense and only its length varies).
//
// Layout: qkv bf16 [T, 3*H*HD] (row = token, q|k|v packed, head-major inside each third - the
// layout the qkv GEMM epilogue writes), O bf16 [T, H*HD], lse2 fp32 [H, T] (log2 domain:
// m*scale*log2e + log2(l)).  Sequences are row ranges [cu[s], cu[s+1]).
//
// One CTA = one 128-row query tile of one (sequence, head), two warpgroups of 64 query rows each.  K_j / V_j tiles of
// 128 keys stream through a two-stage TMA ring (thread 0 refills a stage as soon as both warpgroups are done with it).
// Per tile: S = Q K_j^T (wgmma, both operands in smem), online softmax on the accumulator fragment in registers,
// O += P V_j with P as the register A operand (no shared-memory round trip) and V_j read MN-major.
#include <stdlib.h>

#include "attn_common.cuh"
#include "vjepa_b200.h"

namespace vj {

constexpr int kFwdThreads = 256;
constexpr int kFwdKV = 128;   // keys per tile

struct AttnFwdParams {
  const int* cu_seqlens;
  __nv_bfloat16* out;
  float* lse2;
  int H, T;
  long long ld_out;
  float scale_log2;
};

template <int HD>
struct FwdCfg {
  using A = AttnCfg<HD>;
  static constexpr int TILE = A::template tile_bytes<128>();
  static constexpr int Q_OFF = 0;
  static constexpr int K_OFF = TILE;          // 2 stages
  static constexpr int V_OFF = 3 * TILE;      // 2 stages
  static constexpr int BAR_OFF = 5 * TILE;
  static constexpr int SMEM_BYTES = BAR_OFF + 64 + 1024;
};

template <int HD>
__global__ void __launch_bounds__(kFwdThreads, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQKV, const AttnFwdParams p) {
  using F = FwdCfg<HD>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  const int seq = blockIdx.y, head = blockIdx.z;
  const int row_begin = p.cu_seqlens[seq];
  const int len = p.cu_seqlens[seq + 1] - row_begin;
  const int q0 = blockIdx.x * 128;
  if (q0 >= len) return;
  const int n_kv = (len + kFwdKV - 1) / kFwdKV;

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + F::BAR_OFF);
  const uint32_t bar_q = smem_u32(bars + 0);
  const uint32_t bar_kv0 = smem_u32(bars + 1);   // 2 stages: +0, +8
  const uint32_t sQ = smem_u32(smem + F::Q_OFF), sK = smem_u32(smem + F::K_OFF), sV = smem_u32(smem + F::V_OFF);
  const int HHD = p.H * HD;

  auto load_kv = [&](int j) {   // thread 0 only
    const int st = j & 1;
    mbar_expect_tx(bar_kv0 + 8 * st, 2 * F::TILE);
    attn_load_tile<HD, 128>(sK + st * F::TILE, &tmQKV, bar_kv0 + 8 * st, HHD + head * HD, row_begin + j * kFwdKV);
    attn_load_tile<HD, 128>(sV + st * F::TILE, &tmQKV, bar_kv0 + 8 * st, 2 * HHD + head * HD, row_begin + j * kFwdKV);
  };
  if (threadIdx.x == 0) {
    mbar_init(bar_q, 1);
    mbar_init(bar_kv0, 1);
    mbar_init(bar_kv0 + 8, 1);
    fence_mbar_init();
    tma_prefetch_desc(&tmQKV);
    mbar_expect_tx(bar_q, F::TILE);
    attn_load_tile<HD, 128>(sQ, &tmQKV, bar_q, head * HD, row_begin + q0);
    load_kv(0);
    if (n_kv > 1) load_kv(1);
  }
  __syncthreads();

  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;
  const int r = wg * 64 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);   // this thread's first row in the tile (+8: second)
  float o[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  mbar_wait(bar_q, 0);
  for (int j = 0; j < n_kv; ++j) {
    const int st = j & 1;
    const int valid = min(kFwdKV, len - j * kFwdKV);
    mbar_wait(bar_kv0 + 8 * st, (j >> 1) & 1);
    float s[kFwdKV / 2];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk)
      wgmma_ss<kFwdKV, 0, 0>(s, attn_kmajor_desc<HD, 128>(sQ, wg * 64, kk),
                             attn_kmajor_desc<HD, 128>(sK + st * F::TILE, 0, kk), kk > 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);

    // ---- online softmax on the fragment: s[4c + 2h + e] = row r + 8h, key 8c + 2(lane % 4) + e
    float alpha[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int c = 0; c < kFwdKV / 8; ++c)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int key = 8 * c + 2 * (lane & 3) + e;
          float& v = s[4 * c + 2 * h + e];
          if (key >= valid) v = -INFINITY;
          mx = fmaxf(mx, v);
        }
      mx = quad_max(mx);
      const float m_new = fmaxf(m_run[h], mx);
      alpha[h] = ex2_approx((m_run[h] - m_new) * p.scale_log2);   // 0 on the first tile (m_run = -inf)
      m_run[h] = m_new;
      const float moff = m_new * p.scale_log2;
      float sum = 0.f;
#pragma unroll
      for (int c = 0; c < kFwdKV / 8; ++c)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& v = s[4 * c + 2 * h + e];
          v = ex2_approx(fmaf(v, p.scale_log2, -moff));
          sum += v;
        }
      l_run[h] = l_run[h] * alpha[h] + sum;   // per-thread partial; the quad is summed once at the end
    }
#pragma unroll
    for (int c = 0; c < HD / 8; ++c) {
      o[4 * c + 0] *= alpha[0]; o[4 * c + 1] *= alpha[0];
      o[4 * c + 2] *= alpha[1]; o[4 * c + 3] *= alpha[1];
    }

    // ---- O += P V_j
    wgmma_fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kFwdKV / 16; ++kk) {
      uint32_t a[4];
      acc_to_afrag(s, kk, a);
      wgmma_rs<HD, 1>(o, a, attn_mnmajor_desc<HD, 128>(sV + st * F::TILE, kk), 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    __syncthreads();   // both warpgroups are done with stage st
    if (threadIdx.x == 0 && j + 2 < n_kv) load_kv(j + 2);
  }

  // ---- epilogue: O / l -> bf16, lse2 (log2 domain)
  float inv[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float l = quad_sum(l_run[h]);
    inv[h] = 1.0f / l;
    const int row = q0 + r + 8 * h;
    if ((lane & 3) == 0 && row < len) p.lse2[(long long)head * p.T + row_begin + row] = m_run[h] * p.scale_log2 + log2f(l);
  }
#pragma unroll
  for (int c = 0; c < HD / 8; ++c) {
    o[4 * c + 0] *= inv[0]; o[4 * c + 1] *= inv[0];
    o[4 * c + 2] *= inv[1]; o[4 * c + 3] *= inv[1];
  }
  store_frag_bf16<HD>(o, 1.0f, p.out + (long long)(row_begin + q0) * p.ld_out + head * HD, p.ld_out, r, len - q0);
}

template <int HD>
static int launch_attn_fwd(const void* qkv, void* out, float* lse2, const int* cu, int nseq, int max_len, int H, int T,
                           float scale, cudaStream_t s) {
  using C = AttnCfg<HD>;
  using F = FwdCfg<HD>;
  CUtensorMap tm;
  int rc = make_tmap_2d(&tm, qkv, 0, (uint64_t)3 * H * HD, T, (uint64_t)3 * H * HD * 2, C::BOX_INNER, 128,
                        C::TMAP_SWIZZLE);
  if (rc) return rc;
  auto kern = attn_fwd_kernel<HD>;
  static bool configured = false;
  if (!configured) {
    VJ_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, F::SMEM_BYTES));
    configured = true;
  }
  AttnFwdParams p;
  p.cu_seqlens = cu; p.out = reinterpret_cast<__nv_bfloat16*>(out); p.lse2 = lse2;
  p.H = H; p.T = T; p.ld_out = (long long)H * HD;
  p.scale_log2 = scale * 1.4426950408889634f;
  dim3 grid((max_len + 127) / 128, nseq, H);
  kern<<<grid, kFwdThreads, F::SMEM_BYTES, s>>>(tm, p);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

}  // namespace vj

extern "C" int vj_attn_fwd(const void* qkv, void* out, float* lse2, const int* cu_seqlens, int nseq, int max_len,
                           int H, int HD, int T, float scale, void* stream_) {
  using namespace vj;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(qkv && out && lse2 && cu_seqlens, "vj_attn_fwd: null pointer");
  VJ_CHECK_ARG(nseq > 0 && max_len > 0 && H > 0 && T > 0, "vj_attn_fwd: empty problem");
  VJ_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
               "vj_attn_fwd: pointers must be 16-byte aligned");
  switch (HD) {
    case 32: return launch_attn_fwd<32>(qkv, out, lse2, cu_seqlens, nseq, max_len, H, T, scale, s);
    case 64: return launch_attn_fwd<64>(qkv, out, lse2, cu_seqlens, nseq, max_len, H, T, scale, s);
    case 128: return launch_attn_fwd<128>(qkv, out, lse2, cu_seqlens, nseq, max_len, H, T, scale, s);
    default: set_error("vj_attn_fwd: head dim %d unsupported (32/64/128; pad 24->32 in the weights)", HD); return -1;
  }
}
