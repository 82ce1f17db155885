// Dense (non-causal) variable-length flash attention forward on wgmma (sm_90a).
//
// Replaces F.scaled_dot_product_attention at src/models/utils/modules.py:66-69 (the `mask`
// argument there is ignored - "masked attention" is attention over the gathered token subset,
// so every sequence is dense and only its length varies).
//
// Layout: qkv T [T, 3*H*HD] (row = token, q|k|v packed, head-major inside each third - the
// layout the qkv GEMM epilogue writes), O T [T, H*HD], lse2 fp32 [H, T] (log2 domain:
// m*scale*log2e + log2(l)).  Sequences are row ranges [cu[s], cu[s+1]).  T = bf16 (vj_attn_fwd) or fp16 (vj_attn_fwd_f16,
// frozen evaluation under autocast(float16)); the schedule and the arithmetic are the same, P is packed to T.
//
// One CTA = one query tile of 64 * NWG rows of one (sequence, head); K_j / V_j tiles of 128 keys stream through a 3-stage
// TMA ring.  Warp-specialised, NWG + 1 warpgroups (the FlashAttention-3 schedule):
//   warpgroup 0   : TMA producer (one thread loads Q, then K_j / V_j into stage j % 3 once every active consumer released
//                   it; per-stage full (tx-count) and empty (one arrive per active consumer warp) mbarriers)
//   warpgroups 1..NWG: consumers, 64 query rows each.  S = Q K_j^T (wgmma, both operands in smem), online softmax on the
//                   accumulator fragment in registers, O += P V_j with P as the register A operand (no shared-memory round
//                   trip) and V_j read MN-major.  A consumer whose 64 rows all lie past the sequence's end exits at once.
// Two overlaps keep the tensor cores busy while the exps run:
//   - inside a warpgroup, S_j = Q K_j^T is issued together with O += P_{j-1} V_{j-1} (P_{j-1} held as bf16 fragments), so
//     the softmax of S_j runs under P_{j-1} V_{j-1}; O is rescaled by alpha_j once that MMA has retired;
//   - between the warpgroups, a ring of named barriers makes them take turns issuing (round robin), so one warpgroup's
//     softmax runs under the others' MMAs.
// More consumer warpgroups per CTA put more independent softmax chains on each warp scheduler and share each K / V tile
// among more query rows; NWG is chosen per head dim (fwd_nwg).
// Only the ragged last KV tile of a sequence pays for the key mask.
// The per-row arithmetic and its order over the KV tiles are those of a plain one-tile-at-a-time loop, so O and lse2 do
// not depend on the schedule.
#include <stdlib.h>

#include "attn_common.cuh"
#include "vjepa_b200.h"

namespace vj {

constexpr int kFwdKV = 128;   // keys per tile
constexpr int kFwdStages = 3;

struct AttnFwdParams {
  const int* cu_seqlens;
  void* out;
  float* lse2;
  int H, T;
  long long ld_out;
  float scale_log2;
};

// Consumer warpgroups per CTA, measured per head dim (DESIGN section 6); hd 128's accumulators only fit two.
template <int HD>
constexpr int fwd_nwg() { return HD == 128 ? 2 : 3; }

template <int HD, int NWG>
struct FwdCfg {
  using A = AttnCfg<HD>;
  using W = AttnWarps<NWG>;
  static constexpr int TILE = A::template tile_bytes<kFwdKV>();
  static constexpr int Q_TILE = A::template tile_bytes<W::ROWS>();
  static constexpr int Q_OFF = 0;
  static constexpr int K_OFF = Q_TILE;                        // kFwdStages stages
  static constexpr int V_OFF = K_OFF + kFwdStages * TILE;     // kFwdStages stages
  static constexpr int BAR_OFF = V_OFF + kFwdStages * TILE;   // Q, full[stages], empty[stages]
  static constexpr int SMEM_BYTES = BAR_OFF + 8 * (1 + 2 * kFwdStages) + 1024;
  static_assert(SMEM_BYTES <= 232448, "attention forward shared memory budget exceeded");
};

template <typename T, int HD, int NWG>
__global__ void __launch_bounds__(AttnWarps<NWG>::THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV, const AttnFwdParams p) {
  using F = FwdCfg<HD, NWG>;
  using W = AttnWarps<NWG>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  const int seq = blockIdx.y, head = blockIdx.z;
  const int row_begin = p.cu_seqlens[seq];
  const int len = p.cu_seqlens[seq + 1] - row_begin;
  const int q0 = blockIdx.x * W::ROWS;
  if (q0 >= len) return;
  const int n_wg = attn_active_wgs<NWG>(len, q0);
  const int n_kv = (len + kFwdKV - 1) / kFwdKV;

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + F::BAR_OFF);
  const uint32_t bar_q = smem_u32(bars + 0);
  const uint32_t full0 = smem_u32(bars + 1);                 // stage st: + 8 st
  const uint32_t empty0 = smem_u32(bars + 1 + kFwdStages);
  const uint32_t sQ = smem_u32(smem + F::Q_OFF), sK = smem_u32(smem + F::K_OFF), sV = smem_u32(smem + F::V_OFF);
  const int HHD = p.H * HD;
  const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);   // warp-uniform to the compiler: no divergent wgmma paths

  if (threadIdx.x == 0) {
    mbar_init(bar_q, 1);
    for (int st = 0; st < kFwdStages; ++st) {
      mbar_init(full0 + 8 * st, 1);
      mbar_init(empty0 + 8 * st, 4 * n_wg);   // one arrive per active consumer warp
    }
    fence_mbar_init();
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmKV);
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<W::PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      mbar_expect_tx(bar_q, F::Q_TILE);
      attn_load_tile<HD, W::ROWS>(sQ, &tmQ, bar_q, head * HD, row_begin + q0);
      for (int j = 0; j < n_kv; ++j) {
        const int st = j % kFwdStages;
        mbar_wait(empty0 + 8 * st, ((j / kFwdStages) & 1) ^ 1);
        const uint32_t fb = full0 + 8 * st;
        mbar_expect_tx(fb, 2 * F::TILE);
        attn_load_tile<HD, kFwdKV>(sK + st * F::TILE, &tmKV, fb, HHD + head * HD, row_begin + j * kFwdKV);
        attn_load_tile<HD, kFwdKV>(sV + st * F::TILE, &tmKV, fb, 2 * HHD + head * HD, row_begin + j * kFwdKV);
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers
  const int cw = wg - 1;   // which 64 rows of the query tile
  if (cw >= n_wg) return;
  setmaxnreg_inc<W::CONSUMER_REGS>();
  const int lane = threadIdx.x & 31;
  const int r = cw * 64 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);   // this thread's first row in the tile (+8: second)
  float o[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  float s[kFwdKV / 2];              // S_j, then P_j (fp32)
  uint32_t pf[kFwdKV / 16][4];      // P_{j-1} as T A fragments, read by the in-flight P_{j-1} V_{j-1}
  // Round robin among the n_wg active warpgroups: named barrier 1 + cw opens cw's turn to issue MMAs.
  auto wait_turn = [&]() {
    if (n_wg > 1) named_bar_sync(1 + cw, 256);
  };
  auto pass_turn = [&]() {
    if (n_wg > 1) named_bar_arrive(cw + 1 == n_wg ? 1 : 2 + cw, 256);
  };
  if (cw == n_wg - 1) pass_turn();   // warpgroup 0 issues first

  auto issue_s = [&](int st) {
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk)
      wgmma_ss<kFwdKV, 0, 0, T>(s, attn_kmajor_desc<HD, W::ROWS>(sQ, cw * 64, kk),
                             attn_kmajor_desc<HD, kFwdKV>(sK + st * F::TILE, 0, kk), kk > 0);
    wgmma_commit();
  };
  auto issue_pv = [&](int st) {
#pragma unroll
    for (int kk = 0; kk < kFwdKV / 16; ++kk) wgmma_rs<HD, 1, T>(o, pf[kk], attn_mnmajor_desc<HD, kFwdKV>(sV + st * F::TILE, kk), 1);
    wgmma_commit();
  };
  auto release = [&](int st) {
    __syncwarp();
    if (lane == 0) mbar_arrive(empty0 + 8 * st);
  };
  // ---- online softmax of tile j on the fragment: s[4c + 2h + e] = row r + 8h, key 8c + 2(lane % 4) + e
  auto softmax = [&](int j, float (&alpha)[2]) {
    const int valid = len - j * kFwdKV;
    if (valid < kFwdKV) {   // ragged last tile
#pragma unroll
      for (int c = 0; c < kFwdKV / 8; ++c)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (8 * c + 2 * (lane & 3) + (e & 1) >= valid) s[4 * c + e] = -INFINITY;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int c = 0; c < kFwdKV / 8; ++c)
#pragma unroll
        for (int e = 0; e < 2; ++e) mx = fmaxf(mx, s[4 * c + 2 * h + e]);
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
  };
  auto rescale_o = [&](const float (&alpha)[2]) {
#pragma unroll
    for (int c = 0; c < HD / 8; ++c) {
      o[4 * c + 0] *= alpha[0]; o[4 * c + 1] *= alpha[0];
      o[4 * c + 2] *= alpha[1]; o[4 * c + 3] *= alpha[1];
    }
  };
  auto pack_p = [&]() {
#pragma unroll
    for (int kk = 0; kk < kFwdKV / 16; ++kk) acc_to_afrag<T>(s, kk, pf[kk]);
  };

  mbar_wait(bar_q, 0);
  // tile 0: S_0 alone
  float alpha[2];
  wait_turn();
  mbar_wait(full0, 0);
  wgmma_fence();
  issue_s(0);
  pass_turn();
  wgmma_wait<0>();
  wgmma_fence_regs(s);
  softmax(0, alpha);
  rescale_o(alpha);
  pack_p();
  // tile j: S_j together with P_{j-1} V_{j-1}
  for (int j = 1; j < n_kv; ++j) {
    const int st = j % kFwdStages, st_prev = (j - 1) % kFwdStages;
    wait_turn();
    mbar_wait(full0 + 8 * st, (j / kFwdStages) & 1);
    wgmma_fence_regs(o);
    wgmma_fence();
    issue_s(st);
    issue_pv(st_prev);
    pass_turn();
    wgmma_wait<1>();   // S_j is ready, P_{j-1} V_{j-1} may still run
    wgmma_fence_regs(s);
    softmax(j, alpha);
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    wgmma_fence_regs(pf);
    release(st_prev);
    rescale_o(alpha);
    pack_p();
  }
  // last P V
  wait_turn();
  wgmma_fence_regs(o);
  wgmma_fence();
  issue_pv((n_kv - 1) % kFwdStages);
  pass_turn();
  wgmma_wait<0>();
  wgmma_fence_regs(o);
  wgmma_fence_regs(pf);
  if (cw == 0) wait_turn();   // takes the last warpgroup's last pass, so every turn barrier ends balanced

  // ---- epilogue: O / l -> T, lse2 (log2 domain)
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
  store_frag<HD>(o, 1.0f, reinterpret_cast<T*>(p.out) + (long long)(row_begin + q0) * p.ld_out + head * HD, p.ld_out, r,
                      len - q0);
}

template <typename T, int HD>
static int launch_attn_fwd(const void* qkv, void* out, float* lse2, const int* cu, int nseq, int max_len, int H, int T_,
                           float scale, cudaStream_t s) {
  constexpr int NWG = fwd_nwg<HD>();
  using C = AttnCfg<HD>;
  using F = FwdCfg<HD, NWG>;
  using W = AttnWarps<NWG>;
  const uint64_t width = (uint64_t)3 * H * HD;
  CUtensorMap tmq, tmkv;
  int rc = make_tmap_2d(&tmq, qkv, Elt<T>::kTmap, width, T_, width * 2, C::BOX_INNER, W::ROWS, C::TMAP_SWIZZLE);
  if (!rc) rc = make_tmap_2d(&tmkv, qkv, Elt<T>::kTmap, width, T_, width * 2, C::BOX_INNER, kFwdKV, C::TMAP_SWIZZLE);
  if (rc) return rc;
  auto kern = attn_fwd_kernel<T, HD, NWG>;
  static bool configured = false;
  if (!configured) {
    VJ_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, F::SMEM_BYTES));
    configured = true;
  }
  AttnFwdParams p;
  p.cu_seqlens = cu; p.out = out; p.lse2 = lse2;
  p.H = H; p.T = T_; p.ld_out = (long long)H * HD;
  p.scale_log2 = scale * 1.4426950408889634f;
  dim3 grid((max_len + W::ROWS - 1) / W::ROWS, nseq, H);
  kern<<<grid, W::THREADS, F::SMEM_BYTES, s>>>(tmq, tmkv, p);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

template <typename T>
static int attn_fwd_impl(const void* qkv, void* out, float* lse2, const int* cu_seqlens, int nseq, int max_len, int H,
                         int HD, int T_, float scale, cudaStream_t s) {
  VJ_CHECK_ARG(qkv && out && lse2 && cu_seqlens, "vj_attn_fwd: null pointer");
  VJ_CHECK_ARG(nseq > 0 && max_len > 0 && H > 0 && T_ > 0, "vj_attn_fwd: empty problem");
  VJ_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
               "vj_attn_fwd: pointers must be 16-byte aligned");
  switch (HD) {
    case 32: return launch_attn_fwd<T, 32>(qkv, out, lse2, cu_seqlens, nseq, max_len, H, T_, scale, s);
    case 64: return launch_attn_fwd<T, 64>(qkv, out, lse2, cu_seqlens, nseq, max_len, H, T_, scale, s);
    case 128: return launch_attn_fwd<T, 128>(qkv, out, lse2, cu_seqlens, nseq, max_len, H, T_, scale, s);
    default: set_error("vj_attn_fwd: head dim %d unsupported (32/64/128; pad 24->32 in the weights)", HD); return -1;
  }
}

}  // namespace vj

extern "C" int vj_attn_fwd(const void* qkv, void* out, float* lse2, const int* cu_seqlens, int nseq, int max_len,
                           int H, int HD, int T, float scale, void* stream) {
  return vj::attn_fwd_impl<__nv_bfloat16>(qkv, out, lse2, cu_seqlens, nseq, max_len, H, HD, T, scale,
                                          reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vj_attn_fwd_f16(const void* qkv, void* out, float* lse2, const int* cu_seqlens, int nseq, int max_len,
                               int H, int HD, int T, float scale, void* stream) {
  return vj::attn_fwd_impl<__half>(qkv, out, lse2, cu_seqlens, nseq, max_len, H, HD, T, scale,
                                   reinterpret_cast<cudaStream_t>(stream));
}
