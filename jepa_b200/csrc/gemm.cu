// wgmma GEMM for the V-JEPA hot path (sm_90a).
//
//   D[M,N] = epi( alpha * sum_k A[m,k] * B[n,k] )        bf16 operands, fp32 accumulation in registers
//
// One persistent CTA per SM, warp-specialised, 3 warpgroups:
//   warpgroup 0   : TMA producer   (one thread: cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier tx)
//   warpgroups 1-2: consumers      (each owns 64 of the 128 tile rows: wgmma.mma_async m64nBNk16 from the smem ring,
//                                   then bias / GELU / residual / dGELU straight from the accumulator registers to HBM)
// Operands may be K-major (reduction dim contiguous; nn.Linear forward) or MN-major (reduction dim strided; dgrad reads
// W[N_out,K_in] as B, wgrad reads dY and X transposed) - the smem descriptors and wgmma's transpose bits change, not the
// data in HBM, so no transposes are materialised.  Split-K / stream-K pieces reduce-add into fp32 D.
//
// Replaces the cuBLASLt calls behind nn.Linear on the reference path:
// src/models/utils/modules.py:31-34 (fc1/fc2), :63 (qkv), :76 (proj),
// src/models/predictor.py:194,237 (predictor_embed / predictor_proj),
// src/models/utils/patch_embed.py:54-57 (Conv3d as GEMM) and their autograd backward.

#include <stdlib.h>

#include "common.cuh"
#include "vjepa_b200.h"
#include "wgmma.cuh"

namespace vj {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int kGemmThreads = 384;
// Weight-gradient GEMMs (both operands MN-major) reduce over every token of the batch (K up to ~76k).  They accumulate
// kPromoteKB k-blocks at a time in a fresh register set and add that partial to the running sum with ordinary fp32 adds:
// the tensor core's own accumulation then only ever spans 256 products (its rounding over a full-length K gave rel-L2
// 2.2e-5 against fp64 at K = 76032, this keeps the sum at the plain fp32 summation-order level).
constexpr int kPromoteKB = 4;

struct GemmParams {
  int M, N, K;
  int tiles_m, tiles_n, split_k, kb_total, kb_per_split;
  int stream_k;             // 1: every CTA takes one contiguous range of `sk_chunk` k-blocks of the linearised (tile, k-block)
  long long sk_chunk;       //    space (perfect balance, no wave quantisation); partial tiles reduce-add like split-K ones
  const float* bias;
  int epi;
  const void* aux;
  long long ldaux;
  const int* aux_rowmap;
  int aux_period;
  void* aux_out;
  long long ldauxout;
  void* D;
  long long ldd;
  int reduce_add;
  float alpha;
};

template <int BN>
struct GemmCfg {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = BN == 256 ? 4 : (BN == 128 ? 6 : 8);
  static constexpr int BAR_OFF = STAGES * STAGE_BYTES;
  static constexpr int SMEM_BYTES = BAR_OFF + 2 * STAGES * 8 + 1024;  // +1024 align slack
  static_assert(SMEM_BYTES <= 232448, "GEMM shared memory budget exceeded");
};

// Work decomposition shared by the producer and the consumers.  Classic: work item w = blockIdx.x, blockIdx.x +
// gridDim.x, ... over tiles x split_k.  Stream-K: the CTA walks its contiguous k-block range, one (tile, k-range) piece
// at a time.
struct WorkCursor {
  long long cur, end;
};
VJ_DEVINL WorkCursor work_begin(const GemmParams& p) {
  WorkCursor c;
  if (p.stream_k) {
    const long long total_kb = (long long)p.tiles_m * p.tiles_n * p.kb_total;
    c.cur = (long long)blockIdx.x * p.sk_chunk;
    c.end = min(total_kb, c.cur + p.sk_chunk);
  } else {
    c.cur = blockIdx.x;
    c.end = (long long)p.tiles_m * p.tiles_n * p.split_k;
  }
  return c;
}
VJ_DEVINL bool work_next(const GemmParams& p, WorkCursor& c, int& t, int& kb0, int& kb1) {
  if (c.cur >= c.end) return false;
  if (p.stream_k) {
    t = int(c.cur / p.kb_total);
    kb0 = int(c.cur - (long long)t * p.kb_total);
    const long long take = min((long long)(p.kb_total - kb0), c.end - c.cur);
    kb1 = kb0 + int(take);
    c.cur += take;
  } else {
    const int tiles = p.tiles_m * p.tiles_n;
    const int split = int(c.cur / tiles);
    t = int(c.cur - (long long)split * tiles);
    kb0 = split * p.kb_per_split;
    kb1 = min(p.kb_total, kb0 + p.kb_per_split);
    c.cur += gridDim.x;
  }
  return true;
}

// erf via Abramowitz-Stegun 7.1.26 (|err| < 1.5e-7) - far below the bf16 rounding of the result.
VJ_DEVINL float erf_as(float x) {
  const float ax = fabsf(x);
  const float t = __fdividef(1.0f, fmaf(0.3275911f, ax, 1.0f));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  poly *= t;
  const float r = 1.0f - poly * __expf(-ax * ax);
  return copysignf(r, x);
}
// Exact-erf GELU and its derivative sharing one erf / exp evaluation:  g = x Phi(x),  d = Phi(x) + x pdf(x)
VJ_DEVINL float gelu_and_grad(float x, float& d) {
  const float cdf = 0.5f * (1.0f + erf_as(x * 0.70710678118654752f));
  const float pdf = 0.39894228040143268f * __expf(-0.5f * x * x);
  d = fmaf(x, pdf, cdf);
  return x * cdf;
}
VJ_DEVINL float gelu_grad_fast(float x) {
  float d;
  gelu_and_grad(x, d);
  return d;
}

// EPI is a compile-time epilogue kind so that e.g. the plain / GELU kernels carry none of the aux code.
template <int BN, bool A_MN, bool B_MN, bool OUT_F32, int EPI, bool AUX32>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  constexpr bool kUsesAux = (EPI == VJ_EPI_ADD || EPI == VJ_EPI_DGELU || EPI == VJ_EPI_MUL);
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::BAR_OFF);
  const uint32_t full0 = smem_u32(bars);
  const uint32_t empty0 = smem_u32(bars + STAGES);
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, 8);   // one arrive per consumer warp
    }
    fence_mbar_init();
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      WorkCursor wc = work_begin(p);
      int t, kb0, kb1;
      while (work_next(p, wc, t, kb0, kb1)) {
        const int m0 = (t / p.tiles_n) * BM;
        const int n0 = (t % p.tiles_n) * BN;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(empty0 + 8 * stage, phase ^ 1);
          const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES);
          const uint32_t sb = sa + Cfg::A_BYTES;
          const uint32_t fb = full0 + 8 * stage;
          mbar_expect_tx(fb, Cfg::STAGE_BYTES);
          const int k0 = kb * BK;
          if (!A_MN) {
            tma_load_2d(sa, &tmA, fb, k0, m0);
          } else {
#pragma unroll
            for (int j = 0; j < BM / 64; ++j) tma_load_2d(sa + j * 8192, &tmA, fb, m0 + 64 * j, k0);
          }
          if (!B_MN) {
            tma_load_2d(sb, &tmB, fb, k0, n0);
          } else {
#pragma unroll
            for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * 8192, &tmB, fb, n0 + 64 * j, k0);
          }
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers
  setmaxnreg_inc<232>();
  const int cw = wg - 1;                    // which 64-row half of the tile
  const int warp_in_wg = (threadIdx.x >> 5) & 3;
  const int lane = threadIdx.x & 31;
  constexpr bool kPromote = A_MN && B_MN;
  static_assert(!kPromote || BN <= 128, "promoted accumulation needs two accumulator sets in registers");
  int stage = 0;
  uint32_t phase = 0;
  float acc[BN / 2];
  float part[kPromote ? BN / 2 : 1];
  WorkCursor wc = work_begin(p);
  int t, kb0, kb1;
  while (work_next(p, wc, t, kb0, kb1)) {
    const int m0 = (t / p.tiles_n) * BM;
    const int n0 = (t % p.tiles_n) * BN;
    if constexpr (kPromote) {
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    }
    int prev = -1;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(full0 + 8 * stage, phase);
      const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES) + cw * 8192;   // this warpgroup's 64 rows
      const uint32_t sb = smem_u32(smem + stage * Cfg::STAGE_BYTES) + Cfg::A_BYTES;
      const uint64_t da0 = A_MN ? make_smem_desc(sa, 8192, 1024, 1) : make_smem_desc(sa, 16, 1024, 1);
      const uint64_t db0 = B_MN ? make_smem_desc(sb, 8192, 1024, 1) : make_smem_desc(sb, 16, 1024, 1);
      if constexpr (kPromote) {
        const bool group_first = (kb - kb0) % kPromoteKB == 0;
        const bool group_last = (kb - kb0) % kPromoteKB == kPromoteKB - 1 || kb + 1 == kb1;
        wgmma_fence_regs(part);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < BK / 16; ++kk)
          wgmma_ss<BN, 1, 1>(part, da0 + ((kk * 2048) >> 4), db0 + ((kk * 2048) >> 4), (!group_first || kk > 0) ? 1 : 0);
        wgmma_commit();
        if (group_last) {
          wgmma_wait<0>();
          wgmma_fence_regs(part);
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
        } else {
          wgmma_wait<1>();
        }
      } else {
        wgmma_fence_regs(acc);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < BK / 16; ++kk) {
          const uint32_t koa = A_MN ? kk * 2048 : kk * 32, kob = B_MN ? kk * 2048 : kk * 32;
          wgmma_ss<BN, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da0 + (koa >> 4), db0 + (kob >> 4), (kb > kb0 || kk > 0) ? 1 : 0);
        }
        wgmma_commit();
        wgmma_wait<1>();   // the previous k-block's MMAs have retired: its stage may be refilled
        wgmma_fence_regs(acc);
      }
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(empty0 + 8 * prev);
      }
      prev = stage;
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(empty0 + 8 * prev);

    // ---- epilogue straight from the accumulator fragment: thread holds rows r0 and r0 + 8, column pairs 8j + 2(lane%4)
    const bool add_bias = p.bias != nullptr && kb0 == 0;   // the bias joins the piece holding the tile's first k-block
    const int r0 = m0 + cw * 64 + warp_in_wg * 16 + (lane >> 2);
    const int cq = n0 + 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r0 + 8 * h;
      if (row >= p.M) continue;
      long long arow = row;
      if (kUsesAux && AUX32) {
        if (p.aux_rowmap != nullptr) arow = p.aux_rowmap[row];
        else if (p.aux_period > 0) arow = row % p.aux_period;
      }
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = cq + 8 * j;
        float v0 = acc[4 * j + 2 * h] * p.alpha, v1 = acc[4 * j + 2 * h + 1] * p.alpha;
        if (add_bias) {
          const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
          v0 += b.x;
          v1 += b.y;
        }
        if (kUsesAux) {
          float x0, x1;
          if (AUX32) {
            const float2 x = __ldg(reinterpret_cast<const float2*>(reinterpret_cast<const float*>(p.aux) + arow * p.ldaux + col));
            x0 = x.x; x1 = x.y;
          } else {
            const uint32_t x = __ldg(reinterpret_cast<const unsigned int*>(reinterpret_cast<const __nv_bfloat16*>(p.aux) +
                                                                             arow * p.ldaux + col));
            x0 = bf16_lo(x); x1 = bf16_hi(x);
          }
          if (EPI == VJ_EPI_ADD) { v0 += x0; v1 += x1; }
          else if (EPI == VJ_EPI_MUL) { v0 *= x0; v1 *= x1; }
          else { v0 *= gelu_grad_fast(x0); v1 *= gelu_grad_fast(x1); }
        }
        if (EPI == VJ_EPI_GELU || EPI == VJ_EPI_GELU_GRAD) {
          //   VJ_EPI_GELU      : aux_out = pre-activation
          //   VJ_EPI_GELU_GRAD : aux_out = gelu'(pre) (the backward's epilogue is then a plain multiply)
          float d0, d1;
          const float g0 = gelu_and_grad(v0, d0), g1 = gelu_and_grad(v1, d1);
          if (p.aux_out != nullptr) {
            const uint32_t o = EPI == VJ_EPI_GELU ? pack_bf16x2(v0, v1) : pack_bf16x2(d0, d1);
            *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(p.aux_out) + (long long)row * p.ldauxout + col) = o;
          }
          v0 = g0;
          v1 = g1;
        }
        if (OUT_F32) {
          float2* dst = reinterpret_cast<float2*>(reinterpret_cast<float*>(p.D) + (long long)row * p.ldd + col);
          if (p.reduce_add) atomicAdd(dst, make_float2(v0, v1));
          else *dst = make_float2(v0, v1);
        } else {
          *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(p.D) + (long long)row * p.ldd + col) =
              pack_bf16x2(v0, v1);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
template <int BN, bool A_MN, bool B_MN, bool OUT_F32, int EPI, bool AUX32 = false>
static int launch_gemm(const CUtensorMap& tA, const CUtensorMap& tB, const GemmParams& p, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  auto kern = gemm_kernel<BN, A_MN, B_MN, OUT_F32, EPI, AUX32>;
  static bool configured = false;  // per instantiation
  if (!configured) {
    VJ_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    configured = true;
  }
  const int total = p.tiles_m * p.tiles_n * p.split_k;
  int grid = total < sm_budget() ? total : sm_budget();
  if (p.stream_k) {
    const long long total_kb = (long long)p.tiles_m * p.tiles_n * p.kb_total;
    grid = int((total_kb + p.sk_chunk - 1) / p.sk_chunk);
  }
  kern<<<grid, kGemmThreads, Cfg::SMEM_BYTES, stream>>>(tA, tB, p);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

template <int BN>
static int dispatch_major(int a_mn, int b_mn, int out_f32, int epi, int aux_f32, const CUtensorMap& tA,
                          const CUtensorMap& tB, const GemmParams& p, cudaStream_t s) {
  // instantiated combinations = what the V-JEPA step needs (forward Linear: K/K; dgrad: K/MN; wgrad: MN/MN fp32)
  if (!a_mn && !b_mn) {
    if (epi == VJ_EPI_NONE) return out_f32 ? launch_gemm<BN, false, false, true, VJ_EPI_NONE>(tA, tB, p, s)
                                           : launch_gemm<BN, false, false, false, VJ_EPI_NONE>(tA, tB, p, s);
    if (epi == VJ_EPI_ADD) {
      if (aux_f32) return out_f32 ? launch_gemm<BN, false, false, true, VJ_EPI_ADD, true>(tA, tB, p, s)
                                  : launch_gemm<BN, false, false, false, VJ_EPI_ADD, true>(tA, tB, p, s);
      if (!out_f32) return launch_gemm<BN, false, false, false, VJ_EPI_ADD, false>(tA, tB, p, s);
    }
    if (epi == VJ_EPI_GELU && !out_f32) return launch_gemm<BN, false, false, false, VJ_EPI_GELU>(tA, tB, p, s);
    if (epi == VJ_EPI_GELU_GRAD && !out_f32) return launch_gemm<BN, false, false, false, VJ_EPI_GELU_GRAD>(tA, tB, p, s);
    if (epi == VJ_EPI_DGELU && !out_f32 && !aux_f32) return launch_gemm<BN, false, false, false, VJ_EPI_DGELU>(tA, tB, p, s);
  } else if (!a_mn && b_mn) {
    if (epi == VJ_EPI_NONE) return out_f32 ? launch_gemm<BN, false, true, true, VJ_EPI_NONE>(tA, tB, p, s)
                                           : launch_gemm<BN, false, true, false, VJ_EPI_NONE>(tA, tB, p, s);
    if (epi == VJ_EPI_DGELU && !out_f32 && !aux_f32) return launch_gemm<BN, false, true, false, VJ_EPI_DGELU>(tA, tB, p, s);
    if (epi == VJ_EPI_MUL && !out_f32 && !aux_f32) return launch_gemm<BN, false, true, false, VJ_EPI_MUL>(tA, tB, p, s);
  } else if (a_mn && b_mn) {
    if constexpr (BN <= 128) {
      if (epi == VJ_EPI_NONE) return out_f32 ? launch_gemm<BN, true, true, true, VJ_EPI_NONE>(tA, tB, p, s)
                                             : launch_gemm<BN, true, true, false, VJ_EPI_NONE>(tA, tB, p, s);
    }
  }
  set_error("vj_gemm: combination a_mn=%d b_mn=%d d_f32=%d epi=%d is not instantiated", a_mn, b_mn, out_f32, epi);
  return -1;
}

}  // namespace vj

extern "C" int vj_gemm(const void* A, long long lda, int a_mn, const void* B, long long ldb,
                       int b_mn, void* D, long long ldd, int d_f32, int M, int N, int K,
                       const float* bias, float alpha, int epi, const void* aux, long long ldaux,
                       int aux_f32, const int* aux_rowmap, int aux_period, void* aux_out,
                       long long ldauxout, int split_k, int accumulate, void* stream_) {
  using namespace vj;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(A && B && D, "vj_gemm: null operand");
  VJ_CHECK_ARG(M > 0 && N > 0 && K > 0, "vj_gemm: empty problem M=%d N=%d K=%d", M, N, K);
  VJ_CHECK_ARG(N % 64 == 0, "vj_gemm: N=%d must be a multiple of 64", N);
  // TMA needs 16-byte row strides; the reduction extent itself is free (tails are zero-filled by TMA): for MN-major
  // operands (wgrad: K = token count) K is the OUTER dimension and may be any positive number.
  VJ_CHECK_ARG(lda % 8 == 0 && ldb % 8 == 0, "vj_gemm: lda/ldb must be multiples of 8 elements (16-byte rows)");
  VJ_CHECK_ARG(ldd % (d_f32 ? 4 : 8) == 0, "vj_gemm: ldd misaligned");
  VJ_CHECK_ARG((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(D) & 15) == 0,
               "vj_gemm: operands must be 16-byte aligned");
  VJ_CHECK_ARG(epi >= VJ_EPI_NONE && epi <= VJ_EPI_GELU_GRAD, "vj_gemm: bad epilogue %d", epi);
  VJ_CHECK_ARG(!(accumulate || split_k > 1 || split_k < 0) || d_f32, "vj_gemm: accumulate/split-K needs fp32 D");
  VJ_CHECK_ARG(split_k >= 0 || (epi == VJ_EPI_NONE && accumulate), "vj_gemm: stream-K (split_k < 0) is for accumulating fp32 GEMMs");
  if (epi == VJ_EPI_ADD || epi == VJ_EPI_DGELU || epi == VJ_EPI_MUL) {
    VJ_CHECK_ARG(aux != nullptr, "vj_gemm: epilogue %d needs aux", epi);
    VJ_CHECK_ARG((reinterpret_cast<uintptr_t>(aux) & 15) == 0 && ldaux % (aux_f32 ? 4 : 8) == 0,
                 "vj_gemm: aux misaligned");
  }
  if (a_mn) VJ_CHECK_ARG(M % 8 == 0, "vj_gemm: MN-major A needs M %% 8 == 0");

  // (weight gradients hold two accumulator sets, see kPromoteKB: at most 128 columns per tile)
  const int BN = (N % 256 == 0 && !(a_mn && b_mn)) ? 256 : (N % 128 == 0 ? 128 : 64);
  GemmParams p;
  p.M = M; p.N = N; p.K = K;
  p.tiles_m = (M + BM - 1) / BM;
  p.tiles_n = N / BN;
  p.kb_total = (K + BK - 1) / BK;
  // split_k < 0: stream-K - the linearised (tile, k-block) space is cut into one equal contiguous range per SM, so no SM
  // idles in a ragged last wave (the weight-gradient GEMMs have 32..128 output tiles for 132 SMs); every piece reduce-adds
  p.stream_k = 0;
  p.sk_chunk = 0;
  if (split_k < 0) {
    const long long total_kb = (long long)p.tiles_m * p.tiles_n * p.kb_total;
    const long long ctas = total_kb < sm_budget() ? total_kb : sm_budget();
    p.stream_k = 1;
    p.sk_chunk = (total_kb + ctas - 1) / ctas;
    split_k = 1;
  }
  if (split_k < 1) split_k = 1;
  if (split_k > p.kb_total) split_k = p.kb_total;
  p.kb_per_split = (p.kb_total + split_k - 1) / split_k;
  p.split_k = (p.kb_total + p.kb_per_split - 1) / p.kb_per_split;
  p.bias = bias;
  p.epi = epi;
  p.aux = aux; p.ldaux = ldaux; p.aux_rowmap = aux_rowmap; p.aux_period = aux_period;
  p.aux_out = (epi == VJ_EPI_GELU || epi == VJ_EPI_GELU_GRAD) ? aux_out : nullptr;
  p.ldauxout = ldauxout;
  p.D = D; p.ldd = ldd;
  p.reduce_add = (accumulate || p.split_k > 1 || p.stream_k) ? 1 : 0;
  p.alpha = alpha;

  if (p.aux_out != nullptr)
    VJ_CHECK_ARG((reinterpret_cast<uintptr_t>(aux_out) & 3) == 0 && ldauxout % 2 == 0, "vj_gemm: aux_out misaligned");
  if ((epi == VJ_EPI_ADD || epi == VJ_EPI_DGELU || epi == VJ_EPI_MUL) && !aux_f32) {
    VJ_CHECK_ARG(aux_rowmap == nullptr && aux_period == 0, "vj_gemm: row-mapped / periodic aux must be fp32");
    VJ_CHECK_ARG(p.split_k == 1, "vj_gemm: aux epilogues do not combine with split-K");
  }
  CUtensorMap tA, tB;
  int rc;
  if (!a_mn) rc = make_tmap_2d(&tA, A, 0, K, M, lda * 2, 64, 128, 3);
  else       rc = make_tmap_2d(&tA, A, 0, M, K, lda * 2, 64, 64, 3);
  if (rc) return rc;
  if (!b_mn) rc = make_tmap_2d(&tB, B, 0, K, N, ldb * 2, 64, BN, 3);
  else       rc = make_tmap_2d(&tB, B, 0, N, K, ldb * 2, 64, 64, 3);
  if (rc) return rc;
  switch (BN) {
    case 256: return dispatch_major<256>(a_mn, b_mn, d_f32, epi, aux_f32, tA, tB, p, stream);
    case 128: return dispatch_major<128>(a_mn, b_mn, d_f32, epi, aux_f32, tA, tB, p, stream);
    default:  return dispatch_major<64>(a_mn, b_mn, d_f32, epi, aux_f32, tA, tB, p, stream);
  }
}
