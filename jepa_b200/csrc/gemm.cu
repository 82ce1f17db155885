// wgmma GEMM for the V-JEPA hot path (sm_90a).
//
//   D[M,N] = epi( alpha * sum_k A[m,k] * B[n,k] )        bf16 or fp16 operands, fp32 accumulation in registers
//
// The element type T of the operands and of every 16-bit D / aux / aux_out is a template parameter: bf16 for
// pre-training and bf16 evaluation (vj_gemm), fp16 for frozen evaluation under autocast(float16) (vj_gemm_f16, the
// reference's eval loops).  Only the combinations that evaluation runs are instantiated in fp16.
//
// One persistent CTA per SM, warp-specialised, 3 warpgroups, two schedules:
//
//   gemm_kernel (forward and dgrad: A K-major, B K-major or MN-major) - ping-pong
//     warpgroup 0   : TMA producers (thread 0: A/B k-blocks into a 128B-swizzled smem ring;
//                                    thread 32: the bf16 residual / gelu' tile of the epilogue into its warpgroup's staging)
//     warpgroups 1-2: consumers, each owning whole 128 x BN output tiles, alternating tile by tile.  Two named barriers
//                     hand the tensor cores from one warpgroup to the other, so while one runs the main loop of tile
//                     i+1 the other runs the epilogue of tile i: accumulator (+ staged aux) -> bf16 into swizzled smem
//                     -> TMA store.  fp32 D (split-K / accumulate) and fp32 aux are written / read directly.
//                     Long K (kCoopMinKB, N % 256 == 0): COOP - both warpgroups share a 128 x 256 tile, 64 rows each,
//                     same producers and staged epilogue.
//
//   gemm_wgrad_kernel (weight gradients: both operands MN-major) - cooperative
//     warpgroups 1-2 each own 64 of the 128 tile rows.  These GEMMs hold two accumulator sets (kPromoteKB), reduce over
//     every token and reduce-add fp32 pieces; their epilogue is a few percent of their time.
//
// Operands may be K-major (reduction dim contiguous; nn.Linear forward) or MN-major (reduction dim strided; dgrad reads
// W[N_out,K_in] as B, wgrad reads dY and X transposed) - the smem descriptors and wgmma's transpose bits change, not the
// data in HBM, so no transposes are materialised.  Split-K / stream-K pieces reduce-add into fp32 D.
//
// Replaces the cuBLASLt calls behind nn.Linear on the reference path:
// src/models/utils/modules.py:31-34 (fc1/fc2), :63 (qkv), :76 (proj),
// src/models/predictor.py:194,237 (predictor_embed / predictor_proj),
// src/models/utils/patch_embed.py:54-57 (Conv3d as GEMM) and their autograd backward.

#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "vjepa_b200.h"
#include "wgmma.cuh"

#include <type_traits>

namespace vj {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int kGemmThreads = 384;
constexpr int kSmemBudget = 232448;   // 227 KB of opt-in shared memory per block
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

// Cooperative (weight-gradient) kernel: the ring only.
template <int BN>
struct GemmCfg {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = BN == 128 ? 6 : 8;
  static constexpr int BAR_OFF = STAGES * STAGE_BYTES;
  static constexpr int SMEM_BYTES = BAR_OFF + 2 * STAGES * 8 + 1024;  // +1024 align slack
  static_assert(SMEM_BYTES <= kSmemBudget, "GEMM shared memory budget exceeded");
};

// Forward / dgrad kernel: the ring, then one bf16 staging tile per consumer warpgroup (bf16 D only: its 128 x BN tile
// in ping-pong, its 64 x 256 half of the tile in the cooperative long-K schedule), then the barriers.  The staging tile
// holds the TMA-loaded aux on the way in and the result on the way out, as BN / 64 column blocks of ROWS rows x 128 B,
// 128B-swizzled like the TMA boxes.  The ring takes what is left: 5 stages of 32 KB at BN = 128 with staging (7
// without), 8 stages of 24 KB at BN = 64, 3 stages of 48 KB for the cooperative 128 x 256 tile (4 without staging).
template <int BN, bool STAGED, bool COOP>
struct PingCfg {
  static constexpr int ROWS = COOP ? 64 : BM;          // output rows per consumer warpgroup
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STG_BYTES = STAGED ? ROWS * BN * 2 : 0;
  static constexpr int BAR_BYTES = 256;
  static constexpr int FIT = (kSmemBudget - 1024 - BAR_BYTES - 2 * STG_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = FIT < 8 ? FIT : 8;
  static constexpr int STG_OFF = STAGES * STAGE_BYTES;
  static constexpr int BAR_OFF = STG_OFF + 2 * STG_BYTES;
  static constexpr int SMEM_BYTES = BAR_OFF + BAR_BYTES + 1024;   // +1024 align slack
  static_assert(STAGES >= 3, "GEMM ring too shallow");
  static_assert((2 * STAGES + 4) * 8 <= BAR_BYTES, "GEMM barrier block overflow");
  static_assert(SMEM_BYTES <= kSmemBudget, "GEMM shared memory budget exceeded");
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
// residual add / multiply / dGELU with the aux operand x
template <int EPI>
VJ_DEVINL void apply_aux(float& v0, float& v1, float x0, float x1) {
  if (EPI == VJ_EPI_ADD) { v0 += x0; v1 += x1; }
  else if (EPI == VJ_EPI_MUL) { v0 *= x0; v1 *= x1; }
  else { v0 *= gelu_grad_fast(x0); v1 *= gelu_grad_fast(x1); }
}
// row of the fp32 aux operand for output row `row` (row-mapped: patch embedding's positional table; periodic)
VJ_DEVINL int aux32_row(const GemmParams& p, int row) {
  if (row >= p.M) return 0;
  if (p.aux_rowmap != nullptr) return p.aux_rowmap[row];
  if (p.aux_period > 0) return row % p.aux_period;
  return row;
}

// Direct-from-register epilogue for fp32 D (plain store, or reduce-add for split-K / stream-K / accumulate) and for the
// cooperative weight-gradient kernel's bf16 D.  `acc` is one m64nBN fragment whose rows start at r0: the thread holds
// rows r0 + lane/4 and r0 + lane/4 + 8, column pairs n0 + 8j + 2(lane%4).
template <typename T, int BN, bool OUT_F32, int EPI, bool AUX32>
VJ_DEVINL void epilogue_direct(const GemmParams& p, const float (&acc)[BN / 2], int r0, int n0, bool add_bias, int lane) {
  constexpr bool kUsesAux = (EPI == VJ_EPI_ADD || EPI == VJ_EPI_DGELU || EPI == VJ_EPI_MUL);
  static_assert(!kUsesAux || AUX32, "bf16 aux goes through the staged epilogue");
  const int cq = n0 + 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = r0 + (lane >> 2) + 8 * h;
    if (row >= p.M) continue;
    const long long arow = kUsesAux ? aux32_row(p, row) : 0;
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
        const float2 x = __ldg(reinterpret_cast<const float2*>(reinterpret_cast<const float*>(p.aux) + arow * p.ldaux + col));
        apply_aux<EPI>(v0, v1, x.x, x.y);
      }
      if (OUT_F32) {
        float2* dst = reinterpret_cast<float2*>(reinterpret_cast<float*>(p.D) + (long long)row * p.ldd + col);
        if (p.reduce_add) atomicAdd(dst, make_float2(v0, v1));
        else *dst = make_float2(v0, v1);
      } else {
        *reinterpret_cast<uint32_t*>(reinterpret_cast<T*>(p.D) + (long long)row * p.ldd + col) = Elt<T>::pack(v0, v1);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// forward / dgrad kernel: ping-pong (COOP = false) or, for long K, cooperative on a 128 x 256 tile (COOP = true)
// ---------------------------------------------------------------------------------------------
// EPI is a compile-time epilogue kind so that e.g. the plain / GELU kernels carry none of the aux code.
template <typename T, int BN, bool COOP, bool B_MN, bool OUT_F32, int EPI, bool AUX32>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
            const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmAux,
            const __grid_constant__ CUtensorMap tmAuxOut, const GemmParams p) {
  constexpr bool kUsesAux = (EPI == VJ_EPI_ADD || EPI == VJ_EPI_DGELU || EPI == VJ_EPI_MUL);
  constexpr bool kStaged = !OUT_F32;                  // bf16 D leaves through smem staging and TMA stores
  constexpr bool kAuxTma = kUsesAux && !AUX32;         // bf16 aux arrives in the staging tile by TMA
  constexpr bool kGelu = (EPI == VJ_EPI_GELU || EPI == VJ_EPI_GELU_GRAD);
  static_assert(kStaged || !kAuxTma, "bf16 aux needs the staged epilogue");
  static_assert(kStaged || !kGelu, "GELU epilogues write bf16");
  using Cfg = PingCfg<BN, kStaged, COOP>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int ROWS = Cfg::ROWS;
  constexpr int HALVES = ROWS / 64;                     // m64 accumulator fragments per warpgroup
  constexpr int kBlk = ROWS * 128;                      // one 64-column block of a staging tile
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::BAR_OFF);
  const uint32_t full0 = smem_u32(bars);
  const uint32_t empty0 = smem_u32(bars + STAGES);
  const uint32_t auxfull0 = smem_u32(bars + 2 * STAGES);       // per consumer warpgroup: aux tile landed
  const uint32_t auxempty0 = smem_u32(bars + 2 * STAGES + 2);  //                         staging free for the next aux
  const uint32_t stg0 = smem_u32(smem + Cfg::STG_OFF);
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, COOP ? 8 : 4);   // one arrive per warp of the consuming warpgroup(s)
    }
    for (int c = 0; c < 2; ++c) {
      mbar_init(auxfull0 + 8 * c, 1);
      mbar_init(auxempty0 + 8 * c, 1);
    }
    fence_mbar_init();
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (kStaged) tma_prefetch_desc(&tmD);
    if (kAuxTma) tma_prefetch_desc(&tmAux);
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    WorkCursor wc = work_begin(p);
    int t, kb0, kb1;
    if (threadIdx.x == 0) {
      // ---------------------------------------------------------------- A/B ring, every work item in order
      int stage = 0;
      uint32_t phase = 0;
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
          tma_load_2d(sa, &tmA, fb, k0, m0);
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
    } else if (kAuxTma && threadIdx.x == 32) {
      // ---------------------------------------------------------------- aux tiles: ping-pong item i goes to
      // warpgroup i % 2, a cooperative item's two row halves to both; each as soon as the warpgroup's previous
      // epilogue has released its staging tile
      for (int i = 0; work_next(p, wc, t, kb0, kb1); ++i) {
        const int m0 = (t / p.tiles_n) * BM;
        const int n0 = (t % p.tiles_n) * BN;
#pragma unroll
        for (int h = 0; h < (COOP ? 2 : 1); ++h) {
          const int c = COOP ? h : (i & 1);
          const uint32_t n = uint32_t(COOP ? i : (i >> 1));
          mbar_wait(auxempty0 + 8 * c, (n & 1) ^ 1);
          mbar_expect_tx(auxfull0 + 8 * c, Cfg::STG_BYTES);
#pragma unroll
          for (int j = 0; j < BN / 64; ++j)
            tma_load_2d(stg0 + c * Cfg::STG_BYTES + j * kBlk, &tmAux, auxfull0 + 8 * c, n0 + 64 * j, m0 + ROWS * c * COOP);
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers
  setmaxnreg_inc<232>();
  const int cw = wg - 1;
  const int warp_in_wg = (threadIdx.x >> 5) & 3;
  const int lane = threadIdx.x & 31;
  const bool elected = (threadIdx.x & 127) == 0;
  const uint32_t stg = stg0 + cw * Cfg::STG_BYTES;
  float acc[HALVES][BN / 2];             // ping-pong: rows 0-63 and 64-127 of the tile; cooperative: this warpgroup's 64
  uint32_t ring_pos = 0;                 // k-blocks of all work items so far, this warpgroup's or not
  uint32_t own = 0;                      // this warpgroup's tiles so far
  WorkCursor wc = work_begin(p);
  int t, kb0, kb1;
  for (int i = 0; work_next(p, wc, t, kb0, kb1); ++i) {
    if (!COOP && (i & 1) != cw) {
      ring_pos += kb1 - kb0;
      continue;
    }
    WorkCursor peek = wc;
    int t2, a2, b2;
    const bool has_next = !COOP && work_next(p, peek, t2, a2, b2);
    const int m0 = (t / p.tiles_n) * BM;
    const int n0 = (t % p.tiles_n) * BN;
    const int mw = m0 + (COOP ? 64 * cw : 0);   // first row of this warpgroup's part of the tile

    // ---- main loop, once the other warpgroup has issued its whole tile (ping-pong)
    if (!COOP && i > 0) named_bar_sync(1 + cw, 256);
    int stage = int(ring_pos % STAGES);
    uint32_t phase = (ring_pos / STAGES) & 1;
    int prev = -1;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(full0 + 8 * stage, phase);
      const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES);
      const uint32_t sb = sa + Cfg::A_BYTES;
      const uint64_t da = make_smem_desc(sa + (COOP ? 8192 * cw : 0), 16, 1024, 1);
      const uint64_t db = B_MN ? make_smem_desc(sb, 8192, 1024, 1) : make_smem_desc(sb, 16, 1024, 1);
#pragma unroll
      for (int hh = 0; hh < HALVES; ++hh) wgmma_fence_regs(acc[hh]);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BK / 16; ++kk) {
        const uint32_t kob = B_MN ? kk * 2048 : kk * 32;
        const int scale_d = (kb > kb0 || kk > 0) ? 1 : 0;
#pragma unroll
        for (int hh = 0; hh < HALVES; ++hh)
          wgmma_ss<BN, 0, B_MN ? 1 : 0, T>(acc[hh], da + ((8192 * hh + kk * 32) >> 4), db + (kob >> 4), scale_d);
      }
      wgmma_commit();
      wgmma_wait<1>();   // the previous k-block's MMAs have retired: its stage may be refilled
#pragma unroll
      for (int hh = 0; hh < HALVES; ++hh) wgmma_fence_regs(acc[hh]);
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
    ring_pos += kb1 - kb0;
    if (has_next) named_bar_arrive(1 + (cw ^ 1), 256);   // the tensor cores go to the other warpgroup's next tile
    wgmma_wait<0>();
#pragma unroll
    for (int hh = 0; hh < HALVES; ++hh) wgmma_fence_regs(acc[hh]);
    __syncwarp();
    if (lane == 0) mbar_arrive(empty0 + 8 * prev);

    const bool add_bias = p.bias != nullptr && kb0 == 0;   // the bias joins the piece holding the tile's first k-block
    if constexpr (!kStaged) {
#pragma unroll
      for (int hh = 0; hh < HALVES; ++hh)
        epilogue_direct<T, BN, OUT_F32, EPI, AUX32>(p, acc[hh], mw + 64 * hh + 16 * warp_in_wg, n0, add_bias, lane);
    } else {
      // ---- staged epilogue.  Thread holds rows 16 w + lane/4 (+8, +64, +72) and column pairs 8j + 2(lane%4); under
      // the 128B swizzle the 16-byte chunk j%8 of row r sits at chunk (j%8) ^ (r%8), and r%8 = lane/4 for all four
      // rows - each warp-wide 4-byte access touches 32 distinct banks.
      const int rq = lane >> 2;
      const uint32_t thr = stg + (16 * warp_in_wg + rq) * 128 + 4 * (lane & 3);
      // Staging is free to write: the last TMA store from it was waited for before this warpgroup's turn barrier
      // (ping-pong) or the barrier below (cooperative), or - with a TMA aux - before the staging was released to the
      // aux loader.
      if (kAuxTma) mbar_wait(auxfull0 + 8 * cw, own & 1);
      else if (COOP) named_bar_sync(3 + cw, 128);
      // GELU with aux_out: pass 1 stages aux_out and keeps the activation in acc, pass 2 stages the activation
      const bool two_pass = kGelu && p.aux_out != nullptr;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = n0 + 8 * j + 2 * (lane & 3);
        float2 b = make_float2(0.f, 0.f);
        if (add_bias) b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
        const uint32_t cj = thr + (j >> 3) * kBlk + (((j & 7) ^ rq) << 4);
#pragma unroll
        for (int hh = 0; hh < HALVES; ++hh)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint32_t addr = cj + (64 * hh + 8 * h) * 128;
            float& a0 = acc[hh][4 * j + 2 * h];
            float& a1 = acc[hh][4 * j + 2 * h + 1];
            float v0 = a0 * p.alpha, v1 = a1 * p.alpha;
            if (add_bias) {
              v0 += b.x;
              v1 += b.y;
            }
            if (kAuxTma) {
              uint32_t x;
              asm volatile("ld.shared.b32 %0, [%1];" : "=r"(x) : "r"(addr) : "memory");
              apply_aux<EPI>(v0, v1, Elt<T>::lo(x), Elt<T>::hi(x));
            } else if (kUsesAux) {
              // (fp32 aux: the patch embedding's positional table, once per encoder forward; the row lookup is
              //  repeated per column pair rather than held in registers across the loop)
              const long long arow = aux32_row(p, mw + 64 * hh + 16 * warp_in_wg + rq + 8 * h);
              const float2 x = __ldg(reinterpret_cast<const float2*>(reinterpret_cast<const float*>(p.aux) +
                                                                      arow * p.ldaux + col));
              apply_aux<EPI>(v0, v1, x.x, x.y);
            }
            uint32_t o;
            if (kGelu) {
              //   VJ_EPI_GELU      : aux_out = pre-activation
              //   VJ_EPI_GELU_GRAD : aux_out = gelu'(pre) (the backward's epilogue is then a plain multiply)
              float d0, d1;
              const float g0 = gelu_and_grad(v0, d0), g1 = gelu_and_grad(v1, d1);
              o = EPI == VJ_EPI_GELU ? Elt<T>::pack(v0, v1) : Elt<T>::pack(d0, d1);
              a0 = g0;
              a1 = g1;
              if (!two_pass) o = Elt<T>::pack(g0, g1);
            } else {
              o = Elt<T>::pack(v0, v1);
            }
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(o) : "memory");
          }
      }
      fence_proxy_async_smem();
      named_bar_sync(3 + cw, 128);
      if (two_pass) {
        if (elected) {
#pragma unroll
          for (int j = 0; j < BN / 64; ++j) tma_store_2d(&tmAuxOut, stg + j * kBlk, n0 + 64 * j, mw);
          tma_commit_group();
          tma_wait_group_read<0>();
        }
        named_bar_sync(3 + cw, 128);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const uint32_t cj = thr + (j >> 3) * kBlk + (((j & 7) ^ rq) << 4);
#pragma unroll
          for (int hh = 0; hh < HALVES; ++hh)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const uint32_t o = Elt<T>::pack(acc[hh][4 * j + 2 * h], acc[hh][4 * j + 2 * h + 1]);
              asm volatile("st.shared.b32 [%0], %1;" ::"r"(cj + (64 * hh + 8 * h) * 128), "r"(o) : "memory");
            }
        }
        fence_proxy_async_smem();
        named_bar_sync(3 + cw, 128);
      }
      if (elected) {
        // rows past M are clipped by the tensor map
#pragma unroll
        for (int j = 0; j < BN / 64; ++j) tma_store_2d(&tmD, stg + j * kBlk, n0 + 64 * j, mw);
        tma_commit_group();
        tma_wait_group_read<0>();
        if (kAuxTma) mbar_arrive(auxempty0 + 8 * cw);
      }
    }
    ++own;
  }
}

// ---------------------------------------------------------------------------------------------
// cooperative weight-gradient kernel (both operands MN-major, promoted accumulation)
// ---------------------------------------------------------------------------------------------
template <typename T, int BN, bool OUT_F32>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wgrad_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  static_assert(BN <= 128, "promoted accumulation needs two accumulator sets in registers");
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
#pragma unroll
          for (int j = 0; j < BM / 64; ++j) tma_load_2d(sa + j * 8192, &tmA, fb, m0 + 64 * j, k0);
#pragma unroll
          for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * 8192, &tmB, fb, n0 + 64 * j, k0);
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
  int stage = 0;
  uint32_t phase = 0;
  float acc[BN / 2];
  float part[BN / 2];
  WorkCursor wc = work_begin(p);
  int t, kb0, kb1;
  while (work_next(p, wc, t, kb0, kb1)) {
    const int m0 = (t / p.tiles_n) * BM;
    const int n0 = (t % p.tiles_n) * BN;
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(full0 + 8 * stage, phase);
      const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES) + cw * 8192;   // this warpgroup's 64 rows
      const uint32_t sb = smem_u32(smem + stage * Cfg::STAGE_BYTES) + Cfg::A_BYTES;
      const uint64_t da0 = make_smem_desc(sa, 8192, 1024, 1);
      const uint64_t db0 = make_smem_desc(sb, 8192, 1024, 1);
      const bool group_first = (kb - kb0) % kPromoteKB == 0;
      const bool group_last = (kb - kb0) % kPromoteKB == kPromoteKB - 1 || kb + 1 == kb1;
      wgmma_fence_regs(part);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BK / 16; ++kk)
        wgmma_ss<BN, 1, 1, T>(part, da0 + ((kk * 2048) >> 4), db0 + ((kk * 2048) >> 4), (!group_first || kk > 0) ? 1 : 0);
      wgmma_commit();
      if (group_last) {
        wgmma_wait<0>();
        wgmma_fence_regs(part);
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
      } else {
        wgmma_wait<1>();
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

    const bool add_bias = p.bias != nullptr && kb0 == 0;   // the bias joins the piece holding the tile's first k-block
    epilogue_direct<T, BN, OUT_F32, VJ_EPI_NONE, false>(p, acc, m0 + cw * 64 + warp_in_wg * 16, n0, add_bias, lane);
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static int grid_size(const GemmParams& p) {
  if (p.stream_k) {
    const long long total_kb = (long long)p.tiles_m * p.tiles_n * p.kb_total;
    return int((total_kb + p.sk_chunk - 1) / p.sk_chunk);
  }
  const int total = p.tiles_m * p.tiles_n * p.split_k;
  return total < sm_budget() ? total : sm_budget();
}

struct GemmMaps {
  CUtensorMap A, B, D, aux, aux_out;   // D / aux / aux_out: 16-bit boxes of the staged epilogue (zero if unused)
};

template <typename T, int BN, bool COOP, bool B_MN, bool OUT_F32, int EPI, bool AUX32 = false>
static int launch_gemm(const GemmMaps& m, const GemmParams& p, cudaStream_t stream) {
  constexpr int SMEM = PingCfg<BN, !OUT_F32, COOP>::SMEM_BYTES;
  auto kern = gemm_kernel<T, BN, COOP, B_MN, OUT_F32, EPI, AUX32>;
  static bool configured = false;  // per instantiation
  if (!configured) {
    VJ_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    configured = true;
  }
  kern<<<grid_size(p), kGemmThreads, SMEM, stream>>>(m.A, m.B, m.D, m.aux, m.aux_out, p);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

template <typename T, int BN, bool OUT_F32>
static int launch_gemm_wgrad(const GemmMaps& m, const GemmParams& p, cudaStream_t stream) {
  constexpr int SMEM = GemmCfg<BN>::SMEM_BYTES;
  auto kern = gemm_wgrad_kernel<T, BN, OUT_F32>;
  static bool configured = false;  // per instantiation
  if (!configured) {
    VJ_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    configured = true;
  }
  kern<<<grid_size(p), kGemmThreads, SMEM, stream>>>(m.A, m.B, p);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

template <typename T, int BN, bool COOP>
static int dispatch_major(int a_mn, int b_mn, int out_f32, int epi, int aux_f32, const GemmMaps& m,
                          const GemmParams& p, cudaStream_t s) {
  // instantiated combinations = what the V-JEPA step needs (forward Linear: K/K; dgrad: K/MN; wgrad: MN/MN fp32);
  // in fp16 only what frozen evaluation runs (the encoder's forward, the probe's forward and backward)
  constexpr bool kBf16 = std::is_same<T, __nv_bfloat16>::value;
  if (!a_mn && !b_mn) {
    if (epi == VJ_EPI_NONE) return out_f32 ? launch_gemm<T, BN, COOP, false, true, VJ_EPI_NONE>(m, p, s)
                                           : launch_gemm<T, BN, COOP, false, false, VJ_EPI_NONE>(m, p, s);
    if (epi == VJ_EPI_ADD) {
      if (aux_f32) return out_f32 ? launch_gemm<T, BN, COOP, false, true, VJ_EPI_ADD, true>(m, p, s)
                                  : launch_gemm<T, BN, COOP, false, false, VJ_EPI_ADD, true>(m, p, s);
      if (!out_f32) return launch_gemm<T, BN, COOP, false, false, VJ_EPI_ADD, false>(m, p, s);
    }
    if (epi == VJ_EPI_GELU && !out_f32) return launch_gemm<T, BN, COOP, false, false, VJ_EPI_GELU>(m, p, s);
    if (epi == VJ_EPI_GELU_GRAD && !out_f32) return launch_gemm<T, BN, COOP, false, false, VJ_EPI_GELU_GRAD>(m, p, s);
    if constexpr (kBf16)
      if (epi == VJ_EPI_DGELU && !out_f32 && !aux_f32) return launch_gemm<T, BN, COOP, false, false, VJ_EPI_DGELU>(m, p, s);
  } else if (!a_mn && b_mn) {
    if (epi == VJ_EPI_NONE) return out_f32 ? launch_gemm<T, BN, COOP, true, true, VJ_EPI_NONE>(m, p, s)
                                           : launch_gemm<T, BN, COOP, true, false, VJ_EPI_NONE>(m, p, s);
    if constexpr (kBf16)
      if (epi == VJ_EPI_DGELU && !out_f32 && !aux_f32) return launch_gemm<T, BN, COOP, true, false, VJ_EPI_DGELU>(m, p, s);
    if (epi == VJ_EPI_MUL && !out_f32 && !aux_f32) return launch_gemm<T, BN, COOP, true, false, VJ_EPI_MUL>(m, p, s);
  } else if (a_mn && b_mn) {
    if constexpr (!COOP) {
      if (epi == VJ_EPI_NONE) {
        if (out_f32) return launch_gemm_wgrad<T, BN, true>(m, p, s);
        if constexpr (kBf16) return launch_gemm_wgrad<T, BN, false>(m, p, s);
      }
    }
  }
  set_error("vj_gemm%s: combination a_mn=%d b_mn=%d d_f32=%d epi=%d aux_f32=%d is not instantiated", kBf16 ? "" : "_f16",
            a_mn, b_mn, out_f32, epi, aux_f32);
  return -1;
}

template <typename T>
static int gemm_impl(const void* A, long long lda, int a_mn, const void* B, long long ldb,
                     int b_mn, void* D, long long ldd, int d_f32, int M, int N, int K,
                     const float* bias, float alpha, int epi, const void* aux, long long ldaux,
                     int aux_f32, const int* aux_rowmap, int aux_period, void* aux_out,
                     long long ldauxout, int split_k, int accumulate, void* stream_) {
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

  // Schedule and tile width.  Weight gradients (MN/MN) run cooperatively on 128 x 128 tiles (two 64 x 128 accumulator
  // sets per warpgroup, see kPromoteKB).  Forward / dgrad GEMMs run ping-pong on 128 x 128 tiles (a warpgroup holds the
  // whole tile), so one warpgroup's epilogue hides under the other's main loop - unless K is long enough that the
  // epilogue is a small share of the tile anyway: there the cooperative 128 x 256 tile, which moves fewer smem / L2
  // bytes per FLOP, is faster.  Measured on H100 at step shapes: K <= 1536 (24 k-blocks) ping-pong is faster; at
  // K = 4096 (64 k-blocks) target fc2 + residual ran 582 TFLOP/s ping-pong against 631 on a 128 x 256 tile.  No step
  // GEMM has K between the two.
  // 64-wide tiles when N is an odd multiple of 64.
  constexpr int kCoopMinKB = 48;
  const int kb_total = (K + BK - 1) / BK;
  const bool coop = !(a_mn && b_mn) && N % 256 == 0 && kb_total >= kCoopMinKB;
  const int BN = coop ? 256 : (N % 128 == 0 ? 128 : 64);
  GemmParams p;
  p.M = M; p.N = N; p.K = K;
  p.tiles_m = (M + BM - 1) / BM;
  p.tiles_n = N / BN;
  p.kb_total = kb_total;
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

  // aux_out is written by TMA stores: 16-byte aligned rows
  if (p.aux_out != nullptr)
    VJ_CHECK_ARG((reinterpret_cast<uintptr_t>(aux_out) & 15) == 0 && ldauxout % 8 == 0, "vj_gemm: aux_out misaligned");
  const bool uses_aux = epi == VJ_EPI_ADD || epi == VJ_EPI_DGELU || epi == VJ_EPI_MUL;
  const bool aux_tma = uses_aux && !aux_f32;
  // every split-K piece runs the whole epilogue: an fp32 aux would be added once per piece
  if (uses_aux) VJ_CHECK_ARG(p.split_k == 1, "vj_gemm: aux epilogues do not combine with split-K");
  if (aux_tma) VJ_CHECK_ARG(aux_rowmap == nullptr && aux_period == 0, "vj_gemm: row-mapped / periodic aux must be fp32");
  GemmMaps m;
  memset(&m, 0, sizeof(m));
  int rc;
  constexpr int dt = Elt<T>::kTmap;
  if (!a_mn) rc = make_tmap_2d(&m.A, A, dt, K, M, lda * 2, 64, 128, 3);
  else       rc = make_tmap_2d(&m.A, A, dt, M, K, lda * 2, 64, 64, 3);
  if (rc) return rc;
  if (!b_mn) rc = make_tmap_2d(&m.B, B, dt, K, N, ldb * 2, 64, BN, 3);
  else       rc = make_tmap_2d(&m.B, B, dt, N, K, ldb * 2, 64, 64, 3);
  if (rc) return rc;
  if (!(a_mn && b_mn) && !d_f32) {
    const int rows = coop ? 64 : BM;   // staging rows per consumer warpgroup
    if ((rc = make_tmap_2d(&m.D, D, dt, N, M, ldd * 2, 64, rows, 3))) return rc;
    if (aux_tma && (rc = make_tmap_2d(&m.aux, aux, dt, N, M, ldaux * 2, 64, rows, 3))) return rc;
    if (p.aux_out != nullptr && (rc = make_tmap_2d(&m.aux_out, aux_out, dt, N, M, ldauxout * 2, 64, rows, 3))) return rc;
  }
  if (coop) return dispatch_major<T, 256, true>(a_mn, b_mn, d_f32, epi, aux_f32, m, p, stream);
  return BN == 128 ? dispatch_major<T, 128, false>(a_mn, b_mn, d_f32, epi, aux_f32, m, p, stream)
                   : dispatch_major<T, 64, false>(a_mn, b_mn, d_f32, epi, aux_f32, m, p, stream);
}

}  // namespace vj

extern "C" int vj_gemm(const void* A, long long lda, int a_mn, const void* B, long long ldb,
                       int b_mn, void* D, long long ldd, int d_f32, int M, int N, int K,
                       const float* bias, float alpha, int epi, const void* aux, long long ldaux,
                       int aux_f32, const int* aux_rowmap, int aux_period, void* aux_out,
                       long long ldauxout, int split_k, int accumulate, void* stream) {
  return vj::gemm_impl<__nv_bfloat16>(A, lda, a_mn, B, ldb, b_mn, D, ldd, d_f32, M, N, K, bias, alpha, epi, aux, ldaux,
                                      aux_f32, aux_rowmap, aux_period, aux_out, ldauxout, split_k, accumulate, stream);
}

extern "C" int vj_gemm_f16(const void* A, long long lda, int a_mn, const void* B, long long ldb,
                           int b_mn, void* D, long long ldd, int d_f32, int M, int N, int K,
                           const float* bias, float alpha, int epi, const void* aux, long long ldaux,
                           int aux_f32, const int* aux_rowmap, int aux_period, void* aux_out,
                           long long ldauxout, int split_k, int accumulate, void* stream) {
  return vj::gemm_impl<__half>(A, lda, a_mn, B, ldb, b_mn, D, ldd, d_f32, M, N, K, bias, alpha, epi, aux, ldaux,
                               aux_f32, aux_rowmap, aux_period, aux_out, ldauxout, split_k, accumulate, stream);
}
