// Shared tile geometry and wgmma descriptor helpers of the attention kernels (fwd and bwd).
//
// A [ROWS x HD] bf16 tile of q, k, v, o or dO is loaded by TMA as HD / BOX_INNER boxes of [ROWS x BOX_INNER] (128B swizzle
// for HD >= 64, 64B swizzle for HD = 32), box after box.  The same tile serves as a K-major wgmma operand (reduction over
// HD: Q K^T, dO V^T) and as an MN-major one (reduction over its rows: P V, dS K, P^T dO, dS^T Q).
#pragma once
#include "common.cuh"
#include "wgmma.cuh"

namespace vj {

template <int HD>
struct AttnCfg {
  static constexpr int BOX_INNER = HD >= 64 ? 64 : HD;          // elements per TMA box row
  static constexpr int NBOX = HD / BOX_INNER;                    // boxes per [ROWS x HD] tile
  static constexpr int ROW_BYTES = BOX_INNER * 2;                // 128 (SW128) or 64 (SW64)
  static constexpr int LAYOUT = HD >= 64 ? 1 : 2;                // wgmma descriptor swizzle type
  static constexpr int TMAP_SWIZZLE = HD >= 64 ? 3 : 2;
  static constexpr int SBO = 8 * ROW_BYTES;                      // 8-row group stride
  template <int ROWS>
  static constexpr int tile_bytes() { return ROWS * HD * 2; }
};

// K-major descriptor (reduction over HD) of k-step kk (16 elements) of a [ROWS x HD] tile, starting at row `row0`
template <int HD, int ROWS>
VJ_DEVINL uint64_t attn_kmajor_desc(uint32_t tile, int row0, int kk) {
  using C = AttnCfg<HD>;
  constexpr int steps_per_box = C::BOX_INNER / 16;
  const uint32_t addr = tile + (kk / steps_per_box) * (ROWS * C::ROW_BYTES) + row0 * C::ROW_BYTES + (kk % steps_per_box) * 32;
  return make_smem_desc(addr, 16, C::SBO, C::LAYOUT);
}
// MN-major descriptor (N = HD contiguous, reduction over rows) of k-step kk (16 rows) of a [ROWS x HD] tile
template <int HD, int ROWS>
VJ_DEVINL uint64_t attn_mnmajor_desc(uint32_t tile, int kk) {
  using C = AttnCfg<HD>;
  return make_smem_desc(tile + kk * 16 * C::ROW_BYTES, ROWS * C::ROW_BYTES, C::SBO, C::LAYOUT);
}

// TMA load of rows [r0, r0 + ROWS) of the HD columns starting at column c0 (one box per BOX_INNER columns)
template <int HD, int ROWS>
VJ_DEVINL void attn_load_tile(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int r0) {
  using C = AttnCfg<HD>;
#pragma unroll
  for (int b = 0; b < C::NBOX; ++b) tma_load_2d(dst + b * ROWS * C::ROW_BYTES, m, bar, c0 + b * C::BOX_INNER, r0);
}

// m64k16 A fragment (registers) of k-step kk from an m64nN fp32 accumulator fragment of the same rows: the accumulator's
// column pairs 16kk..16kk+15 are exactly the A operand's k pairs, so P / dS never touch shared memory.
template <int R>
VJ_DEVINL void acc_to_afrag(const float (&d)[R], int kk, uint32_t (&a)[4]) {
  a[0] = pack_bf16x2(d[8 * kk + 0], d[8 * kk + 1]);
  a[1] = pack_bf16x2(d[8 * kk + 2], d[8 * kk + 3]);
  a[2] = pack_bf16x2(d[8 * kk + 4], d[8 * kk + 5]);
  a[3] = pack_bf16x2(d[8 * kk + 6], d[8 * kk + 7]);
}

VJ_DEVINL float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
VJ_DEVINL float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// Stores an m64nHD fp32 accumulator fragment (times `mul`) as bf16 rows: thread holds rows r and r + 8 of the
// warpgroup's 64, column pairs 8j + 2(lane % 4).  Rows at or beyond `rows_valid` are skipped.
template <int HD>
VJ_DEVINL void store_frag_bf16(const float (&d)[HD / 2], float mul, __nv_bfloat16* base, long long ld, int r, int rows_valid) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = r + 8 * h;
    if (row >= rows_valid) continue;
#pragma unroll
    for (int j = 0; j < HD / 8; ++j)
      *reinterpret_cast<uint32_t*>(base + (long long)row * ld + 8 * j + 2 * (lane & 3)) =
          pack_bf16x2(d[4 * j + 2 * h] * mul, d[4 * j + 2 * h + 1] * mul);
  }
}

}  // namespace vj
