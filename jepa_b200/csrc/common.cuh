// Shared device/host helpers for the sm_90a V-JEPA kernels: raw PTX wrappers for
// mbarrier, TMA (cp.async.bulk.tensor), the wgmma shared-memory descriptor and the
// host-side CUtensorMap encoder.  No CUTLASS, no libcuda link dependency (the driver
// entry point is resolved at run time so the library still loads on a GPU-less host).
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#ifndef VJ_DEVINL
#define VJ_DEVINL __device__ __forceinline__
#endif

namespace vj {

// ---------------------------------------------------------------------------------------
// error plumbing (host)
// ---------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);

#define VJ_CHECK_ARG(cond, ...)                 \
  do {                                          \
    if (!(cond)) {                              \
      vj::set_error(__VA_ARGS__);               \
      return -1;                                \
    }                                           \
  } while (0)

#define VJ_CUDA(expr)                                         \
  do {                                                        \
    cudaError_t _e = (expr);                                  \
    if (_e != cudaSuccess) return vj::cuda_fail(_e, #expr);   \
  } while (0)

int num_sms();
int sm_budget();          // num_sms() minus the SMs currently reserved for NCCL (vj_set_sm_limit)
void count_launch(int n);  // bookkeeping for vj_launch_count()

// Encode a 2-D tiled tensor map.  `inner`/`outer` are element counts, `ld_bytes` the byte
// stride of the outer dimension.  swizzle: 0 none, 1 32B, 2 64B, 3 128B.
// dtype: 0 bf16, 1 f32.  Returns 0 on success.
int make_tmap_2d(CUtensorMap* out, const void* ptr, int dtype, uint64_t inner, uint64_t outer,
                 uint64_t ld_bytes, uint32_t box_inner, uint32_t box_outer, int swizzle);

// ---------------------------------------------------------------------------------------
// device: shared-memory addressing, mbarrier
// ---------------------------------------------------------------------------------------
VJ_DEVINL uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

VJ_DEVINL void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
VJ_DEVINL void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
VJ_DEVINL void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
VJ_DEVINL void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
VJ_DEVINL void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
VJ_DEVINL bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
VJ_DEVINL void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---------------------------------------------------------------------------------------
// device: TMA
// ---------------------------------------------------------------------------------------
VJ_DEVINL void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
VJ_DEVINL void tma_load_2d(uint32_t smem_dst, const CUtensorMap* m, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
VJ_DEVINL void tma_store_2d(const CUtensorMap* m, uint32_t smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_src), "r"(c0), "r"(c1)
               : "memory");
}
VJ_DEVINL void tma_reduce_add_2d(const CUtensorMap* m, uint32_t smem_src, int c0, int c1) {
  asm volatile(
      "cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(m)),
      "r"(smem_src), "r"(c0), "r"(c1)
      : "memory");
}
VJ_DEVINL void tma_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
VJ_DEVINL void tma_wait_group_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
VJ_DEVINL void tma_wait_group() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// Explicit shared-space accesses on 32-bit smem addresses.  Pointers derived from the manually aligned
// dynamic-smem base lose their address space in the compiler and degrade to generic LD/ST otherwise.
VJ_DEVINL void sts128(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
VJ_DEVINL void sts128f(uint32_t addr, const float4& v) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
VJ_DEVINL uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}
VJ_DEVINL float4 lds128f(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}
VJ_DEVINL void sts32f(uint32_t addr, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory"); }
VJ_DEVINL float lds32f(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}

// 2^x on the MUFU pipe (ex2.approx.ftz, ~2 ulp): softmax probabilities are rounded to bf16 anyway
VJ_DEVINL float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Shared-memory matrix descriptor of wgmma (sm_90).  Offsets in bytes (16B granules); the tile base must be aligned to
// the swizzle pattern (1024 B for 128B swizzle) so the base-offset field stays 0.
// layout_type: 0 none, 1 128B swizzle, 2 64B swizzle, 3 32B swizzle.
//   K-major, swizzled : LBO unused, SBO = stride between 8-row groups; a K step inside the swizzle atom adds to the address.
//   MN-major, swizzled: LBO = stride between swizzle-atom-wide MN chunks, SBO = stride between groups of 8 K rows.
VJ_DEVINL uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes,
                                  uint32_t layout_type) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(layout_type & 3) << 62;
  return d;
}

// ---------------------------------------------------------------------------------------
// device: small math helpers
// ---------------------------------------------------------------------------------------
VJ_DEVINL uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
// packed bf16 multiply (HMUL2.BF16): both lanes rounded to nearest even
VJ_DEVINL uint32_t mul_bf16x2(uint32_t a, uint32_t b) {
  uint32_t d;
  asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
  return d;
}
VJ_DEVINL float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
VJ_DEVINL float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xFFFF0000u); }

VJ_DEVINL float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
VJ_DEVINL float gelu_erf_grad(float x) {
  const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752f));
  const float pdf = 0.39894228040143268f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}

VJ_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
VJ_DEVINL float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace vj
