// Flat-buffer parameter kernels: fp32 -> bf16 shadow cast, head-dim padding of the predictor's
// qkv/proj weights (hd 24 -> 32 so attention tiles stay wgmma-shaped), the target-encoder EMA
// (app/vjepa/train.py:484-487) and a fused AdamW step (torch.optim.AdamW as configured by
// app/vjepa/utils.py:156-210).  All HBM-bound, 16-byte vectorised, grid = multiple of the SM count.
#include "common.cuh"
#include "vjepa_b200.h"

namespace vj {

static int flat_grid(long long n_vec, int threads) {
  long long g = (n_vec + threads - 1) / threads;
  const long long cap = (long long)num_sms() * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return int(g);
}

__global__ void __launch_bounds__(256) cast_f32_bf16_kernel(const float4* __restrict__ src, uint2* __restrict__ dst,
                                                            long long n4) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 f = src[i];
    uint2 o;
    o.x = pack_bf16x2(f.x, f.y);
    o.y = pack_bf16x2(f.z, f.w);
    dst[i] = o;
  }
}

// view tensors as [outer, G, hd, inner] (unpadded) and [outer, G, hdp, inner] (padded)
template <typename TS, typename TD>
__global__ void __launch_bounds__(256) head_pad_kernel(const TS* __restrict__ src, TD* __restrict__ dst, long long outer,
                                                       int G, int hd, int hdp, long long inner) {
  const long long total = outer * G * hdp * inner;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long in = i % inner;
    long long t = i / inner;
    const int j = int(t % hdp);
    t /= hdp;
    const int g = int(t % G);
    const long long o = t / G;
    float v = 0.f;
    if (j < hd) v = float(src[((o * G + g) * hd + j) * inner + in]);
    dst[i] = TD(v);
  }
}
// unpadded[o,g,j,in] += padded[o,g,j,in]   (fp32 gradients)
__global__ void __launch_bounds__(256) head_unpad_add_kernel(const float* __restrict__ padded, float* __restrict__ dst,
                                                             long long outer, int G, int hd, int hdp, long long inner) {
  const long long total = outer * G * hd * inner;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long in = i % inner;
    long long t = i / inner;
    const int j = int(t % hd);
    t /= hd;
    const int g = int(t % G);
    const long long o = t / G;
    dst[i] += padded[((o * G + g) * hdp + j) * inner + in];
  }
}

// k <- fl(fl(k*m) + fl(om*q)): the reference's param_k.mul_(m).add_((1-m)*param_q), op for op
__global__ void __launch_bounds__(256) ema_kernel(float4* __restrict__ k, const float4* __restrict__ q, long long n4,
                                                  float m, float om) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 a = k[i];
    const float4 b = q[i];
    a.x = __fadd_rn(__fmul_rn(a.x, m), __fmul_rn(om, b.x));
    a.y = __fadd_rn(__fmul_rn(a.y, m), __fmul_rn(om, b.y));
    a.z = __fadd_rn(__fmul_rn(a.z, m), __fmul_rn(om, b.z));
    a.w = __fadd_rn(__fmul_rn(a.w, m), __fmul_rn(om, b.w));
    k[i] = a;
  }
}

// AdamW (decoupled weight decay), torch.optim.AdamW update rule; optional grad unscale (1/loss-scale)
// and skip-on-overflow flag (found_inf != 0 -> no-op), both read from device memory (no host sync).
__global__ void __launch_bounds__(256) adamw_kernel(float4* __restrict__ p, const float4* __restrict__ g,
                                                    float4* __restrict__ m, float4* __restrict__ v, long long n4,
                                                    float lr, float beta1, float beta2, float eps, float wd,
                                                    float bc1, float bc2_sqrt, const float* __restrict__ inv_scale,
                                                    const float* __restrict__ found_inf) {
  if (found_inf != nullptr && *found_inf != 0.f) return;
  const float gs = inv_scale ? *inv_scale : 1.0f;
  const float step_size = lr / bc1;
  const float decay = 1.0f - lr * wd;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 pp = p[i], gg = g[i], mm = m[i], vv = v[i];
#define VJ_ADAM1(c)                                                 \
  {                                                                 \
    const float gr = gg.c * gs;                                     \
    pp.c *= decay;                                                  \
    mm.c = mm.c + (gr - mm.c) * (1.0f - beta1);                     \
    vv.c = vv.c * beta2 + (1.0f - beta2) * gr * gr;                 \
    const float denom = sqrtf(vv.c) / bc2_sqrt + eps;               \
    pp.c -= step_size * (mm.c / denom);                             \
  }
    VJ_ADAM1(x) VJ_ADAM1(y) VJ_ADAM1(z) VJ_ADAM1(w)
#undef VJ_ADAM1
    p[i] = pp; m[i] = mm; v[i] = vv;
  }
}

// sum of squares of a flat fp32 buffer -> out[0] (+=)   (grad-norm logging / clipping)
__global__ void __launch_bounds__(256) sumsq_kernel(const float4* __restrict__ x, long long n4, float* __restrict__ out) {
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 a = x[i];
    acc += a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
  }
  __shared__ float sm[8];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += sm[w];
    atomicAdd(out, s);
  }
}

}  // namespace vj

using namespace vj;

extern "C" int vj_cast_f32_bf16(const float* src, void* dst, long long n, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(src && dst, "vj_cast_f32_bf16: null pointer");
  VJ_CHECK_ARG(n % 4 == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 7) == 0,
               "vj_cast_f32_bf16: n %% 4 and 16-byte alignment required");
  if (n <= 0) return 0;
  cast_f32_bf16_kernel<<<flat_grid(n / 4, 256), 256, 0, s>>>(reinterpret_cast<const float4*>(src),
                                                              reinterpret_cast<uint2*>(dst), n / 4);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_head_pad(const void* src, int src_f32, void* dst, int dst_f32, long long outer, int G, int hd, int hdp,
                           long long inner, int unpad_add, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(src && dst, "vj_head_pad: null pointer");
  VJ_CHECK_ARG(hd > 0 && hdp >= hd && G > 0 && outer > 0 && inner > 0, "vj_head_pad: bad geometry");
  if (unpad_add) {
    VJ_CHECK_ARG(src_f32 && dst_f32, "vj_head_pad: unpad-add is fp32 only");
    head_unpad_add_kernel<<<flat_grid(outer * G * hd * inner, 256), 256, 0, s>>>(
        reinterpret_cast<const float*>(src), reinterpret_cast<float*>(dst), outer, G, hd, hdp, inner);
  } else {
    const int g = flat_grid(outer * G * hdp * inner, 256);
    if (src_f32 && dst_f32)
      head_pad_kernel<float, float><<<g, 256, 0, s>>>(reinterpret_cast<const float*>(src), reinterpret_cast<float*>(dst), outer, G, hd, hdp, inner);
    else if (src_f32)
      head_pad_kernel<float, __nv_bfloat16><<<g, 256, 0, s>>>(reinterpret_cast<const float*>(src), reinterpret_cast<__nv_bfloat16*>(dst), outer, G, hd, hdp, inner);
    else if (!dst_f32)
      head_pad_kernel<__nv_bfloat16, __nv_bfloat16><<<g, 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(src), reinterpret_cast<__nv_bfloat16*>(dst), outer, G, hd, hdp, inner);
    else {
      set_error("vj_head_pad: bf16 -> fp32 not instantiated");
      return -1;
    }
  }
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_ema_update(float* k, const float* q, long long n, float m, float one_minus_m, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(k && q, "vj_ema_update: null pointer");
  VJ_CHECK_ARG(n % 4 == 0 && (reinterpret_cast<uintptr_t>(k) & 15) == 0 && (reinterpret_cast<uintptr_t>(q) & 15) == 0,
               "vj_ema_update: n %% 4 and 16-byte alignment required");
  if (n <= 0) return 0;
  ema_kernel<<<flat_grid(n / 4, 256), 256, 0, s>>>(reinterpret_cast<float4*>(k), reinterpret_cast<const float4*>(q), n / 4,
                                                    m, one_minus_m);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_adamw_step(float* p, const float* g, float* m, float* v, long long n, float lr, float beta1,
                             float beta2, float eps, float weight_decay, int step, const float* inv_scale_dev,
                             const float* found_inf_dev, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(p && g && m && v, "vj_adamw_step: null pointer");
  VJ_CHECK_ARG(n % 4 == 0 && step >= 1, "vj_adamw_step: n %% 4 == 0 and step >= 1 required");
  VJ_CHECK_ARG(((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                 reinterpret_cast<uintptr_t>(v)) & 15) == 0, "vj_adamw_step: 16-byte alignment required");
  if (n <= 0) return 0;
  const double bc1 = 1.0 - pow((double)beta1, (double)step);
  const double bc2 = 1.0 - pow((double)beta2, (double)step);
  adamw_kernel<<<flat_grid(n / 4, 256), 256, 0, s>>>(reinterpret_cast<float4*>(p), reinterpret_cast<const float4*>(g),
                                                      reinterpret_cast<float4*>(m), reinterpret_cast<float4*>(v), n / 4, lr,
                                                      beta1, beta2, eps, weight_decay, float(bc1), float(sqrt(bc2)),
                                                      inv_scale_dev, found_inf_dev);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_sumsq(const float* x, long long n, float* out, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(x && out, "vj_sumsq: null pointer");
  VJ_CHECK_ARG(n % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0, "vj_sumsq: n %% 4 and alignment required");
  if (n <= 0) return 0;
  sumsq_kernel<<<flat_grid(n / 4, 256 * 4), 256, 0, s>>>(reinterpret_cast<const float4*>(x), n / 4, out);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

// ---------------------------------------------------------------------------------------------------
// AdamW over a whole FlatParamStore in ONE launch.  Every 64-element block of the flat buffer carries a
// group id (uint8): hyper-parameters come from a 4-entry table, id 255 = frozen / padding (skipped).
// ---------------------------------------------------------------------------------------------------
namespace vj {
struct AdamGroups {
  float lr[4], wd[4];
};
// STEP_DEV: the step count lives on the device (fp32 scalar, like torch's capturable / fused AdamW): the kernel uses
// *step_dev + 1 and a one-thread tail kernel advances it ONLY when the step was not skipped by the GradScaler, so the
// bias correction and the checkpointed `step` stay exact across overflow skips.  shadow (nullable): bf16 copy of the
// updated parameters, i.e. next step's tensor-core operands, emitted in the same pass (saves the separate cast kernel).
__global__ void __launch_bounds__(256) adamw_flat_kernel(float4* __restrict__ p, const float4* __restrict__ g,
                                                         float4* __restrict__ m, float4* __restrict__ v,
                                                         const unsigned char* __restrict__ gid, long long n4,
                                                         AdamGroups hp, float beta1, float beta2, float eps, float bc1,
                                                         float bc2_sqrt, const float* __restrict__ inv_scale,
                                                         const float* __restrict__ found_inf,
                                                         const float* __restrict__ step_dev, uint2* __restrict__ shadow) {
  if (found_inf != nullptr && *found_inf != 0.f) return;
  const float gs = inv_scale ? *inv_scale : 1.0f;
  if (step_dev != nullptr) {
    const double step = (double)*step_dev + 1.0;       // once per thread, in double like the host path
    bc1 = float(1.0 - pow((double)beta1, step));
    bc2_sqrt = float(sqrt(1.0 - pow((double)beta2, step)));
  }
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const unsigned id = gid[i >> 4];
    if (id > 3) continue;
    const float lr = hp.lr[id];
    const float step_size = lr / bc1;
    const float decay = 1.0f - lr * hp.wd[id];
    float4 pp = p[i], gg = g[i], mm = m[i], vv = v[i];
#define VJ_ADAM1(c)                                                 \
  {                                                                 \
    const float gr = gg.c * gs;                                     \
    pp.c *= decay;                                                  \
    mm.c = mm.c + (gr - mm.c) * (1.0f - beta1);                     \
    vv.c = vv.c * beta2 + (1.0f - beta2) * gr * gr;                 \
    const float denom = sqrtf(vv.c) / bc2_sqrt + eps;               \
    pp.c -= step_size * (mm.c / denom);                             \
  }
    VJ_ADAM1(x) VJ_ADAM1(y) VJ_ADAM1(z) VJ_ADAM1(w)
#undef VJ_ADAM1
    p[i] = pp; m[i] = mm; v[i] = vv;
    if (shadow != nullptr) {
      uint2 o;
      o.x = pack_bf16x2(pp.x, pp.y);
      o.y = pack_bf16x2(pp.z, pp.w);
      shadow[i] = o;
    }
  }
}
__global__ void step_advance_kernel(float* step_dev, const float* __restrict__ found_inf) {
  if (found_inf == nullptr || *found_inf == 0.f) *step_dev += 1.0f;
}
// k = k*m + (1-m)*q with the bf16 shadow of the new k emitted in the same pass (target-encoder EMA, train.py:484-487)
__global__ void __launch_bounds__(256) ema_shadow_kernel(float4* __restrict__ k, const float4* __restrict__ q, long long n4,
                                                         float m, float one_minus_m, uint2* __restrict__ shadow) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 a = k[i];
    const float4 b = q[i];
    // op-for-op like param_k.mul_(m).add_((1.-m)*param_q): two roundings per element, no FMA contraction
    a.x = __fadd_rn(__fmul_rn(a.x, m), __fmul_rn(one_minus_m, b.x));
    a.y = __fadd_rn(__fmul_rn(a.y, m), __fmul_rn(one_minus_m, b.y));
    a.z = __fadd_rn(__fmul_rn(a.z, m), __fmul_rn(one_minus_m, b.z));
    a.w = __fadd_rn(__fmul_rn(a.w, m), __fmul_rn(one_minus_m, b.w));
    k[i] = a;
    uint2 o;
    o.x = pack_bf16x2(a.x, a.y);
    o.y = pack_bf16x2(a.z, a.w);
    shadow[i] = o;
  }
}
}  // namespace vj

extern "C" int vj_adamw_flat(float* p, const float* g, float* m, float* v, const unsigned char* group_ids, long long n,
                             const float* lr4, const float* wd4, float beta1, float beta2, float eps, int step,
                             const float* inv_scale_dev, const float* found_inf_dev, float* step_dev, void* shadow_bf16,
                             void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(p && g && m && v && group_ids && lr4 && wd4, "vj_adamw_flat: null pointer");
  VJ_CHECK_ARG(n % 64 == 0 && (step >= 1 || step_dev != nullptr), "vj_adamw_flat: n %% 64 == 0 and step >= 1 required");
  VJ_CHECK_ARG(((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                 reinterpret_cast<uintptr_t>(v)) & 15) == 0, "vj_adamw_flat: 16-byte alignment required");
  VJ_CHECK_ARG((reinterpret_cast<uintptr_t>(shadow_bf16) & 7) == 0, "vj_adamw_flat: shadow must be 8-byte aligned");
  if (n <= 0) return 0;
  vj::AdamGroups hp;
  for (int i = 0; i < 4; ++i) { hp.lr[i] = lr4[i]; hp.wd[i] = wd4[i]; }   // host arrays
  const int hstep = step >= 1 ? step : 1;
  const double bc1 = 1.0 - pow((double)beta1, (double)hstep);
  const double bc2 = 1.0 - pow((double)beta2, (double)hstep);
  vj::adamw_flat_kernel<<<vj::flat_grid(n / 4, 256), 256, 0, s>>>(
      reinterpret_cast<float4*>(p), reinterpret_cast<const float4*>(g), reinterpret_cast<float4*>(m),
      reinterpret_cast<float4*>(v), group_ids, n / 4, hp, beta1, beta2, eps, float(bc1), float(sqrt(bc2)),
      inv_scale_dev, found_inf_dev, step_dev, reinterpret_cast<uint2*>(shadow_bf16));
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  if (step_dev != nullptr) {
    vj::step_advance_kernel<<<1, 1, 0, s>>>(step_dev, found_inf_dev);
    VJ_CUDA(cudaGetLastError());
    vj::count_launch(1);
  }
  return 0;
}

extern "C" int vj_ema_update_shadow(float* k, const float* q, long long n, float m, float one_minus_m, void* shadow_bf16,
                                    void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(k && q && shadow_bf16, "vj_ema_update_shadow: null pointer");
  VJ_CHECK_ARG(n % 4 == 0 && ((reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(q)) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(shadow_bf16) & 7) == 0, "vj_ema_update_shadow: alignment");
  if (n <= 0) return 0;
  vj::ema_shadow_kernel<<<vj::flat_grid(n / 4, 256), 256, 0, s>>>(reinterpret_cast<float4*>(k), reinterpret_cast<const float4*>(q),
                                                                  n / 4, m, one_minus_m, reinterpret_cast<uint2*>(shadow_bf16));
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}
