// Segmented single-pass reductions over the FLAT gradient / Adam-moment buffers of a FlatParamStore (sm_90a, HBM-bound).
//
// Replaces the per-tensor host-synchronising loops of the reference's logging / clipping helpers:
//   src/utils/logging.py:91-105  grad_logger   : float(torch.norm(p.grad)) for every weight tensor  (~300 syncs / call)
//   src/utils/logging.py:108-118 adamw_logger  : float(exp_avg.abs().mean()), float(exp_avg_sq.abs().mean()) per tensor
//   app/vjepa/train.py:462-471   scaler.unscale_ (torch._amp_foreach_non_finite_check_and_unscale_ over ~450 views) and
//                                torch.nn.utils.clip_grad_norm_
// Every 64-element block of the flat buffer belongs to exactly one parameter tensor (FlatParamStore.ALIGN = 64); a uint16
// table maps blocks to segment (tensor) ids, 0xFFFF = frozen / padding.  One pass: unscale in place, non-finite check,
// per-tensor sum of squares; the clip coefficient is derived on the device and applied by a pass that exits
// immediately when no clipping is needed.  The host reads everything back with ONE copy.
#include "common.cuh"
#include "vjepa_b200.h"

namespace vj {

// MODE 0: sum of squares (optionally after multiplying by *inv_scale, written back when WRITE; non-finite -> *found_inf = 1)
// MODE 1: sum of absolute values
template <int MODE, bool WRITE>
__global__ void __launch_bounds__(256) seg_reduce_kernel(float4* __restrict__ x, const unsigned short* __restrict__ seg,
                                                         long long nblk, const float* __restrict__ inv_scale,
                                                         float* __restrict__ found_inf, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int sub = lane & 15;                    // a half-warp covers one 64-element block
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  const long long w = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  // contiguous, even-sized range of blocks per warp: a warp flushes one atomic per segment it touches
  long long per = (nblk + warps - 1) / warps;
  per = (per + 1) & ~1LL;
  const long long b_begin = w * per;
  const long long b_end = min(nblk, b_begin + per);
  const float gs = (MODE == 0 && inv_scale != nullptr) ? *inv_scale : 1.0f;
  unsigned cur = 0xFFFFu;
  float acc = 0.f;
  bool bad = false;
  for (long long b = b_begin; b < b_end; b += 2) {
    const long long blk = b + (lane >> 4);
    float s = 0.f;
    unsigned sg = 0xFFFFu;
    if (blk < b_end) {
      sg = seg[blk];
      if (sg != 0xFFFFu) {
        float4 v = x[blk * 16 + sub];
        if (MODE == 0) {
          v.x *= gs; v.y *= gs; v.z *= gs; v.w *= gs;
          if (WRITE) x[blk * 16 + sub] = v;
          s = v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
          bad |= !(fabsf(v.x) <= 3.4028234e38f) || !(fabsf(v.y) <= 3.4028234e38f) || !(fabsf(v.z) <= 3.4028234e38f) ||
                 !(fabsf(v.w) <= 3.4028234e38f);
        } else {
          s = fabsf(v.x) + fabsf(v.y) + fabsf(v.z) + fabsf(v.w);
        }
      }
    }
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float s_hi = __shfl_sync(0xffffffffu, s, 16);
    const unsigned sg_hi = __shfl_sync(0xffffffffu, sg, 16);
    if (lane == 0) {
      if (sg != cur) { if (cur != 0xFFFFu) atomicAdd(out + cur, acc); cur = sg; acc = 0.f; }
      acc += s;
      if (sg_hi != cur) { if (cur != 0xFFFFu) atomicAdd(out + cur, acc); cur = sg_hi; acc = 0.f; }
      acc += s_hi;
    }
  }
  if (lane == 0 && cur != 0xFFFFu) atomicAdd(out + cur, acc);
  if (MODE == 0 && found_inf != nullptr && __any_sync(0xffffffffu, bad) && lane == 0) *found_inf = 1.0f;
}

// total = sqrt(sum_i sumsq[i]); coef = min(1, max_norm / (total + 1e-6))   (torch.nn.utils.clip_grad_norm_, L2)
__global__ void clip_coef_kernel(const float* __restrict__ sumsq, int n_seg, float max_norm, float* __restrict__ total_norm,
                                 float* __restrict__ coef) {
  float acc = 0.f;
  for (int i = threadIdx.x; i < n_seg; i += 32) acc += sumsq[i];
  acc = warp_sum(acc);
  if (threadIdx.x == 0) {
    const float t = sqrtf(acc);
    *total_norm = t;
    *coef = fminf(1.0f, max_norm / (t + 1e-6f));
  }
}

__global__ void __launch_bounds__(256) scale_flat_kernel(float4* __restrict__ x, long long n4, const float* __restrict__ coef) {
  const float c = *coef;
  if (c >= 1.0f) return;     // nothing to clip: no memory traffic at all
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 v = x[i];
    v.x *= c; v.y *= c; v.z *= c; v.w *= c;
    x[i] = v;
  }
}

static int reduce_grid(long long nblk) {
  long long g = (nblk / 2 + 7) / 8;        // one block pair per warp at least
  const long long cap = (long long)num_sms() * 8;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return int(g);
}

}  // namespace vj

using namespace vj;

extern "C" int vj_grad_unscale_stats(float* g, const unsigned short* seg, long long n, const float* inv_scale_dev,
                                     float* found_inf_dev, float* sumsq_out, int write_back, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(g && seg && sumsq_out, "vj_grad_unscale_stats: null pointer");
  VJ_CHECK_ARG(n % 64 == 0 && (reinterpret_cast<uintptr_t>(g) & 15) == 0, "vj_grad_unscale_stats: n %% 64 and 16-byte alignment required");
  if (n <= 0) return 0;
  const long long nblk = n / 64;
  if (write_back)
    seg_reduce_kernel<0, true><<<reduce_grid(nblk), 256, 0, s>>>(reinterpret_cast<float4*>(g), seg, nblk, inv_scale_dev,
                                                                found_inf_dev, sumsq_out);
  else
    seg_reduce_kernel<0, false><<<reduce_grid(nblk), 256, 0, s>>>(reinterpret_cast<float4*>(g), seg, nblk, inv_scale_dev,
                                                                 found_inf_dev, sumsq_out);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_seg_abs_sum(const float* x, const unsigned short* seg, long long n, float* out, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(x && seg && out, "vj_seg_abs_sum: null pointer");
  VJ_CHECK_ARG(n % 64 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0, "vj_seg_abs_sum: n %% 64 and 16-byte alignment required");
  if (n <= 0) return 0;
  const long long nblk = n / 64;
  seg_reduce_kernel<1, false><<<reduce_grid(nblk), 256, 0, s>>>(reinterpret_cast<float4*>(const_cast<float*>(x)), seg, nblk,
                                                               nullptr, nullptr, out);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_clip_coef(const float* sumsq, int n_seg, float max_norm, float* total_norm_out, float* coef_out,
                            void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(sumsq && total_norm_out && coef_out && n_seg > 0, "vj_clip_coef: bad arguments");
  clip_coef_kernel<<<1, 32, 0, s>>>(sumsq, n_seg, max_norm, total_norm_out, coef_out);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_scale_flat(float* x, long long n, const float* coef_dev, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(x && coef_dev, "vj_scale_flat: null pointer");
  VJ_CHECK_ARG(n % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0, "vj_scale_flat: n %% 4 and 16-byte alignment required");
  if (n <= 0) return 0;
  long long g = (n / 4 + 255) / 256;
  const long long cap = (long long)num_sms() * 16;
  if (g > cap) g = cap;
  scale_flat_kernel<<<int(g), 256, 0, s>>>(reinterpret_cast<float4*>(x), n / 4, coef_dev);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}
