// GPU input pipeline (SURVEY 8f-3): decoded uint8 frames -> random-resized crop (bilinear) -> horizontal flip ->
// per-channel normalisation -> network input layout, in one pass, so that uint8 frames (not fp32 clips, 4x the bytes)
// cross PCIe and no CPU core touches a pixel.
//
// Replaces, for the non-auto-augment path every shipped pre-training config uses (configs/pretrain/*.yaml):
//   app/vjepa/transforms.py:86-117   VideoTransform.__call__: float conversion, permute, spatial transform, flip, normalise
//   src/datasets/utils/video/transforms.py:545-577  random_resized_crop = crop [i:i+h, j:j+w] +
//       F.interpolate(mode='bilinear', align_corners=False)  (no antialiasing)
//   src/datasets/utils/video/transforms.py:160-190  horizontal_flip (applied AFTER the resize)
//   app/vjepa/transforms.py:140-153  _tensor_normalize_inplace: (x - 255 mean_c) / (255 std_c)
// The random parameters (crop box, flip) are drawn on the host in the reference's RNG call order
// (jepa_b200/transforms.py) and handed over as a small table; the kernel is deterministic.
//
// in  : uint8 frames of clip b at src + src_off[b], layout [T, H_b, W_b, 3] (what decord / the reference's loader yields)
// out : [B, 3, T, S, S] fp32 or bf16 (the Conv3d / vj_im2col_tubelets input layout)
// Bilinear sampling follows ATen's upsample_bilinear2d (align_corners = False): src = max(0, (dst + 0.5) * in/out - 0.5),
// the upper neighbour is clamped to the last row / column of the CROP.
#include "common.cuh"
#include "vjepa_b200.h"

namespace vj {

// (v_c - sub_c) / div_c for the three channels, each step rounded like the reference's fp32 sub_ / div_, stored as TO
// at dst + c * cstride (the channel planes of the [3, T, S, S] layout)
template <typename TO>
__device__ __forceinline__ void normalise_store(TO* dst, long long cstride, const float (&v)[3], float3 sub, float3 div) {
  dst[0] = TO(__fdiv_rn(__fsub_rn(v[0], sub.x), div.x));
  dst[cstride] = TO(__fdiv_rn(__fsub_rn(v[1], sub.y), div.y));
  dst[2 * cstride] = TO(__fdiv_rn(__fsub_rn(v[2], sub.z), div.z));
}

struct ClipParam {     // one per clip, 8 x int32 + 1 x int64 offset (host-built, device-resident)
  long long src_off;   // byte offset of the clip's first frame in `src`
  int H, W;            // decoded frame size
  int i, j, h, w;      // crop box: rows [i, i+h), columns [j, j+w)
  int flip;            // 1: mirror the OUTPUT horizontally
  int pad;
};

template <typename TO>
__global__ void __launch_bounds__(256) clip_preprocess_kernel(const uint8_t* __restrict__ src, const ClipParam* __restrict__ prm,
                                                              TO* __restrict__ out, int T, int S, float3 mean255,
                                                              float3 std255) {
  const int b = blockIdx.z, t = blockIdx.y;
  const ClipParam cp = prm[b];
  const uint8_t* frame = src + cp.src_off + (long long)t * cp.H * cp.W * 3;
  const float sh = float(cp.h) / float(S), sw = float(cp.w) / float(S);
  const long long plane = (long long)S * S;
  TO* ob = out + ((long long)b * 3 * T + t) * plane;      // channel c at + c * T * plane
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < S * S; idx += gridDim.x * blockDim.x) {
    const int y = idx / S, xo = idx - y * S;
    const int x = cp.flip ? (S - 1 - xo) : xo;              // output column xo shows resized column x
    float fy = fmaxf((float(y) + 0.5f) * sh - 0.5f, 0.f);
    float fx = fmaxf((float(x) + 0.5f) * sw - 0.5f, 0.f);
    const int y0 = min(int(fy), cp.h - 1), x0 = min(int(fx), cp.w - 1);
    const int y1 = min(y0 + 1, cp.h - 1), x1 = min(x0 + 1, cp.w - 1);
    const float ly = fy - float(y0), lx = fx - float(x0);
    const float hy = 1.f - ly, hx = 1.f - lx;
    const uint8_t* r0 = frame + ((long long)(cp.i + y0) * cp.W + cp.j) * 3;
    const uint8_t* r1 = frame + ((long long)(cp.i + y1) * cp.W + cp.j) * 3;
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float p00 = float(r0[x0 * 3 + c]), p01 = float(r0[x1 * 3 + c]);
      const float p10 = float(r1[x0 * 3 + c]), p11 = float(r1[x1 * 3 + c]);
      v[c] = hy * (hx * p00 + lx * p01) + ly * (hx * p10 + lx * p11);
    }
    normalise_store(ob + idx, (long long)T * plane, v, mean255, std255);   // sub_ then div_, as the reference
  }
}

// Deterministic evaluation views (evals/video_classification_frozen/utils.py in the reference):
//   EvalVideoTransform (num_views > 1): short side -> S, `num_views` S x S windows along the long side
//   VideoTransform(training=False):     short side -> int(S * 256 / 224), centre S x S crop
// Both resize with resize_clip = cv2.resize(INTER_LINEAR) on uint8 frames (src/datasets/utils/video/functional.py:33-51),
// then ClipToTensor (/ 255) and Normalize ((x - mean) / std) in fp32.  OpenCV's uint8 bilinear resize is fixed point:
// per output column two source columns with 11-bit weights (a0, a1), a horizontal pass into int, per output row two
// source rows with 11-bit weights (b0, b1), and the vertical pass
//   u8 = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2
// (VResizeLinear<uchar, int, short, ...>; its SIMD and scalar paths compute the same expression).  The weights and
// clamped source indices of every resized row / column are computed on the host exactly as OpenCV computes them
// (jepa_b200/transforms.py) and handed over as a table; each thread resamples only the resized pixel its output needs
// (no resized frame is staged).  The no-resize case (short side already at the target) uses weights (2048, 0), which
// the expression maps back to the source byte exactly.
struct ViewJob {        // one (clip, segment, view), host-built, device-resident
  long long src_off;    // byte offset of the clip's first frame [T, H, W, 3] in `src`
  long long out_off;    // element offset of the view's [3, T, S, S] block in `out`
  int H, W;             // decoded frame size
  int ytab, xtab;       // first of the S row / S column entries of this view in `tab`
};

template <typename TO>
__global__ void __launch_bounds__(256) clip_views_kernel(const uint8_t* __restrict__ src, const ViewJob* __restrict__ jobs,
                                                         const int4* __restrict__ tab, TO* __restrict__ out, int T, int S,
                                                         float3 mean, float3 sdev) {
  const int t = blockIdx.y;
  const ViewJob jb = jobs[blockIdx.z];
  const uint8_t* frame = src + jb.src_off + (long long)t * jb.H * jb.W * 3;
  const long long plane = (long long)S * S;
  TO* ob = out + jb.out_off + (long long)t * plane;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < S * S; idx += gridDim.x * blockDim.x) {
    const int y = idx / S, x = idx - y * S;
    const int4 ry = tab[jb.ytab + y];     // (row0, row1, b0, b1)
    const int4 cx = tab[jb.xtab + x];     // (col0, col1, a0, a1)
    const uint8_t* r0 = frame + (long long)ry.x * jb.W * 3;
    const uint8_t* r1 = frame + (long long)ry.y * jb.W * 3;
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int h0 = int(r0[cx.x * 3 + c]) * cx.z + int(r0[cx.y * 3 + c]) * cx.w;
      const int h1 = int(r1[cx.x * 3 + c]) * cx.z + int(r1[cx.y * 3 + c]) * cx.w;
      const int u = ((((ry.z * (h0 >> 4)) >> 16) + ((ry.w * (h1 >> 4)) >> 16) + 2) >> 2) & 255;
      v[c] = __fdiv_rn(float(u), 255.f);   // ClipToTensor: float(u8) / 255
    }
    normalise_store(ob + idx, (long long)T * plane, v, mean, sdev);
  }
}

}  // namespace vj

extern "C" int vj_clip_preprocess(const void* src_u8, const void* params, void* out, int out_f32, int B, int T, int S,
                                  const float* mean3, const float* std3, void* stream_) {
  using namespace vj;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(src_u8 && params && out && mean3 && std3, "vj_clip_preprocess: null pointer");
  VJ_CHECK_ARG(B > 0 && T > 0 && S > 0, "vj_clip_preprocess: empty problem");
  VJ_CHECK_ARG((reinterpret_cast<uintptr_t>(params) & 7) == 0, "vj_clip_preprocess: params must be 8-byte aligned");
  const float3 mean255 = make_float3(mean3[0] * 255.f, mean3[1] * 255.f, mean3[2] * 255.f);       // host arrays
  const float3 istd = make_float3(std3[0] * 255.f, std3[1] * 255.f, std3[2] * 255.f);
  dim3 grid((S * S + 255) / 256, T, B);
  if (grid.x > 64) grid.x = 64;
  if (out_f32)
    clip_preprocess_kernel<float><<<grid, 256, 0, s>>>(reinterpret_cast<const uint8_t*>(src_u8),
                                                       reinterpret_cast<const ClipParam*>(params),
                                                       reinterpret_cast<float*>(out), T, S, mean255, istd);
  else
    clip_preprocess_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(reinterpret_cast<const uint8_t*>(src_u8),
                                                               reinterpret_cast<const ClipParam*>(params),
                                                               reinterpret_cast<__nv_bfloat16*>(out), T, S, mean255, istd);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}

extern "C" int vj_clip_views(const void* src_u8, const void* jobs, const void* tab, void* out, int out_f32, int n_jobs,
                             int T, int S, const float* mean3, const float* std3, void* stream_) {
  using namespace vj;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(src_u8 && jobs && tab && out && mean3 && std3, "vj_clip_views: null pointer");
  VJ_CHECK_ARG(n_jobs > 0 && T > 0 && S > 0, "vj_clip_views: empty problem");
  VJ_CHECK_ARG(n_jobs <= 65535 && T <= 65535, "vj_clip_views: more than 65535 views or frames in one launch");
  VJ_CHECK_ARG((reinterpret_cast<uintptr_t>(jobs) & 7) == 0 && (reinterpret_cast<uintptr_t>(tab) & 15) == 0,
               "vj_clip_views: jobs must be 8-byte and tab 16-byte aligned");
  const float3 mean = make_float3(mean3[0], mean3[1], mean3[2]);       // host arrays, fp32 as torch.as_tensor makes them
  const float3 sdev = make_float3(std3[0], std3[1], std3[2]);
  dim3 grid((S * S + 255) / 256, T, n_jobs);
  if (grid.x > 64) grid.x = 64;
  if (out_f32)
    clip_views_kernel<float><<<grid, 256, 0, s>>>(reinterpret_cast<const uint8_t*>(src_u8),
                                                  reinterpret_cast<const ViewJob*>(jobs), reinterpret_cast<const int4*>(tab),
                                                  reinterpret_cast<float*>(out), T, S, mean, sdev);
  else
    clip_views_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(reinterpret_cast<const uint8_t*>(src_u8),
                                                          reinterpret_cast<const ViewJob*>(jobs),
                                                          reinterpret_cast<const int4*>(tab),
                                                          reinterpret_cast<__nv_bfloat16*>(out), T, S, mean, sdev);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}
