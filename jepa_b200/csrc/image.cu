// Frozen image evaluation transforms on decoded uint8 RGB images of mixed sizes, bit-exact with PIL 12 / torchvision:
//   validation  Resize(int(S * 256 / 224)) (PIL BILINEAR) -> CenterCrop(S) -> ToTensor -> Normalize       (vj_image_views)
//   training    RandomResizedCropAndInterpolation(S, bicubic) -> RandomHorizontalFlip -> AutoAugment 'original'
//               (fill (124, 116, 104)) -> ToTensor -> Normalize -> RandomErasing('pixel')                (vj_image_augment)
// Replaces, per image on the CPU, reference evals/image_classification_frozen/eval.py:392-409 (timm's create_transform
// and the torchvision validation Compose).  Decisions (crop box, flip, AutoAugment ops, erase box and its N(0, 1) noise)
// are drawn on the host in the reference's RNG order (jepa_b200/image_transforms.py) and arrive as tables.
//
// Resampling is PIL's Resample.c for 8-bit images: a horizontal pass into a uint8 intermediate over the source rows the
// vertical pass reads, then the vertical pass.  Per output pixel and axis the host supplies {first tap, tap count,
// int32 weights} (precompute_coeffs + normalize_coeffs_8bpc, 22 fractional bits); a pass PIL skips is an identity table
// ({x, 1, 1 << 22}), which reproduces the copy exactly.  Accumulation starts at 1 << 21 in int32, the result is >> 22
// and clamped.  Only the S x S window that is kept is computed.
//
// Normalisation is torchvision's CPU arithmetic, every step an fp32 round-to-nearest: (v / 255 - mean) / std.
#include "preprocess.cuh"
#include "vjepa_b200.h"

namespace vj {

struct ImgJob {          // per image, 64 bytes (jepa_b200/image_transforms.py IMG_JOB)
  long long src_off;     // byte offset of the image [H, W, 3] in src
  long long tmp_off;     // byte offset of its horizontal-pass rows [nrows, S, 3] in tmp
  int W;                 // source row length in pixels
  int r0, nrows;         // source rows the vertical pass reads: [r0, r0 + nrows)
  int c0;                // source column the horizontal taps count from
  int xtab, ytab;        // int32 offsets of the S column / S row coefficient entries in coefs
  int xk, yk;            // entry strides (2 + taps)
  int flip;              // training: the resized image is written mirrored
  int pad[3];
};

constexpr int kPrec = 22;   // Resample.c PRECISION_BITS for 8-bit images

__device__ __forceinline__ uint8_t clip8(int v) {
  v >>= kPrec;
  return v < 0 ? 0 : (v > 255 ? 255 : (uint8_t)v);
}

__global__ void __launch_bounds__(256) resample_h_kernel(const uint8_t* __restrict__ src, const ImgJob* __restrict__ jobs,
                                                         const int* __restrict__ coefs, uint8_t* __restrict__ tmp, int S) {
  const ImgJob jb = jobs[blockIdx.y];
  const int n = jb.nrows * S;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += gridDim.x * blockDim.x) {
    const int r = idx / S, x = idx - r * S;
    const int* e = coefs + jb.xtab + x * jb.xk;
    const uint8_t* p = src + jb.src_off + ((long long)(jb.r0 + r) * jb.W + jb.c0 + e[0]) * 3;
    int a0 = 1 << (kPrec - 1), a1 = a0, a2 = a0;
    for (int k = 0; k < e[1]; ++k) {
      const int w = e[2 + k];
      a0 += int(p[3 * k]) * w;
      a1 += int(p[3 * k + 1]) * w;
      a2 += int(p[3 * k + 2]) * w;
    }
    uint8_t* o = tmp + jb.tmp_off + (long long)idx * 3;
    o[0] = clip8(a0);
    o[1] = clip8(a1);
    o[2] = clip8(a2);
  }
}

// Vertical pass at output pixel (y, x) of the S x S window, from the horizontal pass's rows
__device__ __forceinline__ void resample_v3(const ImgJob& jb, const int* __restrict__ coefs, const uint8_t* __restrict__ tmp,
                                            int S, int y, int x, int (&v)[3]) {
  const int* e = coefs + jb.ytab + y * jb.yk;
  const uint8_t* p = tmp + jb.tmp_off + ((long long)e[0] * S + x) * 3;
  int a0 = 1 << (kPrec - 1), a1 = a0, a2 = a0;
  for (int k = 0; k < e[1]; ++k) {
    const int w = e[2 + k];
    const uint8_t* q = p + (long long)k * S * 3;
    a0 += int(q[0]) * w;
    a1 += int(q[1]) * w;
    a2 += int(q[2]) * w;
  }
  v[0] = clip8(a0);
  v[1] = clip8(a1);
  v[2] = clip8(a2);
}

// torchvision ToTensor + Normalize of one uint8 RGB pixel into the channel planes of [3, S, S]
template <typename TO>
__device__ __forceinline__ void to_tensor_normalise(TO* dst, long long cstride, const int (&v)[3], float3 mean, float3 std) {
  dst[0] = TO(__fdiv_rn(__fsub_rn(__fdiv_rn(float(v[0]), 255.f), mean.x), std.x));
  dst[cstride] = TO(__fdiv_rn(__fsub_rn(__fdiv_rn(float(v[1]), 255.f), mean.y), std.y));
  dst[2 * cstride] = TO(__fdiv_rn(__fsub_rn(__fdiv_rn(float(v[2]), 255.f), mean.z), std.z));
}

// Validation: vertical pass, then ToTensor + Normalize into out [B, 3, S, S]
template <typename TO>
__global__ void __launch_bounds__(256) resample_v_norm_kernel(const ImgJob* __restrict__ jobs, const int* __restrict__ coefs,
                                                              const uint8_t* __restrict__ tmp, TO* __restrict__ out, int S,
                                                              float3 mean, float3 std) {
  const int b = blockIdx.y;
  const ImgJob jb = jobs[b];
  const long long plane = (long long)S * S;
  TO* ob = out + (long long)b * 3 * plane;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < S * S; idx += gridDim.x * blockDim.x) {
    const int y = idx / S, x = idx - y * S;
    int v[3];
    resample_v3(jb, coefs, tmp, S, y, x, v);
    to_tensor_normalise(ob + idx, plane, v, mean, std);
  }
}

// Training: vertical pass, written (mirrored when flipped) as the uint8 image [S, S, 3] the AutoAugment layers read
__global__ void __launch_bounds__(256) resample_v_u8_kernel(const ImgJob* __restrict__ jobs, const int* __restrict__ coefs,
                                                            const uint8_t* __restrict__ tmp, uint8_t* __restrict__ dst,
                                                            int S) {
  const int b = blockIdx.y;
  const ImgJob jb = jobs[b];
  uint8_t* db = dst + (long long)b * S * S * 3;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < S * S; idx += gridDim.x * blockDim.x) {
    const int y = idx / S, x = idx - y * S;
    int v[3];
    resample_v3(jb, coefs, tmp, S, y, x, v);
    uint8_t* o = db + ((long long)y * S + (jb.flip ? S - 1 - x : x)) * 3;
    o[0] = (uint8_t)v[0];
    o[1] = (uint8_t)v[1];
    o[2] = (uint8_t)v[2];
  }
}

// Training, last pass: ToTensor + Normalize of the AutoAugment output, the erase box copied from the host's noise
template <typename TO>
__global__ void __launch_bounds__(256) image_final_kernel(const uint8_t* __restrict__ buf0, const uint8_t* __restrict__ buf1,
                                                          const AugClip* __restrict__ clips, const float* __restrict__ noise,
                                                          TO* __restrict__ out, int S, float3 mean, float3 std) {
  const int b = blockIdx.y;
  const AugClip cl = clips[b];
  const uint8_t* img = (cl.final_buf ? buf1 : buf0) + cl.off;
  const long long plane = (long long)S * S;
  TO* ob = out + (long long)b * 3 * plane;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < S * S; idx += gridDim.x * blockDim.x) {
    const int y = idx / S, x = idx - y * S;
    if (cl.eh && y >= cl.etop && y < cl.etop + cl.eh && x >= cl.eleft && x < cl.eleft + cl.ew) {
      const long long area = (long long)cl.eh * cl.ew;
      const float* n = noise + cl.seed + (long long)(y - cl.etop) * cl.ew + (x - cl.eleft);
      ob[idx] = TO(n[0]);
      ob[idx + plane] = TO(n[area]);
      ob[idx + 2 * plane] = TO(n[2 * area]);
      continue;
    }
    const uint8_t* p = img + (long long)idx * 3;
    const int v[3] = {p[0], p[1], p[2]};
    to_tensor_normalise(ob + idx, plane, v, mean, std);
  }
}

inline dim3 image_grid(int S, int B) {
  int gx = (S * S + 255) / 256;
  return dim3(gx > 64 ? 64 : gx, B);
}

}  // namespace vj

extern "C" int vj_image_views(const void* src_u8, const void* jobs, const void* coefs, void* tmp, void* out, int out_f32,
                              int B, int S, const float* mean3, const float* std3, void* stream_) {
  using namespace vj;
  static_assert(sizeof(ImgJob) == 64, "record layout shared with jepa_b200/image_transforms.py");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(src_u8 && jobs && coefs && tmp && out && mean3 && std3, "vj_image_views: null pointer");
  VJ_CHECK_ARG(B > 0 && S > 0, "vj_image_views: empty problem");
  VJ_CHECK_ARG(B <= 65535, "vj_image_views: more than 65535 images in one launch");
  VJ_CHECK_ARG((reinterpret_cast<uintptr_t>(jobs) & 15) == 0 && (reinterpret_cast<uintptr_t>(coefs) & 3) == 0,
               "vj_image_views: jobs must be 16-byte and coefs 4-byte aligned");
  const auto* jb = reinterpret_cast<const ImgJob*>(jobs);
  const auto* cf = reinterpret_cast<const int*>(coefs);
  const dim3 grid = image_grid(S, B);
  resample_h_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const uint8_t*>(src_u8), jb, cf, reinterpret_cast<uint8_t*>(tmp), S);
  VJ_CUDA(cudaGetLastError());
  const float3 mean = make_float3(mean3[0], mean3[1], mean3[2]);      // host arrays
  const float3 std = make_float3(std3[0], std3[1], std3[2]);
  const auto* t = reinterpret_cast<const uint8_t*>(tmp);
  if (out_f32)
    resample_v_norm_kernel<float><<<grid, 256, 0, s>>>(jb, cf, t, reinterpret_cast<float*>(out), S, mean, std);
  else
    resample_v_norm_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(jb, cf, t, reinterpret_cast<__nv_bfloat16*>(out), S, mean,
                                                                std);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(2);
  return 0;
}

extern "C" int vj_image_augment(const void* src_u8, const void* jobs, const void* coefs, void* tmp, void* buf0, void* buf1,
                                const void* clips, const void* ops, void* hist, const int* layer_flags, int n_layers,
                                const float* noise, void* out, int out_f32, int B, int S, const float* mean3,
                                const float* std3, const unsigned char* fill3, void* stream_) {
  using namespace vj;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(src_u8 && jobs && coefs && tmp && buf0 && buf1 && clips && out && mean3 && std3 && fill3,
               "vj_image_augment: null pointer");
  VJ_CHECK_ARG(n_layers >= 0 && n_layers <= 16, "vj_image_augment: n_layers must be in [0, 16]");
  VJ_CHECK_ARG(n_layers == 0 || (ops && hist && layer_flags), "vj_image_augment: null ops / hist / layer_flags");
  VJ_CHECK_ARG(B > 0 && S > 0, "vj_image_augment: empty problem");
  VJ_CHECK_ARG(B <= 65535, "vj_image_augment: more than 65535 images in one launch");
  VJ_CHECK_ARG((reinterpret_cast<uintptr_t>(jobs) & 15) == 0 && (reinterpret_cast<uintptr_t>(clips) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(ops) & 15) == 0 && (reinterpret_cast<uintptr_t>(hist) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(coefs) & 3) == 0 && (reinterpret_cast<uintptr_t>(noise) & 3) == 0,
               "vj_image_augment: jobs, clips, ops and hist must be 16-byte and coefs, noise 4-byte aligned");
  const auto* jb = reinterpret_cast<const ImgJob*>(jobs);
  const auto* cf = reinterpret_cast<const int*>(coefs);
  auto* b0 = reinterpret_cast<uint8_t*>(buf0);
  auto* b1 = reinterpret_cast<uint8_t*>(buf1);
  const dim3 grid = image_grid(S, B);
  resample_h_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const uint8_t*>(src_u8), jb, cf, reinterpret_cast<uint8_t*>(tmp), S);
  VJ_CUDA(cudaGetLastError());
  resample_v_u8_kernel<<<grid, 256, 0, s>>>(jb, cf, reinterpret_cast<const uint8_t*>(tmp), b0, S);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(2);
  if (const int rc = ra_layers(b0, b1, clips, ops, hist, layer_flags, n_layers, B, 1,
                               make_uchar3(fill3[0], fill3[1], fill3[2]), s))
    return rc;
  const float3 mean = make_float3(mean3[0], mean3[1], mean3[2]);      // host arrays
  const float3 std = make_float3(std3[0], std3[1], std3[2]);
  const auto* cl = reinterpret_cast<const AugClip*>(clips);
  if (out_f32)
    image_final_kernel<float><<<grid, 256, 0, s>>>(b0, b1, cl, noise, reinterpret_cast<float*>(out), S, mean, std);
  else
    image_final_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(b0, b1, cl, noise, reinterpret_cast<__nv_bfloat16*>(out), S,
                                                           mean, std);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}
