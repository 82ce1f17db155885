// RandAugment (rand-m7-n4-mstd0.5-inc1) and random erasing (mode 'pixel', one box per clip) of the training transforms,
// on decoded uint8 frames, bit-exact with PIL 12 for every op.  Replaces, per frame on the CPU:
//   src/datasets/utils/video/randaugment.py:51-180  the 15 _RAND_INCREASING_TRANSFORMS (PIL ImageOps / ImageEnhance /
//       Image.transform(AFFINE, BICUBIC, fillcolor 128) / Image.rotate)
//   src/datasets/utils/video/randerase.py:116-156   RandomErasing._erase_cube (per-pixel N(0, 1) noise)
//   app/vjepa/transforms.py:86-115, evals/video_classification_frozen/utils.py:251-283  the pipelines around them
// The random decisions are drawn on the host in the reference's RNG order (jepa_b200/transforms.py) and arrive as tables.
//
// Per RandAugment layer: (1) when some clip's op needs one, a histogram pass (3 x 256 RGB bins + 256 bins of the L image
// per frame); (2) one pass over every (clip, frame) that applies the clip's op from one uint8 work buffer into the
// other.  A skipped op costs nothing: the host tracks which buffer holds each clip.  A last pass does the random-resized
// crop, flip, normalisation and erase (crop_bilinear3 / normalise_store, as vj_clip_preprocess).
//
// PIL's arithmetic, as pinned by tests/randaugment_numpy.py (a numpy restatement) against PIL's own outputs:
//   LUT ops    Invert, Posterize, Solarize, SolarizeAdd: integer LUTs.
//   AutoContrast   lo / hi = first / last non-empty bin; lut = trunc(i * (255.0 / (hi - lo)) + (-lo * scale)) in double.
//   Equalize   step = (n - count of the last non-empty bin) // 255; lut[i] = (step // 2 + sum(h[:i])) // step, <= 255.
//   Blends     Image.blend(degenerate, image, f): float32 d + f * (image - d), clipped and truncated.  Degenerate:
//              Color: L = (19595 R + 38470 G + 7471 B + 0x8000) >> 16; Contrast: int(mean(L) + 0.5) from the L
//              histogram; Brightness: 0; Sharpness: SMOOTH = (3 x 3 sum with centre weight 5 + 6) // 13, border copied.
//   Affine     Rotate / Shear / Translate: source = (m0 (x+.5) + m1 (y+.5) + m2, m3 (x+.5) + m4 (y+.5) + m5) in double,
//              outside the frame: the fill colour (128 for RandAugment, the launch's RGB for AutoAugment); else
//              PIL's bicubic (Geometry.c BICUBIC, clamped 4 x 4 taps) in double,
//              clipped and truncated.
// Every float / double operation that must round as PIL's compiled C does is an explicit _rn intrinsic, so no
// multiply-add is contracted.
#include <curand_kernel.h>

#include "preprocess.cuh"
#include "vjepa_b200.h"

namespace vj {

enum RaOp {   // jepa_b200.transforms.RA_OPS
  kAutoContrast, kEqualize, kInvert, kRotate, kPosterize, kSolarize, kSolarizeAdd, kColor, kContrast, kBrightness,
  kSharpness, kShearX, kShearY, kTranslateX, kTranslateY
};

constexpr int kBins = 1024;   // R, G, B, L histograms of one frame

__device__ __forceinline__ int luma(int r, int g, int b) { return (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16; }

__device__ __forceinline__ bool needs_hist(int code) {
  return code == kAutoContrast || code == kEqualize || code == kContrast;
}

__global__ void __launch_bounds__(256) ra_hist_kernel(const uint8_t* __restrict__ buf0, const uint8_t* __restrict__ buf1,
                                                      const AugClip* __restrict__ clips, const AugOp* __restrict__ ops,
                                                      int* __restrict__ hist, int T) {
  const int b = blockIdx.z, t = blockIdx.y;
  const AugOp op = ops[b];
  if (!needs_hist(op.code)) return;
  const AugClip cl = clips[b];
  const long long npx = (long long)cl.H * cl.W;
  const uint8_t* f = (op.in_buf ? buf1 : buf0) + cl.off + t * npx * 3;
  __shared__ int sh[kBins];
  for (int k = threadIdx.x; k < kBins; k += blockDim.x) sh[k] = 0;
  __syncthreads();
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < npx; p += (long long)gridDim.x * blockDim.x) {
    const int r = f[p * 3], g = f[p * 3 + 1], bl = f[p * 3 + 2];
    atomicAdd(&sh[r], 1);
    atomicAdd(&sh[256 + g], 1);
    atomicAdd(&sh[512 + bl], 1);
    atomicAdd(&sh[768 + luma(r, g, bl)], 1);
  }
  __syncthreads();
  int* gh = hist + ((long long)b * T + t) * kBins;
  for (int k = threadIdx.x; k < kBins; k += blockDim.x)
    if (sh[k]) atomicAdd(&gh[k], sh[k]);
}

// PIL's bicubic row / column interpolation (Geometry.c BICUBIC), evaluated left to right in double
__device__ __forceinline__ double cubic(double v1, double v2, double v3, double v4, double d) {
  const double p1 = v2;
  const double p2 = __dadd_rn(-v1, v3);
  const double p3 = __dsub_rn(__dadd_rn(__dmul_rn(2.0, __dsub_rn(v1, v2)), v3), v4);
  const double p4 = __dadd_rn(__dsub_rn(__dadd_rn(-v1, v2), v3), v4);
  return __dadd_rn(p1, __dmul_rn(d, __dadd_rn(p2, __dmul_rn(d, __dadd_rn(p3, __dmul_rn(d, p4))))));
}

__device__ __forceinline__ uint8_t clip_trunc(double v) { return v <= 0.0 ? 0 : (v >= 255.0 ? 255 : (uint8_t)v); }

__device__ __forceinline__ uint8_t blend(int d, int v, float a) {   // Image.blend(degenerate, image, a)
  const float t = __fadd_rn(float(d), __fmul_rn(a, float(v - d)));
  return t <= 0.f ? 0 : (t >= 255.f ? 255 : (uint8_t)t);
}

__global__ void __launch_bounds__(256) ra_apply_kernel(uint8_t* __restrict__ buf0, uint8_t* __restrict__ buf1,
                                                       const AugClip* __restrict__ clips, const AugOp* __restrict__ ops,
                                                       const int* __restrict__ hist, int T, uchar3 fill) {
  const int b = blockIdx.z, t = blockIdx.y;
  const AugOp op = ops[b];
  if (op.code < 0) return;
  const AugClip cl = clips[b];
  const int H = cl.H, W = cl.W;
  const long long npx = (long long)H * W;
  const uint8_t* in = (op.in_buf ? buf1 : buf0) + cl.off + t * npx * 3;
  uint8_t* out = (op.in_buf ? buf0 : buf1) + cl.off + t * npx * 3;

  __shared__ uint8_t lut[3][256];
  __shared__ int scan[3][256], lo[3], hi[3], last[3], nz[3];
  __shared__ long long lsum;
  const int code = op.code, tid = threadIdx.x;
  int mean = 0;
  if (needs_hist(code)) {               // per-frame LUT (AutoContrast, Equalize) or L mean (Contrast)
    const int* h = hist + ((long long)b * T + t) * kBins;
    if (tid < 3) { lo[tid] = 256; hi[tid] = -1; nz[tid] = 0; }
    if (tid == 0) lsum = 0;
    __syncthreads();
    if (code == kContrast) {
      atomicAdd((unsigned long long*)&lsum, (unsigned long long)((long long)tid * h[768 + tid]));
      __syncthreads();
      mean = int(__dadd_rn(__ddiv_rn(double(lsum), double(npx)), 0.5));   // ImageStat mean, int(mean + 0.5)
    } else {
      for (int c = 0; c < 3; ++c) {
        const int v = h[c * 256 + tid];
        scan[c][tid] = v;
        if (v) { atomicMin(&lo[c], tid); atomicMax(&hi[c], tid); atomicAdd(&nz[c], 1); }
      }
      __syncthreads();
      if (code == kEqualize) {
        if (tid < 3) last[tid] = hi[tid] >= 0 ? scan[tid][hi[tid]] : 0;
        for (int o = 1; o < 256; o <<= 1) {       // inclusive prefix sums (Hillis-Steele)
          int v[3];
          for (int c = 0; c < 3; ++c) v[c] = tid >= o ? scan[c][tid - o] : 0;
          __syncthreads();
          for (int c = 0; c < 3; ++c) scan[c][tid] += v[c];
          __syncthreads();
        }
        for (int c = 0; c < 3; ++c) {
          const int step = nz[c] > 1 ? int((npx - last[c]) / 255) : 0;
          const int excl = tid ? scan[c][tid - 1] : 0;
          lut[c][tid] = step ? (uint8_t)min(255, (step / 2 + excl) / step) : (uint8_t)tid;
        }
      } else {
        for (int c = 0; c < 3; ++c) {
          int v = tid;
          if (hi[c] > lo[c]) {
            const double scale = __ddiv_rn(255.0, double(hi[c] - lo[c]));
            const double offset = __dmul_rn(double(-lo[c]), scale);
            const double x = __dadd_rn(__dmul_rn(double(tid), scale), offset);
            v = x < 0.0 ? 0 : min(255, int(x));
          }
          lut[c][tid] = (uint8_t)v;
        }
      }
    }
    __syncthreads();
  }

  const bool geometric = code == kRotate || code >= kShearX;
  const float a = op.fval;
  for (long long p = blockIdx.x * (long long)blockDim.x + tid; p < npx; p += (long long)gridDim.x * blockDim.x) {
    const int y = int(p / W), x = int(p - (long long)y * W);
    const uint8_t* px = in + p * 3;
    uint8_t* o = out + p * 3;
    if (geometric) {
      const double xs = double(x) + 0.5, ys = double(y) + 0.5;
      const double xin = __dadd_rn(__dadd_rn(__dmul_rn(op.m[0], xs), __dmul_rn(op.m[1], ys)), op.m[2]);
      const double yin = __dadd_rn(__dadd_rn(__dmul_rn(op.m[3], xs), __dmul_rn(op.m[4], ys)), op.m[5]);
      if (!(xin >= 0.0 && xin < double(W) && yin >= 0.0 && yin < double(H))) {
        o[0] = fill.x; o[1] = fill.y; o[2] = fill.z;
        continue;
      }
      const double xi = __dsub_rn(xin, 0.5), yi = __dsub_rn(yin, 0.5);
      const double fx = floor(xi), fy = floor(yi);
      const double dx = __dsub_rn(xi, fx), dy = __dsub_rn(yi, fy);
      const int x0 = int(fx) - 1, y0 = int(fy) - 1;
      int cx[4], ry[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        cx[k] = min(max(x0 + k, 0), W - 1) * 3;
        ry[k] = min(max(y0 + k, 0), H - 1);
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        double v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint8_t* row = in + (long long)ry[k] * W * 3 + c;
          v[k] = cubic(row[cx[0]], row[cx[1]], row[cx[2]], row[cx[3]], dx);
        }
        o[c] = clip_trunc(cubic(v[0], v[1], v[2], v[3], dy));
      }
      continue;
    }
    const int r = px[0], g = px[1], bl = px[2];
    int d[3] = {0, 0, 0};
    switch (code) {
      case kAutoContrast:
      case kEqualize:
        o[0] = lut[0][r]; o[1] = lut[1][g]; o[2] = lut[2][bl];
        continue;
      case kInvert:
        o[0] = 255 - r; o[1] = 255 - g; o[2] = 255 - bl;
        continue;
      case kPosterize: {
        const int mask = ~((1 << (8 - op.ival)) - 1) & 255;
        o[0] = r & mask; o[1] = g & mask; o[2] = bl & mask;
        continue;
      }
      case kSolarize:
        o[0] = r < op.ival ? r : 255 - r; o[1] = g < op.ival ? g : 255 - g; o[2] = bl < op.ival ? bl : 255 - bl;
        continue;
      case kSolarizeAdd:
        o[0] = r < 128 ? min(255, r + op.ival) : r;
        o[1] = g < 128 ? min(255, g + op.ival) : g;
        o[2] = bl < 128 ? min(255, bl + op.ival) : bl;
        continue;
      case kColor:
        d[0] = d[1] = d[2] = luma(r, g, bl);
        break;
      case kContrast:
        d[0] = d[1] = d[2] = mean;
        break;
      case kBrightness:
        break;
      case kSharpness:
        if (y == 0 || x == 0 || y == H - 1 || x == W - 1) {
          d[0] = r; d[1] = g; d[2] = bl;
        } else {
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            int s = 0;
#pragma unroll
            for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
              for (int dx = -1; dx <= 1; ++dx) s += int(px[((long long)dy * W + dx) * 3 + c]);
            s += 4 * int(px[c]);
            d[c] = (s + 6) / 13;
          }
        }
        break;
    }
    o[0] = blend(d[0], r, a); o[1] = blend(d[1], g, a); o[2] = blend(d[2], bl, a);
  }
}

// Crop, flip, normalise, erase: [B, 3, T, S, S].  Erase noise: Philox4x32-10 keyed by the clip's seed, one subsequence
// per (frame, output pixel), three normals (Box-Muller) for the three channels.
template <typename TO>
__global__ void __launch_bounds__(256) augment_final_kernel(const uint8_t* __restrict__ buf0,
                                                            const uint8_t* __restrict__ buf1,
                                                            const AugClip* __restrict__ clips, TO* __restrict__ out, int T,
                                                            int S, float3 mean255, float3 std255) {
  const int b = blockIdx.z, t = blockIdx.y;
  const AugClip cl = clips[b];
  const uint8_t* frame = (cl.final_buf ? buf1 : buf0) + cl.off + (long long)t * cl.H * cl.W * 3;
  const float sh = float(cl.h) / float(S), sw = float(cl.w) / float(S);
  const long long plane = (long long)S * S;
  TO* ob = out + ((long long)b * 3 * T + t) * plane;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < S * S; idx += gridDim.x * blockDim.x) {
    const int y = idx / S, xo = idx - y * S;
    if (cl.eh && y >= cl.etop && y < cl.etop + cl.eh && xo >= cl.eleft && xo < cl.eleft + cl.ew) {
      curandStatePhilox4_32_10_t st;
      curand_init(cl.seed, (unsigned long long)t * plane + idx, 0, &st);
      const float4 n = curand_normal4(&st);
      ob[idx] = TO(n.x);
      ob[idx + (long long)T * plane] = TO(n.y);
      ob[idx + 2 * (long long)T * plane] = TO(n.z);
      continue;
    }
    const int x = cl.flip ? (S - 1 - xo) : xo;
    float v[3];
    crop_bilinear3(frame, cl.W, cl.i, cl.j, cl.h, cl.w, sh, sw, y, x, v);
    normalise_store(ob + idx, (long long)T * plane, v, mean255, std255);
  }
}

// The RandAugment / AutoAugment layers of one batch: per layer an optional histogram pass and one apply pass over every
// (clip, frame), ping-ponging between b0 and b1 as the ops' in_buf fields say.  Shared by vj_clip_augment and
// vj_image_augment (image.cu); geometric ops fill uncovered pixels with `fill`.
int ra_layers(uint8_t* b0, uint8_t* b1, const void* clips, const void* ops, void* hist, const int* layer_flags,
              int n_layers, int B, int T, uchar3 fill, cudaStream_t s) {
  const auto* cl = reinterpret_cast<const AugClip*>(clips);
  for (int l = 0; l < n_layers; ++l) {
    if (!(layer_flags[l] & 1)) continue;                 // every op of this layer skipped
    const auto* op = reinterpret_cast<const AugOp*>(ops) + (long long)l * B;
    int* h = reinterpret_cast<int*>(hist) + (long long)l * B * T * kBins;
    const dim3 grid(32, T, B);
    if (layer_flags[l] & 2) {                             // some op of this layer reads the frame's histogram
      VJ_CUDA(cudaMemsetAsync(h, 0, sizeof(int) * (size_t)B * T * kBins, s));
      ra_hist_kernel<<<grid, 256, 0, s>>>(b0, b1, cl, op, h, T);
      VJ_CUDA(cudaGetLastError());
      vj::count_launch(1);
    }
    ra_apply_kernel<<<grid, 256, 0, s>>>(b0, b1, cl, op, h, T, fill);
    VJ_CUDA(cudaGetLastError());
    vj::count_launch(1);
  }
  return 0;
}

}  // namespace vj

extern "C" int vj_clip_augment(void* buf0, void* buf1, const void* clips, const void* ops, void* hist,
                               const int* layer_flags, int n_layers, void* out, int out_f32, int B, int T, int S,
                               const float* mean3, const float* std3, void* stream_) {
  using namespace vj;
  static_assert(sizeof(AugClip) == 64 && sizeof(AugOp) == 64, "record layout shared with jepa_b200/transforms.py");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(buf0 && buf1 && clips && out && mean3 && std3, "vj_clip_augment: null pointer");
  VJ_CHECK_ARG(n_layers >= 0 && n_layers <= 16, "vj_clip_augment: n_layers must be in [0, 16]");
  VJ_CHECK_ARG(n_layers == 0 || (ops && hist && layer_flags), "vj_clip_augment: null ops / hist / layer_flags");
  VJ_CHECK_ARG(B > 0 && T > 0 && S > 0, "vj_clip_augment: empty problem");
  VJ_CHECK_ARG(B <= 65535 && T <= 65535, "vj_clip_augment: more than 65535 clips or frames in one launch");
  VJ_CHECK_ARG((reinterpret_cast<uintptr_t>(clips) & 15) == 0 && (reinterpret_cast<uintptr_t>(ops) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(hist) & 15) == 0,
               "vj_clip_augment: clips, ops and hist must be 16-byte aligned");
  auto* b0 = reinterpret_cast<uint8_t*>(buf0);
  auto* b1 = reinterpret_cast<uint8_t*>(buf1);
  const auto* cl = reinterpret_cast<const AugClip*>(clips);
  if (const int rc = ra_layers(b0, b1, clips, ops, hist, layer_flags, n_layers, B, T, make_uchar3(128, 128, 128), s))
    return rc;
  const float3 mean255 = make_float3(mean3[0] * 255.f, mean3[1] * 255.f, mean3[2] * 255.f);       // host arrays
  const float3 std255 = make_float3(std3[0] * 255.f, std3[1] * 255.f, std3[2] * 255.f);
  dim3 grid((S * S + 255) / 256, T, B);
  if (grid.x > 64) grid.x = 64;
  if (out_f32)
    augment_final_kernel<float><<<grid, 256, 0, s>>>(b0, b1, cl, reinterpret_cast<float*>(out), T, S, mean255, std255);
  else
    augment_final_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(b0, b1, cl, reinterpret_cast<__nv_bfloat16*>(out), T, S,
                                                             mean255, std255);
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}
