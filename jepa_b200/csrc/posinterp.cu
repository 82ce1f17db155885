// Positional-embedding resampling for encoder inputs at a size other than the one the encoder was built for
// (VisionTransformer.interpolate_pos_encoding, src/models/vision_transformer.py:197-246): the fp32 sin-cos table
// [Nt, Nh, Nw, D] becomes [T', H', W', D], the tensor the patch-embed GEMM epilogue adds to every token.
//
//   mode 3  video: F.interpolate(mode='trilinear', scale_factor=(T/Nt, H/Nh, W/Nw), align_corners=False)
//   mode 2  image: F.interpolate(mode='bicubic', scale_factor=sqrt(npatch / N)) on a square grid (Nt = T' = 1)
//
// Bit-exact with torch's CPU kernels (aten/src/ATen/native/cpu/UpSampleKernel.cpp, UpSample.h) as they are compiled
// for x86-64: every operation below is an fp32 round-to-nearest intrinsic, and the places where the compiler fused a
// multiply and an add into one FMA in torch's build are written as __fmaf_rn, the others as separate _rn operations,
// so nvcc contracts nothing on its own.
//   scale        s = (float)(1.0 / scale_factor)  (compute_scales_value; not in / out)
//   source       r = fma(s, dst + 0.5, -0.5)       (area_pixel_compute_source_index)
//   trilinear    r < 0 -> 0; i0 = min(floor(r), in - 1), l1 = clamp(r - i0, 0, 1), i1 = min(i0 + 1, in - 1),
//                l0 = 1 - l1; an axis whose size does not change is a copy (l0 = 1, l1 = 0); corner weights
//                (ld * lh) * lw; the 8 corners are summed as t0 w0 + (t1 w1 + (... + (t6 w6 + t7 w7))) with every
//                step an FMA (cpu_upsample_linear_channels_last: the permuted table is channels-last)
//   bicubic      no clamp of r; taps i0 - 1 .. i0 + 2 clamped into [0, in - 1]; A = -0.75 weights
//                (get_cubic_upsample_coefficients); the W taps are summed first, then the H taps, each as
//                fma(x0, w0, x1 w1) -> fma(x2, w2, .) -> fma(x3, w3, .)  (upsample_generic_Nd_kernel_impl)
// One thread per float4 of an output row: the table is at most tens of MB and the kernel is HBM-bound.
#include "common.cuh"
#include "vjepa_b200.h"

namespace vj {

struct LinTap {
  int i0, i1;
  float l0, l1;
};

VJ_DEVINL float src_coord(float s, int dst) { return __fmaf_rn(s, __fadd_rn(float(dst), 0.5f), -0.5f); }

VJ_DEVINL LinTap linear_tap(int dst, int n_in, int n_out, float s) {
  LinTap t;
  if (n_in == n_out) {  // compute_source_index_and_lambda: same size, plain copy
    t.i0 = t.i1 = dst;
    t.l0 = 1.f;
    t.l1 = 0.f;
    return t;
  }
  float r = src_coord(s, dst);
  if (r < 0.f) r = 0.f;
  t.i0 = min(int(floorf(r)), n_in - 1);
  t.l1 = fminf(fmaxf(__fsub_rn(r, float(t.i0)), 0.f), 1.f);
  t.i1 = t.i0 + (t.i0 < n_in - 1 ? 1 : 0);
  t.l0 = __fsub_rn(1.f, t.l1);
  return t;
}

// cubic_convolution1 / cubic_convolution2 with A = -0.75: (A + 2) = 1.25, (A + 3) = 2.25, 5A = -3.75, 8A = -6, 4A = -3
VJ_DEVINL float cubic1(float x) {
  return __fadd_rn(__fmul_rn(__fmul_rn(__fmaf_rn(1.25f, x, -2.25f), x), x), 1.f);
}
VJ_DEVINL float cubic2(float x) {
  return __fsub_rn(__fmul_rn(__fmaf_rn(__fmaf_rn(-0.75f, x, 3.75f), x, -6.f), x), -3.f);
}

VJ_DEVINL void cubic_taps(int dst, int n_in, float s, int idx[4], float w[4]) {
  const float r = src_coord(s, dst);
  const int i0 = min(int(floorf(r)), n_in - 1);
  const float t = fminf(fmaxf(__fsub_rn(r, float(i0)), 0.f), 1.f);
  const float x2 = __fsub_rn(1.f, t);
  w[0] = cubic2(__fadd_rn(t, 1.f));
  w[1] = cubic1(t);
  w[2] = cubic1(x2);
  w[3] = cubic2(__fadd_rn(x2, 1.f));
#pragma unroll
  for (int j = 0; j < 4; ++j) idx[j] = max(min(i0 + j - 1, n_in - 1), 0);
}

VJ_DEVINL float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

VJ_DEVINL float4 fma4(float4 a, float w, float4 c) {
  return make_float4(__fmaf_rn(a.x, w, c.x), __fmaf_rn(a.y, w, c.y), __fmaf_rn(a.z, w, c.z), __fmaf_rn(a.w, w, c.w));
}

VJ_DEVINL float4 mul4(float4 a, float w) {
  return make_float4(__fmul_rn(a.x, w), __fmul_rn(a.y, w), __fmul_rn(a.z, w), __fmul_rn(a.w, w));
}

// sum of 4 taps: fma(x0, w0, x1 w1), then + x2 w2, + x3 w3 (each an FMA)
VJ_DEVINL float4 sum4(const float4 v[4], const float w[4]) {
  float4 a = fma4(v[0], w[0], mul4(v[1], w[1]));
  a = fma4(v[2], w[2], a);
  return fma4(v[3], w[3], a);
}

__global__ void __launch_bounds__(256) pos_interp_trilinear_kernel(const float* __restrict__ in, float* __restrict__ out,
                                                                   int Nt, int Nh, int Nw, int T, int H, int W, int D,
                                                                   float st, float sh, float sw) {
  const int q = D >> 2;
  const long long total = (long long)T * H * W * q;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = int(i % q) * 4;
  const long long p = i / q;
  const int ow = int(p % W), oh = int((p / W) % H), ot = int(p / ((long long)W * H));
  const LinTap a = linear_tap(ot, Nt, T, st), b = linear_tap(oh, Nh, H, sh), e = linear_tap(ow, Nw, W, sw);
  const float w000 = __fmul_rn(__fmul_rn(a.l0, b.l0), e.l0), w001 = __fmul_rn(__fmul_rn(a.l0, b.l0), e.l1);
  const float w010 = __fmul_rn(__fmul_rn(a.l0, b.l1), e.l0), w011 = __fmul_rn(__fmul_rn(a.l0, b.l1), e.l1);
  const float w100 = __fmul_rn(__fmul_rn(a.l1, b.l0), e.l0), w101 = __fmul_rn(__fmul_rn(a.l1, b.l0), e.l1);
  const float w110 = __fmul_rn(__fmul_rn(a.l1, b.l1), e.l0), w111 = __fmul_rn(__fmul_rn(a.l1, b.l1), e.l1);
  auto at = [&](int t, int h, int w) { return ld4(in + (((long long)t * Nh + h) * Nw + w) * D + c); };
  float4 acc = fma4(at(a.i1, b.i1, e.i1), w111, mul4(at(a.i1, b.i1, e.i0), w110));
  acc = fma4(at(a.i1, b.i0, e.i1), w101, acc);
  acc = fma4(at(a.i1, b.i0, e.i0), w100, acc);
  acc = fma4(at(a.i0, b.i1, e.i1), w011, acc);
  acc = fma4(at(a.i0, b.i1, e.i0), w010, acc);
  acc = fma4(at(a.i0, b.i0, e.i1), w001, acc);
  acc = fma4(at(a.i0, b.i0, e.i0), w000, acc);
  *reinterpret_cast<float4*>(out + p * D + c) = acc;
}

__global__ void __launch_bounds__(256) pos_interp_bicubic_kernel(const float* __restrict__ in, float* __restrict__ out,
                                                                 int Nh, int Nw, int H, int W, int D, float sh, float sw) {
  const int q = D >> 2;
  const long long total = (long long)H * W * q;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = int(i % q) * 4;
  const long long p = i / q;
  const int ow = int(p % W), oh = int(p / W);
  int hi[4], wi[4];
  float hw[4], ww[4];
  cubic_taps(oh, Nh, sh, hi, hw);
  cubic_taps(ow, Nw, sw, wi, ww);
  float4 rows[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float4 v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = ld4(in + ((long long)hi[j] * Nw + wi[k]) * D + c);
    rows[j] = sum4(v, ww);
  }
  *reinterpret_cast<float4*>(out + p * D + c) = sum4(rows, hw);
}

}  // namespace vj

using namespace vj;

// output size of torch's scale_factor path: (int64_t)(in * scale) in double (compute_output_size)
static int scaled_size(int n, double scale) { return int((long long)(double(n) * scale)); }

extern "C" int vj_pos_interp(const float* in, float* out, int Nt, int Nh, int Nw, int T, int H, int W, int D,
                             double scale_t, double scale_h, double scale_w, int mode, void* stream_) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  VJ_CHECK_ARG(in && out, "vj_pos_interp: null pointer");
  VJ_CHECK_ARG(mode == 2 || mode == 3, "vj_pos_interp: mode must be 2 (bicubic) or 3 (trilinear), got %d", mode);
  VJ_CHECK_ARG(Nt > 0 && Nh > 0 && Nw > 0 && T > 0 && H > 0 && W > 0, "vj_pos_interp: empty grid");
  VJ_CHECK_ARG(D > 0 && D % 4 == 0, "vj_pos_interp: D=%d must be a positive multiple of 4", D);
  VJ_CHECK_ARG((reinterpret_cast<uintptr_t>(in) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
               "vj_pos_interp: 16-byte alignment required");
  VJ_CHECK_ARG(scale_t > 0.0 && scale_h > 0.0 && scale_w > 0.0, "vj_pos_interp: scale factors must be positive");
  VJ_CHECK_ARG(scaled_size(Nh, scale_h) == H && scaled_size(Nw, scale_w) == W,
               "vj_pos_interp: output %dx%d is not floor(in * scale) of %dx%d at scales (%g, %g)", H, W, Nh, Nw,
               scale_h, scale_w);
  // s = (float)(1.0 / scale_factor): compute_scales_value in UpSample.h
  const float sh = float(1.0 / scale_h), sw = float(1.0 / scale_w);
  if (mode == 3) {
    VJ_CHECK_ARG(scaled_size(Nt, scale_t) == T, "vj_pos_interp: output depth %d is not floor(%d * %g)", T, Nt, scale_t);
    const long long total = (long long)T * H * W * (D / 4);
    pos_interp_trilinear_kernel<<<unsigned((total + 255) / 256), 256, 0, s>>>(in, out, Nt, Nh, Nw, T, H, W, D,
                                                                              float(1.0 / scale_t), sh, sw);
  } else {
    VJ_CHECK_ARG(Nt == 1 && T == 1, "vj_pos_interp: bicubic (mode 2) resamples a 2-D table (Nt = T = 1)");
    const long long total = (long long)H * W * (D / 4);
    pos_interp_bicubic_kernel<<<unsigned((total + 255) / 256), 256, 0, s>>>(in, out, Nh, Nw, H, W, D, sh, sw);
  }
  VJ_CUDA(cudaGetLastError());
  vj::count_launch(1);
  return 0;
}
