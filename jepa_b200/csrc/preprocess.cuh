// Per-pixel pieces shared by the input-pipeline kernels (preprocess.cu, augment.cu).
#pragma once

#include "common.cuh"

namespace vj {

// (v_c - sub_c) / div_c for the three channels, each step rounded like the reference's fp32 sub_ / div_, stored as TO
// at dst + c * cstride (the channel planes of the [3, T, S, S] layout)
template <typename TO>
__device__ __forceinline__ void normalise_store(TO* dst, long long cstride, const float (&v)[3], float3 sub, float3 div) {
  dst[0] = TO(__fdiv_rn(__fsub_rn(v[0], sub.x), div.x));
  dst[cstride] = TO(__fdiv_rn(__fsub_rn(v[1], sub.y), div.y));
  dst[2 * cstride] = TO(__fdiv_rn(__fsub_rn(v[2], sub.z), div.z));
}

// Resized pixel (y, x) of the random-resized crop [i, i+h) x [j, j+w) of an RGB uint8 frame with row length W, as
// float 0..255 per channel; sh = h / S, sw = w / S for an S x S output.  ATen's upsample_bilinear2d (align_corners =
// False): src = max(0, (dst + 0.5) * in/out - 0.5), the upper neighbour clamped to the last row / column of the crop.
__device__ __forceinline__ void crop_bilinear3(const uint8_t* frame, int W, int i, int j, int h, int w, float sh, float sw,
                                               int y, int x, float (&v)[3]) {
  float fy = fmaxf((float(y) + 0.5f) * sh - 0.5f, 0.f);
  float fx = fmaxf((float(x) + 0.5f) * sw - 0.5f, 0.f);
  const int y0 = min(int(fy), h - 1), x0 = min(int(fx), w - 1);
  const int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
  const float ly = fy - float(y0), lx = fx - float(x0);
  const float hy = 1.f - ly, hx = 1.f - lx;
  const uint8_t* r0 = frame + ((long long)(i + y0) * W + j) * 3;
  const uint8_t* r1 = frame + ((long long)(i + y1) * W + j) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float p00 = float(r0[x0 * 3 + c]), p01 = float(r0[x1 * 3 + c]);
    const float p10 = float(r1[x0 * 3 + c]), p11 = float(r1[x1 * 3 + c]);
    v[c] = hy * (hx * p00 + lx * p01) + ly * (hx * p10 + lx * p11);
  }
}

// Records of vj_clip_augment / vj_image_augment (jepa_b200/transforms.py AUG_CLIP / AUG_OP)
struct AugClip {            // per clip, 64 bytes
  long long off;            // byte offset of the clip's frames [T, H, W, 3] in each work buffer
  int H, W;
  int i, j, h, w;           // crop box
  int flip;                 // mirror the output horizontally
  int final_buf;            // work buffer holding the clip after the last layer (0 or 1)
  int etop, eleft, eh, ew;  // erase box in output coordinates (after the flip); eh == 0: no erase
  unsigned long long seed;  // vj_clip_augment: Philox key of the erase noise; vj_image_augment: element offset of
                            // the host-drawn noise [3, eh, ew] in the noise buffer
};

struct AugOp {              // per (layer, clip), 64 bytes
  double m[6];              // inverse affine matrix of the geometric ops
  int code;                 // RaOp, -1: skipped (the clip stays in in_buf)
  float fval;               // blend factor
  int ival;                 // posterize bits / solarize threshold / solarize-add amount
  int in_buf;               // read from work buffer in_buf, write to 1 - in_buf
};

// RandAugment / AutoAugment layers over B clips of T frames in the work buffers b0 / b1 (augment.cu; records and tables
// as documented at vj_clip_augment).  fill: RGB of the pixels a geometric op leaves uncovered.  Returns 0 or an error.
int ra_layers(uint8_t* b0, uint8_t* b1, const void* clips, const void* ops, void* hist, const int* layer_flags,
              int n_layers, int B, int T, uchar3 fill, cudaStream_t s);

}  // namespace vj
