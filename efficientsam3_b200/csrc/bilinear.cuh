// Bilinear (align_corners=False) sampling shared by every kernel that reads an upsampled mask logit: es3_bilinear_nchw_f32
// (decoder.cu) and the automatic mask generator's mask statistics and RLE (amg.cu).  Those kernels must agree bit for bit on
// each output pixel -- a mask's box, stability score and RLE are thresholds of the same value -- so the source coordinate and
// the two-level lerp are written once, here.
#pragma once
#include "common.cuh"

namespace es3 {

// One axis of the sample: source taps i0 <= i1 and their weights (h = 1 - l on i0, l on i1).  s = in / out.
struct BilinearTap {
  int i0, i1;
  float l, h;
};

__device__ __forceinline__ BilinearTap bilinear_tap(int o, float s, int n) {
  float f = (o + 0.5f) * s - 0.5f;
  if (f < 0.f) f = 0.f;
  const int i0 = min((int)f, n - 1);
  const int i1 = min(i0 + 1, n - 1);
  const float l = f - i0;
  return {i0, i1, l, 1.f - l};
}

// v00 = in[y.i0][x.i0], v01 = in[y.i0][x.i1], v10 = in[y.i1][x.i0], v11 = in[y.i1][x.i1].
__device__ __forceinline__ float bilinear_mix(const BilinearTap& y, const BilinearTap& x, float v00, float v01, float v10,
                                              float v11) {
  return y.h * (x.h * v00 + x.l * v01) + y.l * (x.h * v10 + x.l * v11);
}

}  // namespace es3
