// Block-scaled e4m3 quantisation shared by every FP8 producer (LayerNorm, the bf16 quantiser, the weight packer, the fc1 GEMM
// epilogue).  One fp32 scale covers one block of values (128 consecutive K elements of an activation row, or a 128 x 128 weight
// block); the rule is pinned so that the producers agree bit for bit with each other and with the host emulation in the tests:
//   s = amax / 448 (IEEE fp32 division; s = 1 for an all-zero block),   q = e4m3_rn_satfinite(x / s)   (IEEE division).
#pragma once
#include "common.cuh"

namespace es3 {

constexpr float E4M3_MAX = 448.f;

__device__ __forceinline__ float e4m3_block_scale(float amax) { return amax == 0.f ? 1.f : __fdiv_rn(amax, E4M3_MAX); }

// two values -> two e4m3 codes, lo in the low byte (the lower address)
__device__ __forceinline__ uint32_t e4m3x2(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}

// four consecutive values / s -> four codes in one 32-bit word
__device__ __forceinline__ uint32_t e4m3x4(float a, float b, float c, float d, float s) {
  return e4m3x2(__fdiv_rn(a, s), __fdiv_rn(b, s)) | (e4m3x2(__fdiv_rn(c, s), __fdiv_rn(d, s)) << 16);
}

__device__ __forceinline__ float abs_max4(float a, float b, float c, float d) {
  return fmaxf(fmaxf(fabsf(a), fabsf(b)), fmaxf(fabsf(c), fabsf(d)));
}

}  // namespace es3
