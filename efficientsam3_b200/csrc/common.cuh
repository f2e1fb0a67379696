// Shared device/host helpers for the es3 sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

typedef __nv_bfloat16 bf16;

// ------------------------------------------------------------------------------------ error state
// Every C-ABI export returns 0 on success; the message is read through es3_last_error().
namespace es3 {
void set_error(const char* fmt, ...);
int cuda_status(cudaError_t e, const char* what);
}  // namespace es3

#define ES3_CHECK_CUDA(expr)                                   \
  do {                                                         \
    cudaError_t _e = (expr);                                   \
    if (_e != cudaSuccess) return es3::cuda_status(_e, #expr); \
  } while (0)

#define ES3_REQUIRE(cond, ...)     \
  do {                             \
    if (!(cond)) {                 \
      es3::set_error(__VA_ARGS__); \
      return 1;                    \
    }                              \
  } while (0)

#define ES3_LAUNCH_CHECK(name)                                 \
  do {                                                         \
    cudaError_t _e = cudaGetLastError();                       \
    if (_e != cudaSuccess) return es3::cuda_status(_e, name);  \
  } while (0)

// ------------------------------------------------------------------------------------ activations
// Codes shared with the Python side (efficientsam3_b200/ops.py).
enum Es3Act { ACT_NONE = 0, ACT_RELU = 1, ACT_HSWISH = 2, ACT_GELU = 3, ACT_GELU_TANH = 4, ACT_RELU6 = 5, ACT_SIGMOID = 6 };

__device__ __forceinline__ float es3_act(float x, int act) {
  switch (act) {
    case ACT_RELU: return fmaxf(x, 0.f);
    case ACT_HSWISH: return x * fminf(fmaxf(x + 3.f, 0.f), 6.f) * (1.f / 6.f);
    case ACT_GELU: return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f));
    case ACT_GELU_TANH: {
      float u = 0.7978845608028654f * (x + 0.044715f * x * x * x);
      return 0.5f * x * (1.f + tanhf(u));
    }
    case ACT_RELU6: return fminf(fmaxf(x, 0.f), 6.f);
    case ACT_SIGMOID: return 1.f / (1.f + __expf(-x));
    default: return x;
  }
}

// GELU(erf) with erf from Abramowitz & Stegun 7.1.26 (|abs err| <= 1.5e-7, i.e. below fp32 round-off of the
// product) on MUFU.RCP / MUFU.EX2 instead of libdevice erff (~2x fewer instructions in the fc1 / head epilogues).
__device__ __forceinline__ float es3_gelu_fast(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.f)));   // MUFU.RCP, ~1 ulp
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float e = p * t * __expf(-z * z);          // 1 - erf(z)
  const float erf_abs = 1.f - e;
  return 0.5f * x * (1.f + copysignf(erf_abs, x));
}

// Compile-time activation: a runtime `switch` inside an unrolled epilogue costs a BRX per element -- kernels are
// templated on ACT and dispatched on the host with ES3_DISPATCH_ACT.
template <int ACT>
__device__ __forceinline__ float es3_act_t(float x) {
  if constexpr (ACT == ACT_RELU) return fmaxf(x, 0.f);
  // x * relu6(x + 3) / 6 == x * sat(x / 6 + 0.5): FFMA.SAT + FMUL instead of FADD, 2 FMNMX, 2 FMUL (the
  // 5-op form was a large share of a fused MBConv kernel's instructions)
  else if constexpr (ACT == ACT_HSWISH) return x * __saturatef(fmaf(x, 1.f / 6.f, 0.5f));
  else if constexpr (ACT == ACT_GELU) return es3_gelu_fast(x);
  else if constexpr (ACT == ACT_GELU_TANH) {
    float u = 0.7978845608028654f * (x + 0.044715f * x * x * x);
    return 0.5f * x * (1.f + tanhf(u));
  } else if constexpr (ACT == ACT_RELU6) return fminf(fmaxf(x, 0.f), 6.f);
  else if constexpr (ACT == ACT_SIGMOID) return 1.f / (1.f + __expf(-x));
  else return x;
}

#define ES3_DISPATCH_ACT(act, ACT_CONST, ...)                                            \
  switch (act) {                                                                         \
    case ACT_NONE: { constexpr int ACT_CONST = ACT_NONE; __VA_ARGS__; } break;           \
    case ACT_RELU: { constexpr int ACT_CONST = ACT_RELU; __VA_ARGS__; } break;           \
    case ACT_HSWISH: { constexpr int ACT_CONST = ACT_HSWISH; __VA_ARGS__; } break;       \
    case ACT_GELU: { constexpr int ACT_CONST = ACT_GELU; __VA_ARGS__; } break;           \
    case ACT_GELU_TANH: { constexpr int ACT_CONST = ACT_GELU_TANH; __VA_ARGS__; } break; \
    case ACT_RELU6: { constexpr int ACT_CONST = ACT_RELU6; __VA_ARGS__; } break;         \
    case ACT_SIGMOID: { constexpr int ACT_CONST = ACT_SIGMOID; __VA_ARGS__; } break;     \
    default: es3::set_error("unknown activation code %d", act); return 1;                \
  }

// ------------------------------------------------------------------------------------ bf16 packing
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
// 8 bf16 (one 16-byte vector) <-> 8 floats
__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
  return u;
}

// fp32 pairs: two IEEE fp32 results each, the same roundings as the scalar forms (sm_90 has no packed fp32 instructions,
// so each is two scalar operations; the pair types keep the callers' 64-bit loads and stores).
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ void unpack8_2(const uint4& u, float2* f) {
  f[0] = unpack_bf16x2(u.x); f[1] = unpack_bf16x2(u.y); f[2] = unpack_bf16x2(u.z); f[3] = unpack_bf16x2(u.w);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Image -> token attention (es3_attn_few_keys and its fp32 twin) stages its keys and values in shared memory FEW_KEYS_TILE tokens
// at a time: s [2][cap][D] gets rows row0 .. row0 + nt - 1 of k and v [., ldkv] (K at s, V at s + cap D).  Every thread of the
// block calls it; the barriers keep the previous tile alive until every thread has read it.
constexpr int FEW_KEYS_TILE = 16;
__device__ __forceinline__ void few_keys_load_tile(float* s, const float* __restrict__ k, const float* __restrict__ v, long long ldkv,
                                                   long long row0, int nt, int cap, int D) {
  __syncthreads();
  for (int i = threadIdx.x; i < nt * D; i += blockDim.x) {
    const int t = i / D, c = i % D;
    s[i] = k[(row0 + t) * ldkv + c];
    s[cap * D + i] = v[(row0 + t) * ldkv + c];
  }
  __syncthreads();
}

static inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }
