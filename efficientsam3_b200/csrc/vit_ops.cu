// Token-wise kernels of the SAM3 ViT trunk that are pure HBM streaming (no contraction):
//   * LayerNorm over the channel dim (vitdet.py:597-613 norm1/norm2, ln_pre :828) reading the fp32 residual
//     stream and writing the bf16 GEMM operand; optionally fused with the tiled absolute-position add
//     (get_abs_pos tiling branch, vitdet.py:205-214) for ln_pre
//   * im2col for the 14x14/stride-14 patch embedding (PatchEmbed, vitdet.py:299-336) -> bf16 GEMM operand
//   * [B, HW, C] fp32 tokens -> [B, C, HW] fp32 (the NCHW map ViT.forward returns, vitdet.py:846-857)
#include <cuda_fp16.h>

#include "common.cuh"
#include "fp8.cuh"

namespace es3 {

// One warp per row.  C % 128 == 0, C <= 2048.  x fp32 [M, C]; pos (optional) fp32 [ps*ps, C] tiled over an
// (H, W) token grid; gamma/beta fp32.  Writes y_bf16 and/or y_f32 (either may be null); Q8: writes y_q e4m3 [M, C] and
// y_qs fp32 [M, C / 128] instead (fp8.cuh: vector i of every lane is 128-column block i, so a block's amax is one warp max).
template <int VPL, bool Q8 = false>  // float4 vectors per lane = C / 128
__global__ void layernorm_kernel(const float* __restrict__ x, const float* __restrict__ pos, int ps, int H, int W,
                                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                 bf16* __restrict__ y_bf16, float* __restrict__ y_f32, long long M,
                                 uint8_t* __restrict__ y_q = nullptr, float* __restrict__ y_qs = nullptr) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  constexpr int C = VPL * 128;
  const float4* xr = reinterpret_cast<const float4*>(x + row * C);
  float4 v[VPL];
#pragma unroll
  for (int i = 0; i < VPL; ++i) v[i] = xr[lane + i * 32];
  if (pos != nullptr) {
    const int t = (int)(row % ((long long)H * W));
    const int h = t / W, w = t % W;
    const float4* pr = reinterpret_cast<const float4*>(pos + ((long long)(h % ps) * ps + (w % ps)) * C);
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const float4 p = __ldg(pr + lane + i * 32);
      v[i].x += p.x; v[i].y += p.y; v[i].z += p.z; v[i].w += p.w;
    }
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = warp_sum(s) * (1.f / C);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += (a * a + b * b) + (c * c + d * d);
  }
  const float rstd = rsqrtf(warp_sum(q) * (1.f / C) + eps);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const float4 g = __ldg(g4 + lane + i * 32), bb = __ldg(b4 + lane + i * 32);
    float4 o;
    o.x = (v[i].x - mean) * rstd * g.x + bb.x;
    o.y = (v[i].y - mean) * rstd * g.y + bb.y;
    o.z = (v[i].z - mean) * rstd * g.z + bb.z;
    o.w = (v[i].w - mean) * rstd * g.w + bb.w;
    if constexpr (Q8) {
      const float sc = e4m3_block_scale(warp_max(abs_max4(o.x, o.y, o.z, o.w)));
      reinterpret_cast<uint32_t*>(y_q + row * C)[lane + i * 32] = e4m3x4(o.x, o.y, o.z, o.w, sc);
      if (lane == 0) y_qs[row * VPL + i] = sc;
      continue;
    }
    if (y_f32) reinterpret_cast<float4*>(y_f32 + row * C)[lane + i * 32] = o;
    if (y_bf16) {
      uint2 u;
      u.x = pack_bf16x2(o.x, o.y);
      u.y = pack_bf16x2(o.z, o.w);
      reinterpret_cast<uint2*>(y_bf16 + row * C)[lane + i * 32] = u;
    }
  }
}

// x [B,3,S,S] fp32 -> cols [B*hp*wp, Kp] bf16, column = c*P*P + ky*P + kx (the flattened nn.Conv2d weight
// order), zero for column >= 3*P*P.
__global__ void im2col_patch_kernel(const float* __restrict__ x, bf16* __restrict__ cols, int S, int P, int hp, int wp,
                                    int Kp, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int col = (int)(idx % Kp);
  const long long tok = idx / Kp;
  float v = 0.f;
  if (col < 3 * P * P) {
    const int c = col / (P * P), r = col % (P * P), ky = r / P, kx = r % P;
    const int px = (int)(tok % wp), py = (int)((tok / wp) % hp);
    const long long b = tok / ((long long)wp * hp);
    v = __ldg(x + ((b * 3 + c) * S + (py * P + ky)) * (long long)S + px * P + kx);
  }
  cols[idx] = __float2bfloat16(v);
}

// [B, HW, C] fp32 -> [B, C, HW] fp32
__global__ void tokens_to_nchw_kernel(const float* __restrict__ in, float* __restrict__ out, int HW, int C) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8) {
    const int p = p0 + i, c = c0 + tx;
    tile[i][tx] = (p < HW && c < C) ? in[((long long)b * HW + p) * C + c] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i, p = p0 + tx;
    if (p < HW && c < C) out[((long long)b * C + c) * HW + p] = tile[tx][i];
  }
}

}  // namespace es3

using namespace es3;

extern "C" int es3_layernorm_f32(const float* x, const float* pos, int pos_size, int H, int W, const float* gamma,
                                 const float* beta, float eps, void* y_bf16, float* y_f32, long long M, int C,
                                 void* stream) {
  ES3_REQUIRE(C % 128 == 0 && C <= 2048, "es3_layernorm_f32: C=%d must be a multiple of 128 and <= 2048", C);
  ES3_REQUIRE(pos == nullptr || (pos_size > 0 && H > 0 && W > 0), "es3_layernorm_f32: bad pos tiling");
  const int warps = 8;
  const unsigned blocks = (unsigned)ceil_div(M, warps);
  cudaStream_t st = (cudaStream_t)stream;
#define ES3_LN(V) case V: layernorm_kernel<V><<<blocks, warps * 32, 0, st>>>(x, pos, pos_size, H, W, gamma, beta, eps, (bf16*)y_bf16, y_f32, M); break;
  switch (C / 128) {
    ES3_LN(1) ES3_LN(2) ES3_LN(3) ES3_LN(4) ES3_LN(5) ES3_LN(6) ES3_LN(7) ES3_LN(8) ES3_LN(10) ES3_LN(12) ES3_LN(16)
    default: ES3_REQUIRE(false, "es3_layernorm_f32: C=%d not instantiated", C);
  }
#undef ES3_LN
  ES3_LAUNCH_CHECK("layernorm_kernel");
  return 0;
}

// LayerNorm of the fp32 rows straight to the FP8 GEMM's A operand: e4m3 q [M, C] + fp32 scales [M, C / 128] (fp8.cuh).  The
// statistics and the normalised value are the same arithmetic as es3_layernorm_f32's.
extern "C" int es3_layernorm_f32_e4m3(const float* x, const float* gamma, const float* beta, float eps, void* q, float* scales,
                                      long long M, int C, void* stream) {
  ES3_REQUIRE(C % 128 == 0 && C <= 2048, "es3_layernorm_f32_e4m3: C=%d must be a multiple of 128 and <= 2048", C);
  const int warps = 8;
  const unsigned blocks = (unsigned)ceil_div(M, warps);
  cudaStream_t st = (cudaStream_t)stream;
#define ES3_LNQ(V) case V: layernorm_kernel<V, true><<<blocks, warps * 32, 0, st>>>(x, nullptr, 0, 0, 0, gamma, beta, eps, nullptr, nullptr, M, (uint8_t*)q, scales); break;
  switch (C / 128) {
    ES3_LNQ(8) ES3_LNQ(16)
    default: ES3_REQUIRE(false, "es3_layernorm_f32_e4m3: C=%d not instantiated (1024, 2048)", C);
  }
#undef ES3_LNQ
  ES3_LAUNCH_CHECK("layernorm_kernel<e4m3>");
  return 0;
}

extern "C" int es3_im2col_patch(const float* x, void* cols, int B, int S, int P, int Kp, void* stream) {
  ES3_REQUIRE(B > 0 && S % P == 0 && Kp >= 3 * P * P && Kp % 8 == 0, "es3_im2col_patch: bad B=%d S=%d P=%d Kp=%d", B, S, P, Kp);
  const int hp = S / P;
  const long long total = (long long)B * hp * hp * Kp;
  im2col_patch_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(x, (bf16*)cols, S, P, hp, hp, Kp, total);
  ES3_LAUNCH_CHECK("im2col_patch_kernel");
  return 0;
}

extern "C" int es3_tokens_f32_to_nchw(const float* in, float* out, int B, int HW, int C, void* stream) {
  ES3_REQUIRE(B > 0 && HW > 0 && C > 0, "es3_tokens_f32_to_nchw: bad shape B=%d HW=%d C=%d", B, HW, C);
  dim3 grid(ceil_div(HW, 32), ceil_div(C, 32), B);
  tokens_to_nchw_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in, out, HW, C);
  ES3_LAUNCH_CHECK("tokens_to_nchw_kernel");
  return 0;
}

// fp32 -> fp16 (round to nearest even), 8 elements per thread: the teacher-embedding dump stores fp16
// (save_embedding_image_stage1.py:92 `.to(dtype=torch.float16)`), so the cast runs before the D2H copy and halves it.
namespace es3 {
__global__ void cast_f32_f16_kernel(const float* __restrict__ in, __half* __restrict__ out, long long n) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i + 8 <= n) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(in + i));
    const float4 b = __ldg(reinterpret_cast<const float4*>(in + i + 4));
    __half2 h[4] = {__floats2half2_rn(a.x, a.y), __floats2half2_rn(a.z, a.w), __floats2half2_rn(b.x, b.y), __floats2half2_rn(b.z, b.w)};
    *reinterpret_cast<uint4*>(out + i) = *reinterpret_cast<const uint4*>(h);
  } else {
    for (long long j = i; j < n; ++j) out[j] = __float2half_rn(in[j]);
  }
}
}  // namespace es3

extern "C" int es3_cast_f32_to_f16(const float* in, void* out, long long n, void* stream) {
  ES3_REQUIRE(n >= 0 && ((uintptr_t)in & 15) == 0 && ((uintptr_t)out & 15) == 0, "es3_cast_f32_to_f16: pointers must be 16-byte aligned");
  if (n == 0) return 0;
  const int threads = 256;
  cast_f32_f16_kernel<<<(unsigned)(((n + 7) / 8 + threads - 1) / threads), threads, 0, (cudaStream_t)stream>>>(in, (__half*)out, n);
  ES3_LAUNCH_CHECK("cast_f32_f16_kernel");
  return 0;
}
