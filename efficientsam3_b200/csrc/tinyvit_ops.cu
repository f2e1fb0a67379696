// TinyViT-specific kernels (sam3/sam3/backbones/tiny_vit.py):
//   * window attention with the learned relative-position bias (Attention :219-293) on window partitions with zero
//     padding (TinyViTBlock.forward :344-375): windows are gathered in place from the raster token map; positions
//     outside the map take the per-block constant qkv(LN(0)) vector, exactly like the reference's padded tokens.
//     head_dim 32, N = ws*ws in {49, 196}.  One CTA per (window, head): S = QK^T on mma.sync with the whole
//     score row block in registers, + bias, softmax, PV on mma.sync.
//   * LayerNorm over bf16 rows with arbitrary C % 8 == 0 (C = 448 is not a multiple of 128).
#include <cuda_fp16.h>

#include "ptx.cuh"

namespace es3 {
namespace {
__device__ __forceinline__ void ldsm4t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
}  // namespace

constexpr int WA_HD = 32, WA_RS = WA_HD * 2 + 16;  // smem row: 32 bf16 = 64 B + 16 B pad

struct WinAttnArgs {
  const bf16* qkv;      // [B*H*W, 3*C], per head h: cols [h*96, +32) q | [+32, +64) k | [+64, +96) v
  const bf16* qkv_pad;  // [3*C] value of a zero-padded token (qkv(LN(0)))
  const float* bias;    // [heads][N][N]
  bf16* out;            // [B*H*W, C]
  int H, W, C, ws, nWx, nWin, N;
  float scale;
};

// NT16 = ceil(N / 16): number of 16-row tiles (4 for N=49, 13 for N=196).  The query tiles of a window are split over
// gridDim.z CTAs of blockDim/32 warps each (the 26x4 score registers per thread cap a CTA at ~7 warps); every CTA
// stages the whole window's K / V.
//
// PERSIST (the 14 x 14 windows, N = 196): round 1 launched one CTA per (window, head, half of the query tiles) and every thread
// fetched its 104 + 104 bias values with scalar loads -- 88 KB of L2 traffic and ~26 dependent load batches per CTA per
// launch.  Here a CTA of NT16 warps keeps ONE head: the head's bias table sits in
// shared memory as fp16 (196 rows x 200: the pad makes the (row g, column pair t4) reads conflict-free; fp16 keeps 11 bits of a
// |b| < 8 table, finer than the bf16 rounding of P that follows), loaded once, and the CTA walks the windows
// blockIdx.x, blockIdx.x + gridDim.x, ...
constexpr int WA_BLD = 200;     // fp16 elements per bias row in shared memory

template <int NT16, bool PERSIST>
__global__ void __launch_bounds__(NT16 * 32 > 256 ? NT16 * 32 : 256) win_attn_bias_kernel(const WinAttnArgs a, const int total_windows) {
  constexpr int NP = NT16 * 16;
  extern __shared__ __align__(16) uint8_t smem[];
  uint8_t* s_q = smem;
  uint8_t* s_k = s_q + NP * WA_RS;
  uint8_t* s_v = s_k + NP * WA_RS;
  const __half* s_bias = reinterpret_cast<const __half*>(s_v + NP * WA_RS);      // PERSIST only: [N][WA_BLD]
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = PERSIST ? (tid >> 5) : blockIdx.z * (blockDim.x >> 5) + (tid >> 5);   // query tile handled by this warp
  const int head = blockIdx.y;
  const int ld = 3 * a.C;
  if (PERSIST) {
    __half* sb = const_cast<__half*>(s_bias);
    const float* src = a.bias + (long long)head * a.N * a.N;
    for (int i = tid; i < a.N * a.N; i += blockDim.x) sb[(i / a.N) * WA_BLD + (i % a.N)] = __float2half_rn(src[i]);
  }
  for (int win = blockIdx.x; win < total_windows; win += (PERSIST ? (int)gridDim.x : total_windows)) {
  if (PERSIST) __syncthreads();        // the previous window's tiles are no longer read (and the bias table is complete)
  const int b = win / a.nWin, wi = win % a.nWin;
  const int wy = wi / a.nWx, wx = wi % a.nWx;
  // ---- gather q, k, v rows of this window / head (4 x 16-byte chunks each); rows >= N are zero
  for (int i = tid; i < NP * 12; i += blockDim.x) {
    const int c = i % 12, r = i / 12;         // c: 0..3 q, 4..7 k, 8..11 v
    uint4 val = make_uint4(0, 0, 0, 0);
    if (r < a.N) {
      const int h = wy * a.ws + r / a.ws, w = wx * a.ws + r % a.ws;
      const bf16* src = (h < a.H && w < a.W) ? a.qkv + ((long long)b * a.H * a.W + (long long)h * a.W + w) * ld : a.qkv_pad;
      val = *reinterpret_cast<const uint4*>(src + head * 96 + c * 8);
    }
    uint8_t* dst = (c < 4 ? s_q : (c < 8 ? s_k : s_v)) + r * WA_RS + (c & 3) * 16;
    *reinterpret_cast<uint4*>(dst) = val;
  }
  __syncthreads();
  if (warp >= NT16) { if (PERSIST) continue; else return; }
  const uint32_t u_q = static_cast<uint32_t>(__cvta_generic_to_shared(s_q));
  const uint32_t u_k = static_cast<uint32_t>(__cvta_generic_to_shared(s_k));
  const uint32_t u_v = static_cast<uint32_t>(__cvta_generic_to_shared(s_v));
  const int a_row = lane & 15, a_kh = lane >> 4;
  const int b_n = (lane & 7) + ((lane >> 4) << 3), b_kh = (lane >> 3) & 1;
  const int v_k = (lane & 7) + (((lane >> 3) & 1) << 3), v_n = (lane >> 4) << 3;
  const int g = lane >> 2, t4 = lane & 3;

  // ---- S = Q K^T for this warp's 16 query rows against all NP keys
  uint32_t qf[2][4];
#pragma unroll
  for (int ks = 0; ks < 2; ++ks)
    ptx::ldsm_x4(u_q + (warp * 16 + a_row) * WA_RS + (ks * 16 + a_kh * 8) * 2, qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3]);
  float s[2 * NT16][4];
#pragma unroll
  for (int i = 0; i < 2 * NT16; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
#pragma unroll
  for (int np = 0; np < NT16; ++np) {
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      uint32_t b0, b1, b2, b3;
      ptx::ldsm_x4(u_k + (np * 16 + b_n) * WA_RS + (ks * 16 + b_kh * 8) * 2, b0, b1, b2, b3);
      ptx::mma_16816(s[2 * np], qf[ks], b0, b1);
      ptx::mma_16816(s[2 * np + 1], qf[ks], b2, b3);
    }
  }
  // ---- + bias, mask, softmax (rows g, g+8)
  const int r0 = warp * 16 + g, r1 = r0 + 8;
  const float* bias0 = a.bias + ((long long)head * a.N + min(r0, a.N - 1)) * a.N;
  const float* bias1 = a.bias + ((long long)head * a.N + min(r1, a.N - 1)) * a.N;
  const __half* sb0 = s_bias + min(r0, a.N - 1) * WA_BLD;
  const __half* sb1 = s_bias + min(r1, a.N - 1) * WA_BLD;
  float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
  for (int nt = 0; nt < 2 * NT16; ++nt) {
    const int c0 = nt * 8 + t4 * 2;
    float2 bb0 = make_float2(0.f, 0.f), bb1 = make_float2(0.f, 0.f);
    if (c0 < a.N) {
      if (PERSIST) {
        bb0 = __half22float2(*reinterpret_cast<const __half2*>(sb0 + c0));
        bb1 = __half22float2(*reinterpret_cast<const __half2*>(sb1 + c0));
      } else {       // N = 49: rows are 196 B apart (4-byte aligned only) and the last column pair is half outside
        bb0.x = __ldg(bias0 + c0); bb1.x = __ldg(bias1 + c0);
        if (c0 + 1 < a.N) { bb0.y = __ldg(bias0 + c0 + 1); bb1.y = __ldg(bias1 + c0 + 1); }
      }
    }
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const bool ok = c0 + e < a.N;
      const float v0 = ok ? fmaf(s[nt][e], a.scale, e ? bb0.y : bb0.x) : -INFINITY;
      const float v1 = ok ? fmaf(s[nt][2 + e], a.scale, e ? bb1.y : bb1.x) : -INFINITY;
      s[nt][e] = v0; s[nt][2 + e] = v1;
      mx0 = fmaxf(mx0, v0); mx1 = fmaxf(mx1, v1);
    }
  }
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
  float l0 = 0.f, l1 = 0.f;
  uint32_t pf[NT16][4];
#pragma unroll
  for (int nt = 0; nt < 2 * NT16; ++nt) {
    const float p0 = __expf(s[nt][0] - mx0), p1 = __expf(s[nt][1] - mx0);
    const float p2 = __expf(s[nt][2] - mx1), p3 = __expf(s[nt][3] - mx1);
    l0 += p0 + p1; l1 += p2 + p3;
    pf[nt >> 1][(nt & 1) * 2 + 0] = pack_bf16x2(p0, p1);
    pf[nt >> 1][(nt & 1) * 2 + 1] = pack_bf16x2(p2, p3);
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  // ---- O = P V   (V rows >= N are zero, P columns >= N are zero)
  float o[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
#pragma unroll
  for (int ks = 0; ks < NT16; ++ks) {
#pragma unroll
    for (int np = 0; np < 2; ++np) {
      uint32_t b0, b1, b2, b3;
      ldsm4t(u_v + (ks * 16 + v_k) * WA_RS + (np * 16 + v_n) * 2, b0, b1, b2, b3);
      ptx::mma_16816(o[2 * np], pf[ks], b0, b1);
      ptx::mma_16816(o[2 * np + 1], pf[ks], b2, b3);
    }
  }
  const float i0 = 1.f / l0, i1 = 1.f / l1;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int r = half ? r1 : r0;
    if (r >= a.N) continue;
    const int h = wy * a.ws + r / a.ws, w = wx * a.ws + r % a.ws;
    if (h >= a.H || w >= a.W) continue;   // padded query: the reference crops it away (:373-374)
    bf16* dst = a.out + ((long long)b * a.H * a.W + (long long)h * a.W + w) * a.C + head * WA_HD;
    const float inv = half ? i1 : i0;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
      *reinterpret_cast<uint32_t*>(dst + nt * 8 + t4 * 2) = pack_bf16x2(o[nt][half * 2] * inv, o[nt][half * 2 + 1] * inv);
  }
  }   // windows
}

// LayerNorm over rows of bf16, C % 8 == 0, C <= 1024, values kept in registers.  A row is handled by L = min(32, pow2ceil(C / 8))
// lanes (TinyViT's C = 128 rows are 16 vectors of 8: two rows per warp -- the one-warp-per-row version left half of every warp idle
// on exactly the largest token maps and were far from the memory bound); reductions are xor-shuffles inside
// the L-lane group.
template <int L>
__global__ void __launch_bounds__(256) layernorm_bf16_kernel(const bf16* __restrict__ x, const float* __restrict__ gamma,
                                                             const float* __restrict__ beta, float eps, bf16* __restrict__ y, long long M,
                                                             int C) {
  constexpr int RPW = 32 / L;                                  // rows per warp
  const int lane = threadIdx.x & 31, sub = lane % L;
  const long long row = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * RPW + lane / L;
  const bool live = row < M;
  const int nvec = C >> 3;
  float v[4][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int vi = sub + i * L;
    if (live && vi < nvec) {
      unpack8(__ldg(reinterpret_cast<const uint4*>(x + row * C + vi * 8)), v[i]);
#pragma unroll
      for (int e = 0; e < 8; ++e) s += v[i][e];
    }
  }
#pragma unroll
  for (int o = L / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (live && sub + i * L < nvec) {
#pragma unroll
      for (int e = 0; e < 8; ++e) { const float d = v[i][e] - mean; q += d * d; }
    }
  }
#pragma unroll
  for (int o = L / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / C + eps);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int vi = sub + i * L;
    if (live && vi < nvec) {
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + vi * 8)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + vi * 8) + 1);
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + vi * 8)), b1 = __ldg(reinterpret_cast<const float4*>(beta + vi * 8) + 1);
      const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w}, bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      float o[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = fmaf((v[i][e] - mean) * rstd, gg[e], bb[e]);
      *reinterpret_cast<uint4*>(y + row * C + vi * 8) = pack8(o);
    }
  }
}

}  // namespace es3

using namespace es3;

extern "C" int es3_win_attn_bias_bf16(const void* qkv, const void* qkv_pad, const float* bias, void* out, int B, int H, int W,
                                      int C, int num_heads, int ws, float scale, void* stream) {
  ES3_REQUIRE(C == num_heads * WA_HD, "es3_win_attn_bias_bf16: head_dim must be 32 (C=%d heads=%d)", C, num_heads);
  const int N = ws * ws;
  ES3_REQUIRE(N == 49 || N == 196, "es3_win_attn_bias_bf16: window %d not instantiated (7 or 14)", ws);
  WinAttnArgs a;
  a.qkv = (const bf16*)qkv; a.qkv_pad = (const bf16*)qkv_pad; a.bias = bias; a.out = (bf16*)out;
  a.H = H; a.W = W; a.C = C; a.ws = ws; a.N = N; a.scale = scale;
  const int nWy = ceil_div(H, ws);
  a.nWx = ceil_div(W, ws);
  a.nWin = nWy * a.nWx;
  dim3 grid(B * a.nWin, num_heads);
  cudaStream_t st = (cudaStream_t)stream;
  if (N == 49) {
    const size_t smem = (size_t)3 * 64 * WA_RS;
    win_attn_bias_kernel<4, false><<<grid, 4 * 32, smem, st>>>(a, B * a.nWin);
  } else {
    const size_t smem = (size_t)3 * 208 * WA_RS + (size_t)N * WA_BLD * sizeof(__half);       // 49920 + 78400 B
    ES3_CHECK_CUDA(cudaFuncSetAttribute(win_attn_bias_kernel<13, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    static int sm_count = 0;
    if (sm_count == 0) {
      int dev = 0;
      ES3_CHECK_CUDA(cudaGetDevice(&dev));
      ES3_CHECK_CUDA(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));
    }
    int per_head = sm_count / num_heads;             // one CTA per SM (128 KB of shared memory), every CTA pinned to one head
    if (per_head < 1) per_head = 1;
    if (per_head > B * a.nWin) per_head = B * a.nWin;
    win_attn_bias_kernel<13, true><<<dim3(per_head, num_heads), 13 * 32, smem, st>>>(a, B * a.nWin);
  }
  ES3_LAUNCH_CHECK("win_attn_bias_kernel");
  return 0;
}

extern "C" int es3_layernorm_bf16(const void* x, const float* gamma, const float* beta, float eps, void* y, long long M, int C,
                                  void* stream) {
  ES3_REQUIRE(C % 8 == 0 && C <= 1024, "es3_layernorm_bf16: C=%d must be a multiple of 8 and <= 1024", C);
  ES3_REQUIRE((((uintptr_t)x | (uintptr_t)y | (uintptr_t)gamma | (uintptr_t)beta) & 15) == 0, "es3_layernorm_bf16: 16-byte alignment");
  const int nvec = C / 8;
  cudaStream_t st = (cudaStream_t)stream;
  if (nvec <= 8)
    layernorm_bf16_kernel<8><<<(unsigned)ceil_div(M, 8 * 4), 256, 0, st>>>((const bf16*)x, gamma, beta, eps, (bf16*)y, M, C);
  else if (nvec <= 16)
    layernorm_bf16_kernel<16><<<(unsigned)ceil_div(M, 8 * 2), 256, 0, st>>>((const bf16*)x, gamma, beta, eps, (bf16*)y, M, C);
  else
    layernorm_bf16_kernel<32><<<(unsigned)ceil_div(M, 8), 256, 0, st>>>((const bf16*)x, gamma, beta, eps, (bf16*)y, M, C);
  ES3_LAUNCH_CHECK("layernorm_bf16_kernel");
  return 0;
}
