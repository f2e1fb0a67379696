// LiteMLA on tensor cores (mma.sync bf16, fp32 accumulate) -- reference efficientvit/nn/ops.py:521-671, head dim 16.
//
// Data layout: one NHWC bf16 buffer `ms` of 6*TD channels per pixel (TD = heads*dim):
//   channels [0, 3TD)   = qkv           (written by the qkv 1x1 GEMM with ldo = 6TD)
//   channels [3TD, 6TD) = aggreg(qkv)   (dw5x5 -> grouped 1x1, written by litemla_aggreg_dwpw_kernel)
// which is exactly torch.cat([qkv, aggreg(qkv)], dim=1) (ops.py:656-660); viewed as
// (B, 2*heads, 3*dim, HW), head h owns channels [48h, 48h+48): q | k | v (ops.py:590-606, dim = 16).
//
// Every stage is a small dense contraction:
//  aggreg : depthwise 5x5 as diagonal MMAs, its result rounded to bf16 and fed back as the A fragment of the 16x16 grouped
//           pointwise MMA.
//  kv     : KV[i][j] = sum_p v[p][i] relu(k[p][j])   (M=16, N=16, K=pixels; A and B via ldmatrix.trans),
//           ones row (ops.py:613 F.pad value=1) via a constant A fragment.  Deterministic two-stage reduce.
//  apply  : out[p][d] = sum_j KV[d][j] relu(q[p][j]) / (KV[16] . relu(q[p]) + eps)
//           (M=pixels, N=17->24, K=16), KV split hi+lo bf16 so the fp32 state keeps ~16 mantissa bits.
#include "ptx.cuh"

namespace es3 {
namespace {
__device__ __forceinline__ void ldsm4t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void cpa16(uint32_t saddr, const void* g, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(saddr), "l"(g), "r"(sz) : "memory");
}
__device__ __forceinline__ void cpa_wait_all() { asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ uint32_t relu_bf16x2(uint32_t v) {
  uint32_t r;
  asm("max.bf16x2 %0, %1, %2;" : "=r"(r) : "r"(v), "r"(0u));
  return r;
}
}  // namespace

// ------------------------------------------------------------------------------------------ aggreg
constexpr int AG_TH = 16, AG_TW = 32, AG_IH = AG_TH + 4, AG_IW = AG_TW + 4, AG_PS = 48;  // 16 ch = 32 B + 16 B pad
constexpr int AG_TILE_BYTES = AG_IH * AG_IW * AG_PS;      // 34560

// Aggregation: depthwise 5x5 as 25 x 2 DIAGONAL m16n8k8 MMAs (no structural zeros), its fp32 result rounded to bf16 and re-used
// in registers as the A fragment of ONE 16x16x16 grouped-pointwise MMA pair; the depthwise output is rounded to bf16 exactly
// where the unfused reference path materialises it.
// ms: [B,H,W,ld] bf16.  Reads channels [grp*16, +16) (qkv), writes channels [C3 + grp*16, +16).
// wdw: [C3/16][25][16] bf16 (group, tap, channel);  wpw: [C3][16] bf16 (output channel, input channel within its group).
constexpr int AG2_SMEM = AG_TILE_BYTES + 25 * 16 * 2 + 16 * AG_PS;
__global__ void __launch_bounds__(256, 3) litemla_aggreg_dwpw_kernel(const bf16* ms_in, bf16* ms_out, long long ld,
                                                                  const bf16* __restrict__ wdw, const bf16* __restrict__ wpw,
                                                                  int H, int W, int tiles_x) {
  extern __shared__ __align__(16) uint8_t smem[];
  const uint32_t u_tile = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
  const bf16* s_wd = reinterpret_cast<const bf16*>(smem + AG_TILE_BYTES);   // [25][16]
  const uint32_t u_wp = u_tile + AG_TILE_BYTES + 25 * 16 * 2;               // [16 n][16 k], row stride AG_PS
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tile = blockIdx.x, grp = blockIdx.y, b = blockIdx.z;
  const int oy0 = (tile / tiles_x) * AG_TH, ox0 = (tile % tiles_x) * AG_TW;

  const bf16* xb = ms_in + (long long)b * H * W * ld + grp * 16;
  for (int i = tid; i < AG_IH * AG_IW * 2; i += 256) {
    const int v = i & 1, p = i >> 1;
    const int iy = oy0 - 2 + p / AG_IW, ix = ox0 - 2 + p % AG_IW;
    const bool ok = iy >= 0 && iy < H && ix >= 0 && ix < W;
    cpa16(u_tile + p * AG_PS + v * 16, ok ? xb + ((long long)iy * W + ix) * ld + v * 8 : xb, ok);
  }
  if (tid < 50) cpa16(u_tile + AG_TILE_BYTES + tid * 16, wdw + (long long)grp * 400 + tid * 8, true);
  if (tid >= 64 && tid < 96) {
    const int i = tid - 64, n = i >> 1, v = i & 1;
    cpa16(u_wp + n * AG_PS + v * 16, wpw + ((long long)grp * 16 + n) * 16 + v * 8, true);
  }
  cpa_wait_all();
  __syncthreads();

  const int a_row = lane & 15, a_kh = lane >> 4;
  const int b_n = (lane & 7) + ((lane >> 4) << 3), b_kh = (lane >> 3) & 1;
  const int g = lane >> 2, t4 = lane & 3;
  const uint32_t dshift = (g & 1) ? 16u : 0u;
  const bool dvalid = (g >> 1) == t4;
  float acc[4][2][4];
#pragma unroll
  for (int m = 0; m < 4; ++m)
#pragma unroll
    for (int n = 0; n < 2; ++n) { acc[m][n][0] = acc[m][n][1] = acc[m][n][2] = acc[m][n][3] = 0.f; }

  // warp -> x-half xh (16 pixels) and four CONSECUTIVE output rows y0 .. y0+3: per kx the eight input-row fragments are loaded
  // once and shared by the five ky taps of each output row -- 40 ldmatrix.x4 per warp instead of 100 (the shared-memory pipe was
  // this kernel's busiest unit)
  const int xh = warp & 1, y0 = (warp >> 1) * 4;
#pragma unroll 1
  for (int kx = 0; kx < 5; ++kx) {
    uint32_t af[8][4];
#pragma unroll
    for (int r = 0; r < 8; ++r)
      ptx::ldsm_x4(u_tile + ((y0 + r) * AG_IW + xh * 16 + a_row + kx) * AG_PS + a_kh * 16, af[r][0], af[r][1], af[r][2], af[r][3]);
    // two taps per MMA (m16n8k16 issues at the rate of m16n8k8): (0, kx)+(1, kx), (2, kx)+(3, kx) as k16, (4, kx) as k8 -- 30 MMAs per
    // m-tile instead of 50; the legacy-MMA pipe was this kernel's limiter (60 % busy)
    uint32_t b_lo[5], b_hi[5];
#pragma unroll
    for (int ky = 0; ky < 5; ++ky) {
      const uint32_t w_lo = (uint32_t)__bfloat16_as_ushort(s_wd[(ky * 5 + kx) * 16 + g]);
      const uint32_t w_hi = (uint32_t)__bfloat16_as_ushort(s_wd[(ky * 5 + kx) * 16 + 8 + g]);
      b_lo[ky] = dvalid ? (w_lo << dshift) : 0u;
      b_hi[ky] = dvalid ? (w_hi << dshift) : 0u;
    }
#pragma unroll
    for (int m = 0; m < 4; ++m) {
#pragma unroll
      for (int kp = 0; kp < 2; ++kp) {
        const uint32_t a_lo[4] = {af[m + 2 * kp][0], af[m + 2 * kp][1], af[m + 2 * kp + 1][0], af[m + 2 * kp + 1][1]};
        const uint32_t a_hi[4] = {af[m + 2 * kp][2], af[m + 2 * kp][3], af[m + 2 * kp + 1][2], af[m + 2 * kp + 1][3]};
        ptx::mma_16816(acc[m][0], a_lo, b_lo[2 * kp], b_lo[2 * kp + 1]);
        ptx::mma_16816(acc[m][1], a_hi, b_hi[2 * kp], b_hi[2 * kp + 1]);
      }
      ptx::mma_1688(acc[m][0], af[m + 4][0], af[m + 4][1], b_lo[4]);
      ptx::mma_1688(acc[m][1], af[m + 4][2], af[m + 4][3], b_hi[4]);
    }
  }
  uint32_t p0, p1, p2, p3;
  ptx::ldsm_x4(u_wp + b_n * AG_PS + b_kh * 16, p0, p1, p2, p3);
  bf16* ob = ms_out + (long long)b * H * W * ld + grp * 16;
#pragma unroll
  for (int m = 0; m < 4; ++m) {
    // depthwise result (C fragment of two n-tiles) -> bf16 A fragment of the 16x16x16 grouped pointwise product
    const uint32_t pa[4] = {pack_bf16x2(acc[m][0][0], acc[m][0][1]), pack_bf16x2(acc[m][0][2], acc[m][0][3]),
                            pack_bf16x2(acc[m][1][0], acc[m][1][1]), pack_bf16x2(acc[m][1][2], acc[m][1][3])};
    float o[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
    ptx::mma_16816(o[0], pa, p0, p1);
    ptx::mma_16816(o[1], pa, p2, p3);
    const int oy = oy0 + y0 + m;
    if (oy >= H) continue;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int ox = ox0 + xh * 16 + g + half * 8;
      if (ox >= W) continue;
      bf16* dst = ob + ((long long)oy * W + ox) * ld + t4 * 2;
      *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(o[0][half * 2], o[0][half * 2 + 1]);
      *reinterpret_cast<uint32_t*>(dst + 8) = pack_bf16x2(o[1][half * 2], o[1][half * 2 + 1]);
    }
  }
}

// ------------------------------------------------------------------------------------------ kv
constexpr int KV_PX = 512, KV_RS = 80;  // 32 ch (k|v) = 64 B + 16 B pad

// part: [B][heads2][nchunk][17][16] fp32.  grid (nchunk, heads2, B), block 256 (8 warps x 64 pixels).
__global__ void __launch_bounds__(256) litemla_kv_tc_kernel(const bf16* __restrict__ ms, long long ld,
                                                            float* __restrict__ part, int HW) {
  __shared__ __align__(16) uint8_t s_kv[KV_PX * KV_RS];   // 40960 B; re-used for the cross-warp reduction
  const uint32_t u = static_cast<uint32_t>(__cvta_generic_to_shared(s_kv));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int h = blockIdx.y, b = blockIdx.z, heads2 = gridDim.y, nchunk = gridDim.x;
  const int p_base = blockIdx.x * KV_PX;
  const bf16* src = ms + (long long)b * HW * ld + h * 48 + 16;
  for (int i = tid; i < KV_PX * 4; i += 256) {
    const int v = i & 3, pl = i >> 2;
    const bool ok = p_base + pl < HW;
    cpa16(u + pl * KV_RS + v * 16, ok ? src + (long long)(p_base + pl) * ld + v * 8 : src, ok);
  }
  cpa_wait_all();
  __syncthreads();

  const int g = lane >> 2, t4 = lane & 3;
  float acc[2][4], ones[2][4];
#pragma unroll
  for (int n = 0; n < 2; ++n) {
    acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;
    ones[n][0] = ones[n][1] = ones[n][2] = ones[n][3] = 0.f;
  }
  const uint32_t one2 = (g == 0) ? 0x3F803F80u : 0u;       // bf16 (1, 1): A row 0 = ones, rows 1..15 = 0
  const uint32_t a_ones[4] = {one2, 0u, one2, 0u};
  // A = V^T from [p][i] storage (trans): regs <-> (k0-7,m0-7), (k0-7,m8-15), (k8-15,m0-7), (k8-15,m8-15)
  const int av_p = (lane & 7) + ((lane >> 4) << 3), av_c = 32 + ((lane >> 3) & 1) * 16;
  // B = relu(K) from [p][j] storage (trans): regs <-> (k0-7,n0-7), (k8-15,n0-7), (k0-7,n8-15), (k8-15,n8-15)
  const int bk_p = (lane & 7) + (((lane >> 3) & 1) << 3), bk_c = (lane >> 4) * 16;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    const int p0 = warp * 64 + ks * 16;
    uint32_t af[4], b0, b1, b2, b3;
    ldsm4t(u + (p0 + av_p) * KV_RS + av_c, af[0], af[1], af[2], af[3]);
    ldsm4t(u + (p0 + bk_p) * KV_RS + bk_c, b0, b1, b2, b3);
    b0 = relu_bf16x2(b0); b1 = relu_bf16x2(b1); b2 = relu_bf16x2(b2); b3 = relu_bf16x2(b3);
    ptx::mma_16816(acc[0], af, b0, b1);
    ptx::mma_16816(acc[1], af, b2, b3);
    ptx::mma_16816(ones[0], a_ones, b0, b1);
    ptx::mma_16816(ones[1], a_ones, b2, b3);
  }
  __syncthreads();  // tile no longer needed: reuse smem as red[8 warps][17][16]
  float* red = reinterpret_cast<float*>(s_kv);
  float* mine = red + warp * 17 * 16;
#pragma unroll
  for (int n = 0; n < 2; ++n) {
    const int j = n * 8 + t4 * 2;
    mine[g * 16 + j] = acc[n][0];
    mine[g * 16 + j + 1] = acc[n][1];
    mine[(g + 8) * 16 + j] = acc[n][2];
    mine[(g + 8) * 16 + j + 1] = acc[n][3];
    if (g == 0) {
      mine[16 * 16 + j] = ones[n][0];
      mine[16 * 16 + j + 1] = ones[n][1];
    }
  }
  __syncthreads();
  float* dst = part + (((long long)b * heads2 + h) * nchunk + blockIdx.x) * 17 * 16;
  for (int i = tid; i < 17 * 16; i += 256) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w * 17 * 16 + i];
    dst[i] = s;
  }
}

// ------------------------------------------------------------------------------------------ apply
// grid (ceil(HW/256), heads2, B), block 128: 4 warps x 64 pixels.
__global__ void __launch_bounds__(128) litemla_apply_tc_kernel(const bf16* __restrict__ ms, long long ld,
                                                               const float* __restrict__ part, int nchunk,
                                                               bf16* __restrict__ att, long long ldo, int HW, float eps) {
  __shared__ float skv[17 * 16];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int h = blockIdx.y, b = blockIdx.z, heads2 = gridDim.y;
  const float* src = part + ((long long)b * heads2 + h) * nchunk * 17 * 16;
  for (int i = tid; i < 17 * 16; i += 128) {
    float a = 0.f;
    for (int c = 0; c < nchunk; ++c) a += src[c * 17 * 16 + i];
    skv[i] = a;
  }
  __syncthreads();
  const int g = lane >> 2, t4 = lane & 3;
  // B[k=j][n=d] = KV[d][j], split hi + lo
  uint32_t bh[3][2], bl[3][2];
#pragma unroll
  for (int nt = 0; nt < 3; ++nt) {
    const int d = nt * 8 + g;
#pragma unroll
    for (int kh = 0; kh < 2; ++kh) {
      float v0 = 0.f, v1 = 0.f;
      if (d <= 16) { v0 = skv[d * 16 + kh * 8 + t4 * 2]; v1 = skv[d * 16 + kh * 8 + t4 * 2 + 1]; }
      const uint32_t hi = pack_bf16x2(v0, v1);
      const float2 hf = unpack_bf16x2(hi);
      bh[nt][kh] = hi;
      bl[nt][kh] = pack_bf16x2(v0 - hf.x, v1 - hf.y);
    }
  }
  const bf16* qb = ms + (long long)b * HW * ld + h * 48;
  bf16* ob = att + (long long)b * HW * ldo + h * 16;
#pragma unroll 1
  for (int mt = 0; mt < 4; ++mt) {
    const int p0 = blockIdx.x * 256 + warp * 64 + mt * 16;
    if (p0 >= HW) break;
    const int pa = p0 + g, pb = p0 + g + 8;
    uint32_t af[4] = {0u, 0u, 0u, 0u};
    if (pa < HW) {
      const uint32_t* q = reinterpret_cast<const uint32_t*>(qb + (long long)pa * ld);
      af[0] = relu_bf16x2(__ldg(q + t4));
      af[2] = relu_bf16x2(__ldg(q + 4 + t4));
    }
    if (pb < HW) {
      const uint32_t* q = reinterpret_cast<const uint32_t*>(qb + (long long)pb * ld);
      af[1] = relu_bf16x2(__ldg(q + t4));
      af[3] = relu_bf16x2(__ldg(q + 4 + t4));
    }
    float acc[3][4];
#pragma unroll
    for (int nt = 0; nt < 3; ++nt) {
      acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
      ptx::mma_16816(acc[nt], af, bl[nt][0], bl[nt][1]);
      ptx::mma_16816(acc[nt], af, bh[nt][0], bh[nt][1]);
    }
    // denominators: column 16 (n-tile 2, col 0) lives in lane g*4
    const float den_a = __shfl_sync(0xffffffffu, acc[2][0], g * 4);
    const float den_b = __shfl_sync(0xffffffffu, acc[2][2], g * 4);
    const float ia = 1.f / (den_a + eps), ib = 1.f / (den_b + eps);
    if (pa < HW) {
      uint32_t* o = reinterpret_cast<uint32_t*>(ob + (long long)pa * ldo);
      o[t4] = pack_bf16x2(acc[0][0] * ia, acc[0][1] * ia);
      o[4 + t4] = pack_bf16x2(acc[1][0] * ia, acc[1][1] * ia);
    }
    if (pb < HW) {
      uint32_t* o = reinterpret_cast<uint32_t*>(ob + (long long)pb * ldo);
      o[t4] = pack_bf16x2(acc[0][2] * ib, acc[0][3] * ib);
      o[4 + t4] = pack_bf16x2(acc[1][2] * ib, acc[1][3] * ib);
    }
  }
}

}  // namespace es3

using namespace es3;

// ms: [B,H,W,ld] bf16 with qkv in channels [0,C3) -> writes aggreg(qkv) to channels [C3, 2*C3).
// wdw [C3/16][25][16] bf16 (depthwise taps), wpw [C3][16] bf16 (grouped pointwise).
extern "C" int es3_litemla_aggreg_dwpw(void* ms, long long ld, const void* wdw, const void* wpw, int B, int H, int W, int C3,
                                       void* stream) {
  ES3_REQUIRE(C3 % 16 == 0 && ld % 8 == 0 && ld >= 2 * C3, "es3_litemla_aggreg_dwpw: bad C3=%d ld=%lld", C3, ld);
  static bool configured = false;
  if (!configured) {
    ES3_CHECK_CUDA(cudaFuncSetAttribute(litemla_aggreg_dwpw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AG2_SMEM));
    configured = true;
  }
  const int tiles_x = ceil_div(W, AG_TW), tiles_y = ceil_div(H, AG_TH);
  dim3 grid(tiles_x * tiles_y, C3 / 16, B);
  litemla_aggreg_dwpw_kernel<<<grid, 256, AG2_SMEM, (cudaStream_t)stream>>>((const bf16*)ms, (bf16*)ms + C3, ld, (const bf16*)wdw,
                                                                            (const bf16*)wpw, H, W, tiles_x);
  ES3_LAUNCH_CHECK("litemla_aggreg_dwpw_kernel");
  return 0;
}

// ms: [B,HW,ld] bf16 (ld >= 48*heads2), kv_ws: fp32 workspace of B*heads2*ceil(HW/512)*17*16 floats (es3_litemla_ws_floats): the
// partial KV sums, which es3_litemla_attn_bwd reads.  att: [B,HW,ldo] bf16 output (ldo >= 16*heads2).
extern "C" long long es3_litemla_ws_floats(int B, int HW, int heads2) {
  return (long long)B * heads2 * ceil_div(HW, KV_PX) * 17 * 16;
}

extern "C" int es3_litemla_attn_tc(const void* ms, long long ld, float* kv_ws, void* att, long long ldo, int B, int HW,
                                   int heads2, float eps, void* stream) {
  ES3_REQUIRE(ld >= 48 * heads2 && ld % 8 == 0 && ldo % 8 == 0, "es3_litemla_attn_tc: bad ld=%lld ldo=%lld heads2=%d", ld, ldo, heads2);
  cudaStream_t st = (cudaStream_t)stream;
  const int nchunk = ceil_div(HW, KV_PX);
  litemla_kv_tc_kernel<<<dim3(nchunk, heads2, B), 256, 0, st>>>((const bf16*)ms, ld, kv_ws, HW);
  ES3_LAUNCH_CHECK("litemla_kv_tc_kernel");
  litemla_apply_tc_kernel<<<dim3(ceil_div(HW, 256), heads2, B), 128, 0, st>>>((const bf16*)ms, ld, kv_ws, nchunk,
                                                                             (bf16*)att, ldo, HW, eps);
  ES3_LAUNCH_CHECK("litemla_apply_tc_kernel");
  return 0;
}
