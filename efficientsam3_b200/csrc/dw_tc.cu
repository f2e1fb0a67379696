// Stride-1 depthwise convolution (3x3 | 5x5, NHWC bf16) on the legacy tensor-core path: the standalone form of the depthwise stage of
// the fused MBConv kernels, for the places where the depthwise conv cannot be fused -- RepViT's RepVGGDW, TinyViT's MBConv / local
// conv, every train-mode depthwise (its batch statistics need the whole tensor first) and the backward-data pass, which is the same
// convolution on flipped taps (reference: nn.Conv2d(groups=C) inside efficientvit/nn/ops.py:39-80, repvit.py:84-122, tiny_vit.py:97-133).
//
// Why not the CUDA-core tiled kernel (dw_tiled.cu): it spends 28 thread-instructions per output element -- bf16 -> fp32
// unpacking, fp32 FMAs and the cp.async address arithmetic.  Here the taps are DIAGONAL B operands of mma.sync: ldmatrix delivers the bf16 pixels
// straight into A fragments (no unpacking), two taps share one m16n8k16 (A = [tap-a | tap-b] along k, B = [diag(wa) ; diag(wb)]; k16
// issues at the rate of k8), input rows are shared by the taps of neighbouring output rows.  Per 16 pixels x 16
// channels: 3x3 = 4.5 ldmatrix.x4 + 12 MMAs, 5x5 = 10 ldmatrix.x4 + 30 MMAs, fp32 accumulation; bias / activation epilogue in fp32.
//
// The taps are bf16 operands.  Rounding each fp32 tap to nearest moved tiny_vit_5m's embedding from 1.5e-2 to 2.7e-2 of the fp32
// reference (tolerance 2e-2): on smooth feature maps the output is ~ mean(x) * sum(taps), so the error that matters is the error of the
// tap SUM.  es3_round_taps_sum_bf16 therefore picks, per channel, bf16 taps whose sum stays (nearly) the fp32 sum -- nearest rounding,
// then up to four one-ulp moves of the taps with the largest same-sign rounding error.  CPU oracle experiment (tiny_vit_5m, 512^2):
// nearest 1.9e-2, sum-preserving 3.2e-3 output rel-L2 from the taps alone.  A two-term (hi + lo) split of the taps inside one k16
// MMA was also built and measured: exact, but slower than the CUDA-core kernel for
// 5x5 -- not kept.
//
// CTA: 256 threads, persistent over (8 x 32 pixel tile, channel group, image) items, haloed tile double-buffered with cp.async
// (zero fill = the convolution's padding).  Warp -> (16-channel sub-group, half of the tile's rows).
#include <cstdlib>

#include "ptx.cuh"

namespace es3 {
namespace {
__device__ __forceinline__ void tc_cpa16(uint32_t saddr, const void* g, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(saddr), "l"(g), "r"(sz) : "memory");
}
}  // namespace

constexpr int DTC_TH = 8, DTC_TW = 32;

template <int KS, int CG>
struct DtcCfg {
  static constexpr int IH = DTC_TH + KS - 1, IW = DTC_TW + KS - 1;
  static constexpr int PS = CG * 2 + 16;                       // pixel stride: the 16-byte pad keeps 8 consecutive pixels on distinct bank groups
  static constexpr int TILE = IH * IW * PS;
  static constexpr int WB = (KS * KS + 1) * CG * 4;            // fp32 taps [KS*KS][CG] + bias [CG]
  static constexpr int SMEM = 2 * TILE + 2 * WB;
  static constexpr int NSUB = CG / 16;                         // 16-channel sub-groups
  static constexpr int RB = 8 / NSUB;                          // row blocks per sub-group (8 warps = NSUB x RB)
  static constexpr int ROWS = DTC_TH / RB;                     // output rows per warp
  static_assert(NSUB * RB == 8 && ROWS * RB == DTC_TH, "warp split");
};

// x: [B,H,W,*] bf16, pixel stride ldx, channels [0, C) of the view; w: [KS*KS][C] fp32 tap-major (BN scale folded); bias [C] | null;
// out likewise (ldo).  C % CG == 0.
template <int KS, int CG, int ACT>
__global__ void __launch_bounds__(256, (2 * (DtcCfg<KS, CG>::SMEM + 1024) <= 227 * 1024) ? 2 : 1)
dw_tc_kernel(const bf16* __restrict__ x, long long ldx, const float* __restrict__ w, const float* __restrict__ bias, bf16* __restrict__ out,
             long long ldo, int H, int W, int C, int tiles_x, int tiles_per_img, int n_cg, int total_items) {
  using T = DtcCfg<KS, CG>;
  constexpr int PAD = KS / 2, KK = KS * KS, NV = CG / 8, ROWS = T::ROWS;
  extern __shared__ __align__(16) uint8_t dtc_smem[];
  const uint32_t u_base = static_cast<uint32_t>(__cvta_generic_to_shared(dtc_smem));
  float* s_wb = reinterpret_cast<float*>(dtc_smem + 2 * T::TILE);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int sub = warp % T::NSUB, rb = warp / T::NSUB;         // 16-channel sub-group, row block
  const int g = lane >> 2, t4 = lane & 3;
  const int a_row = lane & 15, a_kh = lane >> 4;
  const uint32_t dshift = (g & 1) ? 16u : 0u;
  const bool dvalid = (g >> 1) == t4;

  auto decode = [&](int item, int& tile, int& c0, int& b) {
    const int cg = item % n_cg;
    const int r = item / n_cg;
    tile = r % tiles_per_img;
    b = r / tiles_per_img;
    c0 = cg * CG;
  };
  auto stage = [&](int item, int buf) {
    int tile, c0, b;
    decode(item, tile, c0, b);
    const int iy0 = (tile / tiles_x) * DTC_TH - PAD, ix0 = (tile % tiles_x) * DTC_TW - PAD;
    const uint32_t u_tile = u_base + buf * T::TILE;
    const bf16* xb = x + (long long)b * H * W * ldx + c0;
    for (int i = tid; i < T::IH * T::IW * NV; i += 256) {
      const int v = i % NV, p = i / NV;
      const int py = p / T::IW, px = p - py * T::IW;
      const int iy = iy0 + py, ix = ix0 + px;
      const bool ok = iy >= 0 && iy < H && ix >= 0 && ix < W;
      tc_cpa16(u_tile + p * T::PS + v * 16, ok ? xb + ((long long)iy * W + ix) * ldx + v * 8 : xb, ok);
    }
    float* s_w = s_wb + buf * (T::WB / 4);
    for (int i = tid; i < KK * CG; i += 256) s_w[i] = w[(long long)(i / CG) * C + c0 + i % CG];
    for (int i = tid; i < CG; i += 256) s_w[KK * CG + i] = bias ? bias[c0 + i] : 0.f;
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  int item = blockIdx.x;
  if (item >= total_items) return;
  stage(item, 0);
  int buf = 0;
  for (; item < total_items; item += gridDim.x, buf ^= 1) {
    const int next = item + gridDim.x;
    if (next < total_items) {
      stage(next, buf ^ 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    int tile, c0, b;
    decode(item, tile, c0, b);
    const int oy0 = (tile / tiles_x) * DTC_TH, ox0 = (tile % tiles_x) * DTC_TW;
    const uint32_t u_tile = u_base + buf * T::TILE;
    const float* s_w = s_wb + buf * (T::WB / 4);
    const float* s_b = s_w + KK * CG;

    // diagonal B fragments of this warp's 16 channels, all taps (bf16-rounded weights)
    uint32_t b_lo[KK], b_hi[KK];
#pragma unroll
    for (int t = 0; t < KK; ++t) {
      const uint32_t w_lo = (uint32_t)__bfloat16_as_ushort(__float2bfloat16(s_w[t * CG + sub * 16 + g]));
      const uint32_t w_hi = (uint32_t)__bfloat16_as_ushort(__float2bfloat16(s_w[t * CG + sub * 16 + 8 + g]));
      b_lo[t] = dvalid ? (w_lo << dshift) : 0u;
      b_hi[t] = dvalid ? (w_hi << dshift) : 0u;
    }
    const float2 bias_lo = *reinterpret_cast<const float2*>(s_b + sub * 16 + t4 * 2);
    const float2 bias_hi = *reinterpret_cast<const float2*>(s_b + sub * 16 + 8 + t4 * 2);
    bf16* ob = out + (long long)b * H * W * ldo + c0 + sub * 16;

#pragma unroll 1
    for (int xh = 0; xh < 2; ++xh) {                          // the two 16-pixel halves of the tile's rows
      float acc[ROWS][2][4];
#pragma unroll
      for (int m = 0; m < ROWS; ++m)
#pragma unroll
        for (int n = 0; n < 2; ++n) { acc[m][n][0] = acc[m][n][1] = acc[m][n][2] = acc[m][n][3] = 0.f; }
#pragma unroll
      for (int kx = 0; kx < KS; ++kx) {
        uint32_t af[ROWS + KS - 1][4];                        // the input rows this warp's ROWS output rows touch, column offset kx
#pragma unroll
        for (int r = 0; r < ROWS + KS - 1; ++r)
          ptx::ldsm_x4(u_tile + ((rb * ROWS + r) * T::IW + xh * 16 + a_row + kx) * T::PS + (sub * 16 + a_kh * 8) * 2, af[r][0], af[r][1], af[r][2],
                       af[r][3]);
#pragma unroll
        for (int m = 0; m < ROWS; ++m) {
#pragma unroll
          for (int kp = 0; kp < KS / 2; ++kp) {               // tap pairs (2 kp, kx) + (2 kp + 1, kx) in one k16 MMA
            const uint32_t a_lo[4] = {af[m + 2 * kp][0], af[m + 2 * kp][1], af[m + 2 * kp + 1][0], af[m + 2 * kp + 1][1]};
            const uint32_t a_hi[4] = {af[m + 2 * kp][2], af[m + 2 * kp][3], af[m + 2 * kp + 1][2], af[m + 2 * kp + 1][3]};
            ptx::mma_16816(acc[m][0], a_lo, b_lo[(2 * kp) * KS + kx], b_lo[(2 * kp + 1) * KS + kx]);
            ptx::mma_16816(acc[m][1], a_hi, b_hi[(2 * kp) * KS + kx], b_hi[(2 * kp + 1) * KS + kx]);
          }
          ptx::mma_1688(acc[m][0], af[m + KS - 1][0], af[m + KS - 1][1], b_lo[(KS - 1) * KS + kx]);   // the odd tap row
          ptx::mma_1688(acc[m][1], af[m + KS - 1][2], af[m + KS - 1][3], b_hi[(KS - 1) * KS + kx]);
        }
      }
#pragma unroll
      for (int m = 0; m < ROWS; ++m) {
        const int oy = oy0 + rb * ROWS + m;
        if (oy >= H) continue;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int ox = ox0 + xh * 16 + g + half * 8;
          if (ox >= W) continue;
          bf16* dst = ob + ((long long)oy * W + ox) * ldo + t4 * 2;
          *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(es3_act_t<ACT>(acc[m][0][half * 2] + bias_lo.x), es3_act_t<ACT>(acc[m][0][half * 2 + 1] + bias_lo.y));
          *reinterpret_cast<uint32_t*>(dst + 8) = pack_bf16x2(es3_act_t<ACT>(acc[m][1][half * 2] + bias_hi.x), es3_act_t<ACT>(acc[m][1][half * 2 + 1] + bias_hi.y));
        }
      }
    }
    __syncthreads();     // this item's buffer is free for the stage() of the next iteration
  }
}

// One thread per channel: out[tap][c] = bf16-representable taps (stored as fp32) with sum_c(out) ~ sum_c(w).
__global__ void round_taps_sum_bf16_kernel(const float* __restrict__ w, float* __restrict__ out, int KK, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float t[25], r[25];
  float sum_w = 0.f, sum_r = 0.f;
#pragma unroll
  for (int i = 0; i < 25; ++i) {
    if (i < KK) {
      t[i] = w[(long long)i * C + c];
      r[i] = __bfloat162float(__float2bfloat16(t[i]));
      sum_w += t[i];
      sum_r += r[i];
    }
  }
  for (int it = 0; it < 4; ++it) {
    const float res = sum_w - sum_r;
    if (res == 0.f) break;
    const float sgn = res > 0.f ? 1.f : -1.f;
    int best = 0;
    float best_score = -INFINITY;
#pragma unroll
    for (int i = 0; i < 25; ++i) {
      if (i < KK) {
        const float score = (t[i] - r[i]) * sgn;
        if (score > best_score) { best_score = score; best = i; }
      }
    }
    float rb = 0.f;
#pragma unroll
    for (int i = 0; i < 25; ++i) if (i == best) rb = r[i];
    const float ulp = __uint_as_float(__float_as_uint(rb) & 0x7f800000u) * 0.0078125f;     // 2^(exponent - 7): one bf16 step at rb
    if (ulp == 0.f) break;
    const float cand = __bfloat162float(__float2bfloat16(rb + sgn * ulp));
    const float new_sum = sum_r - rb + cand;
    if (fabsf(sum_w - new_sum) >= fabsf(res)) break;
#pragma unroll
    for (int i = 0; i < 25; ++i) if (i == best) r[i] = cand;
    sum_r = new_sum;
  }
#pragma unroll
  for (int i = 0; i < 25; ++i)
    if (i < KK) out[(long long)i * C + c] = r[i];
}

template <int KS, int CG, int ACT>
static int launch_dw_tc(const bf16* x, long long ldx, const float* w, const float* bias, bf16* out, long long ldo, int B, int H, int W, int C,
                        cudaStream_t st) {
  using T = DtcCfg<KS, CG>;
  auto kern = dw_tc_kernel<KS, CG, ACT>;
  static bool configured = false;
  if (!configured) {
    ES3_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, T::SMEM));
    configured = true;
  }
  const int tiles_x = ceil_div(W, DTC_TW), tiles_y = ceil_div(H, DTC_TH);
  const int n_cg = C / CG;
  const long long total = (long long)tiles_x * tiles_y * n_cg * B;
  ES3_REQUIRE(total < (1LL << 31), "dw_tc: too many work items");
  static int sm_count = 0;
  if (sm_count == 0) {
    int dev = 0;
    ES3_CHECK_CUDA(cudaGetDevice(&dev));
    ES3_CHECK_CUDA(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));
  }
  const int per_sm = 2 * (T::SMEM + 1024) <= 227 * 1024 ? 2 : 1;
  const long long ctas = (long long)sm_count * per_sm;
  kern<<<(unsigned)(total < ctas ? total : ctas), 256, T::SMEM, st>>>(x, ldx, w, bias, out, ldo, H, W, C, tiles_x, tiles_x * tiles_y, n_cg,
                                                                      (int)total);
  ES3_LAUNCH_CHECK("dw_tc_kernel");
  return 0;
}

}  // namespace es3

using namespace es3;

/* Stride-1 depthwise ks x ks (3 | 5), pad ks/2, C % 32 == 0, on mma.sync with diagonal tap operands.  Same contract as
 * es3_dwconv_tiled_bf16 with stride = 1; the taps are bf16 operands (nearest rounding of what is passed: pass taps prepared by
 * es3_round_taps_sum_bf16 to keep the tap sums, as ops.dwconv does). */
extern "C" int es3_dwconv_tc_bf16(const void* x, long long ldx, const float* w, const float* bias, void* out, long long ldo, int B, int H,
                                  int W, int C, int ks, int act, void* stream) {
  ES3_REQUIRE(C % 32 == 0 && ldx % 8 == 0 && ldo % 8 == 0 && (ks == 3 || ks == 5), "es3_dwconv_tc_bf16: need C %% 32 == 0, ks 3|5 (C=%d ks=%d)", C, ks);
  ES3_REQUIRE(((uintptr_t)x & 15) == 0 && ((uintptr_t)out & 3) == 0, "es3_dwconv_tc_bf16: x must be 16-byte aligned");
  ES3_REQUIRE(act == ACT_NONE || act == ACT_HSWISH || act == ACT_GELU || act == ACT_RELU, "es3_dwconv_tc_bf16: activation %d not instantiated", act);
  cudaStream_t st = (cudaStream_t)stream;
  const bf16* xi = (const bf16*)x;
  bf16* o = (bf16*)out;
#define ES3_DTC_CASE(KS_, CG_)                                                                                    \
  switch (act) {                                                                                                  \
    case ACT_NONE: return launch_dw_tc<KS_, CG_, ACT_NONE>(xi, ldx, w, bias, o, ldo, B, H, W, C, st);             \
    case ACT_RELU: return launch_dw_tc<KS_, CG_, ACT_RELU>(xi, ldx, w, bias, o, ldo, B, H, W, C, st);             \
    case ACT_HSWISH: return launch_dw_tc<KS_, CG_, ACT_HSWISH>(xi, ldx, w, bias, o, ldo, B, H, W, C, st);         \
    default: return launch_dw_tc<KS_, CG_, ACT_GELU>(xi, ldx, w, bias, o, ldo, B, H, W, C, st);                   \
  }
  if (ks == 3) {
    if (C % 64 == 0) { ES3_DTC_CASE(3, 64) } else { ES3_DTC_CASE(3, 32) }
  } else {
    ES3_DTC_CASE(5, 32)
  }
#undef ES3_DTC_CASE
  return 1;
}

/* Per channel, bf16-representable depthwise taps (written as fp32) whose sum stays as close as possible to the fp32 tap sum: w, out
 * [KK][C] tap-major, KK <= 25.  Feed the result to es3_dwconv_tc_bf16 (whose nearest rounding is then the identity). */
extern "C" int es3_round_taps_sum_bf16(const float* w, float* out, int KK, int C, void* stream) {
  ES3_REQUIRE(KK > 0 && KK <= 25 && C > 0, "es3_round_taps_sum_bf16: bad shape (KK=%d C=%d)", KK, C);
  round_taps_sum_bf16_kernel<<<ceil_div(C, 128), 128, 0, (cudaStream_t)stream>>>(w, out, KK, C);
  ES3_LAUNCH_CHECK("round_taps_sum_bf16_kernel");
  return 0;
}
