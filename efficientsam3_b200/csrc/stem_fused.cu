// EfficientViT input stem in ONE kernel, on tensor cores (mma.sync):
//   x1 = hswish(BN(conv3x3_s2(img)))                       input_stem.op_list.0   (efficientvit/backbone.py:49-57)
//   y  = x1 + BN(pw(hswish(BN(dw3x3(x1)))))                input_stem.op_list.1   (ResidualBlock(DSConv), :58-67)
// The two-kernel version (conv.cu: stem_conv3x3_s2 + dsconv_res) was FMA-issue bound (432 + 400 FMAs per pixel)
// and round-tripped x1 through HBM.  Here a CTA owns an 8 x 32 tile of output pixels:
//   phase 0  stage the fp32 NCHW input patch (zero outside the image)
//   phase 1  im2col A fragments (K = 27 padded to 32) gathered from the patch into registers, tile + 1-pixel halo
//   phase 2  x1 = A * W0^T on mma.sync (16 channels), BN + hardswish, zero outside the x1 map (the depthwise's padding),
//            kept in smem as bf16 (the same rounding the unfused path applies when it stores x1)
//   phase 3  depthwise 3x3 as 9 diagonal-B MMAs, BN + hardswish, result re-used in registers as the A operand of the
//            16x16 pointwise MMA, + BN + residual(x1) -> global (NHWC bf16)
#include "ptx.cuh"

namespace es3 {
namespace {
__device__ __forceinline__ void cpa4(uint32_t saddr, const void* g, uint32_t sz) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(saddr), "l"(g), "r"(sz) : "memory");
}
__device__ __forceinline__ void cpa16(uint32_t saddr, const void* g, uint32_t sz) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(saddr), "l"(g), "r"(sz) : "memory");
}
}  // namespace

constexpr int SF_TH = 8, SF_TW = 32, SF_C = 16;
constexpr int SF_XH = SF_TH + 2, SF_XW = SF_TW + 2;            // x1 tile with halo: 10 x 34
constexpr int SF_NPX = SF_XH * SF_XW, SF_NPX_PAD = (SF_NPX + 15) / 16 * 16;   // 340 -> 352
constexpr int SF_IH = 2 * (SF_XH - 1) + 3;                                    // 21 input rows
constexpr int SF_IW = 72;   // 69 input columns (2*33 + 3), widened to 72 with the origin moved one pixel left: 16-byte aligned rows
constexpr int SF_ARS = 32 * 2 + 16;   // im2col row: 32 bf16 + pad
constexpr int SF_XRS = SF_C * 2 + 16; // x1 row: 16 bf16 + pad
constexpr int SF_IN_BYTES = (3 * SF_IH * SF_IW * 4 + 15) / 16 * 16;
constexpr int SF_X_BYTES = SF_NPX_PAD * SF_XRS;
constexpr int SF_SMEM = SF_IN_BYTES + SF_X_BYTES + 16 * SF_ARS + 16 * SF_XRS + (9 * 16 + 6 * 16) * 4;

struct StemArgs {
  const float* img;   // [B,3,H,W]
  bf16* out;          // [B,Ho,Wo,16]
  const bf16* w0;     // [16][32] stem weights, k = ci*9 + ky*3 + kx, zero padded
  const float* s0; const float* b0;    // folded BN after the stem conv
  const float* wdw;   // [9][16] depthwise weights (BN scale folded)
  const float* bdw;   // [16]
  const bf16* wpw;    // [16][16] pointwise weights [n][k]
  const float* spw; const float* bpw;  // folded BN after the pointwise conv
  int H, W, Ho, Wo, tiles_x;
  int vec16;          // image rows are 16-byte aligned (W % 4 == 0, aligned base): 16-byte cp.async
};

__global__ void __launch_bounds__(256) stem_fused_kernel(const StemArgs a) {
  extern __shared__ __align__(16) uint8_t smem[];
  float* s_in = reinterpret_cast<float*>(smem);                     // [3][SF_IH][SF_IW]
  uint8_t* s_x = smem + SF_IN_BYTES;                                 // x1 [SF_NPX_PAD][16]
  uint8_t* s_w0 = s_x + SF_X_BYTES;                                  // [16][32]
  uint8_t* s_wp = s_w0 + 16 * SF_ARS;                                // [16][16]
  float* s_f = reinterpret_cast<float*>(s_wp + 16 * SF_XRS);         // wdw[9][16] | s0 b0 bdw spw bpw (16 each)
  float* s_wdw = s_f;
  float* s_s0 = s_f + 144; float* s_b0 = s_s0 + 16; float* s_bdw = s_b0 + 16; float* s_spw = s_bdw + 16; float* s_bpw = s_spw + 16;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.y;
  const int oy0 = (blockIdx.x / a.tiles_x) * SF_TH, ox0 = (blockIdx.x % a.tiles_x) * SF_TW;
  const int iy0 = 2 * oy0 - 3, ix0 = 2 * ox0 - 4;   // input coords of the patch origin (x: one extra pixel on the left, see SF_IW)

  // ---- phase 0: input patch (4-byte cp.async with zero fill outside the image: every copy of the CTA is in flight
  // before anything waits) + weights
  const float* ib = a.img + (long long)b * 3 * a.H * a.W;
  const uint32_t u_in = static_cast<uint32_t>(__cvta_generic_to_shared(s_in));
  if (a.vec16) {
    // rows are 16-byte aligned and no 4-pixel group straddles the image border: 18 cp.async.16 per row instead of 69 x 4 bytes
    for (int i = tid; i < 3 * SF_IH * (SF_IW / 4); i += 256) {
      const int r = i / (SF_IW / 4), k = i - r * (SF_IW / 4);
      const int c = r / SF_IH, y = r - c * SF_IH;
      const int iy = iy0 + y, ix = ix0 + 4 * k;
      const bool in = iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;
      cpa16(u_in + (r * SF_IW + 4 * k) * 4, ib + ((long long)c * a.H + (in ? iy : 0)) * a.W + (in ? ix : 0), in ? 16u : 0u);
    }
  } else {
    for (int r = warp; r < 3 * SF_IH; r += 8) {
      const int c = r / SF_IH, y = r - c * SF_IH;
      const int iy = iy0 + y;
      const bool rowin = iy >= 0 && iy < a.H;
      const float* src = ib + ((long long)c * a.H + (rowin ? iy : 0)) * a.W;
#pragma unroll
      for (int x = lane; x < SF_IW; x += 32) {
        const int ix = ix0 + x;
        const bool in = rowin && ix >= 0 && ix < a.W;
        cpa4(u_in + (r * SF_IW + x) * 4, src + (in ? ix : 0), in ? 4u : 0u);
      }
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  for (int i = tid; i < 16 * 32; i += 256) *reinterpret_cast<bf16*>(s_w0 + (i >> 5) * SF_ARS + (i & 31) * 2) = a.w0[i];
  for (int i = tid; i < 16 * 16; i += 256) *reinterpret_cast<bf16*>(s_wp + (i >> 4) * SF_XRS + (i & 15) * 2) = a.wpw[i];
  for (int i = tid; i < 144; i += 256) s_wdw[i] = a.wdw[i];
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  if (tid < 16) { s_s0[tid] = a.s0[tid]; s_b0[tid] = a.b0[tid]; s_bdw[tid] = a.bdw[tid]; s_spw[tid] = a.spw[tid]; s_bpw[tid] = a.bpw[tid]; }
  __syncthreads();

  const uint32_t u_x = static_cast<uint32_t>(__cvta_generic_to_shared(s_x));
  const uint32_t u_w0 = static_cast<uint32_t>(__cvta_generic_to_shared(s_w0));
  const uint32_t u_wp = static_cast<uint32_t>(__cvta_generic_to_shared(s_wp));
  const int a_row = lane & 15, a_kh = lane >> 4;
  const int b_n = (lane & 7) + ((lane >> 4) << 3), b_kh = (lane >> 3) & 1;
  const int g = lane >> 2, t4 = lane & 3;

  // ---- phase 2: x1 = im2col * W0^T  (N = 16: two n-tiles; K = 32: two k-steps).  The im2col A fragments are gathered
  // straight from the staged patch: a lane always owns the same 8 k columns, so their patch offsets are loop invariants.
  {
    uint32_t wf[2][4];
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) ptx::ldsm_x4(u_w0 + b_n * SF_ARS + (ks * 16 + b_kh * 8) * 2, wf[ks][0], wf[ks][1], wf[ks][2], wf[ks][3]);
    int koff[8];
    bool kval[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = (j >> 2) * 16 + ((j >> 1) & 1) * 8 + 2 * t4 + (j & 1);
      kval[j] = k < 27;
      const int kk = kval[j] ? k : 0;
      const int ci = kk / 9, r = kk - ci * 9, ky = r / 3, kx = r - ky * 3;
      koff[j] = (ci * SF_IH + ky) * SF_IW + kx + 1;   // +1: the patch origin sits one pixel left of the first tap
    }
    for (int mt = warp; mt < SF_NPX_PAD / 16; mt += 8) {
      float d[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
      const int p0 = min(mt * 16 + g, SF_NPX - 1), p1 = min(mt * 16 + g + 8, SF_NPX - 1);
      const float* q0 = s_in + (2 * (p0 / SF_XW)) * SF_IW + 2 * (p0 % SF_XW);
      const float* q1 = s_in + (2 * (p1 / SF_XW)) * SF_IW + 2 * (p1 % SF_XW);
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        float v[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          v[j] = kval[ks * 4 + j] ? q0[koff[ks * 4 + j]] : 0.f;
          v[4 + j] = kval[ks * 4 + j] ? q1[koff[ks * 4 + j]] : 0.f;
        }
        // A fragment: {row g, k lo pair}, {row g+8, k lo pair}, {row g, k hi pair}, {row g+8, k hi pair}
        const uint32_t af[4] = {pack_bf16x2(v[0], v[1]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[6], v[7])};
        ptx::mma_16816(d[0], af, wf[ks][0], wf[ks][1]);
        ptx::mma_16816(d[1], af, wf[ks][2], wf[ks][3]);
      }
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int p = mt * 16 + g + half * 8;
        const int Y = oy0 - 1 + p / SF_XW, X = ox0 - 1 + p % SF_XW;
        const bool in = p < SF_NPX && Y >= 0 && Y < a.Ho && X >= 0 && X < a.Wo;
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
          const int c = nt * 8 + t4 * 2;
          float v0 = es3_act_t<ACT_HSWISH>(fmaf(d[nt][half * 2], s_s0[c], s_b0[c]));
          float v1 = es3_act_t<ACT_HSWISH>(fmaf(d[nt][half * 2 + 1], s_s0[c + 1], s_b0[c + 1]));
          if (!in) { v0 = 0.f; v1 = 0.f; }
          *reinterpret_cast<uint32_t*>(s_x + p * SF_XRS + c * 2) = pack_bf16x2(v0, v1);
        }
      }
    }
  }
  __syncthreads();

  // ---- phase 3: depthwise (diagonal-B MMAs) -> hswish -> pointwise MMA -> + residual
  {
    // diagonal B fragments of the 9 taps for this lane (explained at the top of mbconv_tc.cu): non-zero only where k == n
    uint32_t dlo[9], dhi[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      uint32_t lo = 0u, hi = 0u;
      if ((g >> 1) == t4) {
        const uint32_t w_lo = (uint32_t)__bfloat16_as_ushort(__float2bfloat16(s_wdw[t * 16 + g]));
        const uint32_t w_hi = (uint32_t)__bfloat16_as_ushort(__float2bfloat16(s_wdw[t * 16 + 8 + g]));
        lo = (g & 1) ? (w_lo << 16) : w_lo;
        hi = (g & 1) ? (w_hi << 16) : w_hi;
      }
      dlo[t] = lo; dhi[t] = hi;
    }
    uint32_t pwf[4];
    ptx::ldsm_x4(u_wp + b_n * SF_XRS + b_kh * 16, pwf[0], pwf[1], pwf[2], pwf[3]);
    bf16* ob = a.out + (long long)b * a.Ho * a.Wo * SF_C;
    for (int mt = warp; mt < SF_TH * (SF_TW / 16); mt += 8) {
      const int ry = mt >> 1, rx0 = (mt & 1) * 16;   // output row / first column inside the tile
      float d[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
      // taps in pairs as m16n8k16 MMAs (A = [tap-a fragment | tap-b fragment] along k, B = [diag(wa) ; diag(wb)]; k16 issues at the rate
      // of k8), tap 8 as m16n8k8: 10 MMAs per m-tile instead of 18
      auto frag = [&](int tap, uint32_t* af) {
        const int ky = tap / 3, kx = tap - ky * 3;
        ptx::ldsm_x4(u_x + ((ry + ky) * SF_XW + rx0 + a_row + kx) * SF_XRS + a_kh * 16, af[0], af[1], af[2], af[3]);
      };
#pragma unroll
      for (int tp = 0; tp < 4; ++tp) {
        uint32_t fa[4], fb[4];
        frag(2 * tp, fa); frag(2 * tp + 1, fb);
        const uint32_t a_lo[4] = {fa[0], fa[1], fb[0], fb[1]};
        const uint32_t a_hi[4] = {fa[2], fa[3], fb[2], fb[3]};
        ptx::mma_16816(d[0], a_lo, dlo[2 * tp], dlo[2 * tp + 1]);
        ptx::mma_16816(d[1], a_hi, dhi[2 * tp], dhi[2 * tp + 1]);
      }
      {
        uint32_t fa[4];
        frag(8, fa);
        ptx::mma_1688(d[0], fa[0], fa[1], dlo[8]);
        ptx::mma_1688(d[1], fa[2], fa[3], dhi[8]);
      }
      // hswish(dw + bias) -> A fragment of the pointwise MMA (C-fragment layout == A-fragment layout)
      uint32_t pa[4];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        const int c = nt * 8 + t4 * 2;
        pa[nt * 2 + 0] = pack_bf16x2(es3_act_t<ACT_HSWISH>(d[nt][0] + s_bdw[c]), es3_act_t<ACT_HSWISH>(d[nt][1] + s_bdw[c + 1]));
        pa[nt * 2 + 1] = pack_bf16x2(es3_act_t<ACT_HSWISH>(d[nt][2] + s_bdw[c]), es3_act_t<ACT_HSWISH>(d[nt][3] + s_bdw[c + 1]));
      }
      float o[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
      ptx::mma_16816(o[0], pa, pwf[0], pwf[1]);
      ptx::mma_16816(o[1], pa, pwf[2], pwf[3]);
      const int oy = oy0 + ry;
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int xl = rx0 + g + half * 8;
        const int ox = ox0 + xl;
        if (oy >= a.Ho || ox >= a.Wo) continue;
        const uint8_t* xc = s_x + ((ry + 1) * SF_XW + xl + 1) * SF_XRS;   // residual: x1 at the centre
        bf16* dst = ob + ((long long)oy * a.Wo + ox) * SF_C;
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
          const int c = nt * 8 + t4 * 2;
          const float2 r = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(xc + c * 2));
          const float v0 = fmaf(o[nt][half * 2], s_spw[c], s_bpw[c]) + r.x;
          const float v1 = fmaf(o[nt][half * 2 + 1], s_spw[c + 1], s_bpw[c + 1]) + r.y;
          *reinterpret_cast<uint32_t*>(dst + c) = pack_bf16x2(v0, v1);
        }
      }
    }
  }
}

}  // namespace es3

using namespace es3;

// Fused EfficientViT-B1 input stem (16 channels).  w0 [16][32] bf16 (k = ci*9+ky*3+kx, zero padded), s0/b0 folded BN;
// wdw [9][16] fp32 (BN scale folded), bdw [16]; wpw [16][16] bf16 [n][k], spw/bpw folded BN.  out [B,Ho,Wo,16] bf16.
extern "C" int es3_stem_fused_c16(const float* img, const void* w0, const float* s0, const float* b0, const float* wdw,
                                  const float* bdw, const void* wpw, const float* spw, const float* bpw, void* out, int B,
                                  int H, int W, void* stream) {
  StemArgs a;
  a.img = img; a.out = (bf16*)out; a.w0 = (const bf16*)w0; a.s0 = s0; a.b0 = b0; a.wdw = wdw; a.bdw = bdw;
  a.wpw = (const bf16*)wpw; a.spw = spw; a.bpw = bpw;
  a.H = H; a.W = W; a.Ho = (H - 1) / 2 + 1; a.Wo = (W - 1) / 2 + 1;
  a.tiles_x = ceil_div(a.Wo, SF_TW);
  a.vec16 = ((W & 3) == 0 && ((uintptr_t)img & 15) == 0) ? 1 : 0;
  static bool configured = false;
  if (!configured) {
    ES3_CHECK_CUDA(cudaFuncSetAttribute(stem_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SF_SMEM));
    configured = true;
  }
  dim3 grid(a.tiles_x * ceil_div(a.Ho, SF_TH), B);
  stem_fused_kernel<<<grid, 256, SF_SMEM, (cudaStream_t)stream>>>(a);
  ES3_LAUNCH_CHECK("stem_fused_kernel");
  return 0;
}
