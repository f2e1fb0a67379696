// Depthwise 3x3 + pointwise projection (+BN, +residual) in ONE wgmma kernel, for the wide MBConv blocks of EfficientViT
// stages 3/4 (Cin 128/256, expanded 512/1024 channels; reference efficientvit/nn/ops.py:315-367) whose expanded tensor does
// not fit the fully fused kernels: the expand 1x1 stays a gemm_tc call, and this kernel replaces
//     dw_tiled_kernel (reads mid, writes dw-out: 2 x 134 MB at stage 3)  +  gemm_tc (reads dw-out)
// with: TMA (4-D map, 1-pixel halo, zero fill = the depthwise's padding) of a 64-channel chunk of `mid` into a 128B-swizzled
// tile -> 9 diagonal m16n8k8 MMAs per (16 px, 8 ch) read with swizzle-aware ldmatrix -> +bias, act -> bf16 written in the
// 128B-swizzled K-major layout of a wgmma A operand -> wgmma accumulating D[128 px x COUT] in registers over the chunks
// (each of the two compute warpgroups holds COUT / 2 columns) -> BN + residual epilogue.  The depthwise output never exists
// in HBM.
//
// Persistent CTAs; warps 0-7 depthwise + wgmma + epilogue, warp 8 lane 0 = TMA (its warpgroup hands its registers to the other
// two); 2-stage ring of (mid chunk, W3 chunk).  A chunk's projection wgmma is retired only after the next chunk's depthwise, so
// the tensor cores run it while the warps do the depthwise.
#include <cuda.h>

#include "ptx.cuh"

namespace es3 {

int encode_map(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_b, const uint32_t* box);

namespace {
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma_16816(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_1688(float* d, uint32_t a0, uint32_t a1, uint32_t b0) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(b0));
}
}  // namespace

constexpr int DP_TH = 8, DP_TW = 16, DP_HH = DP_TH + 2, DP_HW = DP_TW + 2, DP_PIN = DP_HH * DP_HW;   // 8x16 tile, 10x18 halo
constexpr int DP_MC = 64, DP_THREADS = 384;   // two compute warpgroups + one TMA warpgroup

template <int MID, int COUT, int WSTAGES>
struct DPSmem {
  static constexpr int A_STAGE = (DP_PIN * 128 + 1023) / 1024 * 1024;   // 23552
  static constexpr int W_STAGE = COUT * 128;
  static constexpr int OFF_W3 = 2 * A_STAGE, OFF_DW = OFF_W3 + WSTAGES * W_STAGE, OFF_WDW = OFF_DW + 128 * 128;
  static constexpr int OFF_PAR = OFF_WDW + 9 * MID * 2;                  // fp32 b2[MID] s3[COUT] b3[COUT]
  static constexpr int OFF_BAR = OFF_PAR + (MID + 2 * COUT) * 4;
  static constexpr int TOTAL = OFF_BAR + 128;
};

struct DPArgs {
  const bf16* res;     // [B,H,W,COUT] residual or nullptr
  bf16* y;             // [B,H,W,COUT]
  const float* wdw;    // [9][MID] fp32 (BN scale folded)
  const float* b2;     // [MID]
  const float* s3;     // [COUT]
  const float* b3;
  int H, W, tiles_x, tiles_y, total_tiles;
};

template <int MID, int COUT, int WSTAGES, int ACT>
// One CTA per SM of three warpgroups.  The TMA warpgroup drops to 40 registers so that the two compute warpgroups can hold
// 232 each: the (1024, 256) projection keeps 128 fp32 accumulators per thread live across the asynchronous wgmma window, and
// under the 168-register cap of a uniform 288- or 384-thread CTA it spilled 504 bytes per thread.
__global__ void __launch_bounds__(DP_THREADS, 1)
dwproj_tc_kernel(const __grid_constant__ CUtensorMap tm_mid, const __grid_constant__ CUtensorMap tm_w3, const DPArgs a) {
  using L = DPSmem<MID, COUT, WSTAGES>;
  constexpr int NC = MID / DP_MC;
  static_assert(MID % 64 == 0 && NC >= 2 && (COUT == 128 || COUT == 256) && (WSTAGES == 1 || WSTAGES == 2), "shape");
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* s_a = smem;                       // [2][180 rows][128 B] swizzled mid chunks (TMA)
  uint8_t* s_w3 = smem + L::OFF_W3;          // [WSTAGES][COUT][128 B]
  uint8_t* s_dw = smem + L::OFF_DW;          // [128][128 B] swizzled depthwise output = wgmma A operand
  const bf16* s_wdw = reinterpret_cast<const bf16*>(smem + L::OFF_WDW);   // [NC][9][64]
  float* s_b2 = reinterpret_cast<float*>(smem + L::OFF_PAR);
  float *s_s3 = s_b2 + MID, *s_b3 = s_s3 + COUT;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::OFF_BAR);
  uint64_t *bar_a = bars, *bar_w3 = bars + 2, *bar_afree = bars + 4, *bar_w3free = bars + 6;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int my_tiles = (a.total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const int n_total = my_tiles * NC;

  if (tid == 0) {
    if (ptx::smem_u32(smem) & 1023u) { printf("es3: dwproj_tc dynamic smem base not 1024-byte aligned\n"); __trap(); }
    ptx::prefetch_tmap(&tm_mid); ptx::prefetch_tmap(&tm_w3);
    ptx::mbar_init(bar_a, 1); ptx::mbar_init(bar_a + 1, 1);
    ptx::mbar_init(bar_w3, 1); ptx::mbar_init(bar_w3 + 1, 1);
    ptx::mbar_init(bar_afree, 8); ptx::mbar_init(bar_afree + 1, 8);
    ptx::mbar_init(bar_w3free, 8); ptx::mbar_init(bar_w3free + 1, 8);
    ptx::fence_mbar_init();
  }
  for (int i = tid; i < MID; i += DP_THREADS) s_b2[i] = a.b2[i];
  for (int i = tid; i < COUT; i += DP_THREADS) { s_s3[i] = a.s3[i]; s_b3[i] = a.b3[i]; }
  for (int i = tid; i < 9 * MID; i += DP_THREADS) {
    const int c = i % 64, tap = (i / 64) % 9, ch = i / (64 * 9);
    const_cast<bf16*>(s_wdw)[i] = __float2bfloat16(a.wdw[tap * MID + ch * 64 + c]);
  }
  __syncthreads();
  const int tiles_per_img = a.tiles_x * a.tiles_y;

  if (warp >= 8) {
    // ------------------------------------------------------------------------------------ control: TMA (warp 8 lane 0)
    ptx::setmaxnreg_dec<40>();
    if (warp == 8 && lane == 0 && my_tiles > 0) {
      auto load_a = [&](int g) {       // mid chunk g (tile g / NC, channels (g % NC) * 64 ..) with its 1-pixel halo
        const int t = (int)blockIdx.x + (g / NC) * (int)gridDim.x;
        const int bb = t / tiles_per_img, r = t % tiles_per_img, s = g & 1;
        ptx::mbar_arrive_expect_tx(bar_a + s, DP_PIN * 128);
        ptx::tma_load_4d(&tm_mid, bar_a + s, s_a + s * L::A_STAGE, (g % NC) * DP_MC, (r % a.tiles_x) * DP_TW - 1,
                         (r / a.tiles_x) * DP_TH - 1, bb);
      };
      auto load_w = [&](int g) {
        const int s = (WSTAGES == 2) ? (g & 1) : 0;
        ptx::mbar_arrive_expect_tx(bar_w3 + s, L::W_STAGE);
        ptx::tma_load_2d(&tm_w3, bar_w3 + s, s_w3 + s * L::W_STAGE, (g % NC) * DP_MC, 0);
      };
      load_a(0); load_w(0); load_a(1);
      if (WSTAGES == 2) load_w(1);
      // a mid stage is refilled once the depthwise has read it, a W3 stage once the projection that read it retired
#pragma unroll 1
      for (int g = 0; g < n_total; ++g) {
        if (g + 2 < n_total) { ptx::mbar_wait(bar_afree + (g & 1), (uint32_t)((g >> 1) & 1)); load_a(g + 2); }
        if (g + WSTAGES < n_total) {
          const int ws = (WSTAGES == 2) ? (g & 1) : 0;
          ptx::mbar_wait(bar_w3free + ws, (uint32_t)(WSTAGES == 2 ? ((g >> 1) & 1) : (g & 1)));
          load_w(g + WSTAGES);
        }
      }
    }
  } else {
    // ------------------------------------------------------------------------------------ compute warps 0..7 (two warpgroups)
    // warpgroup hsel accumulates the projection's columns hsel * CW .. +CW for all 128 pixels of the tile in registers
    ptx::setmaxnreg_inc<232>();
    constexpr int CW = COUT / 2;
    const int q = warp & 3, hsel = warp >> 2;
    const int g4 = lane >> 2, t4 = lane & 3;
    const int a_row = lane & 15, a_kh = lane >> 4;
    const uint32_t dshift = (g4 & 1) ? 16u : 0u;
    const bool dvalid = (g4 >> 1) == t4;
    const uint32_t u_dw = ptx::smem_u32(s_dw);
    float proj[2][CW / 2];
    int g = 0;
#pragma unroll 1
    for (int it = 0; it < my_tiles; ++it) {
      const int t = (int)blockIdx.x + it * (int)gridDim.x;
      const int b = t / tiles_per_img, tr = t % tiles_per_img;
      const int oy0 = (tr / a.tiles_x) * DP_TH, ox0 = (tr % a.tiles_x) * DP_TW;
#pragma unroll 1
      for (int c = 0; c < NC; ++c, ++g) {
        const int ws = (WSTAGES == 2) ? (g & 1) : 0;
        ptx::mbar_wait(bar_a + (g & 1), (uint32_t)((g >> 1) & 1));
        const uint32_t u_a = ptx::smem_u32(s_a + (g & 1) * L::A_STAGE);
        // ---- depthwise 3x3: warp -> channel group cg (16 ch), four CONSECUTIVE tile rows hsel*4 .. hsel*4+3: per kx the six
        // input-row fragments are loaded once and shared by the three ky taps of each output row (18 ldmatrix.x4 per chunk)
        const int cg = q;
        const bf16* wd = s_wdw + c * 9 * 64 + cg * 16 + g4;
        float dacc[4][2][4];
#pragma unroll
        for (int m = 0; m < 4; ++m)
#pragma unroll
          for (int i = 0; i < 2; ++i) { dacc[m][i][0] = dacc[m][i][1] = dacc[m][i][2] = dacc[m][i][3] = 0.f; }
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          uint32_t af[6][4];
#pragma unroll
          for (int r = 0; r < 6; ++r) {
            const int row = (hsel * 4 + r) * DP_HW + a_row + kx;                // pixel row of the swizzled tile
            ldsm_x4(u_a + row * 128 + (((cg * 2 + a_kh) ^ (row & 7)) << 4), af[r][0], af[r][1], af[r][2], af[r][3]);
          }
          // taps (0, kx) and (1, kx) in one m16n8k16 (same issue rate as m16n8k8), (2, kx) as a k8 MMA: 12 MMAs per m-tile instead of 18
          uint32_t b_lo[3], b_hi[3];
#pragma unroll
          for (int ky = 0; ky < 3; ++ky) {
            const uint32_t w_lo = (uint32_t)__bfloat16_as_ushort(wd[(ky * 3 + kx) * 64]);
            const uint32_t w_hi = (uint32_t)__bfloat16_as_ushort(wd[(ky * 3 + kx) * 64 + 8]);
            b_lo[ky] = dvalid ? (w_lo << dshift) : 0u;
            b_hi[ky] = dvalid ? (w_hi << dshift) : 0u;
          }
#pragma unroll
          for (int m = 0; m < 4; ++m) {
            const uint32_t a_lo[4] = {af[m][0], af[m][1], af[m + 1][0], af[m + 1][1]};
            const uint32_t a_hi[4] = {af[m][2], af[m][3], af[m + 1][2], af[m + 1][3]};
            mma_16816(dacc[m][0], a_lo, b_lo[0], b_lo[1]);
            mma_16816(dacc[m][1], a_hi, b_hi[0], b_hi[1]);
            mma_1688(dacc[m][0], af[m + 2][0], af[m + 2][1], b_lo[2]);
            mma_1688(dacc[m][1], af[m + 2][2], af[m + 2][3], b_hi[2]);
          }
        }
        // The mid stage was read through the generic proxy (ldmatrix) and TMA (async proxy) refills it once bar_afree completes:
        // the mbarrier alone does not order accesses of different proxies, so without this fence the refill could overtake the
        // reads (seen on H100 as run-to-run differences at two CTAs per SM).
        ptx::fence_proxy_async();
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(bar_afree + (g & 1));   // this warp is done reading the mid stage
        if (c > 0) {
          // project(g-1) ran on the tensor cores under this chunk's depthwise; retire it before s_dw is overwritten
          ptx::wg_wait<0>();
          ptx::wg_fence_regs<CW>(&proj[0][0]);
          __syncwarp();
          if (lane == 0) ptx::mbar_arrive(bar_w3free + ((WSTAGES == 2) ? ((g - 1) & 1) : 0));
        }
        ptx::named_bar(1, 256);                                  // project(g-1) of both warpgroups has finished reading s_dw
        const float* b2 = s_b2 + c * DP_MC;
#pragma unroll
        for (int m = 0; m < 4; ++m) {
          const int mt = hsel * 4 + m;
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int p = mt * DP_TW + g4 + half * 8;
#pragma unroll
            for (int nt = 0; nt < 2; ++nt) {
              const int ch = cg * 16 + nt * 8 + t4 * 2;
              const float2 bb = *reinterpret_cast<const float2*>(b2 + ch);
              const float v0 = es3_act_t<ACT>(dacc[m][nt][half * 2 + 0] + bb.x);
              const float v1 = es3_act_t<ACT>(dacc[m][nt][half * 2 + 1] + bb.y);
              const int j = cg * 2 + nt;
              *reinterpret_cast<uint32_t*>(s_dw + p * 128 + ((j ^ (p & 7)) << 4) + t4 * 4) = pack_bf16x2(v0, v1);
            }
          }
        }
        ptx::fence_proxy_async();                                // generic-proxy writes -> visible to wgmma (async proxy)
        ptx::named_bar(1, 256);                                  // s_dw complete
        ptx::mbar_wait(bar_w3 + ws, (uint32_t)(WSTAGES == 2 ? ((g >> 1) & 1) : (g & 1)));
        ptx::wg_fence();
#pragma unroll
        for (int k = 0; k < DP_MC / 16; ++k) {
          const uint64_t db = ptx::make_desc_sw128(ptx::smem_u32(s_w3 + ws * L::W_STAGE) + hsel * CW * 128 + k * 32);
#pragma unroll
          for (int rb = 0; rb < 2; ++rb) {
            const uint64_t da = ptx::make_desc_sw128(u_dw + rb * 8192 + k * 32);
            if constexpr (CW == 128) ptx::wgmma_m64n128<0, 0>(proj[rb], da, db, (c | k) != 0);
            else ptx::wgmma_m64n64<0, 0>(proj[rb], da, db, (c | k) != 0);
          }
        }
        ptx::wg_commit();                                        // retired under the next chunk's depthwise, or below
      }
      ptx::wg_wait<0>();                                         // the tile's last project: the epilogue reads the accumulators
      ptx::wg_fence_regs<CW>(&proj[0][0]);
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(bar_w3free + ((WSTAGES == 2) ? ((g - 1) & 1) : 0));

      // ---- final epilogue: BN3 (+ residual) -> global, from the accumulator fragments
#pragma unroll
      for (int rb = 0; rb < 2; ++rb)
#pragma unroll
        for (int i = 0; i < CW / 2; i += 2) {
          const int r = rb * 64 + ptx::wg_frag_row(q, lane, i), col = hsel * CW + ptx::wg_frag_col(lane, i);
          const int oy = oy0 + r / DP_TW, ox = ox0 + r % DP_TW;
          if (oy < a.H && ox < a.W) {
            const long long pix = (((long long)b * a.H + oy) * a.W + ox) * COUT + col;
            float f0 = fmaf(proj[rb][i], s_s3[col], s_b3[col]), f1 = fmaf(proj[rb][i + 1], s_s3[col + 1], s_b3[col + 1]);
            if (a.res != nullptr) {
              const float2 xr = unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(a.res + pix)));
              f0 += xr.x; f1 += xr.y;
            }
            *reinterpret_cast<uint32_t*>(a.y + pix) = pack_bf16x2(f0, f1);
          }
        }
    }
  }
}

template <int MID, int COUT, int WSTAGES>
static int launch_dwproj(const void* mid, const void* w3, const DPArgs& a, int B, cudaStream_t st) {
  using L = DPSmem<MID, COUT, WSTAGES>;
  CUtensorMap tm_mid, tm_w3;
  {
    uint64_t dims[4] = {(uint64_t)MID, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)B};
    uint64_t str[3] = {(uint64_t)MID * 2, (uint64_t)a.W * MID * 2, (uint64_t)a.H * a.W * MID * 2};
    uint32_t box[4] = {(uint32_t)DP_MC, (uint32_t)DP_HW, (uint32_t)DP_HH, 1u};
    if (encode_map(&tm_mid, mid, 4, dims, str, box)) return 1;
  }
  {
    uint64_t dims[2] = {(uint64_t)MID, (uint64_t)COUT};
    uint64_t str[1] = {(uint64_t)MID * 2};
    uint32_t box[2] = {(uint32_t)DP_MC, (uint32_t)COUT};
    if (encode_map(&tm_w3, w3, 2, dims, str, box)) return 1;
  }
  auto kern = dwproj_tc_kernel<MID, COUT, WSTAGES, ACT_HSWISH>;
  static bool configured = false;
  if (!configured) {
    ES3_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
    configured = true;
  }
  static int sm_count = 0;
  if (sm_count == 0) {
    int dev = 0;
    ES3_CHECK_CUDA(cudaGetDevice(&dev));
    ES3_CHECK_CUDA(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));
  }
  const int ctas = a.total_tiles < sm_count ? a.total_tiles : sm_count;
  kern<<<ctas, DP_THREADS, L::TOTAL, st>>>(tm_mid, tm_w3, a);
  ES3_LAUNCH_CHECK("dwproj_tc_kernel");
  return 0;
}

}  // namespace es3

using namespace es3;

// y = [res +] s3 * (act(dw3x3(mid) + b2) . W3^T) + b3 for mid [B,H,W,Mid] bf16 (stride 1, zero padding), hardswish.
// Instantiated: (Mid, Cout) = (512, 128), (1024, 256).  Returns -1 (no error set) for any other shape.
extern "C" int es3_dwproj_tc_bf16(const void* mid, const float* wdw, const float* b2, const void* w3, const float* s3, const float* b3,
                                  const void* residual, void* y, int B, int H, int W, int Mid, int Cout, int act, void* stream) {
  if (!(act == ACT_HSWISH && ((Mid == 512 && Cout == 128) || (Mid == 1024 && Cout == 256)))) return -1;
  ES3_REQUIRE(B > 0 && H > 0 && W > 0, "es3_dwproj_tc_bf16: bad shape");
  ES3_REQUIRE((((uintptr_t)mid | (uintptr_t)w3 | (uintptr_t)y | (uintptr_t)residual) & 15) == 0, "es3_dwproj_tc_bf16: 16-byte alignment");
  DPArgs a;
  a.res = (const bf16*)residual; a.y = (bf16*)y; a.wdw = wdw; a.b2 = b2; a.s3 = s3; a.b3 = b3;
  a.H = H; a.W = W; a.tiles_x = ceil_div(W, DP_TW); a.tiles_y = ceil_div(H, DP_TH);
  a.total_tiles = B * a.tiles_x * a.tiles_y;
  cudaStream_t st = (cudaStream_t)stream;
  if (Mid == 512) return launch_dwproj<512, 128, 2>(mid, w3, a, B, st);
  return launch_dwproj<1024, 256, 2>(mid, w3, a, B, st);
}
