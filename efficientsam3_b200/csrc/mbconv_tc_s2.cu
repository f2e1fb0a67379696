// Fused stride-2 MBConv on wgmma (the stage-opening blocks 16->64->32 @512^2, 32->128->64 @256^2, 64->256->128 @128^2 of
// efficientvit_b1: y = BN3(pw2(act(BN2(dw3x3_s2(act(BN1(pw1(x)))))))), no residual; reference efficientvit/nn/ops.py:315-367).
// Same machinery as mbconv_tc.cu (TMA-staged swizzled input tile, wgmma expand into registers, BN+act epilogue into a
// pixel-major smem tile, diagonal m16n8k8 depthwise into the swizzled A operand of the projecting wgmma that accumulates over
// chunks), with the geometry of a stride-2 block: a 4 x 16 output tile needs a 9 x 33 input tile = 297 pixels = five 64-row
// wgmma blocks, so the expanded tensor is processed in 32-channel chunks to keep its tile (297 x 32 bf16) at 24 KB and two
// CTAs on an SM.  Project K-steps per chunk: 2 (32 channels); the W3 box still loads 64 K-columns (128-byte swizzled rows), the
// upper half is simply not referenced.
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
__device__ __forceinline__ void compute_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
}  // namespace

constexpr int S2_TH = 4, S2_TW = 16;                       // output tile (64 pixels = rows 0..63 of the project wgmma)
constexpr int S2_IH = 2 * S2_TH + 1, S2_IW = 2 * S2_TW + 1;  // 9 x 33 input pixels
constexpr int S2_PIN = S2_IH * S2_IW;                      // 297
constexpr int S2_MC = 32;                                  // expanded-channel chunk
constexpr int S2_RS_MID = S2_MC * 2 + 16;                  // 80-byte rows: conflict-free 16-byte stores / ldmatrix
// s_mid keeps the EVEN and ODD input columns of every input row in separate planes (even column 2j -> slot j, odd column 2j+1 ->
// slot S2_ODD + j).  A stride-2 tap then walks CONSECUTIVE 80-byte rows (8 rows -> 8 distinct 4-bank groups); walking every other
// row of an interleaved tile (160-byte stride) made every ldmatrix 2-way conflicted.  S2_ODD = 20 also keeps the expand epilogue's 16-byte stores (lanes alternate planes) apart.
constexpr int S2_ODD = 20, S2_PW = S2_ODD + S2_TW;           // slots per input row: 17 even | 3 unused | 16 odd
constexpr int S2_THREADS = 384;                           // two compute warpgroups + one TMA warpgroup

template <int MID, int COUT, int WSTAGES>
struct S2Smem {
  // 38912: the 297 input rows.  The expand reads five 64-row blocks (320 rows): rows 304..319 fall on the depthwise weights and
  // per-channel parameters that follow, which are written once before the main loop and read-only after (a whole 320-row
  // buffer would not leave room for two CTAs per SM at (64, 256, 128)).
  static constexpr int IN = (S2_PIN * 128 + 1023) / 1024 * 1024;
  static constexpr int W1 = 2 * S2_MC * 128;
  static constexpr int W3_STAGE = COUT * 128;
  static constexpr int OFF_WDW = IN;                                   // bf16 [MID/32][9][32]
  static constexpr int OFF_PAR = OFF_WDW + 9 * MID * 2;
  static constexpr int OFF_BAR = OFF_PAR + (3 * MID + 2 * COUT) * 4;
  static constexpr int OFF_W1 = (OFF_BAR + 128 + 1023) / 1024 * 1024;
  static constexpr int OFF_W3 = OFF_W1 + W1, OFF_DW = OFF_W3 + WSTAGES * W3_STAGE, OFF_MID = OFF_DW + 128 * 128;
  static constexpr int TOTAL = OFF_MID + (S2_IH * S2_PW * S2_RS_MID + 15) / 16 * 16;
  static_assert(5 * 64 * 128 <= OFF_BAR, "the padding rows of the A operand must fall on the read-only parameters");
  static_assert(2 * (TOTAL + 1024) <= 233472, "two CTAs per SM");
};

struct S2Args {
  bf16* y;             // [B,Ho,Wo,COUT]
  const float* s1;     // [MID]
  const float* b1;
  const float* wdw;    // [9][MID] fp32 (BN2 scale folded)
  const float* b2;
  const float* s3;     // [COUT]
  const float* b3;
  int H, W, Ho, Wo, tiles_x, tiles_y, total_tiles;
};

// MINB CTAs per SM; the TMA warpgroup gives its registers to the compute warpgroups (setmaxnreg), as in mbconv_tc.cu.
template <int MINB>
struct S2Regs {
  static constexpr int TMA = MINB == 1 ? 40 : 24, MMA = MINB == 1 ? 232 : 104;
};

template <int CIN, int MID, int COUT, int WSTAGES, int ACT, int MINB>
__global__ void __launch_bounds__(S2_THREADS, MINB)
mbconv_tc_s2_kernel(const __grid_constant__ CUtensorMap tm_in, const __grid_constant__ CUtensorMap tm_w1,
                    const __grid_constant__ CUtensorMap tm_w3, const S2Args a) {
  using L = S2Smem<MID, COUT, WSTAGES>;
  constexpr int NC = MID / S2_MC;
  static_assert(CIN % 16 == 0 && CIN <= 64 && MID % 32 == 0 && NC >= 2 && (COUT == 32 || COUT == 64 || COUT == 128), "shape");
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* s_in = smem;
  uint8_t* s_w1 = smem + L::OFF_W1;
  uint8_t* s_w3 = smem + L::OFF_W3;
  uint8_t* s_dw = smem + L::OFF_DW;
  uint8_t* s_mid = smem + L::OFF_MID;
  const bf16* s_wdw = reinterpret_cast<const bf16*>(smem + L::OFF_WDW);
  float* s_par = reinterpret_cast<float*>(smem + L::OFF_PAR);
  float *s_s1 = s_par, *s_b1 = s_par + MID, *s_b2 = s_par + 2 * MID, *s_s3 = s_par + 3 * MID, *s_b3 = s_s3 + COUT;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::OFF_BAR);
  uint64_t *bar_in = bars, *bar_w1 = bars + 1, *bar_w3 = bars + 3, *bar_infree = bars + 5, *bar_w1free = bars + 6,
           *bar_w3free = bars + 8;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int my_tiles = (a.total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const int n_total = my_tiles * NC;

  if (tid == 0) {
    if (ptx::smem_u32(smem) & 1023u) { printf("es3: mbconv_tc_s2 dynamic smem base not 1024-byte aligned\n"); __trap(); }
    ptx::prefetch_tmap(&tm_in); ptx::prefetch_tmap(&tm_w1); ptx::prefetch_tmap(&tm_w3);
    ptx::mbar_init(bar_in, 1);
    ptx::mbar_init(bar_w1, 1); ptx::mbar_init(bar_w1 + 1, 1);
    ptx::mbar_init(bar_w3, 1); ptx::mbar_init(bar_w3 + 1, 1);
    ptx::mbar_init(bar_infree, 8);
    ptx::mbar_init(bar_w1free, 8); ptx::mbar_init(bar_w1free + 1, 8);
    ptx::mbar_init(bar_w3free, 8); ptx::mbar_init(bar_w3free + 1, 8);
    ptx::fence_mbar_init();
  }
  for (int i = tid; i < MID; i += S2_THREADS) { s_s1[i] = a.s1[i]; s_b1[i] = a.b1[i]; s_b2[i] = a.b2[i]; }
  for (int i = tid; i < COUT; i += S2_THREADS) { s_s3[i] = a.s3[i]; s_b3[i] = a.b3[i]; }
  for (int i = tid; i < 9 * MID; i += S2_THREADS) {      // bf16 depthwise weights, [chunk][tap][32]
    const int c = i % S2_MC, tap = (i / S2_MC) % 9, ch = i / (S2_MC * 9);
    const_cast<bf16*>(s_wdw)[i] = __float2bfloat16(a.wdw[tap * MID + ch * S2_MC + c]);
  }
  __syncthreads();
  const int tiles_per_img = a.tiles_x * a.tiles_y;
  constexpr uint32_t W1_BYTES = S2_MC * 128, W3_BYTES = L::W3_STAGE;

  if (warp >= 8) {
    // ------------------------------------------------------------------------------------ control: TMA (warp 8 lane 0)
    ptx::setmaxnreg_dec<S2Regs<MINB>::TMA>();
    if (warp == 8 && lane == 0 && my_tiles > 0) {
      auto load_in = [&](int t) {
        const int bb = t / tiles_per_img, r = t % tiles_per_img;
        ptx::mbar_arrive_expect_tx(bar_in, S2_PIN * 128);
        ptx::tma_load_4d(&tm_in, bar_in, s_in, 0, 2 * (r % a.tiles_x) * S2_TW - 1, 2 * (r / a.tiles_x) * S2_TH - 1, bb);
      };
      auto load_w1 = [&](int g) {
        const int s = g & 1;
        ptx::mbar_arrive_expect_tx(bar_w1 + s, W1_BYTES);
        ptx::tma_load_2d(&tm_w1, bar_w1 + s, s_w1 + s * W1_BYTES, 0, (g % NC) * S2_MC);
      };
      auto load_w3 = [&](int g) {
        const int s = (WSTAGES == 2) ? (g & 1) : 0;
        ptx::mbar_arrive_expect_tx(bar_w3 + s, W3_BYTES);
        ptx::tma_load_2d(&tm_w3, bar_w3 + s, s_w3 + s * W3_BYTES, (g % NC) * S2_MC, 0);
      };
      load_in((int)blockIdx.x);
      load_w1(0); load_w3(0); load_w1(1);
      if (WSTAGES == 2) load_w3(1);
      // each stage is refilled as soon as the compute warps report the MMA that read it retired
#pragma unroll 1
      for (int g = 0; g < n_total; ++g) {
        const int it = g / NC, c = g % NC;
        if (g + 2 < n_total) { ptx::mbar_wait(bar_w1free + (g & 1), (uint32_t)((g >> 1) & 1)); load_w1(g + 2); }
        if (c == NC - 1 && it + 1 < my_tiles) {
          ptx::mbar_wait(bar_infree, (uint32_t)(it & 1));
          load_in((int)blockIdx.x + (it + 1) * (int)gridDim.x);
        }
        if (g + WSTAGES < n_total) {
          const int ws = (WSTAGES == 2) ? (g & 1) : 0;
          ptx::mbar_wait(bar_w3free + ws, (uint32_t)(WSTAGES == 2 ? ((g >> 1) & 1) : (g & 1)));
          load_w3(g + WSTAGES);
        }
      }
    }
  } else {
    // ------------------------------------------------------------------------------------ compute warps 0..7 (two warpgroups)
    // expand: warpgroup 0 takes the 64-row blocks 0, 2, 4 of the 297 input pixels, warpgroup 1 blocks 1, 3;
    // project: warpgroup hsel takes output columns hsel * PN .. +PN (COUT 32: warpgroup 0 alone)
    ptx::setmaxnreg_inc<S2Regs<MINB>::MMA>();
    const int q = warp & 3, hsel = warp >> 2;
    const int g4 = lane >> 2, t4 = lane & 3;
    const int a_row = lane & 15, a_kh = lane >> 4;
    const uint32_t u_mid = ptx::smem_u32(s_mid), u_in = ptx::smem_u32(s_in), u_dw = ptx::smem_u32(s_dw);
    const uint32_t dshift = (g4 & 1) ? 16u : 0u;
    const bool dvalid = (g4 >> 1) == t4;
    constexpr int PN = COUT >= 64 ? COUT / 2 : COUT;
    const bool pact = COUT >= 64 || hsel == 0;
    const int pc0 = COUT >= 64 ? hsel * PN : 0;
    float proj[PN / 2];
    int g = 0;

#pragma unroll 1
    for (int it = 0; it < my_tiles; ++it) {
      const int t = (int)blockIdx.x + it * (int)gridDim.x;
      const int b = t / tiles_per_img, tr = t % tiles_per_img;
      const int oy0 = (tr / a.tiles_x) * S2_TH, ox0 = (tr % a.tiles_x) * S2_TW;
      const int iy0 = 2 * oy0 - 1, ix0 = 2 * ox0 - 1;
#pragma unroll 1
      for (int c = 0; c < NC; ++c, ++g) {
        const int st = g & 1, ws = (WSTAGES == 2) ? (g & 1) : 0;
        // ---- expand: D_exp[rows of my blocks][32] = s_in x W1c^T
        if (c == 0) ptx::mbar_wait(bar_in, (uint32_t)(it & 1));
        ptx::mbar_wait(bar_w1 + st, (uint32_t)((g >> 1) & 1));
        float ex[3][16];
        ptx::wg_fence();
#pragma unroll
        for (int k = 0; k < CIN / 16; ++k) {
          const uint64_t db = ptx::make_desc_sw128(ptx::smem_u32(s_w1 + st * W1_BYTES) + k * 32);
#pragma unroll
          for (int j = 0; j < 3; ++j) {
            // warpgroup 1 has two blocks; its third MMA repeats block 3 and is discarded, so no wgmma sits on a divergent path
            const int mb = (j == 2 && hsel == 1) ? 3 : 2 * j + hsel;
            ptx::wgmma_m64n32<0, 0>(ex[j], ptx::make_desc_sw128(u_in + mb * 8192 + k * 32), db, k != 0);
          }
        }
        ptx::wg_commit();
        ptx::wg_wait<0>();                                   // also retires project(g-1), still in flight unless c == 0
        ptx::wg_fence_regs<48>(&ex[0][0]);
        __syncwarp();
        if (lane == 0) {
          ptx::mbar_arrive(bar_w1free + st);
          if (c == NC - 1) ptx::mbar_arrive(bar_infree);
          if (c > 0) ptx::mbar_arrive(bar_w3free + ((WSTAGES == 2) ? (st ^ 1) : 0));
        }
        compute_bar_sync();                                // every warp is done reading s_mid for the previous chunk
        // ---- expand epilogue: BN1 + act, zero outside the image, bf16 -> s_mid (even / odd column planes)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          if (j == 2 && hsel == 1) break;
          const int mb = 2 * j + hsel;
#pragma unroll
          for (int i = 0; i < 16; i += 2) {
            const int row = mb * 64 + ptx::wg_frag_row(q, lane, i), col = ptx::wg_frag_col(lane, i);
            if (row < S2_PIN) {
              const int iy = iy0 + row / S2_IW, ix = ix0 + row % S2_IW;
              const bool in = iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;   // outside the image: the depthwise's zero padding
              const int lx = row % S2_IW;
              const float2 sc = *reinterpret_cast<const float2*>(s_s1 + c * S2_MC + col);
              const float2 bi = *reinterpret_cast<const float2*>(s_b1 + c * S2_MC + col);
              const float v0 = in ? es3_act_t<ACT>(fmaf(ex[j][i], sc.x, bi.x)) : 0.f;
              const float v1 = in ? es3_act_t<ACT>(fmaf(ex[j][i + 1], sc.y, bi.y)) : 0.f;
              *reinterpret_cast<uint32_t*>(s_mid + ((row / S2_IW) * S2_PW + ((lx & 1) ? S2_ODD + (lx >> 1) : (lx >> 1))) * S2_RS_MID +
                                           col * 2) = pack_bf16x2(v0, v1);
            }
          }
        }
        compute_bar_sync();                                // s_mid complete (and project(g-1) of both warpgroups retired)

        // ---- depthwise 3x3 stride 2 (diagonal m16n8k8 MMAs): warp -> channel group cg (16 of the 32), output row mt
        {
          const int cg = warp & 1, mt = warp >> 1;
          const bf16* wd = s_wdw + c * 9 * S2_MC + cg * 16 + g4;
          float dacc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
          // taps in pairs (0,1) (2,3) (4,5) (6,7) as m16n8k16 MMAs -- A = [tap-a fragment | tap-b fragment] along k, B = [diag(wa) ; diag(wb)]
          // -- and tap 8 as m16n8k8: 10 MMAs instead of 18 (k16 issues at the rate of k8)
          auto frag = [&](int tap, uint32_t* af) {
            const int ky = tap / 3, kx = tap - ky * 3;
            // input column 2 * a_row + kx: kx = 0 / 2 -> even slots a_row / a_row + 1, kx = 1 -> odd slot a_row
            ldsm_x4(u_mid + ((2 * mt + ky) * S2_PW + a_row + (kx == 1 ? S2_ODD : (kx >> 1))) * S2_RS_MID + (cg * 16 + a_kh * 8) * 2,
                    af[0], af[1], af[2], af[3]);
          };
          auto bfrag = [&](int tap, uint32_t& b_lo, uint32_t& b_hi) {
            const uint32_t w_lo = (uint32_t)__bfloat16_as_ushort(wd[tap * S2_MC]);
            const uint32_t w_hi = (uint32_t)__bfloat16_as_ushort(wd[tap * S2_MC + 8]);
            b_lo = dvalid ? (w_lo << dshift) : 0u;
            b_hi = dvalid ? (w_hi << dshift) : 0u;
          };
#pragma unroll
          for (int tp = 0; tp < 4; ++tp) {
            uint32_t fa[4], fb[4], la, ha, lb, hb;
            frag(2 * tp, fa); frag(2 * tp + 1, fb);
            bfrag(2 * tp, la, ha); bfrag(2 * tp + 1, lb, hb);
            const uint32_t a_lo[4] = {fa[0], fa[1], fb[0], fb[1]};
            const uint32_t a_hi[4] = {fa[2], fa[3], fb[2], fb[3]};
            mma_16816(dacc[0], a_lo, la, lb);
            mma_16816(dacc[1], a_hi, ha, hb);
          }
          {
            uint32_t fa[4], la, ha;
            frag(8, fa); bfrag(8, la, ha);
            mma_1688(dacc[0], fa[0], fa[1], la);
            mma_1688(dacc[1], fa[2], fa[3], ha);
          }
          const float* b2 = s_b2 + c * S2_MC;
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int p = mt * S2_TW + g4 + half * 8;      // output pixel = A-operand row (0..63) of the project wgmma
#pragma unroll
            for (int nt = 0; nt < 2; ++nt) {
              const int ch = cg * 16 + nt * 8 + t4 * 2;
              const float2 bb = *reinterpret_cast<const float2*>(b2 + ch);
              const float v0 = es3_act_t<ACT>(dacc[nt][half * 2 + 0] + bb.x);
              const float v1 = es3_act_t<ACT>(dacc[nt][half * 2 + 1] + bb.y);
              const int j = cg * 2 + nt;                    // 16-byte chunk 0..3 of the 128-byte row, XOR-swizzled by row % 8
              *reinterpret_cast<uint32_t*>(s_dw + p * 128 + ((j ^ (p & 7)) << 4) + t4 * 4) = pack_bf16x2(v0, v1);
            }
          }
        }
        ptx::fence_proxy_async();                           // generic-proxy writes -> visible to wgmma (async proxy)
        compute_bar_sync();                                // s_dw complete
        // ---- project: D_proj[64 px][pc0 .. +PN] += s_dw x W3c^T (K = 32 of the 64-column W3 box), accumulated in registers
        // (COUT 32: warpgroup 1 repeats warpgroup 0's MMAs and does not store them -- no wgmma on a divergent path)
        ptx::mbar_wait(bar_w3 + ws, (uint32_t)(WSTAGES == 2 ? ((g >> 1) & 1) : (g & 1)));
        ptx::wg_fence();
#pragma unroll
        for (int k = 0; k < S2_MC / 16; ++k) {
          const uint64_t da = ptx::make_desc_sw128(u_dw + k * 32);
          const uint64_t db = ptx::make_desc_sw128(ptx::smem_u32(s_w3 + ws * W3_BYTES) + pc0 * 128 + k * 32);
          if constexpr (PN == 64) ptx::wgmma_m64n64<0, 0>(proj, da, db, (c | k) != 0);
          else ptx::wgmma_m64n32<0, 0>(proj, da, db, (c | k) != 0);
        }
        ptx::wg_commit();                                  // retired by the next chunk's expand wait, or below
      }
      ptx::wg_wait<0>();                                   // the tile's last project: the final epilogue reads the accumulators
      ptx::wg_fence_regs<PN / 2>(proj);
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(bar_w3free + ((WSTAGES == 2) ? ((g - 1) & 1) : 0));

      // ---- final epilogue: BN3 -> global, from the accumulator fragments
      if (pact) {
#pragma unroll
        for (int i = 0; i < PN / 2; i += 2) {
          const int r = ptx::wg_frag_row(q, lane, i), col = pc0 + ptx::wg_frag_col(lane, i);
          const int oy = oy0 + r / S2_TW, ox = ox0 + r % S2_TW;
          if (oy < a.Ho && ox < a.Wo) {
            const long long pix = (((long long)b * a.Ho + oy) * a.Wo + ox) * COUT + col;
            *reinterpret_cast<uint32_t*>(a.y + pix) =
                pack_bf16x2(fmaf(proj[i], s_s3[col], s_b3[col]), fmaf(proj[i + 1], s_s3[col + 1], s_b3[col + 1]));
          }
        }
      }
    }
  }
}

template <int CIN, int MID, int COUT, int WSTAGES, int MINB>
static int launch_mbconv_tc_s2(const void* x, const void* w1, const void* w3, const S2Args& a, int B, cudaStream_t st) {
  using L = S2Smem<MID, COUT, WSTAGES>;
  CUtensorMap tm_in, tm_w1, tm_w3;
  {
    uint64_t dims[4] = {(uint64_t)CIN, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)B};
    uint64_t str[3] = {(uint64_t)CIN * 2, (uint64_t)a.W * CIN * 2, (uint64_t)a.H * a.W * CIN * 2};
    uint32_t box[4] = {64u, (uint32_t)S2_IW, (uint32_t)S2_IH, 1u};
    if (encode_map(&tm_in, x, 4, dims, str, box)) return 1;
  }
  {
    uint64_t dims[2] = {(uint64_t)CIN, (uint64_t)MID};
    uint64_t str[1] = {(uint64_t)CIN * 2};
    uint32_t box[2] = {64u, (uint32_t)S2_MC};
    if (encode_map(&tm_w1, w1, 2, dims, str, box)) return 1;
  }
  {
    uint64_t dims[2] = {(uint64_t)MID, (uint64_t)COUT};
    uint64_t str[1] = {(uint64_t)MID * 2};
    uint32_t box[2] = {64u, (uint32_t)COUT};
    if (encode_map(&tm_w3, w3, 2, dims, str, box)) return 1;
  }
  auto kern = mbconv_tc_s2_kernel<CIN, MID, COUT, WSTAGES, ACT_HSWISH, MINB>;
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
  const int ctas = a.total_tiles < MINB * sm_count ? a.total_tiles : MINB * sm_count;
  kern<<<ctas, S2_THREADS, L::TOTAL, st>>>(tm_in, tm_w1, tm_w3, a);
  ES3_LAUNCH_CHECK("mbconv_tc_s2_kernel");
  return 0;
}

}  // namespace es3

using namespace es3;

// Same contract as es3_mbconv_fused_bf16 for the stride-2, no-residual, hardswish blocks with (Cin, Mid, Cout) in
// {(16,64,32), (32,128,64), (64,256,128)}.  Returns -1 (no error set) for any other shape.
extern "C" int es3_mbconv_tc_s2_bf16(const void* x, void* y, const void* w1, const float* s1, const float* b1, const float* wdw,
                                     const float* b2, const void* w3, const float* s3, const float* b3, int B, int H, int W, int Cin,
                                     int Mid, int Cout, int stride, int residual, int act, void* stream) {
  const bool ok = stride == 2 && !residual && act == ACT_HSWISH &&
                  ((Cin == 16 && Mid == 64 && Cout == 32) || (Cin == 32 && Mid == 128 && Cout == 64) || (Cin == 64 && Mid == 256 && Cout == 128));
  if (!ok) return -1;
  ES3_REQUIRE(B > 0 && H > 0 && W > 0, "es3_mbconv_tc_s2_bf16: bad shape");
  ES3_REQUIRE((((uintptr_t)x | (uintptr_t)w1 | (uintptr_t)w3 | (uintptr_t)y) & 15) == 0, "es3_mbconv_tc_s2_bf16: 16-byte alignment");
  S2Args a;
  a.y = (bf16*)y; a.s1 = s1; a.b1 = b1; a.wdw = wdw; a.b2 = b2; a.s3 = s3; a.b3 = b3;
  a.H = H; a.W = W; a.Ho = (H - 1) / 2 + 1; a.Wo = (W - 1) / 2 + 1;
  a.tiles_x = ceil_div(a.Wo, S2_TW); a.tiles_y = ceil_div(a.Ho, S2_TH);
  a.total_tiles = B * a.tiles_x * a.tiles_y;
  cudaStream_t st = (cudaStream_t)stream;
  // two CTAs per SM (104 registers) where that does not spill, one (232 registers) for (64, 256, 128)
  if (Cin == 16) return launch_mbconv_tc_s2<16, 64, 32, 2, 2>(x, w1, w3, a, B, st);
  if (Cin == 32) return launch_mbconv_tc_s2<32, 128, 64, 2, 2>(x, w1, w3, a, B, st);
  return launch_mbconv_tc_s2<64, 256, 128, 1, 1>(x, w1, w3, a, B, st);
}
