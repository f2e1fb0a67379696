// Fused MBConv on wgmma (stride 1, residual): y = x + BN3(pw2(act(BN2(dw3x3(act(BN1(pw1(x)))))))) with the 4x-expanded
// tensor kept on the SM (reference efficientvit/nn/ops.py:315-367 MBConv inside ResidualBlock :740-770).
//
// Why a second fused kernel: in mbconv_fused.cu all three contractions run on mma.sync, with every phase separated by
// __syncthreads.  Here the two pointwise GEMMs are warpgroup MMAs (wgmma) from TMA-staged, 128B-swizzled operands:
//
//   TMA (4-D map, halo + zero fill)  ->  s_in  [10x18 px][64 ch]  128B-swizzled K-major A operand
//   per 64-channel chunk of the expanded tensor:
//     expand   D_exp[192 x 64] = s_in (three 64-row blocks) x W1c^T             wgmma, SS, fp32 in registers
//     epilogue BN1 + act (+ zero outside the image = the depthwise's padding) -> bf16 s_mid (pixel-major)
//     dw3x3    9 diagonal-B mma.sync per (16 px, 16 ch) from s_mid -> +bias, act -> bf16 s_dw, written in the
//              128B-swizzled K-major layout a wgmma A operand needs (fence.proxy.async before handing it over)
//     project  D_proj[128 x COUT] += s_dw x W3c^T                                  wgmma, SS, accumulating over chunks in registers
//   final     D_proj fragments -> BN3 + residual (x re-read from global / L2) -> global
//
// Warps 0-7 (two warpgroups) issue the MMAs and do the elementwise / depthwise work, warp 8 lane 0 of the third warpgroup issues
// TMA (that warpgroup hands its registers to the other two); chunk weights sit in a 2-stage ring refilled as soon as the MMA that
// read a stage retires, so the weight loads overlap the depthwise.  A chunk's project wgmma is retired only by the next chunk's
// expand wait, so it runs on the tensor cores while the warps wait for the next weights and issue the next expand.
// CTAs are persistent: parameters and barriers are set up once, the weight ring runs across tiles and the next tile's input
// TMA is issued as soon as the current tile's last expand retires.
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
// m16n8k8: a diagonal 8x8 B has no structural zeros to multiply (the k16 form wasted half of every MMA)
__device__ __forceinline__ void mma_1688(float* d, uint32_t a0, uint32_t a1, uint32_t b0) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(b0));
}
__device__ __forceinline__ void compute_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
}  // namespace

constexpr int MT_TH = 8, MT_TW = 16;                    // output tile
constexpr int MT_HH = MT_TH + 2, MT_HW = MT_TW + 2;      // haloed input tile: 10 x 18
constexpr int MT_PIN = MT_HH * MT_HW;                    // 180 pixels
constexpr int MT_MC = 64;                                // expanded-channel chunk
constexpr int MT_RS_MID = MT_MC * 2 + 16;                // s_mid row stride (bytes)
constexpr int MT_THREADS = 384;                          // two compute warpgroups + one TMA warpgroup

template <int MID, int COUT>
struct MTSmem {
  static constexpr int IN = 3 * 64 * 128;   // the three 64-row expand blocks (rows 180..191 are padding, never written by TMA)
  static constexpr int W1 = 2 * MT_MC * 128;
  static constexpr int W3 = 2 * COUT * 128;
  static constexpr int DW = 128 * 128;
  static constexpr int MIDB = MT_PIN * MT_RS_MID;
  static constexpr int OFF_W1 = IN, OFF_W3 = OFF_W1 + W1, OFF_DW = OFF_W3 + W3, OFF_MID = OFF_DW + DW;
  static constexpr int OFF_WDW = OFF_MID + (MIDB + 15) / 16 * 16;   // bf16 [MID/64][9][64]
  static constexpr int OFF_PAR = OFF_WDW + 9 * MID * 2;              // fp32 s1[MID] b1[MID] b2[MID] s3[COUT] b3[COUT]
  static constexpr int OFF_BAR = OFF_PAR + (3 * MID + 2 * COUT) * 4;
  static constexpr int TOTAL = OFF_BAR + 128;   // 9 mbarriers
  static_assert(IN >= MT_PIN * 128 && 2 * (TOTAL + 1024) <= 233472, "input tile / two CTAs per SM");
};

struct MTArgs {
  const bf16* x;       // [B,H,W,CIN] (the TMA map reads it; the final epilogue re-reads the residual)
  bf16* y;             // [B,H,W,COUT]
  const float* s1;     // [MID]
  const float* b1;
  const float* wdw;    // [9][MID] fp32 (BN2 scale folded)
  const float* b2;     // [MID]
  const float* s3;     // [COUT]
  const float* b3;
  int H, W, tiles_x, tiles_y, total_tiles;
};

// MINB CTAs per SM.  The TMA warpgroup gives its registers to the two compute warpgroups (setmaxnreg): 40 / 232 at one CTA per
// SM, 24 / 104 at two, against a uniform 168 / 80.
template <int MINB>
struct MTRegs {
  static constexpr int TMA = MINB == 1 ? 40 : 24, MMA = MINB == 1 ? 232 : 104;
};

template <int CIN, int MID, int COUT, int ACT, int MINB>
__global__ void __launch_bounds__(MT_THREADS, MINB)
mbconv_tc_kernel(const __grid_constant__ CUtensorMap tm_in, const __grid_constant__ CUtensorMap tm_w1,
                 const __grid_constant__ CUtensorMap tm_w3, const MTArgs a) {
  using L = MTSmem<MID, COUT>;
  constexpr int NC = MID / MT_MC;
  static_assert(CIN == COUT && CIN % 16 == 0 && CIN <= 64 && MID % 64 == 0 && NC >= 2 && (COUT == 32 || COUT == 64), "shape");
  // (no integer round trip on the pointer: the compiler must keep seeing shared-space addresses, or every access below
  //  turns into a generic LD/ST -- the first version of this kernel spent its time in long-scoreboard stalls on those)
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
  // persistent: this CTA owns tiles blockIdx.x, blockIdx.x + gridDim.x, ... of the B * tiles_y * tiles_x tiles
  const int my_tiles = (a.total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const int n_total = my_tiles * NC;                      // chunks this CTA will run (the weight ring spans tiles)

  if (tid == 0) {
    if (ptx::smem_u32(smem) & 1023u) { printf("es3: mbconv_tc dynamic smem base not 1024-byte aligned\n"); __trap(); }
    ptx::prefetch_tmap(&tm_in); ptx::prefetch_tmap(&tm_w1); ptx::prefetch_tmap(&tm_w3);
    ptx::mbar_init(bar_in, 1);
    ptx::mbar_init(bar_w1, 1); ptx::mbar_init(bar_w1 + 1, 1);
    ptx::mbar_init(bar_w3, 1); ptx::mbar_init(bar_w3 + 1, 1);
    ptx::mbar_init(bar_infree, 8);
    ptx::mbar_init(bar_w1free, 8); ptx::mbar_init(bar_w1free + 1, 8);
    ptx::mbar_init(bar_w3free, 8); ptx::mbar_init(bar_w3free + 1, 8);
    ptx::fence_mbar_init();
  }
  // per-channel parameters and the depthwise weights (bf16, [chunk][tap][64]) -- once per CTA
  for (int i = tid; i < MID; i += MT_THREADS) { s_s1[i] = a.s1[i]; s_b1[i] = a.b1[i]; s_b2[i] = a.b2[i]; }
  for (int i = tid; i < COUT; i += MT_THREADS) { s_s3[i] = a.s3[i]; s_b3[i] = a.b3[i]; }
  for (int i = tid; i < 9 * MID; i += MT_THREADS) {
    const int c = i % 64, tap = (i / 64) % 9, ch = i / (64 * 9);
    const_cast<bf16*>(s_wdw)[i] = __float2bfloat16(a.wdw[tap * MID + ch * 64 + c]);
  }
  __syncthreads();
  const int tiles_per_img = a.tiles_x * a.tiles_y;

  if (warp >= 8) {
    // ------------------------------------------------------------------------------------ control: TMA (warp 8 lane 0)
    ptx::setmaxnreg_dec<MTRegs<MINB>::TMA>();
    if (warp == 8 && lane == 0 && my_tiles > 0) {
      constexpr uint32_t W1_BYTES = MT_MC * 128, W3_BYTES = COUT * 128;
      auto load_in = [&](int t) {
        const int bb = t / tiles_per_img, r = t % tiles_per_img;
        ptx::mbar_arrive_expect_tx(bar_in, MT_PIN * 128);
        ptx::tma_load_4d(&tm_in, bar_in, s_in, 0, (r % a.tiles_x) * MT_TW - 1, (r / a.tiles_x) * MT_TH - 1, bb);
      };
      auto load_w1 = [&](int gc) {
        const int s = gc & 1;
        ptx::mbar_arrive_expect_tx(bar_w1 + s, W1_BYTES);
        ptx::tma_load_2d(&tm_w1, bar_w1 + s, s_w1 + s * W1_BYTES, 0, (gc % NC) * MT_MC);
      };
      auto load_w3 = [&](int gc) {
        const int s = gc & 1;
        ptx::mbar_arrive_expect_tx(bar_w3 + s, W3_BYTES);
        ptx::tma_load_2d(&tm_w3, bar_w3 + s, s_w3 + s * W3_BYTES, (gc % NC) * MT_MC, 0);
      };
      load_in((int)blockIdx.x);
      load_w1(0); load_w3(0); load_w1(1); load_w3(1);
      // each stage is refilled as soon as the compute warps report the MMA that read it retired; the next tile's input as soon
      // as the tile's last expand retired (the residual is re-read from global, not from s_in)
#pragma unroll 1
      for (int g = 0; g < n_total; ++g) {
        const int it = g / NC, c = g % NC, st = g & 1;
        const uint32_t par = (uint32_t)((g >> 1) & 1);
        if (g + 2 < n_total) { ptx::mbar_wait(bar_w1free + st, par); load_w1(g + 2); }
        if (c == NC - 1 && it + 1 < my_tiles) {
          ptx::mbar_wait(bar_infree, (uint32_t)(it & 1));
          load_in((int)blockIdx.x + (it + 1) * (int)gridDim.x);
        }
        if (g + 2 < n_total) { ptx::mbar_wait(bar_w3free + st, par); load_w3(g + 2); }
      }
    }
  } else {
    // ------------------------------------------------------------------------------------ compute warps 0..7 (two warpgroups)
    // warpgroup hsel: expand columns hsel*32 .. +32 of the chunk; project columns hsel*32 .. (COUT 64) or rows hsel*64 .. (COUT 32)
    ptx::setmaxnreg_inc<MTRegs<MINB>::MMA>();
    const int q = warp & 3, hsel = warp >> 2;            // warp inside the warpgroup; warpgroup = column half / m-tile parity (dw)
    const int g = lane >> 2, t4 = lane & 3;
    const int a_row = lane & 15, a_kh = lane >> 4;
    const uint32_t u_mid = ptx::smem_u32(s_mid), u_in = ptx::smem_u32(s_in), u_dw = ptx::smem_u32(s_dw);
    const uint32_t dshift = (g & 1) ? 16u : 0u;
    const bool dvalid = (g >> 1) == t4;
    constexpr uint32_t W1_BYTES = MT_MC * 128, W3_BYTES = COUT * 128;
    constexpr int PRB = COUT == 64 ? 2 : 1;               // 64-row blocks of the project accumulator this warpgroup holds
    const int prb0 = COUT == 64 ? 0 : hsel, pcol0 = COUT == 64 ? hsel * 32 : 0;
    float proj[PRB][16];
    int gc = 0;

#pragma unroll 1
    for (int it = 0; it < my_tiles; ++it) {
      const int t = (int)blockIdx.x + it * (int)gridDim.x;
      const int b = t / tiles_per_img, tr = t % tiles_per_img;
      const int oy0 = (tr / a.tiles_x) * MT_TH, ox0 = (tr % a.tiles_x) * MT_TW;
      const int iy0 = oy0 - 1, ix0 = ox0 - 1;
#pragma unroll 1
      for (int c = 0; c < NC; ++c, ++gc) {
        const int st = gc & 1;
        // ---- expand: D_exp[192 x 32] = s_in (three 64-row blocks; rows >= 180 are padding) x W1c[hsel*32 .. +32]^T
        if (c == 0) ptx::mbar_wait(bar_in, (uint32_t)(it & 1));
        ptx::mbar_wait(bar_w1 + st, (uint32_t)((gc >> 1) & 1));
        float ex[3][16];
        ptx::wg_fence();
#pragma unroll
        for (int k = 0; k < CIN / 16; ++k) {
          const uint64_t db = ptx::make_desc_sw128(ptx::smem_u32(s_w1 + st * W1_BYTES) + hsel * 4096 + k * 32);
#pragma unroll
          for (int mb = 0; mb < 3; ++mb) ptx::wgmma_m64n32<0, 0>(ex[mb], ptx::make_desc_sw128(u_in + mb * 8192 + k * 32), db, k != 0);
        }
        ptx::wg_commit();
        ptx::wg_wait<0>();                                 // also retires project(gc-1), still in flight unless c == 0
        ptx::wg_fence_regs<48>(&ex[0][0]);
        __syncwarp();
        if (lane == 0) {
          ptx::mbar_arrive(bar_w1free + st);
          if (c == NC - 1) ptx::mbar_arrive(bar_infree);
          if (c > 0) ptx::mbar_arrive(bar_w3free + (st ^ 1));
        }
        compute_bar_sync();                              // every warp is done reading s_mid for the previous chunk
        // ---- expand epilogue: BN1 + act, zero outside the image, bf16 -> s_mid[row][hsel*32 .. +32)
#pragma unroll
        for (int mb = 0; mb < 3; ++mb)
#pragma unroll
          for (int i = 0; i < 16; i += 2) {
            const int row = mb * 64 + ptx::wg_frag_row(q, lane, i), col = hsel * 32 + ptx::wg_frag_col(lane, i);
            if (row < MT_PIN) {
              const int iy = iy0 + row / MT_HW, ix = ix0 + row % MT_HW;
              const bool in = iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;   // outside the image: the depthwise's zero padding
              const float2 sc = *reinterpret_cast<const float2*>(s_s1 + c * MT_MC + col);
              const float2 bi = *reinterpret_cast<const float2*>(s_b1 + c * MT_MC + col);
              const float v0 = in ? es3_act_t<ACT>(fmaf(ex[mb][i], sc.x, bi.x)) : 0.f;
              const float v1 = in ? es3_act_t<ACT>(fmaf(ex[mb][i + 1], sc.y, bi.y)) : 0.f;
              *reinterpret_cast<uint32_t*>(s_mid + row * MT_RS_MID + col * 2) = pack_bf16x2(v0, v1);
            }
          }
        compute_bar_sync();                              // s_mid complete (and project(gc-1) of both warpgroups retired)

        // ---- depthwise 3x3 on tensor cores (diagonal-B MMAs): warp -> channel group cg (16 ch), output rows hsel*4 .. hsel*4+3.
        // Four CONSECUTIVE output rows share their input rows: per kx the warp loads the 6 input-row fragments once and feeds
        // them to the 3 ky taps of each output row -- 18 ldmatrix.x4 per chunk instead of 36 (the kernel's busiest unit is the
        // shared-memory pipe; ldmatrix was 2/3 of its loads).
        {
          const int cg = q;
          const bf16* wd = s_wdw + c * 9 * 64 + cg * 16 + g;
          float dacc[4][2][4];
#pragma unroll
          for (int m = 0; m < 4; ++m)
#pragma unroll
            for (int i = 0; i < 2; ++i) { dacc[m][i][0] = dacc[m][i][1] = dacc[m][i][2] = dacc[m][i][3] = 0.f; }
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) {
            uint32_t af[6][4];
#pragma unroll
            for (int r = 0; r < 6; ++r)
              ldsm_x4(u_mid + ((hsel * 4 + r) * MT_HW + a_row + kx) * MT_RS_MID + (cg * 16 + a_kh * 8) * 2, af[r][0], af[r][1], af[r][2], af[r][3]);
            // two taps per MMA: m16n8k16 issues at the rate of m16n8k8, so the taps (0, kx) and
            // (1, kx) share one instruction -- A = [tap-0 fragment | tap-1 fragment] along k, B = [diag(w0) ; diag(w1)] -- and (2, kx)
            // stays a k8 MMA: 12 MMAs per 16 pixels x 16 channels instead of 18
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
              mma_16816(dacc[m][0], a_lo, b_lo[0], b_lo[1]);                   // channels cg*16 + 0..7, taps ky = 0, 1
              mma_16816(dacc[m][1], a_hi, b_hi[0], b_hi[1]);                   // channels cg*16 + 8..15
              mma_1688(dacc[m][0], af[m + 2][0], af[m + 2][1], b_lo[2]);       // tap ky = 2
              mma_1688(dacc[m][1], af[m + 2][2], af[m + 2][3], b_hi[2]);
            }
          }
          const float* b2 = s_b2 + c * MT_MC;
#pragma unroll
          for (int m = 0; m < 4; ++m) {
            const int mt = hsel * 4 + m;
#pragma unroll
            for (int half = 0; half < 2; ++half) {
              const int p = mt * MT_TW + g + half * 8;     // output pixel = A-operand row of the project wgmma
#pragma unroll
              for (int nt = 0; nt < 2; ++nt) {
                const int ch = cg * 16 + nt * 8 + t4 * 2;
                const float2 bb = *reinterpret_cast<const float2*>(b2 + ch);
                const float v0 = es3_act_t<ACT>(dacc[m][nt][half * 2 + 0] + bb.x);
                const float v1 = es3_act_t<ACT>(dacc[m][nt][half * 2 + 1] + bb.y);
                const int j = cg * 2 + nt;                  // 16-byte chunk inside the 128-byte row; XOR-swizzled by row % 8
                *reinterpret_cast<uint32_t*>(s_dw + p * 128 + ((j ^ (p & 7)) << 4) + t4 * 4) = pack_bf16x2(v0, v1);
              }
            }
          }
        }
        ptx::fence_proxy_async();                         // generic-proxy writes -> visible to wgmma (async proxy)
        compute_bar_sync();                              // s_dw complete
        // ---- project: D_proj[rows][pcol0 .. +32] += s_dw x W3c^T, accumulated over the chunks in registers
        ptx::mbar_wait(bar_w3 + st, (uint32_t)((gc >> 1) & 1));
        ptx::wg_fence();
#pragma unroll
        for (int k = 0; k < MT_MC / 16; ++k) {
          const uint64_t db = ptx::make_desc_sw128(ptx::smem_u32(s_w3 + st * W3_BYTES) + pcol0 * 128 + k * 32);
#pragma unroll
          for (int rb = 0; rb < PRB; ++rb)
            ptx::wgmma_m64n32<0, 0>(proj[rb], ptx::make_desc_sw128(u_dw + (prb0 + rb) * 8192 + k * 32), db, (c | k) != 0);
        }
        ptx::wg_commit();                                // retired by the next chunk's expand wait, or below
      }
      ptx::wg_wait<0>();                                 // the tile's last project: the final epilogue reads the accumulators
      ptx::wg_fence_regs<PRB * 16>(&proj[0][0]);
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(bar_w3free + ((gc - 1) & 1));

      // ---- final epilogue: BN3 + residual (x re-read from global / L2) -> global, from the accumulator fragments
#pragma unroll
      for (int rb = 0; rb < PRB; ++rb)
#pragma unroll
        for (int i = 0; i < 16; i += 2) {
          const int r = (prb0 + rb) * 64 + ptx::wg_frag_row(q, lane, i), col = pcol0 + ptx::wg_frag_col(lane, i);
          const int oy = oy0 + r / MT_TW, ox = ox0 + r % MT_TW;
          if (oy < a.H && ox < a.W) {
            const long long pix = (((long long)b * a.H + oy) * a.W + ox) * COUT + col;
            const float2 xr = unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(a.x + pix)));
            const float f0 = fmaf(proj[rb][i], s_s3[col], s_b3[col]) + xr.x;
            const float f1 = fmaf(proj[rb][i + 1], s_s3[col + 1], s_b3[col + 1]) + xr.y;
            *reinterpret_cast<uint32_t*>(a.y + pix) = pack_bf16x2(f0, f1);
          }
        }
    }
  }
}

template <int CIN, int MID, int COUT, int MINB>
static int launch_mbconv_tc(const void* x, void* y, const void* w1, const void* w3, const MTArgs& a, int B, cudaStream_t st) {
  using L = MTSmem<MID, COUT>;
  CUtensorMap tm_in, tm_w1, tm_w3;
  {
    uint64_t dims[4] = {(uint64_t)CIN, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)B};
    uint64_t str[3] = {(uint64_t)CIN * 2, (uint64_t)a.W * CIN * 2, (uint64_t)a.H * a.W * CIN * 2};
    uint32_t box[4] = {64u, (uint32_t)MT_HW, (uint32_t)MT_HH, 1u};
    if (encode_map(&tm_in, x, 4, dims, str, box)) return 1;
  }
  {
    uint64_t dims[2] = {(uint64_t)CIN, (uint64_t)MID};
    uint64_t str[1] = {(uint64_t)CIN * 2};
    uint32_t box[2] = {64u, (uint32_t)MT_MC};
    if (encode_map(&tm_w1, w1, 2, dims, str, box)) return 1;
  }
  {
    uint64_t dims[2] = {(uint64_t)MID, (uint64_t)COUT};
    uint64_t str[1] = {(uint64_t)MID * 2};
    uint32_t box[2] = {(uint32_t)MT_MC, (uint32_t)COUT};
    if (encode_map(&tm_w3, w3, 2, dims, str, box)) return 1;
  }
  auto kern = mbconv_tc_kernel<CIN, MID, COUT, ACT_HSWISH, MINB>;
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
  const int ctas = a.total_tiles < MINB * sm_count ? a.total_tiles : MINB * sm_count;   // persistent
  kern<<<ctas, MT_THREADS, L::TOTAL, st>>>(tm_in, tm_w1, tm_w3, a);
  ES3_LAUNCH_CHECK("mbconv_tc_kernel");
  return 0;
}

}  // namespace es3

using namespace es3;

// Same contract as es3_mbconv_fused_bf16 for the stride-1 residual blocks (Cin == Cout in {32, 64}, Mid = 4 Cin, hardswish).
// Returns -1 (no error set) for any other shape.
extern "C" int es3_mbconv_tc_bf16(const void* x, void* y, const void* w1, const float* s1, const float* b1, const float* wdw,
                                  const float* b2, const void* w3, const float* s3, const float* b3, int B, int H, int W, int Cin,
                                  int Mid, int Cout, int stride, int residual, int act, void* stream) {
  if (!(stride == 1 && residual && act == ACT_HSWISH && Cin == Cout && Mid == 4 * Cin && (Cin == 32 || Cin == 64))) return -1;
  ES3_REQUIRE(B > 0 && H > 0 && W > 0, "es3_mbconv_tc_bf16: bad shape");
  ES3_REQUIRE((((uintptr_t)x | (uintptr_t)w1 | (uintptr_t)w3 | (uintptr_t)y) & 15) == 0, "es3_mbconv_tc_bf16: 16-byte alignment");
  MTArgs a;
  a.x = (const bf16*)x; a.y = (bf16*)y; a.s1 = s1; a.b1 = b1; a.wdw = wdw; a.b2 = b2; a.s3 = s3; a.b3 = b3;
  a.H = H; a.W = W; a.tiles_x = ceil_div(W, MT_TW); a.tiles_y = ceil_div(H, MT_TH);
  a.total_tiles = B * a.tiles_x * a.tiles_y;
  cudaStream_t st = (cudaStream_t)stream;
  // (32, 128, 32) fits 104 registers and runs faster with a second CTA per SM to overlap its phases; (64, 256, 64) needs more
  // than 104 (it spills and ptxas serialises its wgmma) and runs at one CTA per SM
  if (Cin == 32) return launch_mbconv_tc<32, 128, 32, 2>(x, y, w1, w3, a, B, st);
  return launch_mbconv_tc<64, 256, 64, 1>(x, y, w1, w3, a, B, st);
}
