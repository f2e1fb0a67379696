// Block-scaled FP8 (e4m3) GEMM for sm_90a, and the quantisers that feed it: the opt-in FP8 route of the frozen SAM3 ViT teacher's
// four linear layers (qkv, proj, fc1, fc2; model/vitdet.py ViT.enable_fp8).
//
//   out[m, n] = epi( sum_kb  sA[m, kb] * sW[n / 128, kb] * sum_{k in kb} qA[m, k] * qW[n, k]  + bias[n] )
//
// qA: e4m3 [M][K] (K contiguous), sA: fp32 [M][K / 128] -- one scale per row per 128-element K block
// qW: e4m3 [N][K] (K contiguous, the nn.Linear layout), sW: fp32 [N / 128][K / 128] -- one scale per 128 x 128 block
// (quantisation rule: fp8.cuh).  A scale block is one 128-byte swizzled TMA row, so no scale ever crosses a CTA.
//
// Structure (persistent CTAs, 128 x 128 output tiles, 288 threads, one CTA per SM):
//   warpgroups 0, 1: MMA + epilogue -- warpgroup c owns rows [64 c, 64 c + 64) of the tile.  Per 128-wide K block it runs four
//                    wgmma m64n128k32 into a partial accumulator, waits for them, and adds partial * sA[row] * sW into the fp32
//                    main accumulator.  The promotion is required: the tensor core's accumulation of e4m3 products is not full
//                    fp32, and over K = 4736 its error would grow with K.  The epilogue runs from the main accumulator's registers.
//   warp 8         : TMA producer   -- cp.async.bulk.tensor into a STAGES-deep 128B-swizzled smem ring (full/empty mbarriers);
//                    it runs ahead into the next tile while the MMA warpgroups drain the epilogue of this one.
// Epilogues: bias + 2-D axial RoPE -> bf16 (qkv), bias (+ fp32 residual) -> fp32 (proj, fc2), bias + GELU(erf) -> e4m3 + per-row
// scales of the 128-column block (fc1: fc2 reads it as its A operand at one byte per element), and bias + GELU(erf) -> fp32 (the
// fc1 arithmetic before quantisation, for checking it).
#include <cstdio>
#include <cstdlib>

#include "fp8.cuh"
#include "ptx.cuh"

namespace es3 {
namespace fp8 {

constexpr int BM = 128, BN = 128, BK = 128;  // BK: 128 e4m3 = 128 B = one swizzle row = one scale block
constexpr int STAGES = 6;
constexpr int TILE_BYTES = BM * BK;          // A and B tiles are both 128 x 128 bytes
constexpr int STAGE_BYTES = 2 * TILE_BYTES;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES;   // 192 KB; the buffer is declared __align__(1024)
constexpr int MMA_WARPS = 8;
constexpr int TMA_WARP = MMA_WARPS;
constexpr int THREADS = (MMA_WARPS + 1) * 32;

enum Out { OUT_BF16 = 0, OUT_F32 = 1, OUT_E4M3 = 2 };

struct Args {
  int M, N, num_kb, tiles_n;
  const float* sA;      // [M][num_kb]
  const float* sW;      // [N / 128][num_kb]
  const float* bias;    // [N] or null
  const float* residual;  // fp32 [M][ldr] or null (OUT_F32 only)
  long long ldr;
  void* out;
  long long ldo;
  float* out_scales;    // OUT_E4M3: [M][N / 128]
  const float2* rope;   // OUT_BF16: (cos, sin) [positions][32] for columns [0, rope_cols), or null
  int rope_cols, rope_H, rope_W, rope_win;
};

template <int OUT, int ACT>
__global__ void __launch_bounds__(THREADS, 1) gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmA,
                                                              const __grid_constant__ CUtensorMap tmB, const Args args,
                                                              const int num_tiles) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ __align__(8) uint64_t full_bar[STAGES];
  __shared__ __align__(8) uint64_t empty_bar[STAGES];

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    if (ptx::smem_u32(smem) & 1023u) __trap();   // the 128B swizzle atoms need 1024-byte aligned stages
    ptx::prefetch_tmap(&tmA);
    ptx::prefetch_tmap(&tmB);
#pragma unroll
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], MMA_WARPS);   // one arrival per MMA warp
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();

  if (warp == TMA_WARP) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int n0 = (tile % args.tiles_n) * BN, m0 = (tile / args.tiles_n) * BM;
        for (int kb = 0; kb < args.num_kb; ++kb) {
          ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          ptx::mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);
          // the maps address the bytes as bf16 pairs (see es3_gemm_fp8): 128 bytes along K are 64 elements
          ptx::tma_load_2d(&tmA, &full_bar[stage], sa, kb * (BK / 2), m0);
          ptx::tma_load_2d(&tmB, &full_bar[stage], sa + TILE_BYTES, kb * (BK / 2), n0);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- MMA warpgroups (+ epilogue)
  const int wg = warp >> 2, wq = warp & 3;
  const int rfrag = 16 * wq + (lane >> 2);          // fragment rows rfrag and rfrag + 8 of this warpgroup's 64-row half
  const int cfrag = 2 * (lane & 3);                 // fragment columns 8 j + cfrag, + 1
  float acc[64], part[64];
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int n0 = (tile % args.tiles_n) * BN, m0 = (tile / args.tiles_n) * BM;
    const int row0 = m0 + 64 * wg + rfrag, row1 = row0 + 8;
    const bool ok0 = row0 < args.M, ok1 = row1 < args.M;
    const float* sa0 = args.sA + (long long)(ok0 ? row0 : 0) * args.num_kb;
    const float* sa1 = args.sA + (long long)(ok1 ? row1 : 0) * args.num_kb;
    const float* sw = args.sW + (long long)(n0 / BN) * args.num_kb;
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < args.num_kb; ++kb) {
      // the scales are read before the wait, so their latency hides behind the TMA / the previous block's promotion
      const float w_s = __ldg(sw + kb);
      const float s0 = ok0 ? __ldg(sa0 + kb) * w_s : 0.f;
      const float s1 = ok1 ? __ldg(sa1 + kb) * w_s : 0.f;
      ptx::mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = ptx::smem_u32(smem + stage * STAGE_BYTES) + wg * 8192;   // 64 rows x 128 B further on
      const uint32_t sb = ptx::smem_u32(smem + stage * STAGE_BYTES + TILE_BYTES);
      ptx::wg_fence();
#pragma unroll
      for (int k = 0; k < BK / 32; ++k)
        ptx::wgmma_m64n128k32_e4m3(part, ptx::make_desc_sw128(sa + k * 32), ptx::make_desc_sw128(sb + k * 32), k != 0);
      ptx::wg_commit();
      ptx::wg_wait<0>();
      ptx::wg_fence_regs<64>(part);
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&empty_bar[stage]);
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = fmaf(part[i], (i & 2) ? s1 : s0, acc[i]);
    }

    // ---------------------------------------------------------------- epilogue, from registers
    // element i of the fragment: row rfrag + 8 ((i >> 1) & 1), column 8 (i >> 2) + cfrag + (i & 1)
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      float2 b = make_float2(0.f, 0.f);
      if (args.bias != nullptr) b = __ldg(reinterpret_cast<const float2*>(args.bias + n0 + 8 * j + cfrag));
      acc[4 * j] = es3_act_t<ACT>(acc[4 * j] + b.x);
      acc[4 * j + 1] = es3_act_t<ACT>(acc[4 * j + 1] + b.y);
      acc[4 * j + 2] = es3_act_t<ACT>(acc[4 * j + 2] + b.x);
      acc[4 * j + 3] = es3_act_t<ACT>(acc[4 * j + 3] + b.y);
    }
    if constexpr (OUT == OUT_BF16) {
      if (args.rope != nullptr && n0 < args.rope_cols) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = h ? row1 : row0;
          const int t = (int)(row % (args.rope_H * args.rope_W));
          const int y = t / args.rope_W, x = t - y * args.rope_W;
          const int pidx = args.rope_win ? (y % args.rope_win) * args.rope_win + (x % args.rope_win) : t;
          const float2* tp = args.rope + (long long)pidx * 32;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const float2 cs = __ldg(tp + (((8 * j + cfrag) & 63) >> 1));   // n0 is a multiple of 64: a head starts at column 0
            const float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
            acc[4 * j + 2 * h] = x0 * cs.x - x1 * cs.y;
            acc[4 * j + 2 * h + 1] = x0 * cs.y + x1 * cs.x;
          }
        }
      }
      bf16* out = reinterpret_cast<bf16*>(args.out);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!(h ? ok1 : ok0)) continue;
        bf16* o = out + (long long)(h ? row1 : row0) * args.ldo + n0 + cfrag;
#pragma unroll
        for (int j = 0; j < 16; ++j) *reinterpret_cast<uint32_t*>(o + 8 * j) = pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      }
    } else if constexpr (OUT == OUT_F32) {
      float* out = reinterpret_cast<float*>(args.out);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!(h ? ok1 : ok0)) continue;
        const long long row = h ? row1 : row0;
        float* o = out + row * args.ldo + n0 + cfrag;
        const float* r = args.residual != nullptr ? args.residual + row * args.ldr + n0 + cfrag : nullptr;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          float2 v = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
          if (r != nullptr) {
            const float2 rr = __ldg(reinterpret_cast<const float2*>(r + 8 * j));
            v.x += rr.x; v.y += rr.y;
          }
          *reinterpret_cast<float2*>(o + 8 * j) = v;
        }
      }
    } else {
      // a row's 128 columns of this tile are one scale block, spread over the four lanes of a quad (32 values each)
      uint8_t* out = reinterpret_cast<uint8_t*>(args.out);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float amax = 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j) amax = fmaxf(amax, fmaxf(fabsf(acc[4 * j + 2 * h]), fabsf(acc[4 * j + 2 * h + 1])));
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
        const float s = e4m3_block_scale(amax);
        if (!(h ? ok1 : ok0)) continue;
        const long long row = h ? row1 : row0;
        uint8_t* o = out + row * args.ldo + n0 + cfrag;
#pragma unroll
        for (int j = 0; j < 16; ++j)
          *reinterpret_cast<uint16_t*>(o + 8 * j) =
              (uint16_t)e4m3x2(__fdiv_rn(acc[4 * j + 2 * h], s), __fdiv_rn(acc[4 * j + 2 * h + 1], s));
        if ((lane & 3) == 0) args.out_scales[row * (args.N / BN) + n0 / BN] = s;
      }
    }
  }
}

template <int OUT, int ACT>
static int launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const Args& args, int num_tiles, cudaStream_t stream) {
  static int sm_count = 0;
  if (sm_count == 0) {
    ES3_CHECK_CUDA(cudaFuncSetAttribute(gemm_fp8_kernel<OUT, ACT>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    int dev = 0, occ = 0;
    ES3_CHECK_CUDA(cudaGetDevice(&dev));
    ES3_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gemm_fp8_kernel<OUT, ACT>, THREADS, SMEM_BYTES));
    ES3_REQUIRE(occ >= 1, "gemm_fp8_kernel: does not fit an SM (%d B of dynamic shared memory)", SMEM_BYTES);
    int n = 0;
    ES3_CHECK_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
    sm_count = n;
  }
  const dim3 grid((unsigned)(num_tiles < sm_count ? num_tiles : sm_count));
  gemm_fp8_kernel<OUT, ACT><<<grid, THREADS, SMEM_BYTES, stream>>>(tmA, tmB, args, num_tiles);
  ES3_LAUNCH_CHECK("gemm_fp8_kernel");
  return 0;
}

// ---------------------------------------------------------------------------------------------- quantisers
// bf16 [M][C] (row stride lda) -> e4m3 [M][C] + fp32 scales [M][C / 128].  One warp per (row, 128-column block), 4 values a lane.
__global__ void quantize_bf16_e4m3_kernel(const bf16* __restrict__ x, long long lda, uint8_t* __restrict__ q,
                                          float* __restrict__ scales, long long M, int nb) {
  const long long w = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= M * nb) return;
  const int lane = threadIdx.x & 31;
  const long long row = w / nb;
  const int b = (int)(w - row * nb);
  const uint2 u = __ldg(reinterpret_cast<const uint2*>(x + row * lda + b * 128) + lane);
  const float2 v0 = unpack_bf16x2(u.x), v1 = unpack_bf16x2(u.y);
  const float s = e4m3_block_scale(warp_max(abs_max4(v0.x, v0.y, v1.x, v1.y)));
  reinterpret_cast<uint32_t*>(q + row * (long long)nb * 128 + b * 128)[lane] = e4m3x4(v0.x, v0.y, v1.x, v1.y, s);
  if (lane == 0) scales[w] = s;
}

// weights [N][K] (bf16 or fp32) -> e4m3 [N][K] + fp32 scales [ceil(N / 128)][K / 128].  One CTA of 256 threads per 128 x 128
// block; rows past N take no part in the block's amax.
template <typename T>
__global__ void pack_weight_e4m3_kernel(const T* __restrict__ w, uint8_t* __restrict__ q, float* __restrict__ scales, int N, int K) {
  __shared__ float red[8];
  const int nb = blockIdx.y, kb = blockIdx.x;
  const int rows = min(128, N - nb * 128);
  auto load4 = [&](int e, float* v) {
    const long long off = (long long)(nb * 128 + e / 32) * K + kb * 128 + 4 * (e % 32);
    if constexpr (sizeof(T) == 4) {
      const float4 f = __ldg(reinterpret_cast<const float4*>(w + off));
      v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
    } else {
      const uint2 u = __ldg(reinterpret_cast<const uint2*>(w + off));
      const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y);
      v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
    }
  };
  float amax = 0.f;
  for (int e = threadIdx.x; e < rows * 32; e += blockDim.x) {
    float v[4];
    load4(e, v);
    amax = fmaxf(amax, abs_max4(v[0], v[1], v[2], v[3]));
  }
  amax = warp_max(amax);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = amax;
  __syncthreads();
  amax = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) amax = fmaxf(amax, red[i]);
  const float s = e4m3_block_scale(amax);
  for (int e = threadIdx.x; e < rows * 32; e += blockDim.x) {
    float v[4];
    load4(e, v);
    const long long off = (long long)(nb * 128 + e / 32) * K + kb * 128 + 4 * (e % 32);
    *reinterpret_cast<uint32_t*>(q + off) = e4m3x4(v[0], v[1], v[2], v[3], s);
  }
  if (threadIdx.x == 0) scales[nb * gridDim.x + kb] = s;
}

}  // namespace fp8
}  // namespace es3

using namespace es3;

// out_kind: 0 bf16, 1 fp32, 2 e4m3 (+ out_scales).  act: ACT_NONE or ACT_GELU.  Instantiated: bf16 / none (rope optional),
// fp32 / none (residual optional), e4m3 / gelu, fp32 / gelu.  N % 128 == 0, K % 128 == 0; scale tensors contiguous.
extern "C" int es3_gemm_fp8(const void* A, long long lda, const float* sA, const void* W, long long ldw, const float* sW,
                            void* out, long long ldo, int out_kind, float* out_scales, int M, int N, int K, const float* bias,
                            int act, const float* residual, long long ldr, const float* rope, int rope_cols, int rope_H,
                            int rope_W, int rope_win, void* stream) {
  using namespace fp8;
  ES3_REQUIRE(M > 0 && N > 0 && K > 0, "es3_gemm_fp8: bad shape M=%d N=%d K=%d", M, N, K);
  ES3_REQUIRE(N % BN == 0 && K % BK == 0, "es3_gemm_fp8: N=%d and K=%d must be multiples of 128", N, K);
  ES3_REQUIRE(lda >= K && ldw >= K && lda % 16 == 0 && ldw % 16 == 0, "es3_gemm_fp8: lda/ldw must be >= K and multiples of 16 bytes");
  ES3_REQUIRE(((uintptr_t)A & 15) == 0 && ((uintptr_t)W & 15) == 0 && ((uintptr_t)out & 15) == 0,
              "es3_gemm_fp8: A, W and out must be 16-byte aligned");
  ES3_REQUIRE(sA != nullptr && sW != nullptr, "es3_gemm_fp8: operand scales missing");
  ES3_REQUIRE(((uintptr_t)bias & 7) == 0, "es3_gemm_fp8: bias must be 8-byte aligned");
  ES3_REQUIRE(ldo >= N && ldo % 16 == 0, "es3_gemm_fp8: ldo=%lld must be >= N and a multiple of 16", ldo);
  ES3_REQUIRE(residual == nullptr || (out_kind == OUT_F32 && act == ACT_NONE && ldr >= N && ldr % 2 == 0 && ((uintptr_t)residual & 7) == 0),
              "es3_gemm_fp8: a residual needs an fp32 output without activation and an 8-byte aligned row stride");
  ES3_REQUIRE(rope == nullptr || (out_kind == OUT_BF16 && act == ACT_NONE && rope_cols % BN == 0 && rope_cols <= N && rope_H > 0 &&
                                  rope_W > 0 && ((uintptr_t)rope & 7) == 0),
              "es3_gemm_fp8: bad rope arguments (bf16 output, no activation, rope_cols %% 128 == 0)");
  ES3_REQUIRE(out_kind != OUT_E4M3 || out_scales != nullptr, "es3_gemm_fp8: an e4m3 output needs out_scales");
  CUtensorMap tmA, tmB;
  // e4m3 has no tensor-map data type of its own; a row of bytes is mapped as bf16 pairs (TMA moves bytes: the box of 64 x 2 B is
  // the same 128-byte swizzle row, and zero fill is zero bytes)
  {
    uint64_t dims[2] = {(uint64_t)K / 2, (uint64_t)M};
    uint64_t str[1] = {(uint64_t)lda};
    uint32_t box[2] = {BK / 2, BM};
    if (encode_map(&tmA, A, 2, dims, str, box)) return 1;
  }
  {
    uint64_t dims[2] = {(uint64_t)K / 2, (uint64_t)N};
    uint64_t str[1] = {(uint64_t)ldw};
    uint32_t box[2] = {BK / 2, BN};
    if (encode_map(&tmB, W, 2, dims, str, box)) return 1;
  }
  Args a;
  memset(&a, 0, sizeof(a));
  a.M = M; a.N = N; a.num_kb = K / BK; a.tiles_n = N / BN;
  a.sA = sA; a.sW = sW; a.bias = bias;
  a.residual = residual; a.ldr = ldr;
  a.out = out; a.ldo = ldo; a.out_scales = out_scales;
  a.rope = (const float2*)rope; a.rope_cols = rope_cols; a.rope_H = rope_H; a.rope_W = rope_W; a.rope_win = rope_win;
  const int num_tiles = ceil_div(M, BM) * a.tiles_n;
  cudaStream_t st = (cudaStream_t)stream;
  if (out_kind == OUT_BF16 && act == ACT_NONE) return launch<OUT_BF16, ACT_NONE>(tmA, tmB, a, num_tiles, st);
  if (out_kind == OUT_F32 && act == ACT_NONE) return launch<OUT_F32, ACT_NONE>(tmA, tmB, a, num_tiles, st);
  if (out_kind == OUT_F32 && act == ACT_GELU) return launch<OUT_F32, ACT_GELU>(tmA, tmB, a, num_tiles, st);
  if (out_kind == OUT_E4M3 && act == ACT_GELU) return launch<OUT_E4M3, ACT_GELU>(tmA, tmB, a, num_tiles, st);
  set_error("es3_gemm_fp8: output kind %d with activation %d is not instantiated", out_kind, act);
  return 1;
}

// bf16 [M][C] (row stride lda elements) -> e4m3 [M][C] contiguous + fp32 scales [M][C / 128]
extern "C" int es3_quantize_bf16_e4m3(const void* x, long long lda, void* q, float* scales, long long M, int C, void* stream) {
  ES3_REQUIRE(M > 0 && C > 0 && C % 128 == 0 && lda >= C && lda % 4 == 0 && ((uintptr_t)x & 7) == 0 && ((uintptr_t)q & 3) == 0,
              "es3_quantize_bf16_e4m3: need C %% 128 == 0 (C=%d), lda >= C, lda %% 4 == 0, aligned pointers", C);
  const int nb = C / 128, warps = 8;
  fp8::quantize_bf16_e4m3_kernel<<<(unsigned)ceil_div(M * nb, warps), warps * 32, 0, (cudaStream_t)stream>>>(
      (const bf16*)x, lda, (uint8_t*)q, scales, M, nb);
  ES3_LAUNCH_CHECK("quantize_bf16_e4m3_kernel");
  return 0;
}

// weights [N][K] contiguous, bf16 (w_f32 = 0) or fp32 (w_f32 = 1) -> e4m3 [N][K] + fp32 scales [ceil(N / 128)][K / 128]
extern "C" int es3_pack_weight_e4m3(const void* w, int w_f32, void* q, float* scales, int N, int K, void* stream) {
  ES3_REQUIRE(N > 0 && K > 0 && K % 128 == 0 && ((uintptr_t)w & 15) == 0 && ((uintptr_t)q & 3) == 0,
              "es3_pack_weight_e4m3: need K %% 128 == 0 (K=%d) and aligned pointers", K);
  const dim3 grid(K / 128, ceil_div(N, 128));
  if (w_f32) fp8::pack_weight_e4m3_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>((const float*)w, (uint8_t*)q, scales, N, K);
  else fp8::pack_weight_e4m3_kernel<bf16><<<grid, 256, 0, (cudaStream_t)stream>>>((const bf16*)w, (uint8_t*)q, scales, N, K);
  ES3_LAUNCH_CHECK("pack_weight_e4m3_kernel");
  return 0;
}
