// Weight gradient of the pointwise (1x1) convolutions on wgmma:  dW[n][k] += sum_m dz[m][n] * x[m][k]
// (autograd of nn.Conv2d(k=1) / nn.Linear inside the student's training step, stage1/train_image_encoder_stage1.py:199-227).
//
// It is a dense contraction over the PIXEL index m (33 K .. 8 M rows) with small outputs (N, K <= 1024): a split-K GEMM whose two
// operands both have the contraction index as their slow dimension.  The round-1 kernel (es3_wgrad_pw, mma.sync + ldmatrix.trans)
// stays the route for shapes this kernel does not take.  Here:
//
//   TMA    box {64 channels, 64 pixels} of dz and of x  ->  128B-swizzled tiles [64 px][128 B]: exactly the MN-major ("transposed")
//          shared-memory operand layout of a wgmma -- no transpose pass, no ldmatrix
//   wgmma  D[128 (n) x KT (k)] += A^T B with both operands MN-major (transpose immediates 1, 1), K = 16 pixels per
//          instruction, one 64 x 64 block per instruction, accumulating over this CTA's pixel range in registers (KT <= 128)
//   split  grid = (n-tiles x k-tiles, nsplit): each CTA owns one output tile and one contiguous pixel range; partial tiles go to a
//          workspace and a second kernel adds them into dW in a fixed order (deterministic: no atomics)
//
// Warp roles: warps 0-3 = MMA warpgroup, which also stores its partial tile from the fragments; warp 4 = TMA producer.
// Channel counts below a 64-wide tile read zeros (TMA out-of-bounds fill) or neighbouring columns of a strided view; rows / columns
// past N / K are never stored.  Shapes with N % 64 != 0 or K % 64 != 0 stay on es3_wgrad_pw (the entry point returns -1).
#include <cuda.h>

#include "ptx.cuh"

namespace es3 {

constexpr int WG_PX = 64;                 // pixels per stage (4 wgmma k-steps)
constexpr int WG_TILE = WG_PX * 128;      // one [64 px][64 ch] tile: 8 KB
constexpr int WG_STAGES = 4;
constexpr int WG_THREADS = 160;

template <int KT>
struct WGSmem {
  static constexpr int A_BYTES = 2 * WG_TILE;               // 128 dz channels
  static constexpr int B_BYTES = (KT / 64) * WG_TILE;       // KT x channels
  static constexpr int STAGE = A_BYTES + B_BYTES;
  static constexpr int TOTAL = WG_STAGES * STAGE;
};

struct WGArgs {
  long long M;
  int N, K, tiles_k, nsplit;
  long long px_per_split;     // multiple of WG_PX
  float* ws;                  // [nsplit][N][K]
};

template <int KT>
__global__ void __launch_bounds__(WG_THREADS, 1)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap tm_dz, const __grid_constant__ CUtensorMap tm_x, const WGArgs a) {
  static_assert(KT == 64 || KT == 128, "one warpgroup holds 128 x KT fp32 accumulators in registers");
  using L = WGSmem<KT>;
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ __align__(8) uint64_t full_bar[WG_STAGES];
  __shared__ __align__(8) uint64_t empty_bar[WG_STAGES];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = ((int)blockIdx.x / a.tiles_k) * 128, k0 = ((int)blockIdx.x % a.tiles_k) * KT;
  const int split = blockIdx.y;
  const long long px0 = (long long)split * a.px_per_split;
  long long px1 = px0 + a.px_per_split;
  if (px1 > a.M) px1 = a.M;
  const int nblk = px1 > px0 ? (int)((px1 - px0 + WG_PX - 1) / WG_PX) : 0;

  if (threadIdx.x == 0) {
    if (ptx::smem_u32(smem) & 1023u) { printf("es3: wgrad_tc dynamic smem base not 1024-byte aligned\n"); __trap(); }
    ptx::prefetch_tmap(&tm_dz); ptx::prefetch_tmap(&tm_x);
#pragma unroll
    for (int s = 0; s < WG_STAGES; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], 4); }
    ptx::fence_mbar_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int b = 0; b < nblk; ++b) {
        ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sa = smem + stage * L::STAGE;
        uint8_t* sb = sa + L::A_BYTES;
        const int px = (int)(px0 + (long long)b * WG_PX);          // M < 2^31 (checked on the host)
        ptx::mbar_arrive_expect_tx(&full_bar[stage], L::STAGE);
        ptx::tma_load_2d(&tm_dz, &full_bar[stage], sa, n0, px);
        ptx::tma_load_2d(&tm_dz, &full_bar[stage], sa + WG_TILE, n0 + 64, px);
#pragma unroll
        for (int c = 0; c < KT / 64; ++c) ptx::tma_load_2d(&tm_x, &full_bar[stage], sb + c * WG_TILE, k0 + c * 64, px);
        if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ---- MMA warpgroup: d[h][c] = rows n0 + 64 h .., columns k0 + 64 c ..
    float d[2][KT / 64][32];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int c = 0; c < KT / 64; ++c)
#pragma unroll
        for (int i = 0; i < 32; ++i) d[h][c][i] = 0.f;
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int b = 0; b < nblk; ++b) {
      ptx::mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = ptx::smem_u32(smem + stage * L::STAGE), sb = sa + L::A_BYTES;
      ptx::wg_fence();
#pragma unroll
      for (int ks = 0; ks < WG_PX / 16; ++ks)      // 16 pixels = 2 atoms of 1024 B
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int c = 0; c < KT / 64; ++c)
            ptx::wgmma_m64n64<1, 1>(d[h][c], ptx::make_desc_sw128(sa + h * WG_TILE + ks * 2048),
                                    ptx::make_desc_sw128(sb + c * WG_TILE + ks * 2048), 1u);
      ptx::wg_commit();
      ptx::wg_wait<1>();
      if (prev >= 0 && lane == 0) ptx::mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
    }
    ptx::wg_wait<0>();
    ptx::wg_fence_regs<KT>(&d[0][0][0]);
    // ---- partial tile -> workspace (a CTA with no pixels writes its zeros: the reduction reads every split)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int c = 0; c < KT / 64; ++c) {
        if (k0 + c * 64 >= a.K) continue;
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
          const int n = n0 + h * 64 + ptx::wg_frag_row(warp, lane, i), k = k0 + c * 64 + ptx::wg_frag_col(lane, i);
          if (n < a.N)
            *reinterpret_cast<float2*>(a.ws + ((long long)split * a.N + n) * a.K + k) = make_float2(d[h][c][i], d[h][c][i + 1]);
        }
      }
  }
}

// dW[n * ldn + k] += sum over the splits, in split order
__global__ void wgrad_tc_reduce_kernel(const float* __restrict__ ws, int nsplit, int N, int K, float* __restrict__ dW, long long ldn) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * K) return;
  float acc = 0.f;
  for (int s = 0; s < nsplit; ++s) acc += ws[(long long)s * N * K + i];
  const int n = (int)(i / K), k = (int)(i % K);
  dW[(long long)n * ldn + k] += acc;
}

static void wgrad_tc_plan(long long M, int N, int K, int* kt, int* tiles, int* nsplit, long long* pps) {
  *kt = K >= 128 ? 128 : 64;
  const int tn = (N + 127) / 128, tk = (K + *kt - 1) / *kt;
  *tiles = tn * tk;
  long long blocks = (M + WG_PX - 1) / WG_PX;
  static int sm_count = 0;
  if (sm_count == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
      sm_count = 132;
  }
  int ns = sm_count / *tiles;                  // one CTA per SM (128 KB of operand stages)
  if (ns < 1) ns = 1;
  if (ns > blocks) ns = (int)blocks;
  long long bps = (blocks + ns - 1) / ns;      // pixel blocks per split
  *nsplit = (int)((blocks + bps - 1) / bps);
  *pps = bps * WG_PX;
}

template <int KT>
static int launch_wgrad_tc(const CUtensorMap& tm_dz, const CUtensorMap& tm_x, const WGArgs& a, int tiles, cudaStream_t st) {
  using L = WGSmem<KT>;
  ES3_CHECK_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<KT>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
  wgrad_tc_kernel<KT><<<dim3(tiles, a.nsplit), WG_THREADS, L::TOTAL, st>>>(tm_dz, tm_x, a);
  ES3_LAUNCH_CHECK("wgrad_tc_kernel");
  return 0;
}

}  // namespace es3

using namespace es3;

extern "C" long long es3_wgrad_tc_ws_floats(long long M, int N, int K) {
  int kt, tiles, nsplit;
  long long pps;
  wgrad_tc_plan(M, N, K, &kt, &tiles, &nsplit, &pps);
  return (long long)nsplit * N * K;
}

/* dW[n * ldn + k] += sum_m dz[m * lddz + n] * x[m * ldx + k], dz / x bf16 with unit channel stride, dW fp32.
 * Returns -1 (no error set) when the shape is not on this kernel (N or K not a multiple of 64, unaligned strides): the caller then
 * uses es3_wgrad_pw.  ws: es3_wgrad_tc_ws_floats(M, N, K) floats. */
extern "C" int es3_wgrad_tc(const void* dz, long long lddz, const void* x, long long ldx, long long M, int N, int K, float* ws,
                            float* dW, long long ldn, void* stream) {
  if (N % 64 != 0 || K % 64 != 0 || N < 64 || K < 64 || lddz % 8 != 0 || ldx % 8 != 0 || M < WG_PX || M >= (1LL << 31) ||
      (((uintptr_t)dz | (uintptr_t)x) & 15) != 0)
    return -1;
  int kt, tiles, nsplit;
  long long pps;
  wgrad_tc_plan(M, N, K, &kt, &tiles, &nsplit, &pps);
  CUtensorMap tm_dz, tm_x;
  {
    uint64_t dims[2] = {(uint64_t)N, (uint64_t)M};
    uint64_t str[1] = {(uint64_t)lddz * 2};
    uint32_t box[2] = {64u, (uint32_t)WG_PX};
    if (encode_map(&tm_dz, dz, 2, dims, str, box)) return 1;
  }
  {
    uint64_t dims[2] = {(uint64_t)K, (uint64_t)M};
    uint64_t str[1] = {(uint64_t)ldx * 2};
    uint32_t box[2] = {64u, (uint32_t)WG_PX};
    if (encode_map(&tm_x, x, 2, dims, str, box)) return 1;
  }
  WGArgs a;
  a.M = M; a.N = N; a.K = K; a.tiles_k = (K + kt - 1) / kt; a.nsplit = nsplit; a.px_per_split = pps; a.ws = ws;
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (kt == 128) rc = launch_wgrad_tc<128>(tm_dz, tm_x, a, tiles, st);
  else rc = launch_wgrad_tc<64>(tm_dz, tm_x, a, tiles, st);
  if (rc) return rc;
  const long long total = (long long)N * K;
  wgrad_tc_reduce_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(ws, nsplit, N, K, dW, ldn);
  ES3_LAUNCH_CHECK("wgrad_tc_reduce_kernel");
  return 0;
}
