// Flash attention on wgmma for the SAM3 ViT trunk (head_dim 64), windowed or global.
//   O = softmax(Q K^T / 8) V            reference: F.scaled_dot_product_attention, vitdet.py:502
//
// One CTA = one 128-row query tile of one (image, window, head):
//   warp 8 / warp 9  : K / V producers -- cp.async row gather (windows are gathered in place, no window_partition
//                      copy) into 128B-swizzled smem tiles, 2-stage ring
//   warps 0-3 / 4-7  : two consumer warpgroups, query rows 0..63 / 64..127 of the tile; per key tile
//                        S  = Q K^T          wgmma, A = Q smem, B = K smem, both K-major, 64 x BN x 64, fp32 in registers
//                        online softmax on the S fragment (row max / sum across the four threads of a quad)
//                        O += P V            wgmma, A = P from registers (bf16), B = V smem MN-major, 64 x 64 x BN
#include <cstdlib>

#include "ptx.cuh"

namespace es3 {

constexpr int FA_BM = 128, FA_D = 64, FA_STG = 2;   // KV tile rows BN is a template parameter (128 or 96)
constexpr int FA_TILE_BYTES = 128 * 128;  // 128 rows x 64 bf16
constexpr int FA_THREADS = 10 * 32;

struct FaArgs {
  const bf16* qkv;
  bf16* out;
  int H, W, C, win, nwx, nwin, L;
  float scale_log2;
};

__device__ __forceinline__ long long fa_token_row(const FaArgs& a, int b, int wi, int l) {
  if (a.win == 0) return (long long)b * a.H * a.W + l;
  const int wy = wi / a.nwx, wx = wi % a.nwx;
  const int i = l / a.win, j = l % a.win;
  return (long long)b * a.H * a.W + (long long)(wy * a.win + i) * a.W + wx * a.win + j;
}

__device__ __forceinline__ void fa_cp16(uint32_t saddr, const void* g, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(saddr), "l"(g), "r"(sz) : "memory");
}
__device__ __forceinline__ void fa_cp_wait_all() { asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory"); }

// 128-byte-swizzled placement of 16-byte chunk c of row r inside a 1024-byte-aligned tile (what TMA SWIZZLE_128B
// would write, and what the wgmma SW128 descriptors expect).
__device__ __forceinline__ uint32_t fa_sw(uint32_t tile, int r, int c) { return tile + r * 128 + ((c ^ (r & 7)) << 4); }

__device__ __forceinline__ float fa_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// BN = keys per tile: 128 in general; 96 for 24x24 windows (576 = 6 x 96: no padded columns).
template <int FA_BN>
__global__ void __launch_bounds__(FA_THREADS, 1) attn_tc_kernel(const FaArgs a) {
  extern __shared__ uint8_t fa_raw[];
  __shared__ __align__(8) uint64_t kv_full[FA_STG], kv_empty[FA_STG];

  const uint32_t smem0 = (ptx::smem_u32(fa_raw) + 1023u) & ~1023u;
  const uint32_t u_q = smem0;                          // [128 x 128 B]
  const uint32_t u_kv = smem0 + FA_TILE_BYTES;         // [stage][K | V]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int head = blockIdx.y;
  const int b = blockIdx.z / a.nwin, wi = blockIdx.z % a.nwin;
  const int q0 = blockIdx.x * FA_BM;
  const int ld = 3 * a.C;
  const bf16* qbase = a.qkv + head * FA_D;
  const bf16* kbase = qbase + a.C;
  const bf16* vbase = qbase + 2 * a.C;
  const int ntiles = (a.L + FA_BN - 1) / FA_BN;

  if (tid == 0) {
    for (int s = 0; s < FA_STG; ++s) { ptx::mbar_init(&kv_full[s], 2); ptx::mbar_init(&kv_empty[s], 8); }
    ptx::fence_mbar_init();
  }
  // Q tile, gathered by everyone
  for (int i = tid; i < FA_BM * 8; i += FA_THREADS) {
    const int c = i & 7, r = i >> 3;
    const int l = q0 + r;
    const bool ok = l < a.L;
    const long long row = ok ? fa_token_row(a, b, wi, l) : 0;
    fa_cp16(fa_sw(u_q, r, c), qbase + row * ld + c * 8, ok);
  }
  fa_cp_wait_all();
  ptx::fence_proxy_async();
  __syncthreads();

  if (warp >= 8) {
    // ------------------------------------------------------------------ K (warp 8) / V (warp 9) producers
    const bf16* base = (warp == 8) ? kbase : vbase;
    const uint32_t off = (warp == 8) ? 0 : FA_TILE_BYTES;
    int stage = 0;
    uint32_t phase = 0;
    for (int j = 0; j < ntiles; ++j) {
      ptx::mbar_wait(&kv_empty[stage], phase ^ 1);
      const uint32_t tile = u_kv + stage * 2 * FA_TILE_BYTES + off;
#pragma unroll
      for (int k = 0; k < FA_BN / 32; ++k) {
        const int r = lane + 32 * k;
        const int l = j * FA_BN + r;
        const bool ok = l < a.L;
        const bf16* src = base + (ok ? fa_token_row(a, b, wi, l) : 0) * ld;
#pragma unroll
        for (int c = 0; c < 8; ++c) fa_cp16(fa_sw(tile, r, c), src + c * 8, ok);
      }
      fa_cp_wait_all();
      ptx::fence_proxy_async();
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&kv_full[stage]);
      if (++stage == FA_STG) { stage = 0; phase ^= 1; }
    }
  } else {
    // ------------------------------------------------------------------ consumer warpgroups: query rows wg*64 .. +64
    const int wg = warp >> 2, wq = warp & 3;
    const uint32_t u_qg = u_q + wg * 8192;             // 64 rows = 8 swizzle atoms
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // rows lane/4 and lane/4 + 8 of the warp's 16
    int stage = 0;
    uint32_t phase = 0;
    for (int j = 0; j < ntiles; ++j) {
      ptx::mbar_wait(&kv_full[stage], phase);
      const uint32_t u_k = u_kv + stage * 2 * FA_TILE_BYTES, u_v = u_k + FA_TILE_BYTES;
      float sacc[FA_BN / 2];
      ptx::wg_fence();
#pragma unroll
      for (int k = 0; k < FA_D / 16; ++k) {
        const uint64_t dq = ptx::make_desc_sw128(u_qg + k * 32), dk = ptx::make_desc_sw128(u_k + k * 32);
        if constexpr (FA_BN == 128) ptx::wgmma_m64n128<0, 0>(sacc, dq, dk, k != 0);
        else ptx::wgmma_m64n96<0, 0>(sacc, dq, dk, k != 0);
      }
      ptx::wg_commit();
      ptx::wg_wait<0>();
      ptx::wg_fence_regs<FA_BN / 2>(sacc);
      const int col0 = j * FA_BN;
      if (col0 + FA_BN > a.L) {                        // partial key tile: columns past L do not exist
#pragma unroll
        for (int i = 0; i < FA_BN / 2; ++i)
          if (col0 + ptx::wg_frag_col(lane, i) >= a.L) sacc[i] = -INFINITY;
      }
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < FA_BN / 2; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], sacc[i]);
      float corr[2], m_new[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
        m_new[h] = fmaxf(m_run[h], mx[h] * a.scale_log2);
        corr[h] = fa_exp2(m_run[h] - m_new[h]);
        m_run[h] = m_new[h];
      }
      float rs[2] = {0.f, 0.f};
      uint32_t pk[FA_BN / 4];
#pragma unroll
      for (int i = 0; i < FA_BN / 2; i += 2) {
        const int h = (i >> 1) & 1;
        const float p0 = fa_exp2(fmaf(sacc[i], a.scale_log2, -m_new[h]));       // exp2(-inf) = 0 for the masked columns
        const float p1 = fa_exp2(fmaf(sacc[i + 1], a.scale_log2, -m_new[h]));
        rs[h] += p0 + p1;
        pk[i >> 1] = pack_bf16x2(p0, p1);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) l_run[h] = l_run[h] * corr[h] + rs[h];      // per-thread partial sums, quad-reduced at the end
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] *= corr[(i >> 1) & 1];
      // P as the A operand: key columns 16 kk .. +16 are the accumulator's n8 blocks 2 kk and 2 kk + 1
      ptx::wg_fence();
#pragma unroll
      for (int kk = 0; kk < FA_BN / 16; ++kk) {
        const uint32_t af[4] = {pk[4 * kk], pk[4 * kk + 1], pk[4 * kk + 2], pk[4 * kk + 3]};
        ptx::wgmma_m64n64_rs<1>(o, af, ptx::make_desc_sw128(u_v + kk * 2048));   // 16 key rows = 2 atoms of 1024 B
      }
      ptx::wg_commit();
      ptx::wg_wait<0>();
      ptx::wg_fence_regs<32>(o);
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&kv_empty[stage]);   // K_j / V_j no longer needed
      if (++stage == FA_STG) { stage = 0; phase ^= 1; }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
      l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int l = q0 + wg * 64 + ptx::wg_frag_row(wq, lane, 2 * h);
      if (l < a.L) {
        const float inv = 1.f / l_run[h];
        bf16* op = a.out + fa_token_row(a, b, wi, l) * a.C + head * FA_D;
#pragma unroll
        for (int i = 2 * h; i < 32; i += 4)
          *reinterpret_cast<uint32_t*>(op + ptx::wg_frag_col(lane, i)) = pack_bf16x2(o[i] * inv, o[i + 1] * inv);
      }
    }
  }
}

}  // namespace es3

using namespace es3;

// wgmma flash attention; same contract as es3_attention_bf16 (which dispatches here for L >= 128).
extern "C" int es3_attention_tc_bf16(const void* qkv, void* out, int B, int H, int W, int C, int num_heads, int win,
                                     float scale, void* stream) {
  ES3_REQUIRE(B > 0 && H > 0 && W > 0 && win >= 0, "es3_attention_tc_bf16: bad shape B=%d H=%d W=%d win=%d", B, H, W, win);
  ES3_REQUIRE(C == num_heads * FA_D, "es3_attention_tc_bf16: head_dim must be 64 (C=%d heads=%d)", C, num_heads);
  // cp.async moves 16-byte chunks of qkv; the output is stored as bf16 pairs
  ES3_REQUIRE(((uintptr_t)qkv & 15) == 0 && ((uintptr_t)out & 3) == 0,
              "es3_attention_tc_bf16: qkv must be 16-byte and out 4-byte aligned");
  ES3_REQUIRE(win == 0 || (H % win == 0 && W % win == 0), "es3_attention_tc_bf16: H,W must be multiples of the window");
  FaArgs a;
  a.qkv = (const bf16*)qkv; a.out = (bf16*)out; a.H = H; a.W = W; a.C = C; a.win = win;
  a.nwx = win ? W / win : 1;
  a.nwin = win ? (H / win) * (W / win) : 1;
  a.L = win ? win * win : H * W;
  a.scale_log2 = scale * 1.4426950408889634f;
  const int smem = 1024 + FA_TILE_BYTES + FA_STG * 2 * FA_TILE_BYTES;
  static bool configured = false;
  if (!configured) {
    ES3_CHECK_CUDA(cudaFuncSetAttribute(attn_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    ES3_CHECK_CUDA(cudaFuncSetAttribute(attn_tc_kernel<96>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid(ceil_div(a.L, FA_BM), num_heads, B * a.nwin);
  // 24x24 windows (L = 576 = 6 x 96) and other multiples of 96 that are not multiples of 128: 96-key tiles, no padding
  const bool bn96 = a.L % 96 == 0 && a.L % 128 != 0;
  if (bn96) attn_tc_kernel<96><<<grid, FA_THREADS, smem, st>>>(a);
  else attn_tc_kernel<128><<<grid, FA_THREADS, smem, st>>>(a);
  ES3_LAUNCH_CHECK("attn_tc_kernel");
  return 0;
}
