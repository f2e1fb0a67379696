// Windowed / global multi-head softmax attention for the SAM3 ViT trunk (head_dim 64), flash-style:
//   O = softmax(Q K^T / sqrt(64)) V         reference: F.scaled_dot_product_attention, vitdet.py:502
// Q, K (already RoPE-rotated by the QKV GEMM epilogue) and V live interleaved in the qkv activation
// [tokens, 3*C] bf16 exactly as nn.Linear(dim, 3*dim) lays them out (vitdet.py:480-483):
//   q(head h) = cols [h*64, h*64+64), k = C + ..., v = 2C + ...
// Tokens stay in raster order [B, H, W]: window_partition / window_unpartition (vitdet.py:93-139) are
// never materialised -- a window's token l = (i, j) is the row b*H*W + (wy*win+i)*W + wx*win+j, and the
// kernel gathers 128-byte rows with cp.async.
//
// One CTA = 64 query rows of one (image, window, head); 4 warps x 16 rows.  K/V tiles of 64 rows are
// double-buffered in shared memory; S = QK^T and O += PV run on mma.sync.m16n8k16 (bf16 in, fp32
// accumulate), the online softmax lives in registers, P is re-used from the S accumulators as the A
// operand (no smem round trip).  The wgmma flash attention (attention_tc.cu) serves sequences of >= 128 tokens.
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
__device__ __forceinline__ void cpa_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cpa_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
}  // namespace

constexpr int AT_BN = 64, AT_D = 64, AT_RS = AT_D * 2 + 16;  // smem row stride (bytes)

struct AttnArgs {
  const bf16* qkv;  // [B*H*W, 3*C]
  bf16* out;        // [B*H*W, C]
  int H, W, C, win; // win == 0: global attention over H*W tokens
  int nwx, nwin, L; // windows per row, windows per image, tokens per window
  float scale_log2; // softmax scale * log2(e)
};

__device__ __forceinline__ long long token_row(const AttnArgs& a, int b, int wi, int l) {
  if (a.win == 0) return (long long)b * a.H * a.W + l;
  const int wy = wi / a.nwx, wx = wi % a.nwx;
  const int i = l / a.win, j = l % a.win;
  return (long long)b * a.H * a.W + (long long)(wy * a.win + i) * a.W + wx * a.win + j;
}

// CAUSAL: token l attends to tokens <= l only (the additive triu(-inf) mask of the text encoders, mobile_clip.py:825-831,
// text_encoder_ve.py:220-226); KV tiles wholly above the diagonal of this CTA's query rows are not loaded.
// MT = 16-row query tiles per warp.  K/V fragments loaded by ldmatrix are reused for all MT tiles: on this part
// one m16n8k16 MMA (1 tensor-pipe cycle per SM at 2048 FMA/clk) consumes a 256-byte B fragment, i.e. 2 cycles of the
// 128 B/clk shared-memory pipe -- with MT = 1 the kernel is smem-bandwidth-bound.
template <int MT, bool CAUSAL = false>
__global__ void __launch_bounds__(128) attn_fwd_kernel(const AttnArgs a) {
  constexpr int AT_BM = 64 * MT;
  extern __shared__ __align__(16) uint8_t at_smem[];
  uint8_t* s_q = at_smem;
  uint8_t (*s_k)[AT_BN * AT_RS] = reinterpret_cast<uint8_t (*)[AT_BN * AT_RS]>(at_smem + AT_BM * AT_RS);
  uint8_t (*s_v)[AT_BN * AT_RS] = reinterpret_cast<uint8_t (*)[AT_BN * AT_RS]>(at_smem + AT_BM * AT_RS + 2 * AT_BN * AT_RS);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int qt = blockIdx.x, head = blockIdx.y;
  const int b = blockIdx.z / a.nwin, wi = blockIdx.z % a.nwin;
  const int ld = 3 * a.C;
  const bf16* qbase = a.qkv + head * AT_D;
  const bf16* kbase = qbase + a.C;
  const bf16* vbase = qbase + 2 * a.C;
  const uint32_t u_q = static_cast<uint32_t>(__cvta_generic_to_shared(s_q));
  const uint32_t u_k = static_cast<uint32_t>(__cvta_generic_to_shared(&s_k[0][0]));
  const uint32_t u_v = static_cast<uint32_t>(__cvta_generic_to_shared(&s_v[0][0]));

  // ---- async loads: Q tile, then KV tile 0
  for (int i = tid; i < AT_BM * 8; i += 128) {
    const int r = i >> 3, v = i & 7;
    const int l = qt * AT_BM + r;
    const bool ok = l < a.L;
    const long long row = ok ? token_row(a, b, wi, l) : 0;
    cpa16(u_q + r * AT_RS + v * 16, qbase + row * ld + v * 8, ok);
  }
  auto load_kv = [&](int t, int buf) {
    for (int i = tid; i < AT_BN * 8; i += 128) {
      const int r = i >> 3, v = i & 7;
      const int l = t * AT_BN + r;
      const bool ok = l < a.L;
      const long long row = ok ? token_row(a, b, wi, l) : 0;
      cpa16(u_k + buf * (AT_BN * AT_RS) + r * AT_RS + v * 16, kbase + row * ld + v * 8, ok);
      cpa16(u_v + buf * (AT_BN * AT_RS) + r * AT_RS + v * 16, vbase + row * ld + v * 8, ok);
    }
  };
  load_kv(0, 0);
  cpa_commit();

  const int a_row = lane & 15, a_kh = lane >> 4;                       // A / non-trans x4 addressing
  const int b_n = (lane & 7) + ((lane >> 4) << 3), b_kh = (lane >> 3) & 1;   // B from [n][k] storage
  const int v_k = (lane & 7) + (((lane >> 3) & 1) << 3), v_n = (lane >> 4) << 3;  // B from [k][n] storage (.trans)
  const int g = lane >> 2, t4 = lane & 3;

  float o[MT][8][4];
  float m_run[MT][2], l_run[MT][2];
  uint32_t qf[MT][4][4];
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { o[mt][i][0] = o[mt][i][1] = o[mt][i][2] = o[mt][i][3] = 0.f; }
    m_run[mt][0] = m_run[mt][1] = -INFINITY;
    l_run[mt][0] = l_run[mt][1] = 0.f;
  }

  int ntiles = (a.L + AT_BN - 1) / AT_BN;
  if (CAUSAL) ntiles = min(ntiles, (qt * AT_BM + AT_BM - 1) / AT_BN + 1);
  for (int t = 0; t < ntiles; ++t) {
    const int buf = t & 1;
    if (t + 1 < ntiles) {
      load_kv(t + 1, buf ^ 1);
      cpa_commit();
      cpa_wait<1>();
    } else {
      cpa_wait<0>();
    }
    __syncthreads();
    if (t == 0) {
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
          ptx::ldsm_x4(u_q + ((warp * MT + mt) * 16 + a_row) * AT_RS + (ks * 16 + a_kh * 8) * 2, qf[mt][ks][0], qf[mt][ks][1],
                       qf[mt][ks][2], qf[mt][ks][3]);
    }
    // ---- S = Q K^T (K fragments shared by the MT query tiles)
    float s[MT][8][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int i = 0; i < 8; ++i) { s[mt][i][0] = s[mt][i][1] = s[mt][i][2] = s[mt][i][3] = 0.f; }
    const uint32_t kb = u_k + buf * (AT_BN * AT_RS);
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t b0, b1, b2, b3;
        ptx::ldsm_x4(kb + (np * 16 + b_n) * AT_RS + (ks * 16 + b_kh * 8) * 2, b0, b1, b2, b3);
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
          ptx::mma_16816(s[mt][2 * np], qf[mt][ks], b0, b1);
          ptx::mma_16816(s[mt][2 * np + 1], qf[mt][ks], b2, b3);
        }
      }
    }
    // ---- online softmax (rows g and g+8 of each 16-row tile)
    const int col0 = t * AT_BN;
    uint32_t pf[MT][4][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int col = col0 + nt * 8 + t4 * 2 + (e & 1);
          float v = s[mt][nt][e] * a.scale_log2;
          if (col >= a.L) v = -INFINITY;
          if (CAUSAL && col > qt * AT_BM + (warp * MT + mt) * 16 + g + ((e >> 1) << 3)) v = -INFINITY;
          s[mt][nt][e] = v;
          mx[e >> 1] = fmaxf(mx[e >> 1], v);
        }
      }
      float corr[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        const float m_new = fmaxf(m_run[mt][r], mx[r]);
        corr[r] = fast_exp2(m_run[mt][r] - m_new);   // first tile: exp2(-inf) = 0
        m_run[mt][r] = m_new;
        l_run[mt][r] *= corr[r];
      }
      float rs[2] = {0.f, 0.f};
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const float p0 = fast_exp2(s[mt][nt][0] - m_run[mt][0]), p1 = fast_exp2(s[mt][nt][1] - m_run[mt][0]);
        const float p2 = fast_exp2(s[mt][nt][2] - m_run[mt][1]), p3 = fast_exp2(s[mt][nt][3] - m_run[mt][1]);
        rs[0] += p0 + p1;
        rs[1] += p2 + p3;
        pf[mt][nt >> 1][(nt & 1) * 2 + 0] = pack_bf16x2(p0, p1);
        pf[mt][nt >> 1][(nt & 1) * 2 + 1] = pack_bf16x2(p2, p3);
      }
      l_run[mt][0] += rs[0];
      l_run[mt][1] += rs[1];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        o[mt][nt][0] *= corr[0]; o[mt][nt][1] *= corr[0];
        o[mt][nt][2] *= corr[1]; o[mt][nt][3] *= corr[1];
      }
    }
    // ---- O += P V (V fragments shared by the MT query tiles)
    const uint32_t vb = u_v + buf * (AT_BN * AT_RS);
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {      // 16 kv rows per step
#pragma unroll
      for (int np = 0; np < 4; ++np) {    // two 8-wide d tiles per ldmatrix
        uint32_t b0, b1, b2, b3;
        ldsm4t(vb + (ks * 16 + v_k) * AT_RS + (np * 16 + v_n) * 2, b0, b1, b2, b3);
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
          ptx::mma_16816(o[mt][2 * np], pf[mt][ks], b0, b1);
          ptx::mma_16816(o[mt][2 * np + 1], pf[mt][ks], b2, b3);
        }
      }
    }
    __syncthreads();  // all warps done with buf before the next iteration's prefetch overwrites it
  }

  // ---- normalise, stage through smem (Q tile is dead), 16-byte stores
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l_run[mt][r] += __shfl_xor_sync(0xffffffffu, l_run[mt][r], 1);
      l_run[mt][r] += __shfl_xor_sync(0xffffffffu, l_run[mt][r], 2);
    }
    const float inv0 = 1.f / l_run[mt][0], inv1 = 1.f / l_run[mt][1];
    const int r0 = (warp * MT + mt) * 16 + g;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      *reinterpret_cast<uint32_t*>(s_q + r0 * AT_RS + (nt * 8 + t4 * 2) * 2) = pack_bf16x2(o[mt][nt][0] * inv0, o[mt][nt][1] * inv0);
      *reinterpret_cast<uint32_t*>(s_q + (r0 + 8) * AT_RS + (nt * 8 + t4 * 2) * 2) = pack_bf16x2(o[mt][nt][2] * inv1, o[mt][nt][3] * inv1);
    }
  }
  __syncthreads();
  for (int i = tid; i < AT_BM * 8; i += 128) {
    const int r = i >> 3, v = i & 7;
    const int l = qt * AT_BM + r;
    if (l < a.L) {
      const long long row = token_row(a, b, wi, l);
      *reinterpret_cast<uint4*>(a.out + row * a.C + head * AT_D + v * 8) = *reinterpret_cast<const uint4*>(s_q + r * AT_RS + v * 16);
    }
  }
}

}  // namespace es3

using namespace es3;

// qkv [B*H*W, 3*C] bf16 (q|k|v, heads of 64 inside each) -> out [B*H*W, C] bf16.
// win > 0: attention inside non-overlapping win x win windows (H, W multiples of win); win == 0: global.
extern "C" int es3_attention_tc_bf16(const void* qkv, void* out, int B, int H, int W, int C, int num_heads, int win,
                                     float scale, void* stream);

// Dispatcher: sequences of >= 128 tokens run the wgmma kernel (attention_tc.cu); shorter windows (only
// reached by reduced-size test configurations) use the warp-level mma.sync kernel below.
extern "C" int es3_attention_mma_bf16(const void* qkv, void* out, int B, int H, int W, int C, int num_heads, int win,
                                      float scale, void* stream);
extern "C" int es3_attention_bf16(const void* qkv, void* out, int B, int H, int W, int C, int num_heads, int win,
                                  float scale, void* stream) {
  const int L = win ? win * win : H * W;
  if (L >= 128) return es3_attention_tc_bf16(qkv, out, B, H, W, C, num_heads, win, scale, stream);
  return es3_attention_mma_bf16(qkv, out, B, H, W, C, num_heads, win, scale, stream);
}

template <bool CAUSAL>
static int attention_mma(const void* qkv, void* out, int B, int H, int W, int C, int num_heads, int win, float scale,
                         void* stream) {
  const char* name = CAUSAL ? "es3_attention_causal_bf16" : "es3_attention_mma_bf16";
  ES3_REQUIRE(B > 0 && H > 0 && W > 0 && win >= 0, "%s: bad shape B=%d H=%d W=%d win=%d", name, B, H, W, win);
  ES3_REQUIRE(C == num_heads * AT_D, "%s: head_dim must be 64 (C=%d heads=%d)", name, C, num_heads);
  // cp.async loads and the output's uint4 stores move 16 bytes at a time
  ES3_REQUIRE(((uintptr_t)qkv & 15) == 0 && ((uintptr_t)out & 15) == 0, "%s: qkv and out must be 16-byte aligned", name);
  ES3_REQUIRE(win == 0 || (H % win == 0 && W % win == 0), "%s: H,W must be multiples of the window (%d,%d,%d)", name, H, W, win);
  AttnArgs a;
  a.qkv = (const bf16*)qkv; a.out = (bf16*)out; a.H = H; a.W = W; a.C = C; a.win = win;
  a.nwx = win ? W / win : 1;
  a.nwin = win ? (H / win) * (W / win) : 1;
  a.L = win ? win * win : H * W;
  a.scale_log2 = scale * 1.4426950408889634f;
  // two 16-row query tiles per warp (128-row CTA tile) whenever the sequence fills it; one otherwise
  const bool mt2 = a.L >= 128;
  const int bm = mt2 ? 128 : 64;
  const size_t smem = (size_t)(bm + 4 * AT_BN) * AT_RS;
  static bool configured = false;
  if (!configured) {
    ES3_CHECK_CUDA(cudaFuncSetAttribute(attn_fwd_kernel<1, CAUSAL>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    ES3_CHECK_CUDA(cudaFuncSetAttribute(attn_fwd_kernel<2, CAUSAL>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    configured = true;
  }
  dim3 grid(ceil_div(a.L, bm), num_heads, B * a.nwin);
  if (mt2) attn_fwd_kernel<2, CAUSAL><<<grid, 128, smem, (cudaStream_t)stream>>>(a);
  else attn_fwd_kernel<1, CAUSAL><<<grid, 128, smem, (cudaStream_t)stream>>>(a);
  ES3_LAUNCH_CHECK("attn_fwd_kernel");
  return 0;
}

extern "C" int es3_attention_mma_bf16(const void* qkv, void* out, int B, int H, int W, int C, int num_heads, int win,
                                      float scale, void* stream) {
  return attention_mma<false>(qkv, out, B, H, W, C, num_heads, win, scale, stream);
}

// Causal self-attention over B sequences of L tokens (the mma.sync kernel with CAUSAL = true; sequences are one row
// of L tokens, global attention).
extern "C" int es3_attention_causal_bf16(const void* qkv, void* out, int B, int L, int C, int num_heads, float scale,
                                         void* stream) {
  ES3_REQUIRE(L >= 1, "es3_attention_causal_bf16: L must be >= 1 (L=%d)", L);
  return attention_mma<true>(qkv, out, B, 1, L, C, num_heads, 0, scale, stream);
}
