// FP8 (e4m3) flash attention on wgmma for the SAM3 ViT teacher (head_dim 64), windowed or global: the attention of
// ViT.enable_fp8(attention=True).  Same contract as es3_attention_tc_bf16: bf16 qkv [B*H*W, 3C] (q | k | v, heads of 64, RoPE
// already applied) -> bf16 [B*H*W, C]; windows are gathered in place, any L, the last key tile masked.
//
// Quantisation happens on the device with power-of-two scales: multiplying by 2^-k is exact, so the host reproduces every code bit
// for bit (tests/emu_fp8_attention.py) and no IEEE division is needed:
//   s = 2^k,  k = ceil(log2(amax / 448)) clamped to >= -126  (s = 1 for an all-zero block),   q = e4m3_rn_satfinite(x * 2^-k)
// with the blocks
//   Q: one (query token, head), 64 values     K: one (key token, head)     V: one (key tile, head, channel), the tile's BN keys
//   P: the softmax numerators p = exp2(t - m) in [0, 1] as e4m3(p * 2^8); no scale.
// Then  S = (qQ . qK) sQ[row] sK[col]  and, per key tile,  pv[d] = sum_j P_j qV[j, d]  into a fresh fp32 accumulator, promoted as
//   o[d] = (o[d] + pv[d] sV[d]) corr,   l = (l + sum_j P_j) corr,   out = o / l      (the common 2^8 of P cancels in o / l).
// The row sum comes out of the same MMA: V^T carries a 65th row of 1.0 codes (an m64n72 PV product), so l is the sum of exactly the
// P codes that entered the MMA, accumulated the same way as o.
//
// Two launches.  quantize_kv_kernel quantises K and V once per (image, window, head, key tile) into a workspace: K rows as they
// are (K-major), V transposed (V^T: channels x keys, keys contiguous), with their scales.  Every query tile of the same window reads
// those codes, so the quantisation is paid once per key instead of once per (query tile, key).  attn_fp8_kernel then runs one CTA
// per 128-row query tile of one (image, window, head), 384 threads:
//   warpgroup 0     : producer -- cp.async copies the e4m3 tiles and scales of key tile j into a STG-deep ring (128B-swizzled for
//                     the wgmma descriptors) and publishes tile j - LAG on its full mbarrier once its own copies of it have landed,
//                     so LAG tiles are in flight while the consumers work.
//   warpgroups 1, 2 : consumers, query rows 0..63 / 64..127 of the tile.  Q is quantised once into shared memory.  Per key tile j
//                     a consumer issues S_j = Q K_j^T (m64nBNk32, both operands in shared memory) and then PV_{j-1} (m64n72k32,
//                     P from registers) without waiting in between, runs the softmax of S_j while PV_{j-1} is in the tensor core,
//                     and only then waits for PV_{j-1} to promote it.  The two consumers interleave on the tensor core by
//                     themselves; the producer gives them its registers (setmaxnreg).
// e4m3 wgmma reads P as the A operand in a layout that is not the fp32 accumulator's: thread t of a quad holds columns
// 8 n + 2 t, + 1 of S but must supply A columns 4 t .. 4 t + 3.  Instead of moving values between lanes, the keys inside every
// 16-key group are permuted in V^T: A column 4 t + c carries key 8 (c >> 1) + 2 t + (c & 1), which is where the producer writes
// that key's V.  The product sums over keys, so the permutation is invisible in the result.
#include <cstdlib>

#include "fp8.cuh"
#include "ptx.cuh"

namespace es3 {
namespace fa8 {

constexpr int BM = 128, D = 64, STG = 6, LAG = 2;   // LAG: key tiles in flight between a copy and its publication
constexpr int THREADS = 3 * 128;
constexpr int ROW_BYTES = 128;                        // every tile row is one 128-byte swizzle row
constexpr int Q_BYTES = BM * ROW_BYTES;               // e4m3 Q, 64 codes in each 128-byte row
constexpr int STAGING_BYTES = 2 * 128 * ROW_BYTES;    // bf16 K | V of one key tile (up to 128 keys), in the pre-pass
constexpr int KQ_BYTES = 128 * ROW_BYTES;             // e4m3 K, 64 codes a row
constexpr int VT_ROWS = 72;                           // 64 channels, the row of 1.0 codes, 7 zero rows (N = 72)
constexpr int VT_OFF = KQ_BYTES;
constexpr int SK_OFF = VT_OFF + VT_ROWS * ROW_BYTES;  // fp32 sK[128]
constexpr int SV_OFF = SK_OFF + 128 * 4;              // fp32 sV[64]
constexpr int RING_BYTES = 26 * 1024;                 // SV_OFF + 256 rounded up to the 1024-byte swizzle atom
constexpr int SMEM_BYTES = 1024 + Q_BYTES + STG * RING_BYTES;
constexpr int PRE_SMEM_BYTES = 1024 + STAGING_BYTES;
// setmaxnreg moves registers inside the CTA's allocation (168 a thread at 384 threads, one CTA per SM): the consumers' increase
// can only be granted out of what the producer hands back, so the split must fit the launch allocation
constexpr int LAUNCH_REGS = 168, PRODUCER_REGS = 40, CONSUMER_REGS = 232;
static_assert(128 * PRODUCER_REGS + 256 * CONSUMER_REGS <= LAUNCH_REGS * THREADS, "register split exceeds the CTA's allocation");
constexpr uint32_t E4M3_ONE = 0x38383838u;

struct Args {
  const bf16* qkv;
  bf16* out;
  uint8_t* kq;          // workspace: e4m3 K [group][tiles * BN][64], group = (image * windows + window) * heads + head
  uint8_t* vt;          //            e4m3 V^T [group][tile][64][BN]
  float* sk;            //            [group][tiles * BN]
  float* sv;            //            [group][tile][64]
  int H, W, C, win, nwx, nwin, L;
  float scale_log2;
};

__device__ __forceinline__ long long token_row(const Args& a, int b, int wi, int l) {
  if (a.win == 0) return (long long)b * a.H * a.W + l;
  const int wy = wi / a.nwx, wx = wi - wy * a.nwx;
  const int i = l / a.win, j = l - i * a.win;
  return (long long)b * a.H * a.W + (long long)(wy * a.win + i) * a.W + wx * a.win + j;
}

__device__ __forceinline__ void cp16(uint32_t saddr, const void* g, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(saddr), "l"(g), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// staging: bf16 row r (a key) of 128 bytes, 16-byte chunk c.  XOR with r & 7 spreads a warp's row-per-lane reads (K) over the
// banks; XOR with 2 ((r >> 5) & 3) does the same for the column reads of V, whose lanes sit 32 rows apart.
__device__ __forceinline__ uint32_t stg_off(int r, int c) { return r * ROW_BYTES + ((c ^ (r & 7) ^ (((r >> 5) & 3) << 1)) << 4); }
// e4m3 tiles: the 128B swizzle of the wgmma descriptors (8-row atoms of 1024 B)
__device__ __forceinline__ uint32_t sw_off(int r, int c) { return r * ROW_BYTES + ((c ^ (r & 7)) << 4); }

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// lane-wise max of two pairs of non-negative bf16
__device__ __forceinline__ uint32_t bmax2(uint32_t a, uint32_t b) {
  uint32_t r;
  asm("max.bf16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
  return r;
}
__device__ __forceinline__ float bf_lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf_hi(uint32_t u) { return __uint_as_float(u & 0xFFFF0000u); }

// k = ceil(log2(amax / 448)) for amax > 0, from the bits: amax = 1.f 2^e is above 448 2^(e - 8) = 1.75 2^e exactly when f > 0.75
__device__ __forceinline__ int scale_exp(float amax) {
  if (amax == 0.f) return 0;
  const uint32_t b = __float_as_uint(amax);
  return max((int)(b >> 23) - 135 + ((b & 0x7FFFFFu) > 0x600000u ? 1 : 0), -126);
}
__device__ __forceinline__ float exp2i(int k) { return __uint_as_float((uint32_t)(k + 127) << 23); }

// four bf16 (two words) * inv -> four e4m3 codes in one word
__device__ __forceinline__ uint32_t codes4(uint32_t u0, uint32_t u1, float inv) {
  return e4m3x2(bf_lo(u0) * inv, bf_hi(u0) * inv) | (e4m3x2(bf_lo(u1) * inv, bf_hi(u1) * inv) << 16);
}

template <int R>
__device__ __forceinline__ void fence_u32(uint32_t* r) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+r"(r[i])::"memory");
}

// Pre-pass: quantise one key tile (BN keys) of one (image, window, head) into the workspace, once for every query tile that reads
// it.  K rows stay K-major ([key][64] codes + sK[key]); V is written transposed ([channel][BN] codes, the keys of every 16-key group
// permuted as the P fragment needs; see the header) with sV[channel].  Keys past L are zero codes with scale 1.
template <int BN>
__global__ void __launch_bounds__(128) quantize_kv_kernel(const Args a) {
  extern __shared__ uint8_t raw[];
  const uint32_t s_raw = ptx::smem_u32(raw);
  const uint32_t s0 = (s_raw + 1023u) & ~1023u;
  uint8_t* g0 = raw + (s0 - s_raw);
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int j = blockIdx.x, head = blockIdx.y;
  const int b = blockIdx.z / a.nwin, wi = blockIdx.z % a.nwin;
  const int ntiles = gridDim.x;
  const long long grp = (long long)blockIdx.z * gridDim.y + head;
  const int ld = 3 * a.C;
  {
    const bf16* kbase = a.qkv + head * D + a.C;
    const int c = t & 7;
#pragma unroll
    for (int r = t >> 3; r < BN; r += 16) {
      const int l = j * BN + r;
      const bool ok = l < a.L;
      const bf16* src = kbase + (ok ? token_row(a, b, wi, l) : 0) * ld + c * 8;
      cp16(s0 + stg_off(r, c), src, ok);
      cp16(s0 + 128 * ROW_BYTES + stg_off(r, c), src + a.C, ok);
    }
    cp_commit();
    cp_wait<0>();
    __syncthreads();
  }
  const uint8_t* kst = g0;
  const uint8_t* vst = kst + 128 * ROW_BYTES;
  // ---- K: thread t quantises key row t (64 values, one block)
  if (t < BN) {
    uint4 ch[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) ch[c] = *reinterpret_cast<const uint4*>(kst + stg_off(t, c));
    uint32_t m = 0;
#pragma unroll
    for (int c = 0; c < 8; ++c)
      m = bmax2(m, bmax2(bmax2(ch[c].x & 0x7FFF7FFFu, ch[c].y & 0x7FFF7FFFu), bmax2(ch[c].z & 0x7FFF7FFFu, ch[c].w & 0x7FFF7FFFu)));
    const int k = scale_exp(fmaxf(bf_lo(m), bf_hi(m)));
    const float inv = exp2i(-k);
    uint4* dst = reinterpret_cast<uint4*>(a.kq + (grp * ntiles * BN + (long long)j * BN + t) * D);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const uint4 x = ch[2 * c], y = ch[2 * c + 1];
      dst[c] = make_uint4(codes4(x.x, x.y, inv), codes4(x.z, x.w, inv), codes4(y.x, y.y, inv), codes4(y.z, y.w, inv));
    }
    a.sk[grp * ntiles * BN + (long long)j * BN + t] = exp2i(k);
  }
  // ---- V: channels 2 cp, 2 cp + 1 over the 32 keys 32 q .. 32 q + 31; the four q of a channel pair are neighbouring lanes
  {
    const int cp = (warp << 3) + (lane >> 2), q = lane & 3;
    const bool act = q < BN / 32;
    uint32_t v[32];
    uint32_t m = 0;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int key = 32 * q + i;
      v[i] = act ? *reinterpret_cast<const uint32_t*>(vst + stg_off(key, cp >> 2) + 4 * (cp & 3)) : 0u;
      m = bmax2(m, v[i] & 0x7FFF7FFFu);
    }
    m = bmax2(m, __shfl_xor_sync(0xffffffffu, m, 1));
    m = bmax2(m, __shfl_xor_sync(0xffffffffu, m, 2));
    const int k0 = scale_exp(bf_lo(m)), k1 = scale_exp(bf_hi(m));
    const float inv0 = exp2i(-k0), inv1 = exp2i(-k1);
    if (act) {
      uint8_t* vt = a.vt + (grp * ntiles + j) * D * BN;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int d = 2 * cp + h;
        const float inv = h ? inv1 : inv0;
        auto val = [&](int i) { return h ? bf_hi(v[i]) : bf_lo(v[i]); };
#pragma unroll
        for (int g = 0; g < 2; ++g) {
          uint32_t w[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {   // A column 4 u + c of the 16-key group holds key 8 (c >> 1) + 2 u + (c & 1)
            const int k = 16 * g + 2 * u;
            w[u] = e4m3x2(val(k) * inv, val(k + 1) * inv) | (e4m3x2(val(k + 8) * inv, val(k + 9) * inv) << 16);
          }
          *reinterpret_cast<uint4*>(vt + d * BN + (2 * q + g) * 16) = make_uint4(w[0], w[1], w[2], w[3]);
        }
      }
      if (q == 0) {
        float* sv = a.sv + (grp * ntiles + j) * D;
        sv[2 * cp] = exp2i(k0);
        sv[2 * cp + 1] = exp2i(k1);
      }
    }
  }
}

template <int BN>
__global__ void __launch_bounds__(THREADS, 1) attn_fp8_kernel(const Args a) {
  extern __shared__ uint8_t raw[];
  __shared__ __align__(8) uint64_t full[STG], empty[STG];
  __shared__ float sq[BM];

  const uint32_t s_raw = ptx::smem_u32(raw);
  const uint32_t s0 = (s_raw + 1023u) & ~1023u;
  uint8_t* g0 = raw + (s0 - s_raw);                   // the same aligned base as a generic pointer
  const uint32_t u_q = s0, u_ring = s0 + Q_BYTES;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int head = blockIdx.y;
  const int b = blockIdx.z / a.nwin, wi = blockIdx.z % a.nwin;
  const int q0 = blockIdx.x * BM;
  const int ld = 3 * a.C;
  const bf16* qbase = a.qkv + head * D;
  const int ntiles = (a.L + BN - 1) / BN;

  if (tid == 0) {
    for (int s = 0; s < STG; ++s) { ptx::mbar_init(&full[s], 128); ptx::mbar_init(&empty[s], 8); }
    ptx::fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ================================================================== producer warpgroup: copies only
    ptx::setmaxnreg_dec<PRODUCER_REGS>();
    const int t = tid;
    // the constant rows of every V^T stage: row 64 = 1.0 codes (the row sum), rows 65..71 = 0
    for (int i = t; i < STG * 8 * 8; i += 128) {
      const int s = i >> 6, r = (i >> 3) & 7, c = i & 7;
      *reinterpret_cast<uint4*>(g0 + (u_ring - s0) + s * RING_BYTES + VT_OFF + (64 + r) * ROW_BYTES + c * 16) =
          r == 0 ? make_uint4(E4M3_ONE, E4M3_ONE, E4M3_ONE, E4M3_ONE) : make_uint4(0, 0, 0, 0);
    }
    const long long grp = (long long)blockIdx.z * gridDim.y + head;
    const uint8_t* kq = a.kq + grp * ntiles * BN * D;
    const uint8_t* vt = a.vt + grp * ntiles * D * BN;
    const float* sk = a.sk + grp * ntiles * BN;
    const float* sv = a.sv + grp * ntiles * D;
    constexpr int NK = BN * 4, NV = D * (BN / 16), NSK = BN / 4, NSV = D / 4;   // 16-byte chunks of one key tile
    int stage = 0;
    uint32_t phase = 0;
    for (int j = 0; j < ntiles; ++j) {
      ptx::mbar_wait(&empty[stage], phase ^ 1);
      const uint32_t ring = u_ring + stage * RING_BYTES;
      for (int i = t; i < NK + NV + NSK + NSV; i += 128) {
        if (i < NK) {
          const int r = i >> 2, c = i & 3;
          cp16(ring + sw_off(r, c), kq + ((long long)j * BN + r) * D + c * 16, true);
        } else if (i < NK + NV) {
          const int d = (i - NK) / (BN / 16), c = (i - NK) % (BN / 16);
          cp16(ring + VT_OFF + sw_off(d, c), vt + ((long long)j * D + d) * BN + c * 16, true);
        } else if (i < NK + NV + NSK) {
          const int c = i - NK - NV;
          cp16(ring + SK_OFF + c * 16, sk + (long long)j * BN + 4 * c, true);
        } else {
          const int c = i - NK - NV - NSK;
          cp16(ring + SV_OFF + c * 16, sv + (long long)j * D + 4 * c, true);
        }
      }
      cp_commit();
      // tile j - LAG has landed (this thread's copies of it): publish it to the consumers
      if (j >= LAG) {
        cp_wait<LAG>();
        ptx::fence_proxy_async();                     // generic-proxy writes -> visible to the wgmma (async proxy) reads
        const int ps = (stage + STG - LAG) % STG;
        ptx::mbar_arrive(&full[ps]);
      }
      if (++stage == STG) { stage = 0; phase ^= 1; }
    }
    cp_wait<0>();
    ptx::fence_proxy_async();
    for (int j = ntiles > LAG ? ntiles - LAG : 0; j < ntiles; ++j) ptx::mbar_arrive(&full[j % STG]);
    return;
  }

  // ==================================================================== consumer warpgroups
  ptx::setmaxnreg_inc<CONSUMER_REGS>();
  const int wg = (warp >> 2) - 1, wq = warp & 3, tw = tid & 127;
  // ---- Q: thread tw quantises half (32 values) of row tw / 2 of this warpgroup's 64; the two halves share the block's amax
  {
    const int r = tw >> 1, hf = tw & 1;
    const int l = q0 + wg * 64 + r;
    uint4 x[4];
    if (l < a.L) {
      const uint4* src = reinterpret_cast<const uint4*>(qbase + token_row(a, b, wi, l) * ld + hf * 32);
#pragma unroll
      for (int i = 0; i < 4; ++i) x[i] = __ldg(src + i);
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) x[i] = make_uint4(0, 0, 0, 0);
    }
    uint32_t m = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i)
      m = bmax2(m, bmax2(bmax2(x[i].x & 0x7FFF7FFFu, x[i].y & 0x7FFF7FFFu), bmax2(x[i].z & 0x7FFF7FFFu, x[i].w & 0x7FFF7FFFu)));
    m = bmax2(m, __shfl_xor_sync(0xffffffffu, m, 1));
    const int k = scale_exp(fmaxf(bf_lo(m), bf_hi(m)));
    const float inv = exp2i(-k);
    const int row = wg * 64 + r;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const uint4 p = x[2 * c], n = x[2 * c + 1];
      *reinterpret_cast<uint4*>(g0 + sw_off(row, 2 * hf + c)) =
          make_uint4(codes4(p.x, p.y, inv), codes4(p.z, p.w, inv), codes4(n.x, n.y, inv), codes4(n.z, n.w, inv));
    }
    if (hf == 0) sq[row] = exp2i(k);
    ptx::fence_proxy_async();
    ptx::named_bar(2 + wg, 128);
  }
  const int g = lane >> 2, t4 = lane & 3;
  float rowscale[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) rowscale[h] = sq[wg * 64 + 16 * wq + g + 8 * h] * a.scale_log2;
  const uint64_t dq = ptx::make_desc_sw128(u_q + wg * 8192);

  float o[32], pv[36], s[BN / 2];
  uint32_t pk[BN / 8];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  auto issue_s = [&](int st) {
    const uint64_t dk = ptx::make_desc_sw128(u_ring + st * RING_BYTES);
#pragma unroll
    for (int k = 0; k < D / 32; ++k) {
      if constexpr (BN == 128) ptx::wgmma_m64n128k32_e4m3(s, ptx::desc_advance(dq, 32 * k), ptx::desc_advance(dk, 32 * k), k != 0);
      else ptx::wgmma_m64n96k32_e4m3(s, ptx::desc_advance(dq, 32 * k), ptx::desc_advance(dk, 32 * k), k != 0);
    }
    ptx::wg_commit();
  };
  auto issue_pv = [&](int st) {
    const uint64_t dv = ptx::make_desc_sw128(u_ring + st * RING_BYTES + VT_OFF);
#pragma unroll
    for (int k = 0; k < BN / 32; ++k) ptx::wgmma_m64n72k32_e4m3_rs(pv, pk + 4 * k, ptx::desc_advance(dv, 32 * k), k != 0);
    ptx::wg_commit();
  };
  // S_j (in s) -> p * 2^8 (in s); returns the rescale of the running sums in corr
  auto softmax = [&](int j, int st, float* corr) {
    const float* sk = reinterpret_cast<const float*>(g0 + (u_ring - s0) + st * RING_BYTES + SK_OFF);
#pragma unroll
    for (int n = 0; n < BN / 8; ++n) {
      const float2 kk = *reinterpret_cast<const float2*>(sk + 8 * n + 2 * t4);
      s[4 * n] *= kk.x; s[4 * n + 1] *= kk.y; s[4 * n + 2] *= kk.x; s[4 * n + 3] *= kk.y;
    }
    const int col0 = j * BN;
    if (col0 + BN > a.L) {                            // partial key tile: columns past L do not exist
#pragma unroll
      for (int i = 0; i < BN / 2; ++i)
        if (col0 + ptx::wg_frag_col(lane, i) >= a.L) s[i] = -INFINITY;
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
    float bias[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      const float m_new = fmaxf(m_run[h], mx[h] * rowscale[h]);
      corr[h] = ex2(m_run[h] - m_new);
      m_run[h] = m_new;
      bias[h] = 8.f - m_new;                          // p * 2^8 = exp2(t - m + 8)
    }
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) s[i] = ex2(fmaf(s[i], rowscale[(i >> 1) & 1], bias[(i >> 1) & 1]));   // masked -> 0
  };
  // accumulator columns 16 kk .. 16 kk + 15 of rows r / r + 8 -> the A fragment of k-step kk / 2 (see the header)
  auto pack = [&]() {
#pragma unroll
    for (int kk = 0; kk < BN / 32; ++kk) {
      const float* x = s + 16 * kk;
      pk[4 * kk + 0] = e4m3x2(x[0], x[1]) | (e4m3x2(x[4], x[5]) << 16);
      pk[4 * kk + 1] = e4m3x2(x[2], x[3]) | (e4m3x2(x[6], x[7]) << 16);
      pk[4 * kk + 2] = e4m3x2(x[8], x[9]) | (e4m3x2(x[12], x[13]) << 16);
      pk[4 * kk + 3] = e4m3x2(x[10], x[11]) | (e4m3x2(x[14], x[15]) << 16);
    }
  };
  auto promote = [&](int st, const float* corr) {
    const float* sv = reinterpret_cast<const float*>(g0 + (u_ring - s0) + st * RING_BYTES + SV_OFF);
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      const float2 vv = *reinterpret_cast<const float2*>(sv + 8 * n + 2 * t4);
      o[4 * n] = (o[4 * n] + pv[4 * n] * vv.x) * corr[0];
      o[4 * n + 1] = (o[4 * n + 1] + pv[4 * n + 1] * vv.y) * corr[0];
      o[4 * n + 2] = (o[4 * n + 2] + pv[4 * n + 2] * vv.x) * corr[1];
      o[4 * n + 3] = (o[4 * n + 3] + pv[4 * n + 3] * vv.y) * corr[1];
    }
    // column 64 (the 1.0 row) of lane t4 == 0 is the row sum; the other lanes' columns 64.. are the zero rows
    l_run[0] = (l_run[0] + pv[32]) * corr[0];
    l_run[1] = (l_run[1] + pv[34]) * corr[1];
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(&empty[st]);       // K_j / V_j of this stage no longer needed by this warp
  };

  int stage = 0;
  uint32_t phase = 0;
  float corr[2];
  ptx::mbar_wait(&full[0], 0);
  ptx::wg_fence();
  issue_s(0);
  ptx::wg_wait<0>();
  ptx::wg_fence_regs<BN / 2>(s);
  softmax(0, 0, corr);
  pack();
  int pstage = 0;
  if (++stage == STG) { stage = 0; phase ^= 1; }
  for (int j = 1; j < ntiles; ++j) {
    ptx::mbar_wait(&full[stage], phase);
    ptx::wg_fence();
    fence_u32<BN / 8>(pk);
    issue_s(stage);                                   // S_j ...
    issue_pv(pstage);                                 // ... and PV_{j-1} back to back
    ptx::wg_wait<1>();
    ptx::wg_fence_regs<BN / 2>(s);
    softmax(j, stage, corr);                          // overlaps PV_{j-1}
    ptx::wg_wait<0>();
    ptx::wg_fence_regs<36>(pv);
    fence_u32<BN / 8>(pk);
    promote(pstage, corr);
    pack();
    pstage = stage;
    if (++stage == STG) { stage = 0; phase ^= 1; }
  }
  ptx::wg_fence();
  fence_u32<BN / 8>(pk);
  issue_pv(pstage);
  ptx::wg_wait<0>();
  ptx::wg_fence_regs<36>(pv);
  fence_u32<BN / 8>(pk);
  const float one[2] = {1.f, 1.f};
  promote(pstage, one);

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
      bf16* op = a.out + token_row(a, b, wi, l) * a.C + head * D;
#pragma unroll
      for (int i = 2 * h; i < 32; i += 4)
        *reinterpret_cast<uint32_t*>(op + ptx::wg_frag_col(lane, i)) = pack_bf16x2(o[i] * inv, o[i + 1] * inv);
    }
  }
}

}  // namespace fa8
}  // namespace es3

using namespace es3;

// Workspace of es3_attention_fp8 in floats: the e4m3 K and V^T codes of every key tile and their scales.
static long long ws_bytes(int B, int H, int W, int num_heads, int win) {
  const int L = win ? win * win : H * W;
  const int bn = (L % 96 == 0 && L % 128 != 0) ? 96 : 128;
  const long long groups = (long long)B * (win ? (H / win) * (W / win) : 1) * num_heads;
  const long long keys = (long long)ceil_div(L, bn) * bn;
  return groups * keys * (2 * fa8::D + 4) + groups * ceil_div(L, bn) * fa8::D * 4;
}
extern "C" long long es3_attention_fp8_ws_floats(int B, int H, int W, int num_heads, int win) {
  if (B <= 0 || H <= 0 || W <= 0 || num_heads <= 0 || win < 0 || (win && (H % win || W % win))) return 0;
  return (ws_bytes(B, H, W, num_heads, win) + 3) / 4;
}

// FP8 flash attention; the contract of es3_attention_tc_bf16 (head_dim 64, the window divides H and W, scale > 0) plus a workspace
// of es3_attention_fp8_ws_floats(B, H, W, num_heads, win) floats, 16-byte aligned.
extern "C" int es3_attention_fp8(const void* qkv, void* out, void* ws, int B, int H, int W, int C, int num_heads, int win,
                                 float scale, void* stream) {
  using namespace fa8;
  ES3_REQUIRE(B > 0 && H > 0 && W > 0 && win >= 0, "es3_attention_fp8: bad shape B=%d H=%d W=%d win=%d", B, H, W, win);
  ES3_REQUIRE(C == num_heads * D, "es3_attention_fp8: head_dim must be 64 (C=%d heads=%d)", C, num_heads);
  ES3_REQUIRE(win == 0 || (H % win == 0 && W % win == 0), "es3_attention_fp8: H,W must be multiples of the window");
  ES3_REQUIRE(scale > 0.f && scale < INFINITY, "es3_attention_fp8: scale must be positive and finite (%g)", (double)scale);
  ES3_REQUIRE(((uintptr_t)qkv & 15) == 0 && ((uintptr_t)out & 3) == 0 && ws != nullptr && ((uintptr_t)ws & 15) == 0,
              "es3_attention_fp8: qkv and the workspace must be 16-byte aligned");
  Args a;
  a.qkv = (const bf16*)qkv; a.out = (bf16*)out; a.H = H; a.W = W; a.C = C; a.win = win;
  a.nwx = win ? W / win : 1;
  a.nwin = win ? (H / win) * (W / win) : 1;
  a.L = win ? win * win : H * W;
  a.scale_log2 = scale * 1.4426950408889634f;
  const bool bn96 = a.L % 96 == 0 && a.L % 128 != 0;   // 24x24 windows (576 = 6 x 96) and L = 5184 (54 x 96): no padded keys
  const int bn = bn96 ? 96 : 128, ntiles = ceil_div(a.L, bn);
  const long long groups = (long long)B * a.nwin * num_heads, keys = (long long)ntiles * bn;
  a.kq = (uint8_t*)ws;
  a.vt = a.kq + groups * keys * D;
  a.sk = (float*)(a.vt + groups * keys * D);
  a.sv = a.sk + groups * keys;
  int dev = 0;
  ES3_CHECK_CUDA(cudaGetDevice(&dev));
  static uint64_t configured = 0;                      // one bit per device: the attribute is per device
  if (dev >= 64 || !(configured >> dev & 1)) {
    ES3_CHECK_CUDA(cudaFuncSetAttribute(attn_fp8_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    ES3_CHECK_CUDA(cudaFuncSetAttribute(attn_fp8_kernel<96>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    if (dev < 64) configured |= 1ull << dev;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 pgrid(ntiles, num_heads, B * a.nwin), grid(ceil_div(a.L, BM), num_heads, B * a.nwin);
  if (bn96) {
    quantize_kv_kernel<96><<<pgrid, 128, PRE_SMEM_BYTES, st>>>(a);
    ES3_LAUNCH_CHECK("quantize_kv_kernel");
    attn_fp8_kernel<96><<<grid, THREADS, SMEM_BYTES, st>>>(a);
  } else {
    quantize_kv_kernel<128><<<pgrid, 128, PRE_SMEM_BYTES, st>>>(a);
    ES3_LAUNCH_CHECK("quantize_kv_kernel");
    attn_fp8_kernel<128><<<grid, THREADS, SMEM_BYTES, st>>>(a);
  }
  ES3_LAUNCH_CHECK("attn_fp8_kernel");
  return 0;
}
