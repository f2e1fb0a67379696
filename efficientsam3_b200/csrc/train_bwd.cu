// Student backward (SURVEY.md §8 A19/A20: the `loss.backward()` half of train_one_epoch,
// stage1/train_image_encoder_stage1.py:154-268) -- the kernels the train-mode forward and the backward of the
// EfficientViT student need beyond the inference kernels:
//
//   train-mode BatchNorm2d (efficientvit/nn/ops.py:39-80 ConvLayer.norm in .train(): batch statistics + running-stat update)
//     es3_bn_stats            per-channel mean / invstd over the rows of a raw conv output  (two-stage, deterministic)
//     es3_affine_act          a = act(scale[c] * z + shift[c]) (+ residual)                (the normalise + activation pass)
//     es3_bn_act_bwd_reduce   g = da * act'(u); per-channel sum g, sum g z -> dgamma, dbeta and the dz coefficients
//     es3_bn_act_bwd_apply    dz = A[c] g + B[c] z + C[c]   (batch BN, eval BN and bias-only layers share it)
//   convolution gradients
//     es3_wgrad_pw            dW[n][k] = sum_m dz[m][n] x[m][k]: 1x1 convs, and one tap of a dense 3x3 (spatially shifted x)
//                             -- mma.sync m16n8k16 with both operands through ldmatrix.trans (contraction over pixels)
//     es3_dwconv_bwd_data     depthwise conv input gradient for any stride (stride 1 can also use es3_dwconv with flipped taps)
//     es3_dwconv_wgrad        depthwise conv weight gradient
//     es3_stem_wgrad          weight gradient of the 3 -> C stride-2 stem conv on the fp32 NCHW image
//     (input gradients of 1x1 / dense 3x3 convs are es3_gemm_bf16 / es3_conv3x3_bf16 calls on transposed / flipped weights)
//   es3_bilinear_bwd          adjoint of es3_bilinear_nhwc_to_nchw (F.interpolate backward, stage1/model.py:204-210)
//   es3_litemla_attn_bwd      backward of the ReLU linear attention (ops.py:592-621), head dim 16
//   es3_add_bf16              out = a + b on (row-strided) bf16 matrices: gradient fan-in at residual joins
//
// Gradients of activations are bf16 (the reference's AMP path keeps them fp16), parameter gradients fp32 and ACCUMULATED
// (+=) into their destination, all reductions are two-stage with a fixed order: no atomics, bit-reproducible.
#include "col_reduce.cuh"
#include "ptx.cuh"

namespace es3 {
namespace {

// ------------------------------------------------------------------------------------------ activation derivative
template <int ACT>
__device__ __forceinline__ float act_grad_t(float u) {
  if constexpr (ACT == ACT_RELU) return u > 0.f ? 1.f : 0.f;
  // aten hardswish_backward: 0 below -3, x/3 + 0.5 on [-3, 3], 1 above
  else if constexpr (ACT == ACT_HSWISH) return u < -3.f ? 0.f : (u <= 3.f ? fmaf(u, 1.f / 3.f, 0.5f) : 1.f);
  else if constexpr (ACT == ACT_GELU)
    return 0.5f * (1.f + erff(u * 0.70710678118654752440f)) + u * 0.3989422804014327f * __expf(-0.5f * u * u);
  else if constexpr (ACT == ACT_RELU6) return (u > 0.f && u < 6.f) ? 1.f : 0.f;
  else return 1.f;
}

#define ES3_DISPATCH_ACT_BWD(act, ACT_CONST, ...)                                                       \
  switch (act) {                                                                                        \
    case ACT_NONE: { constexpr int ACT_CONST = ACT_NONE; __VA_ARGS__; } break;                          \
    case ACT_RELU: { constexpr int ACT_CONST = ACT_RELU; __VA_ARGS__; } break;                          \
    case ACT_HSWISH: { constexpr int ACT_CONST = ACT_HSWISH; __VA_ARGS__; } break;                      \
    case ACT_GELU: { constexpr int ACT_CONST = ACT_GELU; __VA_ARGS__; } break;                          \
    case ACT_RELU6: { constexpr int ACT_CONST = ACT_RELU6; __VA_ARGS__; } break;                        \
    default: es3::set_error("activation code %d has no backward instantiated", act); return 1;          \
  }

__device__ __forceinline__ void cpa16(uint32_t saddr, const void* g, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(saddr), "l"(g), "r"(sz) : "memory");
}
__device__ __forceinline__ void cpa_wait_all() { asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void ldsm4t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}

// ------------------------------------------------------------------------------------------ per-channel column reductions
// z (and da) are [M][C] bf16, contiguous.  grid (nblk, ceil(CV / CVB)), block 256.  A thread owns one 8-channel vector
// (cv) and every `lanes`-th row of the block's row range; the lanes are then tree-reduced through shared memory.
// STATS: s0 = sum (z - k), s1 = sum (z - k)^2 with the per-channel pivot k = z[row 0] (shifted sums: no cancellation in
// E[z^2] - E[z]^2 when |mean| >> std).   else: g = da * act'(scale z + shift), s0 = sum g, s1 = sum g z.
// part: [nblk][2][C] fp32.
constexpr int CR_THREADS = 256;

// The loads are DECOUPLED from the registers: every thread streams its rows through a private ring of CRR_STAGES 16-byte
// shared-memory slots per tensor with cp.async (it reads back only what it copied itself, so no barrier is involved) and keeps
// CRR_STAGES - 1 rows in flight whatever the register pressure of the arithmetic.  With three resident CTAs that is
// 3 x 256 x 5 x 32 B = 120 KB per SM in flight.
constexpr int CRR_STAGES = 6;
template <int ACT, bool STATS>
__global__ void __launch_bounds__(CR_THREADS, 3) col_reduce_ring_kernel(const bf16* __restrict__ z, const bf16* __restrict__ da,
                                                                     const float* __restrict__ scale, const float* __restrict__ shift,
                                                                     long long M, int C, int CVB, long long rows_per_block,
                                                                     float* __restrict__ part) {
  __shared__ float red[CR_THREADS][17];
  extern __shared__ __align__(16) uint4 crr_ring[];          // [CRR_STAGES][STATS ? 1 : 2][CR_THREADS]
  constexpr int NT = STATS ? 1 : 2;
  const int tid = threadIdx.x;
  const int lanes = CR_THREADS / CVB;
  const int cvl = tid % CVB, pl = tid / CVB;
  const int cv = blockIdx.y * CVB + cvl;
  const bool active = pl < lanes && cv * 8 < C;
  float s0[8], s1[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) s0[i] = s1[i] = 0.f;
  if (active) {
    float sc[8], sh[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      sc[i] = (!STATS && scale) ? scale[cv * 8 + i] : 1.f;
      sh[i] = (!STATS && shift) ? shift[cv * 8 + i] : 0.f;
    }
    float piv[8];
    if constexpr (STATS) unpack8(__ldg(reinterpret_cast<const uint4*>(z + cv * 8)), piv);
    const long long r0 = (long long)blockIdx.x * rows_per_block + pl;
    const long long r1 = min(M, (long long)blockIdx.x * rows_per_block + rows_per_block);
    const long long n = r0 < r1 ? (r1 - r0 + lanes - 1) / lanes : 0;      // rows of this thread: r0, r0 + lanes, ...
    const uint32_t u_ring = static_cast<uint32_t>(__cvta_generic_to_shared(crr_ring)) + tid * 16;
    auto issue = [&](long long k) {
      if (k < n) {
        const long long off = (r0 + k * lanes) * C + cv * 8;
        const uint32_t slot = u_ring + (uint32_t)((k % CRR_STAGES) * NT) * (CR_THREADS * 16);
        cpa16(slot, z + off, true);
        if constexpr (!STATS) cpa16(slot + CR_THREADS * 16, da + off, true);
      }
      asm volatile("cp.async.commit_group;" ::: "memory");       // one group per row slot, empty past the end: the wait count stays fixed
    };
#pragma unroll
    for (int k = 0; k < CRR_STAGES - 1; ++k) issue(k);
    for (long long k = 0; k < n; ++k) {
      issue(k + CRR_STAGES - 1);
      asm volatile("cp.async.wait_group %0;" ::"n"(CRR_STAGES - 1) : "memory");
      const uint4* slot = crr_ring + (size_t)((k % CRR_STAGES) * NT) * CR_THREADS + tid;
      float fz[8];
      unpack8(slot[0], fz);
      if constexpr (STATS) {
#pragma unroll
        for (int i = 0; i < 8; ++i) { const float d = fz[i] - piv[i]; s0[i] += d; s1[i] = fmaf(d, d, s1[i]); }
      } else {
        float fd[8];
        unpack8(slot[CR_THREADS], fd);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float g = fd[i] * act_grad_t<ACT>(fmaf(sc[i], fz[i], sh[i]));
          s0[i] += g;
          s1[i] = fmaf(g, fz[i], s1[i]);
        }
      }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) { red[tid][i] = s0[i]; red[tid][8 + i] = s1[i]; }
  __syncthreads();
  int top = 1;
  while (top < lanes) top <<= 1;
  for (int stride = top >> 1; stride > 0; stride >>= 1) {
    if (pl < stride && pl + stride < lanes) {
#pragma unroll
      for (int i = 0; i < 16; ++i) red[tid][i] += red[tid + stride * CVB][i];
    }
    __syncthreads();
  }
  if (pl == 0 && cv * 8 < C) {
    float* p0 = part + ((long long)blockIdx.x * 2) * C + cv * 8;
    float* p1 = p0 + C;
#pragma unroll
    for (int i = 0; i < 8; ++i) { p0[i] = red[tid][i]; p1[i] = red[tid][8 + i]; }
  }
}

// Second stage of the column reductions: sum_block_partials (col_reduce.cuh).

// batch statistics, folded (scale, shift) for the normalise pass, running-stat update (nn.BatchNorm2d: momentum on the
// UNBIASED variance).  grid ceil(C / 8), block 256.
__global__ void __launch_bounds__(256) bn_stats_finalize_kernel(const bf16* __restrict__ z, const float* __restrict__ part, int nblk, int C,
                                                                long long M, float eps, float momentum, const float* __restrict__ gamma,
                                                                const float* __restrict__ beta, float* __restrict__ mean,
                                                                float* __restrict__ invstd, float* __restrict__ scale, float* __restrict__ shift,
                                                                float* __restrict__ running_mean, float* __restrict__ running_var,
                                                                long long* __restrict__ num_batches_tracked) {
  if (blockIdx.x == 0 && threadIdx.x == 0 && num_batches_tracked) num_batches_tracked[0] += 1;
  double s, q;
  int c;
  if (!sum_block_partials(part, nblk, C, s, q, c)) return;
  const double dm = s / (double)M;                       // mean of (z - pivot)
  const double mu = (double)__bfloat162float(z[c]) + dm;
  double var = q / (double)M - dm * dm;
  if (var < 0.0) var = 0.0;
  const float is = (float)(1.0 / sqrt(var + (double)eps));
  mean[c] = (float)mu;
  invstd[c] = is;
  const float sc = (gamma ? gamma[c] : 1.f) * is;
  scale[c] = sc;
  shift[c] = (beta ? beta[c] : 0.f) - (float)mu * sc;
  if (running_mean) running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)mu;
  if (running_var) {
    const double unbiased = M > 1 ? var * (double)M / (double)(M - 1) : var;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unbiased;
  }
}

// mode 0: no norm (scale = 1 or given, shift = conv bias): A = scale, dbeta (= d bias) += sum g
// mode 1: eval-mode BN (running stats): A = scale; dbeta += sum g; dgamma += invstd (sum g z - mean sum g)
// mode 2: batch-stat BN: additionally B, C carry the mean / variance terms of the BN backward.
// coef: [3][C] = A | B | C with dz = A g + B z + C.   grid ceil(C / 8), block 256.
__global__ void __launch_bounds__(256) bn_bwd_finalize_kernel(const float* __restrict__ part, int nblk, int C, long long M, int mode,
                                                              const float* __restrict__ scale, const float* __restrict__ mean,
                                                              const float* __restrict__ invstd, float* __restrict__ coef,
                                                              float* __restrict__ dgamma, float* __restrict__ dbeta) {
  double sg, sgz;
  int c;
  if (!sum_block_partials(part, nblk, C, sg, sgz, c)) return;
  const float sc = scale ? scale[c] : 1.f;
  float A = sc, Bc = 0.f, Cc = 0.f;
  if (mode != 0) {
    const double mu = (double)mean[c], is = (double)invstd[c];
    const double dgam = is * (sgz - mu * sg);
    if (dgamma) dgamma[c] += (float)dgam;
    if (mode == 2) {
      const double mg = sg / (double)M, mgx = dgam / (double)M;
      Bc = (float)(-(double)sc * is * mgx);
      Cc = (float)(-(double)sc * mg + (double)sc * is * mu * mgx);
    }
  }
  if (dbeta) dbeta[c] += (float)sg;
  coef[c] = A;
  coef[C + c] = Bc;
  coef[2 * C + c] = Cc;
}

// ------------------------------------------------------------------------------------------ elementwise passes
// Elementwise passes over [M][C] bf16.  Same thread map as the reductions: grid (nblk, ceil(CV / CVB)), a thread owns one
// 8-channel vector (its per-channel coefficients are loaded ONCE into registers) and every `lanes`-th row of the block's
// row range.  (The first version recomputed cv per element and re-read 3-5 coefficient scalars per value through
// LDG.32.)
__device__ __forceinline__ void load8f(const float* p, float* f, float fill) {
  if (p) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = fill;
  }
}

// a[m][c] = act(scale[c] z[m][c] + shift[c]) (+ residual[m][c])
template <int ACT>
__global__ void __launch_bounds__(256) affine_act_kernel(const bf16* __restrict__ z, const float* __restrict__ scale,
                                                         const float* __restrict__ shift, const bf16* __restrict__ residual,
                                                         bf16* __restrict__ out, long long M, int C, int CVB, long long rows_per_block) {
  const int tid = threadIdx.x, lanes = 256 / CVB;
  const int cv = blockIdx.y * CVB + tid % CVB, pl = tid / CVB;
  if (pl >= lanes || cv * 8 >= C) return;
  float sc[8], sh[8];
  load8f(scale ? scale + cv * 8 : nullptr, sc, 1.f);
  load8f(shift ? shift + cv * 8 : nullptr, sh, 0.f);
  const long long r0 = (long long)blockIdx.x * rows_per_block, r1 = min(M, r0 + rows_per_block);
  for (long long r = r0 + pl; r < r1; r += lanes) {
    const long long off = r * C + cv * 8;
    float f[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(z + off)), f);
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = es3_act_t<ACT>(fmaf(sc[k], f[k], sh[k]));
    if (residual) {
      float rr[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(residual + off)), rr);
#pragma unroll
      for (int k = 0; k < 8; ++k) f[k] += rr[k];
    }
    *reinterpret_cast<uint4*>(out + off) = pack8(f);
  }
}

// dz = A[c] * (da * act'(scale z + shift)) + B[c] * z + C[c]
template <int ACT>
__global__ void __launch_bounds__(256) bn_act_bwd_apply_kernel(const bf16* __restrict__ da, const bf16* __restrict__ z,
                                                               const float* __restrict__ scale, const float* __restrict__ shift,
                                                               const float* __restrict__ coef, bf16* __restrict__ dz, long long M, int C,
                                                               int CVB, long long rows_per_block) {
  const int tid = threadIdx.x, lanes = 256 / CVB;
  const int cv = blockIdx.y * CVB + tid % CVB, pl = tid / CVB;
  if (pl >= lanes || cv * 8 >= C) return;
  float sc[8], sh[8], cA[8], cB[8], cC[8];
  load8f(scale ? scale + cv * 8 : nullptr, sc, 1.f);
  load8f(shift ? shift + cv * 8 : nullptr, sh, 0.f);
  load8f(coef + cv * 8, cA, 0.f);
  load8f(coef + C + cv * 8, cB, 0.f);
  load8f(coef + 2 * C + cv * 8, cC, 0.f);
  const long long r0 = (long long)blockIdx.x * rows_per_block, r1 = min(M, r0 + rows_per_block);
  for (long long r = r0 + pl; r < r1; r += lanes) {
    const long long off = r * C + cv * 8;
    float fz[8], fd[8], o[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(z + off)), fz);
    unpack8(__ldg(reinterpret_cast<const uint4*>(da + off)), fd);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float g = fd[k] * act_grad_t<ACT>(fmaf(sc[k], fz[k], sh[k]));
      o[k] = fmaf(cA[k], g, fmaf(cB[k], fz[k], cC[k]));
    }
    *reinterpret_cast<uint4*>(dz + off) = pack8(o);
  }
}

// out[m][c] = a[m][c] + b[m][c]; row strides in elements (channel-sliced views), C % 8 == 0.
__global__ void add_bf16_kernel(const bf16* __restrict__ a, long long lda, const bf16* __restrict__ b, long long ldb,
                                bf16* __restrict__ out, long long ldo, long long M, int CV) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * CV) return;
  const long long m = i / CV;
  const int cv = (int)(i % CV);
  float fa[8], fb[8];
  unpack8(__ldg(reinterpret_cast<const uint4*>(a + m * lda + cv * 8)), fa);
  unpack8(__ldg(reinterpret_cast<const uint4*>(b + m * ldb + cv * 8)), fb);
#pragma unroll
  for (int k = 0; k < 8; ++k) fa[k] += fb[k];
  *reinterpret_cast<uint4*>(out + m * ldo + cv * 8) = pack8(fa);
}

// out[(i / inner) * ld_outer + (i % inner) * ld_inner] += sum_b part[b * n + i]   (fixed order over b).
// block 256 = 32 outputs x 8 lanes (lane l adds partials l, l + 8, ...), grid ceil(n / 32).
__global__ void __launch_bounds__(256) sum_partials_kernel(const float* __restrict__ part, int nblk, long long n, int inner,
                                                           long long ld_outer, long long ld_inner, float* __restrict__ out) {
  __shared__ float red[8][33];
  const int il = threadIdx.x & 31, lane = threadIdx.x >> 5;
  const long long i = (long long)blockIdx.x * 32 + il;
  float s = 0.f;
  if (i < n)
    for (int b = lane; b < nblk; b += 8) s += part[(long long)b * n + i];
  red[lane][il] = s;
  __syncthreads();
  if (lane == 0 && i < n) {
    float t = 0.f;
#pragma unroll
    for (int l = 0; l < 8; ++l) t += red[l][il];
    out[(i / inner) * ld_outer + (i % inner) * ld_inner] += t;
  }
}

// ------------------------------------------------------------------------------------------ pointwise weight gradient
// part[split][n][k] = sum over the split's row chunks of dz[m][n] * x[shift(m)][k].
// CTA tile: 64 (n) x 64 (k) outputs, 256-row chunks staged with cp.async; warp w contracts rows [32 w, 32 w + 32) of the
// chunk for the whole tile (4 x 8 m16n8 accumulator tiles), the 8 warps are summed through shared memory at the end.
// Both operands are [row = pixel][channel] in shared memory and go through ldmatrix.trans (the contraction index is the
// row), exactly the v^T k pattern of litemla_kv_tc_kernel.  shift: x row of output pixel (b, y, x) is (b, y+dy, x+dx),
// zero outside the H x W map (one tap of a 3x3 conv); dy = dx = 0 and H = 0 for plain 1x1 convs.
// MT / NP: the CTA tile is (16 MT) n x (16 NP) k outputs, MT, NP in {1, 2, 4} (narrow layers do not pay for a 64 x 64 tile:
// wgrad_pw[N=16,K=16] wasted most of the fixed tile).
constexpr int WG_ROWS = 256;
template <int MT, int NP>
struct WgCfg {
  static constexpr int TN = MT * 16, TK = NP * 16;
  static constexpr int VPR = (MT + NP) * 2;                 // 16-byte vectors per staged row
  static constexpr int RS = (MT + NP) * 32 + 16;            // row stride in bytes: odd multiple of 16 -> ldmatrix conflict-free
  static constexpr int RED = 8 * 16 * TK * 4;               // cross-warp reduction buffer (one 16-row slab)
  static constexpr int SMEM = (WG_ROWS * RS > RED) ? WG_ROWS * RS : RED;
};

template <int MT, int NP>
__global__ void __launch_bounds__(256) wgrad_pw_kernel(const bf16* __restrict__ dz, long long lddz, const bf16* __restrict__ x,
                                                       long long ldx, long long M, int N, int K, int H, int W, int dy, int dx,
                                                       float* __restrict__ part) {
  using Cfg = WgCfg<MT, NP>;
  extern __shared__ __align__(16) uint8_t wg_smem[];
  const uint32_t u = static_cast<uint32_t>(__cvta_generic_to_shared(wg_smem));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n0 = blockIdx.y * Cfg::TN, k0 = blockIdx.z * Cfg::TK;
  const long long nchunks = (M + WG_ROWS - 1) / WG_ROWS;
  float acc[MT][2 * NP][4];
#pragma unroll
  for (int a = 0; a < MT; ++a)
#pragma unroll
    for (int b = 0; b < 2 * NP; ++b) acc[a][b][0] = acc[a][b][1] = acc[a][b][2] = acc[a][b][3] = 0.f;
  const int av_p = (lane & 7) + ((lane >> 4) << 3), av_cb = ((lane >> 3) & 1) * 16;
  const int bk_p = (lane & 7) + (((lane >> 3) & 1) << 3), bk_cb = (lane >> 4) * 16;
  const bool shifted = H > 0;

  for (long long chunk = blockIdx.x; chunk < nchunks; chunk += gridDim.x) {
    const long long row0 = chunk * WG_ROWS;
    __syncthreads();   // every warp is done with the previous chunk
    for (int i = tid; i < WG_ROWS * Cfg::VPR; i += 256) {
      const int rl = i / Cfg::VPR, v = i % Cfg::VPR;
      const long long r = row0 + rl;
      const bf16* src = dz;
      bool ok = r < M;
      if (v < MT * 2) {
        const int c = n0 + v * 8;
        ok = ok && c < N;
        if (ok) src = dz + r * lddz + c;
      } else {
        const int c = k0 + (v - MT * 2) * 8;
        ok = ok && c < K;
        long long rs = r;
        if (ok && shifted) {
          const int px = (int)(r % W), py = (int)((r / W) % H);
          const int yy = py + dy, xx = px + dx;
          ok = yy >= 0 && yy < H && xx >= 0 && xx < W;
          rs = r + (long long)dy * W + dx;
        }
        if (ok) src = x + rs * ldx + c;
      }
      cpa16(u + rl * Cfg::RS + v * 16, src, ok);
    }
    cpa_wait_all();
    __syncthreads();
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      const int p0 = warp * 32 + ks * 16;
      uint32_t af[MT][4];
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
        ldsm4t(u + (p0 + av_p) * Cfg::RS + mt * 32 + av_cb, af[mt][0], af[mt][1], af[mt][2], af[mt][3]);
#pragma unroll
      for (int np = 0; np < NP; ++np) {
        uint32_t b0, b1, b2, b3;
        ldsm4t(u + (p0 + bk_p) * Cfg::RS + Cfg::TN * 2 + np * 32 + bk_cb, b0, b1, b2, b3);
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
          ptx::mma_16816(acc[mt][2 * np], af[mt], b0, b1);
          ptx::mma_16816(acc[mt][2 * np + 1], af[mt], b2, b3);
        }
      }
    }
  }
  // cross-warp sum, one 16-row slab (mt) at a time: red[8 warps][16][TK] fp32 inside the staging buffer
  float* red = reinterpret_cast<float*>(wg_smem);
  const int g = lane >> 2, t4 = lane & 3;
  float* dst = part + (long long)blockIdx.x * N * K;
#pragma unroll   // static indices: acc stays in registers
  for (int mt = 0; mt < MT; ++mt) {
    __syncthreads();
    float* mine = red + warp * 16 * Cfg::TK;
#pragma unroll
    for (int nt = 0; nt < 2 * NP; ++nt) {
      const int col = nt * 8 + t4 * 2;
      mine[g * Cfg::TK + col] = acc[mt][nt][0];
      mine[g * Cfg::TK + col + 1] = acc[mt][nt][1];
      mine[(g + 8) * Cfg::TK + col] = acc[mt][nt][2];
      mine[(g + 8) * Cfg::TK + col + 1] = acc[mt][nt][3];
    }
    __syncthreads();
    for (int i = tid; i < 16 * Cfg::TK; i += 256) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) s += red[w * 16 * Cfg::TK + i];
      const int n = n0 + mt * 16 + i / Cfg::TK, k = k0 + i % Cfg::TK;
      if (n < N && k < K) dst[(long long)n * K + k] = s;
    }
  }
}

// ------------------------------------------------------------------------------------------ depthwise conv gradients
// dx[b,iy,ix,c] = sum_{ky,kx} dz[b,oy,ox,c] w[ky*KS+kx][c] over the (oy, ox) with oy*stride + ky - pad == iy (same for x).
__global__ void dw_bwd_data_kernel(const bf16* __restrict__ dz, const float* __restrict__ w, bf16* __restrict__ dxo, int B, int H,
                                   int W, int C, int Ho, int Wo, int ks, int stride) {
  const int CV = C >> 3;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * H * W * CV) return;
  const int cv = (int)(i % CV);
  const long long p = i / CV;
  const int ix = (int)(p % W), iy = (int)((p / W) % H), b = (int)(p / ((long long)W * H));
  const int pad = ks >> 1;
  float acc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) acc[k] = 0.f;
  for (int ky = 0; ky < ks; ++ky) {
    const int ty = iy + pad - ky;
    if (ty < 0 || ty % stride) continue;
    const int oy = ty / stride;
    if (oy >= Ho) continue;
    for (int kx = 0; kx < ks; ++kx) {
      const int tx = ix + pad - kx;
      if (tx < 0 || tx % stride) continue;
      const int ox = tx / stride;
      if (ox >= Wo) continue;
      float f[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(dz + (((long long)b * Ho + oy) * Wo + ox) * C + cv * 8)), f);
      const float4 w0 = __ldg(reinterpret_cast<const float4*>(w + (long long)(ky * ks + kx) * C + cv * 8));
      const float4 w1 = __ldg(reinterpret_cast<const float4*>(w + (long long)(ky * ks + kx) * C + cv * 8 + 4));
      acc[0] = fmaf(f[0], w0.x, acc[0]); acc[1] = fmaf(f[1], w0.y, acc[1]);
      acc[2] = fmaf(f[2], w0.z, acc[2]); acc[3] = fmaf(f[3], w0.w, acc[3]);
      acc[4] = fmaf(f[4], w1.x, acc[4]); acc[5] = fmaf(f[5], w1.y, acc[5]);
      acc[6] = fmaf(f[6], w1.z, acc[6]); acc[7] = fmaf(f[7], w1.w, acc[7]);
    }
  }
  *reinterpret_cast<uint4*>(dxo + p * C + cv * 8) = pack8(acc);
}

// part[blk][tap][c] = sum over the block's output pixels of dz[p][c] * x[src(p, tap)][c].
// grid (nblk, ceil(CG / CGB)), block 256: thread = (VEC-channel group, pixel lane); VEC = 8 (one 16-byte load per operand,
// 3x3: 72 accumulators) or 4 (5x5: 100 accumulators).  x may be a channel slice (pixel stride ldx).
// (First version: 2 channels per thread, LDG.32 per tap.)
template <int VEC>
__device__ __forceinline__ void ldvec(const bf16* p, float* f) {
  if constexpr (VEC == 8) {
    unpack8(__ldg(reinterpret_cast<const uint4*>(p)), f);
  } else {
    const uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
    const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y;
  }
}

template <int KS, int VEC>
__global__ void __launch_bounds__(256) dw_wgrad_kernel(const bf16* __restrict__ dz, const bf16* __restrict__ x, long long ldx, int B,
                                                       int H, int W, int C, int Ho, int Wo, int stride, int CGB,
                                                       long long pix_per_block, float* __restrict__ part) {
  __shared__ float red[256][VEC + 1];
  constexpr int KK = KS * KS, PAD = KS / 2;
  const int tid = threadIdx.x;
  const int lanes = 256 / CGB;
  const int cgl = tid % CGB, pl = tid / CGB;
  const int cg = blockIdx.y * CGB + cgl;
  const bool active = pl < lanes && cg * VEC < C;
  float acc[KK][VEC];
#pragma unroll
  for (int t = 0; t < KK; ++t)
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[t][v] = 0.f;
  const long long total = (long long)B * Ho * Wo;
  const long long p0 = (long long)blockIdx.x * pix_per_block, p1 = min(total, p0 + pix_per_block);
  if (active) {
    for (long long p = p0 + pl; p < p1; p += lanes) {
      const int ox = (int)(p % Wo), oy = (int)((p / Wo) % Ho), b = (int)(p / ((long long)Wo * Ho));
      float g[VEC];
      ldvec<VEC>(dz + p * C + cg * VEC, g);
#pragma unroll
      for (int ky = 0; ky < KS; ++ky) {
        const int iy = oy * stride + ky - PAD;
        if (iy < 0 || iy >= H) continue;
#pragma unroll
        for (int kx = 0; kx < KS; ++kx) {
          const int ix = ox * stride + kx - PAD;
          if (ix < 0 || ix >= W) continue;
          float xv[VEC];
          ldvec<VEC>(x + (((long long)b * H + iy) * W + ix) * ldx + cg * VEC, xv);
#pragma unroll
          for (int v = 0; v < VEC; ++v) acc[ky * KS + kx][v] = fmaf(g[v], xv[v], acc[ky * KS + kx][v]);
        }
      }
    }
  }
  int top = 1;
  while (top < lanes) top <<= 1;
#pragma unroll   // static indices keep acc[][] in registers
  for (int t = 0; t < KK; ++t) {
#pragma unroll
    for (int v = 0; v < VEC; ++v) red[tid][v] = acc[t][v];
    __syncthreads();
    for (int s = top >> 1; s > 0; s >>= 1) {
      if (pl < s && pl + s < lanes) {
#pragma unroll
        for (int v = 0; v < VEC; ++v) red[tid][v] += red[tid + s * CGB][v];
      }
      __syncthreads();
    }
    if (pl == 0 && cg * VEC < C) {
      float* d = part + ((long long)blockIdx.x * KK + t) * C + cg * VEC;
#pragma unroll
      for (int v = 0; v < VEC; ++v) d[v] = red[tid][v];
    }
    __syncthreads();
  }
}

// Stride-1 version with register reuse along x: a thread owns a strip of P consecutive output pixels of one row; per kernel
// row it loads the P + KS - 1 input vectors of the strip once and every one of them feeds up to KS taps
// (loads per pixel and kernel row: (P + KS - 1) / P instead of KS -- the per-pixel kernel above is LSU-bound at
// far from the memory bound).  Work unit = (image, output row, strip); same partial-sum layout.
template <int KS, int VEC, int P>
__global__ void __launch_bounds__(256) dw_wgrad_strip_kernel(const bf16* __restrict__ dz, const bf16* __restrict__ x, long long ldx, int B,
                                                             int H, int W, int C, int CGB, long long strips_per_block,
                                                             float* __restrict__ part) {
  __shared__ float red[256][VEC + 1];
  constexpr int KK = KS * KS, PAD = KS / 2, XW = P + KS - 1;
  const int tid = threadIdx.x;
  const int lanes = 256 / CGB;
  const int cgl = tid % CGB, pl = tid / CGB;
  const int cg = blockIdx.y * CGB + cgl;
  const bool active = pl < lanes && cg * VEC < C;
  float acc[KK][VEC];
#pragma unroll
  for (int t = 0; t < KK; ++t)
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[t][v] = 0.f;
  const int spr = (W + P - 1) / P;                           // strips per row (stride 1: Ho = H, Wo = W)
  const long long total = (long long)B * H * spr;
  const long long s0 = (long long)blockIdx.x * strips_per_block, s1 = min(total, s0 + strips_per_block);
  if (active) {
    for (long long sidx = s0 + pl; sidx < s1; sidx += lanes) {
      const int xs = (int)(sidx % spr), oy = (int)((sidx / spr) % H), b = (int)(sidx / ((long long)spr * H));
      const int ox0 = xs * P;
      float g[P][VEC];
#pragma unroll
      for (int j = 0; j < P; ++j) {
        if (ox0 + j < W) {
          ldvec<VEC>(dz + (((long long)b * H + oy) * W + ox0 + j) * C + cg * VEC, g[j]);
        } else {
#pragma unroll
          for (int v = 0; v < VEC; ++v) g[j][v] = 0.f;
        }
      }
#pragma unroll
      for (int ky = 0; ky < KS; ++ky) {
        const int iy = oy + ky - PAD;
        if (iy < 0 || iy >= H) continue;
        const bf16* xrow = x + ((long long)b * H + iy) * W * ldx + cg * VEC;
        float xr[XW][VEC];
#pragma unroll
        for (int j = 0; j < XW; ++j) {
          const int ix = ox0 - PAD + j;
          if (ix >= 0 && ix < W) {
            ldvec<VEC>(xrow + (long long)ix * ldx, xr[j]);
          } else {
#pragma unroll
            for (int v = 0; v < VEC; ++v) xr[j][v] = 0.f;
          }
        }
#pragma unroll
        for (int kx = 0; kx < KS; ++kx)
#pragma unroll
          for (int j = 0; j < P; ++j)
#pragma unroll
            for (int v = 0; v < VEC; ++v) acc[ky * KS + kx][v] = fmaf(g[j][v], xr[j + kx][v], acc[ky * KS + kx][v]);
      }
    }
  }
  int top = 1;
  while (top < lanes) top <<= 1;
#pragma unroll   // static indices keep acc[][] in registers
  for (int t = 0; t < KK; ++t) {
#pragma unroll
    for (int v = 0; v < VEC; ++v) red[tid][v] = acc[t][v];
    __syncthreads();
    for (int s = top >> 1; s > 0; s >>= 1) {
      if (pl < s && pl + s < lanes) {
#pragma unroll
        for (int v = 0; v < VEC; ++v) red[tid][v] += red[tid + s * CGB][v];
      }
      __syncthreads();
    }
    if (pl == 0 && cg * VEC < C) {
      float* d = part + ((long long)blockIdx.x * KK + t) * C + cg * VEC;
#pragma unroll
      for (int v = 0; v < VEC; ++v) d[v] = red[tid][v];
    }
    __syncthreads();
  }
}

// Sliding-window version (stride 1 | 2, C % 32 == 0; the route for these shapes).  A CTA owns a 32-channel slab and walks 8 x 32
// output-pixel tiles: the dz tile and the haloed x tile are staged once with cp.async (zero fill outside the map).  A thread owns one
// channel pair and a 16-pixel run of ONE output row, keeps the KS x KS input window of the current pixel in registers (as channel-pair float2s) and slides it along x -- STRIDE new columns (KS x STRIDE shared-memory
// reads) per pixel instead of KS x KS, every multiply-add a packed FFMA2.  Per pixel and channel pair: 3x3 s1  4 LDS + 9 FFMA2 (was
// 10 LDS + 18 FFMA), 5x5 s1  6 + 25 (was 26 + 50), 3x3 s2  7 + 9.
// The two half-warps of a warp walk output rows py and py + 1: the row strides are padded so that their reads fall into opposite
// 64-byte halves of the 128-byte bank window.
constexpr int DWW_TH = 8, DWW_TW = 32, DWW_CS = 32;
constexpr int dww_pad(int rs0, int stride) {
  for (int p = 0; p < 128; p += 16)
    if ((stride * (rs0 + p)) % 128 == 64) return p;
  return 0;
}
template <int KS, int STRIDE>
struct DwwCfg {
  static constexpr int IH = (DWW_TH - 1) * STRIDE + KS, IW = (DWW_TW - 1) * STRIDE + KS;
  static constexpr int X_RS = IW * 64 + dww_pad(IW * 64, STRIDE);      // bytes per staged input row (64 B per pixel = 32 channels)
  static constexpr int DZ_RS = DWW_TW * 64 + dww_pad(DWW_TW * 64, 1);
  static constexpr int X_BYTES = IH * X_RS, DZ_BYTES = DWW_TH * DZ_RS;
  static constexpr int RED_BYTES = 8 * KS * KS * DWW_CS * 4;
  static constexpr int SMEM = (X_BYTES + DZ_BYTES > RED_BYTES) ? X_BYTES + DZ_BYTES : RED_BYTES;
  static_assert((STRIDE * X_RS) % 128 == 64 && DZ_RS % 128 == 64 && X_RS % 16 == 0, "row strides must split the half-warps across the banks");
};

template <int KS, int STRIDE>
__global__ void __launch_bounds__(256, (2 * (DwwCfg<KS, STRIDE>::SMEM + 1024) <= 227 * 1024) ? 2 : 1)
dw_wgrad_win_kernel(const bf16* __restrict__ dz, const bf16* __restrict__ x, long long ldx, int B, int H, int W, int C, int Ho, int Wo,
                    int tiles_x, int tiles_y, float* __restrict__ part) {
  using Cfg = DwwCfg<KS, STRIDE>;
  constexpr int KK = KS * KS, PAD = KS / 2;
  extern __shared__ __align__(16) uint8_t dww_smem[];
  const uint32_t u_x = static_cast<uint32_t>(__cvta_generic_to_shared(dww_smem));
  const uint32_t u_dz = u_x + Cfg::X_BYTES;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cp = lane & 15, half = lane >> 4;
  const int py = (warp >> 1) * 2 + half, x0 = (warp & 1) * 16;   // this thread's output row and first output column inside the tile
  const int c0 = blockIdx.y * DWW_CS;
  float2 acc[KK];
#pragma unroll
  for (int t = 0; t < KK; ++t) acc[t] = make_float2(0.f, 0.f);
  const long long ntiles = (long long)B * tiles_y * tiles_x;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int tx = (int)(tile % tiles_x), ty = (int)((tile / tiles_x) % tiles_y), b = (int)(tile / ((long long)tiles_x * tiles_y));
    const int oy0 = ty * DWW_TH, ox0 = tx * DWW_TW;
    __syncthreads();                                         // previous tile fully consumed
    for (int i = tid; i < Cfg::IH * Cfg::IW * 4; i += 256) {
      const int v = i & 3, pix = i >> 2;
      const int ly = pix / Cfg::IW, lx = pix - ly * Cfg::IW;
      const int iy = oy0 * STRIDE - PAD + ly, ix = ox0 * STRIDE - PAD + lx;
      const bool ok = iy >= 0 && iy < H && ix >= 0 && ix < W;
      cpa16(u_x + ly * Cfg::X_RS + lx * 64 + v * 16, ok ? x + (((long long)b * H + iy) * W + ix) * ldx + c0 + v * 8 : x, ok);
    }
    for (int i = tid; i < DWW_TH * DWW_TW * 4; i += 256) {
      const int v = i & 3, pix = i >> 2;
      const int ly = pix / DWW_TW, lx = pix % DWW_TW;
      const int oy = oy0 + ly, ox = ox0 + lx;
      const bool ok = oy < Ho && ox < Wo;
      cpa16(u_dz + ly * Cfg::DZ_RS + lx * 64 + v * 16, ok ? dz + (((long long)b * Ho + oy) * Wo + ox) * C + c0 + v * 8 : dz, ok);
    }
    cpa_wait_all();
    __syncthreads();
    const uint8_t* xrow = dww_smem + (py * STRIDE) * Cfg::X_RS + (x0 * STRIDE) * 64 + cp * 4;
    const uint8_t* grow = dww_smem + Cfg::X_BYTES + py * Cfg::DZ_RS + x0 * 64 + cp * 4;
    float2 win[KS][KS];                                      // input column c of the run lives in slot c % KS
#pragma unroll
    for (int c = 0; c < KS - STRIDE; ++c)
#pragma unroll
      for (int ky = 0; ky < KS; ++ky) win[ky][c % KS] = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(xrow + ky * Cfg::X_RS + c * 64));
#pragma unroll
    for (int px = 0; px < 16; ++px) {
#pragma unroll
      for (int n = 0; n < STRIDE; ++n) {
        const int c = px * STRIDE + KS - STRIDE + n;
#pragma unroll
        for (int ky = 0; ky < KS; ++ky) win[ky][c % KS] = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(xrow + ky * Cfg::X_RS + c * 64));
      }
      const float2 g = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(grow + px * 64));
#pragma unroll
      for (int ky = 0; ky < KS; ++ky)
#pragma unroll
        for (int kx = 0; kx < KS; ++kx) acc[ky * KS + kx] = ffma2(g, win[ky][(px * STRIDE + kx) % KS], acc[ky * KS + kx]);
    }
  }
  // the two half-warps (same channel pair, different rows), then the 8 warps through shared memory: red[warp][tap][32 channels]
#pragma unroll
  for (int t = 0; t < KK; ++t) {
    acc[t].x += __shfl_xor_sync(0xffffffffu, acc[t].x, 16);
    acc[t].y += __shfl_xor_sync(0xffffffffu, acc[t].y, 16);
  }
  __syncthreads();
  float* red = reinterpret_cast<float*>(dww_smem);
  if (half == 0) {
#pragma unroll
    for (int t = 0; t < KK; ++t) *reinterpret_cast<float2*>(red + (warp * KK + t) * DWW_CS + cp * 2) = acc[t];
  }
  __syncthreads();
  for (int i = tid; i < KK * DWW_CS; i += 256) {
    float sum = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) sum += red[w * KK * DWW_CS + i];
    const int t = i / DWW_CS, c = i % DWW_CS;
    part[((long long)blockIdx.x * KK + t) * C + c0 + c] = sum;
  }
}

// ------------------------------------------------------------------------------------------ SqueezeExcite backward (batched)
// Per-image column reductions / per-image affine of the SqueezeExcite backward in ONE launch each (the training graph's first
// version loops over the batch with es3_bn_act_bwd_reduce / es3_affine_act: ~100 launches per SE block at batch 32).
// GPU parity: tests/test_zz_train_gpu.py::test_se_bwd_batched.
//   se_dgate:  part[chunk][b][c] = sum over the chunk's pixels of dy[b][p][c] * x[b][p][c]          grid (nchunk, B), block 256
//   se_apply:  dx[b][p][c] = dy[b][p][c] * gate[b][c] + add[b][c]                                    one thread per 8-channel vector
__global__ void __launch_bounds__(256) se_dgate_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x, int HW, int C, int CVB,
                                                       int px_per_chunk, float* __restrict__ part) {
  __shared__ float red[256][9];
  const int tid = threadIdx.x, lanes = 256 / CVB;
  const int cvl = tid % CVB, pl = tid / CVB;
  const int b = blockIdx.y, B = gridDim.y;
  const int p0 = blockIdx.x * px_per_chunk, p1 = min(HW, p0 + px_per_chunk);
  for (int cv0 = 0; cv0 * 8 < C; cv0 += CVB) {              // C > 2048: several passes over the chunk
    const int cv = cv0 + cvl;
    float s[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i] = 0.f;
    if (pl < lanes && cv * 8 < C) {
      for (int p = p0 + pl; p < p1; p += lanes) {
        const long long off = ((long long)b * HW + p) * C + cv * 8;
        float a[8], v[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(dy + off)), a);
        unpack8(__ldg(reinterpret_cast<const uint4*>(x + off)), v);
#pragma unroll
        for (int i = 0; i < 8; ++i) s[i] = fmaf(a[i], v[i], s[i]);
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) red[tid][i] = s[i];
    __syncthreads();
    int top = 1;
    while (top < lanes) top <<= 1;
    for (int st = top >> 1; st > 0; st >>= 1) {
      if (pl < st && pl + st < lanes) {
#pragma unroll
        for (int i = 0; i < 8; ++i) red[tid][i] += red[tid + st * CVB][i];
      }
      __syncthreads();
    }
    if (pl == 0 && cv * 8 < C) {
      float* d = part + ((long long)blockIdx.x * B + b) * C + cv * 8;
#pragma unroll
      for (int i = 0; i < 8; ++i) d[i] = red[tid][i];
    }
    __syncthreads();
  }
}

__global__ void se_apply_kernel(const bf16* __restrict__ dy, const float* __restrict__ gate, const float* __restrict__ add,
                                bf16* __restrict__ dx, int HW, int CV, long long total_vec) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total_vec) return;
  const int cv = (int)(i % CV);
  const int b = (int)(i / ((long long)CV * HW));
  const int C = CV * 8;
  float f[8], g[8], a[8];
  unpack8(__ldg(reinterpret_cast<const uint4*>(dy) + i), f);
  load8f(gate + (long long)b * C + cv * 8, g, 1.f);
  load8f(add + (long long)b * C + cv * 8, a, 0.f);
#pragma unroll
  for (int k = 0; k < 8; ++k) f[k] = fmaf(f[k], g[k], a[k]);
  reinterpret_cast<uint4*>(dx)[i] = pack8(f);
}

// ------------------------------------------------------------------------------------------ stem conv weight gradient
// img [B,3,H,W] fp32 NCHW; dz [B,Ho,Wo,COUT] bf16 (3x3, stride 2, pad 1).  part[blk][n][27] with 27 = ci*9 + ky*3 + kx.
// 128-pixel chunks staged in shared memory: dz rows as fp32 and the 27-tap patches (28th column = 0).  A compute thread owns a
// (channel pair, tap pair): per pixel two 8-byte broadcast reads feed four FMAs (round 1: one thread per weight, two 4-byte reads per
// FMA, the patch gather paid a div / mod chain per ELEMENT and the block synchronised every 64 pixels).  The
// gather now resolves (b, oy, ox) once per (pixel, input channel) and reads that channel's 3 x 3 window.
constexpr int SW_PX = 128, SW_MAXC = 32;
__global__ void __launch_bounds__(256) stem_wgrad_kernel(const float* __restrict__ img, const bf16* __restrict__ dz, int B, int H, int W,
                                                         int Ho, int Wo, int COUT, int chunks_per_block, float* __restrict__ part) {
  __shared__ __align__(16) float s_dz[SW_PX][SW_MAXC + 2];
  __shared__ __align__(16) float s_patch[SW_PX][28];
  const int tid = threadIdx.x;
  const int npair = COUT >> 1;                       // COUT is even (checked on the host)
  const int n2 = tid / 14, tp = tid % 14;
  const bool owner = n2 < npair;
  const long long total = (long long)B * Ho * Wo;
  float a00 = 0.f, a01 = 0.f, a10 = 0.f, a11 = 0.f;   // [channel 2 n2 + i][tap 2 tp + j]
  for (int ch = 0; ch < chunks_per_block; ++ch) {
    const long long p0 = ((long long)blockIdx.x * chunks_per_block + ch) * SW_PX;
    if (p0 >= total) break;
    __syncthreads();
    for (int i = tid; i < SW_PX * (COUT / 8); i += 256) {
      const int pp = i / (COUT / 8), v = i % (COUT / 8);
      const long long p = p0 + pp;
      float f[8];
      if (p < total) unpack8(__ldg(reinterpret_cast<const uint4*>(dz + p * COUT) + v), f);
      else {
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = 0.f;
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) s_dz[pp][v * 8 + e] = f[e];
    }
    for (int i = tid; i < SW_PX * 3; i += 256) {
      const int pp = i % SW_PX, ci = i / SW_PX;
      const long long p = p0 + pp;
      float v[9];
#pragma unroll
      for (int k = 0; k < 9; ++k) v[k] = 0.f;
      if (p < total) {
        const int ox = (int)(p % Wo), oy = (int)((p / Wo) % Ho), b = (int)(p / ((long long)Wo * Ho));
        const float* plane = img + ((long long)b * 3 + ci) * H * W;
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
          const int iy = oy * 2 - 1 + ky;
          if (iy < 0 || iy >= H) continue;
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) {
            const int ix = ox * 2 - 1 + kx;
            if (ix >= 0 && ix < W) v[ky * 3 + kx] = __ldg(plane + (long long)iy * W + ix);
          }
        }
      }
#pragma unroll
      for (int k = 0; k < 9; ++k) s_patch[pp][ci * 9 + k] = v[k];
      if (ci == 0) s_patch[pp][27] = 0.f;
    }
    __syncthreads();
    if (owner) {
#pragma unroll 8
      for (int pp = 0; pp < SW_PX; ++pp) {
        const float2 d = *reinterpret_cast<const float2*>(&s_dz[pp][2 * n2]);
        const float2 t = *reinterpret_cast<const float2*>(&s_patch[pp][2 * tp]);
        a00 = fmaf(d.x, t.x, a00); a01 = fmaf(d.x, t.y, a01);
        a10 = fmaf(d.y, t.x, a10); a11 = fmaf(d.y, t.y, a11);
      }
    }
  }
  if (owner) {
    float* o = part + (long long)blockIdx.x * COUT * 27;
    o[(2 * n2) * 27 + 2 * tp] = a00;
    o[(2 * n2 + 1) * 27 + 2 * tp] = a10;
    if (2 * tp + 1 < 27) {
      o[(2 * n2) * 27 + 2 * tp + 1] = a01;
      o[(2 * n2 + 1) * 27 + 2 * tp + 1] = a11;
    }
  }
}

// ------------------------------------------------------------------------------------------ padded transpose
// in [B,H,W,C] bf16 NHWC -> out [C][Mp] bf16, Mp = B * (H+2) * Wp (Wp >= W + 2, multiple of 8):
//   out[c][(b (H+2) + y + 1) Wp + x + 1 - dx] = in[b,y,x,c], zero everywhere else (the caller clears `out`).
// With the zero frame around every image a 3x3 tap becomes a pure column offset of the transposed operand, so the
// weight gradient of a dense 3x3 conv is nine tensor-core GEMMs over the pixel index: dW[ky][kx] = dYp^T[:, P] . Ap_dx^T[:, P + (ky-1) Wp]
// (dx = kx - 1 is baked into the copy so that every TMA base address stays 16-byte aligned).
// grid (ceil(C / 64), H, B), block 256: 32-pixel x 64-channel tiles through shared memory.
__global__ void __launch_bounds__(256) transpose_pad_kernel(const bf16* __restrict__ in, bf16* __restrict__ out, int H, int W, int C,
                                                            int Wp, int dx, long long Mp) {
  __shared__ __align__(16) bf16 tile[32][72];
  const int c0 = blockIdx.x * 64, y = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x;
  const long long prow = ((long long)b * (H + 2) + y + 1) * Wp + 1 - dx;   // column of pixel x = 0
  for (int x0 = 0; x0 < W; x0 += 32) {
    __syncthreads();
    {
      const int xl = tid >> 3, v = tid & 7;
      uint4 u = make_uint4(0, 0, 0, 0);
      if (x0 + xl < W && c0 + v * 8 < C)
        u = __ldg(reinterpret_cast<const uint4*>(in + (((long long)b * H + y) * W + x0 + xl) * C + c0 + v * 8));
      *reinterpret_cast<uint4*>(&tile[xl][v * 8]) = u;
    }
    __syncthreads();
    const int c = tid >> 2, part = tid & 3;
    if (c0 + c < C) {
      bf16* dst = out + (long long)(c0 + c) * Mp + prow + x0 + part * 8;
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (x0 + part * 8 + i < W) dst[i] = tile[part * 8 + i][c];
    }
  }
}

// ------------------------------------------------------------------------------------------ bilinear adjoint
// dout [B,C,Ho,Wo] fp32 NCHW -> din [B,Hi,Wi,C] bf16 NHWC, adjoint of bilinear_nhwc_to_nchw_kernel (same source-index
// arithmetic).  grid (C/32, Hi, B), block 256: 32 channels x one input row; the result goes through shared memory so
// the NHWC store is 64-byte contiguous per pixel.
constexpr int BB_CB = 32, BB_MAXT = 12;    // channels per block; candidate outputs per input pixel and axis (up-scaling by <= 4)
__global__ void __launch_bounds__(256) bilinear_bwd_kernel(const float* __restrict__ dout, bf16* __restrict__ din, int Hi, int Wi, int C,
                                                           int Ho, int Wo, float sy, float sx) {
  extern __shared__ float bb_tile[];   // [Wi][BB_CB + 1] | wx table [Wi][BB_MAXT] | ox0 [Wi] | wy [BB_MAXT]
  float* s_wx = bb_tile + Wi * (BB_CB + 1);
  int* s_ox0 = reinterpret_cast<int*>(s_wx + Wi * BB_MAXT);
  float* s_wy = reinterpret_cast<float*>(s_ox0 + Wi);
  const int c0 = blockIdx.x * BB_CB, iy = blockIdx.y, b = blockIdx.z;
  // candidate output rows: every oy whose source interval [y0, y1] can contain iy
  int oy_lo = (int)floorf(((float)iy - 1.f + 0.5f) / sy - 0.5f) - 1;
  int oy_hi = (int)ceilf(((float)iy + 1.f + 0.5f) / sy - 0.5f) + 1;
  oy_lo = max(oy_lo, 0);
  oy_hi = min(oy_hi, Ho - 1);
  if (oy_hi - oy_lo + 1 > BB_MAXT) oy_hi = oy_lo + BB_MAXT - 1;      // (host checks the scale: never taken)
  // The interpolation weights depend on (iy, oy) and (ix, ox) only -- not on the channel: they are built once per block (round 1
  // recomputed floorf / ceilf / the clamped source index for every (channel, ix, oy, ox) candidate).
  for (int t = threadIdx.x; t <= oy_hi - oy_lo; t += 256) {
    const int oy = oy_lo + t;
    float fy = (oy + 0.5f) * sy - 0.5f;
    if (fy < 0.f) fy = 0.f;
    const int y0 = min((int)fy, Hi - 1), y1 = min(y0 + 1, Hi - 1);
    const float ly = fy - (float)y0, hy = 1.f - ly;
    s_wy[t] = (y0 == iy ? hy : 0.f) + (y1 == iy ? ly : 0.f);
  }
  for (int ix = threadIdx.x; ix < Wi; ix += 256) {
    int ox_lo = (int)floorf(((float)ix - 1.f + 0.5f) / sx - 0.5f) - 1;
    int ox_hi = (int)ceilf(((float)ix + 1.f + 0.5f) / sx - 0.5f) + 1;
    ox_lo = max(ox_lo, 0);
    ox_hi = min(ox_hi, Wo - 1);
    s_ox0[ix] = ox_lo;
    for (int t = 0; t < BB_MAXT; ++t) {
      const int ox = ox_lo + t;
      float wx = 0.f;
      if (ox <= ox_hi) {
        float fx = (ox + 0.5f) * sx - 0.5f;
        if (fx < 0.f) fx = 0.f;
        const int x0 = min((int)fx, Wi - 1), x1 = min(x0 + 1, Wi - 1);
        const float lx = fx - (float)x0, hx = 1.f - lx;
        wx = (x0 == ix ? hx : 0.f) + (x1 == ix ? lx : 0.f);
      }
      s_wx[ix * BB_MAXT + t] = wx;
    }
  }
  __syncthreads();
  const int ny = oy_hi - oy_lo + 1;
  for (int idx = threadIdx.x; idx < BB_CB * Wi; idx += 256) {
    const int ix = idx % Wi, cl = idx / Wi;
    const int c = c0 + cl;
    float acc = 0.f;
    if (c < C) {
      const int ox_lo = s_ox0[ix];
      const float* plane = dout + ((long long)b * C + c) * Ho * Wo;
      for (int t = 0; t < ny; ++t) {
        const float wy = s_wy[t];
        if (wy == 0.f) continue;
        const float* rowp = plane + (long long)(oy_lo + t) * Wo + ox_lo;
        float ra = 0.f;
#pragma unroll
        for (int u = 0; u < BB_MAXT; ++u) {
          const float wx = s_wx[ix * BB_MAXT + u];
          if (wx != 0.f) ra = fmaf(wx, __ldg(rowp + u), ra);       // wx == 0 also covers ox beyond the row
        }
        acc = fmaf(wy, ra, acc);
      }
    }
    bb_tile[ix * (BB_CB + 1) + cl] = acc;
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < BB_CB * Wi; idx += 256) {
    const int cl = idx % BB_CB, ix = idx / BB_CB;
    if (c0 + cl < C) din[(((long long)b * Hi + iy) * Wi + ix) * C + c0 + cl] = __float2bfloat16(bb_tile[ix * (BB_CB + 1) + cl]);
  }
}

// ------------------------------------------------------------------------------------------ LiteMLA attention backward
// Forward (ops.py:592-621, head dim 16): q' = relu(q), k' = relu(k), vpad = [v, 1]; KV[j][i] = sum_n vpad[n][j] k'[n][i]
// (17 x 16); o[n][j] = sum_i KV[j][i] q'[n][i]; y[n][j] = o[n][j] / (o[n][16] + eps), j < 16.
// Backward, with r = 1 / (o16 + eps):   do[j] = dy[j] r (j < 16),  do[16] = -r sum_j dy[j] y[j]
//   dKV[j][i] = sum_n do[n][j] q'[n][i];  dq'[i] = sum_j KV[j][i] do[j];  dv[j] = sum_i dKV[j][i] k'[i];
//   dk'[i] = sum_j vpad[j] dKV[j][i];  dq = dq' [q > 0], dk = dk' [k > 0].
// ms [B][HW][ld] bf16 with head h at channels [48 h, 48 h + 48) = q | k | v; dy [B][HW][lddy] bf16, head h at [16 h, +16).
constexpr int LB_PX = 128;

__device__ __forceinline__ void load16(const bf16* p, float* f) {
  unpack8(__ldg(reinterpret_cast<const uint4*>(p)), f);
  unpack8(__ldg(reinterpret_cast<const uint4*>(p) + 1), f + 8);
}

// The partial KV / dKV sums are reduced ONCE per (image, head) by this kernel (fixed chunk order); round 1 had every CTA of the two
// kernels below re-sum all chunks from global memory (43 KB of L2 reads per CTA, 0.7 GB per launch at stage 3).
__global__ void __launch_bounds__(288) litemla_sum_partials_kernel(const float* __restrict__ src, int nchunk, float* __restrict__ dst) {
  const int i = threadIdx.x;
  if (i >= 17 * 16) return;
  const float* p = src + (long long)blockIdx.x * nchunk * 17 * 16 + i;
  float a = 0.f;
  for (int c = 0; c < nchunk; ++c) a += p[(long long)c * 17 * 16];
  dst[(long long)blockIdx.x * 17 * 16 + i] = a;
}

__device__ __forceinline__ void load_kv_sum(const float* __restrict__ src, float* s_dst, int tid, int nthr) {
  for (int i = tid; i < 17 * 16; i += nthr) s_dst[i] = src[i];
}

// do[0..16] for one token from q' (fp32, already relu'd), dy and KV
__device__ __forceinline__ void token_do(const float* skv, const float* q, const float* dy, float eps, float* dof) {
  float o[17];
#pragma unroll
  for (int j = 0; j < 17; ++j) {
    float a = 0.f;
#pragma unroll
    for (int i4 = 0; i4 < 4; ++i4) {       // warp-uniform 16-byte reads: one LDS.128 broadcast per four FMAs
      const float4 w = *reinterpret_cast<const float4*>(skv + j * 16 + i4 * 4);
      a = fmaf(w.x, q[i4 * 4], a); a = fmaf(w.y, q[i4 * 4 + 1], a); a = fmaf(w.z, q[i4 * 4 + 2], a); a = fmaf(w.w, q[i4 * 4 + 3], a);
    }
    o[j] = a;
  }
  const float r = 1.f / (o[16] + eps);
  float dot = 0.f;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    dof[j] = dy[j] * r;
    dot = fmaf(dy[j], o[j] * r, dot);
  }
  dof[16] = -r * dot;
}

// grid (ceil(HW / 128), heads2, B), block 288.  dkv_part [B][heads2][nchunk_b][17][16].
__global__ void __launch_bounds__(288) litemla_dkv_kernel(const bf16* __restrict__ ms, long long ld, const bf16* __restrict__ dy,
                                                          long long lddy, const float* __restrict__ kv_part, int nchunk_f,
                                                          float* __restrict__ dkv_part, int HW, float eps) {
  __shared__ __align__(16) float skv[17 * 16];
  __shared__ float s_q[LB_PX][17];
  __shared__ float s_do[LB_PX][17];
  const int tid = threadIdx.x;
  const int h = blockIdx.y, b = blockIdx.z, heads2 = gridDim.y;
  load_kv_sum(kv_part + ((long long)b * heads2 + h) * 17 * 16, skv, tid, 288);       // kv_part: already summed over the chunks
  (void)nchunk_f;
  __syncthreads();
  if (tid < LB_PX) {
    const int n = blockIdx.x * LB_PX + tid;
    float q[16], dyv[16], dof[17];
    if (n < HW) {
      load16(ms + ((long long)b * HW + n) * ld + h * 48, q);
      load16(dy + ((long long)b * HW + n) * lddy + h * 16, dyv);
#pragma unroll
      for (int i = 0; i < 16; ++i) q[i] = fmaxf(q[i], 0.f);
      token_do(skv, q, dyv, eps, dof);
    } else {
#pragma unroll
      for (int i = 0; i < 16; ++i) q[i] = 0.f;
#pragma unroll
      for (int j = 0; j < 17; ++j) dof[j] = 0.f;
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) s_q[tid][i] = q[i];
#pragma unroll
    for (int j = 0; j < 17; ++j) s_do[tid][j] = dof[j];
  }
  __syncthreads();
  if (tid < 17 * 16) {
    const int j = tid >> 4, i = tid & 15;
    float a = 0.f;
#pragma unroll 8
    for (int n = 0; n < LB_PX; ++n) a = fmaf(s_do[n][j], s_q[n][i], a);
    dkv_part[(((long long)b * heads2 + h) * gridDim.x + blockIdx.x) * 17 * 16 + tid] = a;
  }
}

// grid (ceil(HW / 128), heads2, B), block 128: thread = token.  dms [B][HW][ld] bf16 (same layout as ms).
__global__ void __launch_bounds__(128) litemla_dqkv_kernel(const bf16* __restrict__ ms, long long ld, const bf16* __restrict__ dy,
                                                           long long lddy, const float* __restrict__ kv_part, int nchunk_f,
                                                           const float* __restrict__ dkv_part, int nchunk_b, bf16* __restrict__ dms,
                                                           long long lddms, int HW, float eps) {
  __shared__ __align__(16) float skv[17 * 16];      // KV [j][i]
  __shared__ __align__(16) float sdkv[17 * 16];     // dKV [j][i]
  __shared__ __align__(16) float skvT[16 * 20];     // KV^T [i][j], j padded 17 -> 20
  __shared__ __align__(16) float sdkvT[16 * 20];    // dKV^T [i][j]
  const int tid = threadIdx.x;
  const int h = blockIdx.y, b = blockIdx.z, heads2 = gridDim.y;
  load_kv_sum(kv_part + ((long long)b * heads2 + h) * 17 * 16, skv, tid, 128);       // both already summed over their chunks
  load_kv_sum(dkv_part + ((long long)b * heads2 + h) * 17 * 16, sdkv, tid, 128);
  (void)nchunk_f; (void)nchunk_b;
  __syncthreads();
  for (int t = tid; t < 16 * 20; t += 128) {
    const int i = t / 20, j = t % 20;
    skvT[t] = j < 17 ? skv[j * 16 + i] : 0.f;
    sdkvT[t] = j < 17 ? sdkv[j * 16 + i] : 0.f;
  }
  __syncthreads();
  const int n = blockIdx.x * LB_PX + tid;
  if (n >= HW) return;
  const bf16* row = ms + ((long long)b * HW + n) * ld + h * 48;
  float q[16], k[16], v[20], dyv[16], dof[20], qr[16];
  load16(row, q);
  load16(row + 16, k);
  load16(row + 32, v);
  v[16] = 1.f; v[17] = v[18] = v[19] = 0.f;          // vpad = [v, 1] (+ zero pad to a multiple of 4)
  load16(dy + ((long long)b * HW + n) * lddy + h * 16, dyv);
#pragma unroll
  for (int i = 0; i < 16; ++i) qr[i] = fmaxf(q[i], 0.f);
  token_do(skv, qr, dyv, eps, dof);
  dof[17] = dof[18] = dof[19] = 0.f;
  float dq[16], dk[16], dv[16];
  // every shared-memory operand below is one warp-uniform LDS.128 per four FMAs (round 1: one LDS.32 per FMA)
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    float a = 0.f, c = 0.f;
#pragma unroll
    for (int j4 = 0; j4 < 5; ++j4) {
      const float4 w = *reinterpret_cast<const float4*>(skvT + i * 20 + j4 * 4);
      const float4 d = *reinterpret_cast<const float4*>(sdkvT + i * 20 + j4 * 4);
      a = fmaf(w.x, dof[j4 * 4], a); a = fmaf(w.y, dof[j4 * 4 + 1], a); a = fmaf(w.z, dof[j4 * 4 + 2], a); a = fmaf(w.w, dof[j4 * 4 + 3], a);
      c = fmaf(d.x, v[j4 * 4], c); c = fmaf(d.y, v[j4 * 4 + 1], c); c = fmaf(d.z, v[j4 * 4 + 2], c); c = fmaf(d.w, v[j4 * 4 + 3], c);
    }
    dq[i] = q[i] > 0.f ? a : 0.f;
    dk[i] = k[i] > 0.f ? c : 0.f;
  }
  float kr[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) kr[i] = fmaxf(k[i], 0.f);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    float a = 0.f;
#pragma unroll
    for (int i4 = 0; i4 < 4; ++i4) {
      const float4 d = *reinterpret_cast<const float4*>(sdkv + j * 16 + i4 * 4);
      a = fmaf(d.x, kr[i4 * 4], a); a = fmaf(d.y, kr[i4 * 4 + 1], a); a = fmaf(d.z, kr[i4 * 4 + 2], a); a = fmaf(d.w, kr[i4 * 4 + 3], a);
    }
    dv[j] = a;
  }
  uint4* o = reinterpret_cast<uint4*>(dms + ((long long)b * HW + n) * lddms + h * 48);
  o[0] = pack8(dq); o[1] = pack8(dq + 8);
  o[2] = pack8(dk); o[3] = pack8(dk + 8);
  o[4] = pack8(dv); o[5] = pack8(dv + 8);
}

static int pick_blocks(long long rows, int lanes, int max_blocks) {
  // enough blocks to fill the GPU, but at least ~16 rows per lane and block.  (64 rows per lane made every deep-stage reduction a
  // 32-iteration dependent load chain on 8..128 CTAs.)
  long long want = (rows + (long long)lanes * 16 - 1) / ((long long)lanes * 16);
  if (want < 1) want = 1;
  if (want > max_blocks) want = max_blocks;
  return (int)want;
}

}  // namespace
}  // namespace es3

using namespace es3;

// ------------------------------------------------------------------------------------------ C ABI
extern "C" long long es3_col_reduce_ws_floats(long long M, int C) {
  const int CV = C / 8, CVB = CV < CR_THREADS ? CV : CR_THREADS;
  const int nblk = pick_blocks(M, CR_THREADS / (CVB > 0 ? CVB : 1), 1184);
  return (long long)nblk * 2 * C;
}

static int col_reduce_geometry(long long M, int C, int* CVB, int* nblk, long long* rpb, int* gy) {
  const int CV = C / 8;
  *CVB = CV < CR_THREADS ? CV : CR_THREADS;
  *nblk = pick_blocks(M, CR_THREADS / *CVB, 1184);
  *rpb = (M + *nblk - 1) / *nblk;
  *gy = (CV + *CVB - 1) / *CVB;
  return 0;
}

// elementwise passes: up to 16 CTAs per SM worth of blocks, at least 8 rows per lane
static int elementwise_geometry(long long M, int C, int* CVB, int* nblk, long long* rpb, int* gy) {
  const int CV = C / 8;
  *CVB = CV < 256 ? CV : 256;
  const int lanes = 256 / *CVB;
  long long want = (M + (long long)lanes * 8 - 1) / ((long long)lanes * 8);
  if (want < 1) want = 1;
  if (want > 132 * 16) want = 132 * 16;
  *nblk = (int)want;
  *rpb = (M + *nblk - 1) / *nblk;
  *gy = (CV + *CVB - 1) / *CVB;
  return 0;
}

int es3::col_reduce_partials(bool stats, int act, const void* z, const void* da, const float* scale, const float* shift,
                              long long M, int C, float* ws, int* nblk_out, cudaStream_t st) {
  int CVB, nblk, gy;
  long long rpb;
  col_reduce_geometry(M, C, &CVB, &nblk, &rpb, &gy);
  *nblk_out = nblk;
  if (stats) {
    constexpr int RING = CRR_STAGES * 1 * CR_THREADS * 16;
    col_reduce_ring_kernel<ACT_NONE, true><<<dim3(nblk, gy), CR_THREADS, RING, st>>>((const bf16*)z, nullptr, nullptr, nullptr, M, C, CVB, rpb, ws);
    ES3_LAUNCH_CHECK("col_reduce_ring_kernel<stats>");
    return 0;
  }
  ES3_DISPATCH_ACT_BWD(act, A, {
    constexpr int RING = CRR_STAGES * 2 * CR_THREADS * 16;                       // 48 KB: needs the opt-in above the default 48 KB with `red`
    static bool configured = false;
    if (!configured) {
      ES3_CHECK_CUDA(cudaFuncSetAttribute(col_reduce_ring_kernel<A, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, RING));
      configured = true;
    }
    col_reduce_ring_kernel<A, false><<<dim3(nblk, gy), CR_THREADS, RING, st>>>((const bf16*)z, (const bf16*)da, scale, shift, M, C, CVB, rpb, ws);
  })
  ES3_LAUNCH_CHECK("col_reduce_ring_kernel<bwd>");
  return 0;
}

extern "C" int es3_bn_stats(const void* z, long long M, int C, float eps, float momentum, const float* gamma, const float* beta,
                            float* ws, float* mean, float* invstd, float* scale, float* shift, float* running_mean,
                            float* running_var, long long* num_batches_tracked, void* stream) {
  ES3_REQUIRE(M > 0 && C > 0 && C % 8 == 0, "es3_bn_stats: need M > 0 and C %% 8 == 0 (M=%lld C=%d)", M, C);
  ES3_REQUIRE(((uintptr_t)z & 15) == 0, "es3_bn_stats: z must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  int nblk;
  const int rc = col_reduce_partials(true, ACT_NONE, z, nullptr, nullptr, nullptr, M, C, ws, &nblk, st);
  if (rc) return rc;
  bn_stats_finalize_kernel<<<ceil_div(C, 8), 256, 0, st>>>((const bf16*)z, ws, nblk, C, M, eps, momentum, gamma, beta, mean, invstd, scale, shift,
                                                            running_mean, running_var, num_batches_tracked);
  ES3_LAUNCH_CHECK("bn_stats_finalize_kernel");
  return 0;
}

extern "C" int es3_affine_act(const void* z, const float* scale, const float* shift, int act, const void* residual, void* out,
                              long long M, int C, void* stream) {
  ES3_REQUIRE(M > 0 && C % 8 == 0, "es3_affine_act: need C %% 8 == 0 (C=%d)", C);
  int CVB, nblk, gy;
  long long rpb;
  elementwise_geometry(M, C, &CVB, &nblk, &rpb, &gy);
  cudaStream_t st = (cudaStream_t)stream;
  ES3_DISPATCH_ACT(act, A, {
    affine_act_kernel<A><<<dim3(nblk, gy), 256, 0, st>>>((const bf16*)z, scale, shift, (const bf16*)residual, (bf16*)out, M, C, CVB, rpb);
  })
  ES3_LAUNCH_CHECK("affine_act_kernel");
  return 0;
}

extern "C" int es3_bn_act_bwd_reduce(const void* da, const void* z, const float* scale, const float* shift, int act, int mode,
                                     const float* mean, const float* invstd, long long M, int C, float* ws, float* coef,
                                     float* dgamma, float* dbeta, void* stream) {
  ES3_REQUIRE(M > 0 && C > 0 && C % 8 == 0, "es3_bn_act_bwd_reduce: need C %% 8 == 0 (C=%d)", C);
  ES3_REQUIRE(mode >= 0 && mode <= 2, "es3_bn_act_bwd_reduce: mode %d", mode);
  ES3_REQUIRE(mode == 0 || (mean && invstd), "es3_bn_act_bwd_reduce: BN modes need mean / invstd");
  cudaStream_t st = (cudaStream_t)stream;
  int nblk;
  const int rc = col_reduce_partials(false, act, z, da, scale, shift, M, C, ws, &nblk, st);
  if (rc) return rc;
  bn_bwd_finalize_kernel<<<ceil_div(C, 8), 256, 0, st>>>(ws, nblk, C, M, mode, scale, mean, invstd, coef, dgamma, dbeta);
  ES3_LAUNCH_CHECK("bn_bwd_finalize_kernel");
  return 0;
}

extern "C" int es3_bn_act_bwd_apply(const void* da, const void* z, const float* scale, const float* shift, int act,
                                    const float* coef, void* dz, long long M, int C, void* stream) {
  ES3_REQUIRE(M > 0 && C % 8 == 0, "es3_bn_act_bwd_apply: need C %% 8 == 0 (C=%d)", C);
  int CVB, nblk, gy;
  long long rpb;
  elementwise_geometry(M, C, &CVB, &nblk, &rpb, &gy);
  cudaStream_t st = (cudaStream_t)stream;
  ES3_DISPATCH_ACT_BWD(act, A, {
    bn_act_bwd_apply_kernel<A><<<dim3(nblk, gy), 256, 0, st>>>((const bf16*)da, (const bf16*)z, scale, shift, coef, (bf16*)dz, M, C, CVB, rpb);
  })
  ES3_LAUNCH_CHECK("bn_act_bwd_apply_kernel");
  return 0;
}

extern "C" int es3_add_bf16(const void* a, long long lda, const void* b, long long ldb, void* out, long long ldo, long long M, int C,
                            void* stream) {
  ES3_REQUIRE(M > 0 && C % 8 == 0 && lda % 8 == 0 && ldb % 8 == 0 && ldo % 8 == 0, "es3_add_bf16: C / strides must be multiples of 8");
  const long long total = M * (C / 8);
  add_bf16_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)a, lda, (const bf16*)b, ldb, (bf16*)out,
                                                                                    ldo, M, C / 8);
  ES3_LAUNCH_CHECK("add_bf16_kernel");
  return 0;
}

static int wg_pick(int c) { return c <= 16 ? 1 : (c <= 32 ? 2 : 4); }

static int wgrad_splits(long long M, int N, int K) {
  const int mt = wg_pick(N), np = wg_pick(K);
  const long long nchunks = (M + WG_ROWS - 1) / WG_ROWS;
  const long long tiles = (long long)ceil_div(N, mt * 16) * ceil_div(K, np * 16);
  const long long target = (mt + np <= 3) ? 4 * 132 : 2 * 132;      // light CTAs: several per SM
  long long s = (target + tiles - 1) / tiles;
  if (s > nchunks) s = nchunks;
  if (s < 1) s = 1;
  return (int)s;
}

extern "C" long long es3_wgrad_pw_ws_floats(long long M, int N, int K) { return (long long)wgrad_splits(M, N, K) * N * K; }

template <int MT, int NP>
static int wgrad_launch(const bf16* dz, long long lddz, const bf16* x, long long ldx, long long M, int N, int K, int H, int W, int dy,
                        int dx, float* ws, int splits, cudaStream_t st) {
  using Cfg = WgCfg<MT, NP>;
  static bool configured = false;
  if (!configured) {
    ES3_CHECK_CUDA(cudaFuncSetAttribute(wgrad_pw_kernel<MT, NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM));
    configured = true;
  }
  wgrad_pw_kernel<MT, NP><<<dim3(splits, ceil_div(N, Cfg::TN), ceil_div(K, Cfg::TK)), 256, Cfg::SMEM, st>>>(dz, lddz, x, ldx, M, N, K, H, W,
                                                                                                          dy, dx, ws);
  ES3_LAUNCH_CHECK("wgrad_pw_kernel");
  return 0;
}

/* dW[n * ldn + k * ldk] += sum_m dz[m][n] * x[shift(m)][k] */
extern "C" int es3_wgrad_pw(const void* dz, long long lddz, const void* x, long long ldx, long long M, int N, int K, int H, int W,
                            int dy, int dx, float* ws, float* dW, long long ldn, long long ldk, void* stream) {
  ES3_REQUIRE(M > 0 && N % 8 == 0 && K % 8 == 0 && lddz % 8 == 0 && ldx % 8 == 0, "es3_wgrad_pw: N/K/strides must be multiples of 8 (N=%d K=%d)", N, K);
  ES3_REQUIRE(((uintptr_t)dz & 15) == 0 && ((uintptr_t)x & 15) == 0, "es3_wgrad_pw: operands must be 16-byte aligned");
  ES3_REQUIRE((H == 0 && dy == 0 && dx == 0) || (H > 0 && W > 0 && M % ((long long)H * W) == 0), "es3_wgrad_pw: bad shift geometry");
  const int splits = wgrad_splits(M, N, K);
  cudaStream_t st = (cudaStream_t)stream;
  const bf16* a = (const bf16*)dz;
  const bf16* b = (const bf16*)x;
  const int mt = wg_pick(N), np = wg_pick(K);
  int rc = 1;
#define ES3_WG(MT_, NP_) if (mt == MT_ && np == NP_) rc = wgrad_launch<MT_, NP_>(a, lddz, b, ldx, M, N, K, H, W, dy, dx, ws, splits, st)
  ES3_WG(1, 1); ES3_WG(1, 2); ES3_WG(1, 4); ES3_WG(2, 1); ES3_WG(2, 2); ES3_WG(2, 4); ES3_WG(4, 1); ES3_WG(4, 2); ES3_WG(4, 4);
#undef ES3_WG
  if (rc != 0) return rc;
  const long long n = (long long)N * K;
  sum_partials_kernel<<<(unsigned)ceil_div(n, 32), 256, 0, st>>>(ws, splits, n, K, ldn, ldk, dW);
  ES3_LAUNCH_CHECK("sum_partials_kernel");
  return 0;
}

// 3x3, stride 2 (the stage openers: 4 launches, 2 GB of dx per EV-M step): one thread per 2 x 2 block of input pixels and 8 channels.
// With z(oy,ox) = sum w[ky][kx] x(2 oy - 1 + ky, 2 ox - 1 + kx) the block (2m + a, 2n + b) reads only dz(m..m+1, n..n+1):
//   dx(2m  ,2n  ) = w11 dz00                      dx(2m  ,2n+1) = w12 dz00 + w10 dz01
//   dx(2m+1,2n  ) = w21 dz00 + w01 dz10           dx(2m+1,2n+1) = w22 dz00 + w20 dz01 + w02 dz10 + w00 dz11
// four 16-byte loads and four 16-byte stores per thread (the generic kernel above walked nine taps with a modulo test per tap and
// re-read the weights from global memory for every tap).
__global__ void __launch_bounds__(256) dw_bwd_data_s2k3_kernel(const bf16* __restrict__ dz, const float* __restrict__ w,
                                                               bf16* __restrict__ dxo, int B, int H, int W, int C, int Ho, int Wo) {
  const int CV = C >> 3;
  const int Hb = (H + 1) >> 1, Wb = (W + 1) >> 1;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * Hb * Wb * CV) return;
  const int cv = (int)(i % CV);
  const long long p = i / CV;
  const int n = (int)(p % Wb), m = (int)((p / Wb) % Hb), b = (int)(p / ((long long)Wb * Hb));
  float d[4][8];
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int oy = m + (t >> 1), ox = n + (t & 1);
    if (oy < Ho && ox < Wo) unpack8(__ldg(reinterpret_cast<const uint4*>(dz + (((long long)b * Ho + oy) * Wo + ox) * C + cv * 8)), d[t]);
    else {
#pragma unroll
      for (int e = 0; e < 8; ++e) d[t][e] = 0.f;
    }
  }
  float wk[9][8];
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(w + (long long)t * C + cv * 8));
    const float4 w1 = __ldg(reinterpret_cast<const float4*>(w + (long long)t * C + cv * 8 + 4));
    wk[t][0] = w0.x; wk[t][1] = w0.y; wk[t][2] = w0.z; wk[t][3] = w0.w; wk[t][4] = w1.x; wk[t][5] = w1.y; wk[t][6] = w1.z; wk[t][7] = w1.w;
  }
  float o[4][8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    o[0][e] = wk[4][e] * d[0][e];
    o[1][e] = fmaf(wk[5][e], d[0][e], wk[3][e] * d[1][e]);
    o[2][e] = fmaf(wk[7][e], d[0][e], wk[1][e] * d[2][e]);
    o[3][e] = fmaf(wk[8][e], d[0][e], fmaf(wk[6][e], d[1][e], fmaf(wk[2][e], d[2][e], wk[0][e] * d[3][e])));
  }
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int iy = 2 * m + (t >> 1), ix = 2 * n + (t & 1);
    if (iy < H && ix < W) *reinterpret_cast<uint4*>(dxo + (((long long)b * H + iy) * W + ix) * C + cv * 8) = pack8(o[t]);
  }
}

extern "C" int es3_dwconv_bwd_data(const void* dz, const float* w, void* dx, int B, int H, int W, int C, int ks, int stride,
                                   void* stream) {
  ES3_REQUIRE(C % 8 == 0 && (ks == 3 || ks == 5) && (stride == 1 || stride == 2), "es3_dwconv_bwd_data: unsupported C=%d ks=%d stride=%d", C, ks, stride);
  const int pad = ks / 2;
  const int Ho = (H + 2 * pad - ks) / stride + 1, Wo = (W + 2 * pad - ks) / stride + 1;
  if (ks == 3 && stride == 2) {
    const long long blocks = (long long)B * ((H + 1) / 2) * ((W + 1) / 2) * (C / 8);
    dw_bwd_data_s2k3_kernel<<<(unsigned)ceil_div(blocks, 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)dz, w, (bf16*)dx, B, H, W, C, Ho,
                                                                                              Wo);
    ES3_LAUNCH_CHECK("dw_bwd_data_s2k3_kernel");
    return 0;
  }
  const long long total = (long long)B * H * W * (C / 8);
  dw_bwd_data_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)dz, w, (bf16*)dx, B, H, W, C, Ho, Wo,
                                                                                       ks, stride);
  ES3_LAUNCH_CHECK("dw_bwd_data_kernel");
  return 0;
}

constexpr int DWS_P3 = 4, DWS_P5 = 8;   // strip lengths of the stride-1 kernels (3x3: 8 channels / thread, 5x5: 4 channels / thread)

// units = output pixels (stride 2, per-pixel kernel) or strips (stride 1, strip kernel)
static int dw_wgrad_geometry(int B, int Ho, int Wo, int C, int ks, int stride, int* CGB, int* nblk, long long* upb, int* gy) {
  const int vec = ks == 3 ? 8 : 4;
  const int CG = C / vec;
  *CGB = CG < 256 ? CG : 256;
  const int lanes = 256 / *CGB;
  long long total = (long long)B * Ho * Wo;
  if (stride == 1) {
    const int P = ks == 3 ? DWS_P3 : DWS_P5;
    total = (long long)B * Ho * ((Wo + P - 1) / P);
    long long want = (total + (long long)lanes * 8 - 1) / ((long long)lanes * 8);     // >= 8 strips per lane and block
    if (want < 1) want = 1;
    if (want > 1184) want = 1184;
    *nblk = (int)want;
  } else {
    *nblk = pick_blocks(total, lanes, 1184);
  }
  *upb = (total + *nblk - 1) / *nblk;
  *gy = (CG + *CGB - 1) / *CGB;
  return 0;
}

extern "C" long long es3_dwconv_wgrad_ws_floats(int B, int H, int W, int C, int ks, int stride) {
  const int pad = ks / 2;
  const int Ho = (H + 2 * pad - ks) / stride + 1, Wo = (W + 2 * pad - ks) / stride + 1;
  int CPB, nblk, gy;
  long long ppb;
  dw_wgrad_geometry(B, Ho, Wo, C, ks, stride, &CPB, &nblk, &ppb, &gy);
  return (long long)nblk * ks * ks * C;
}

/* dW[c * ks*ks + tap] += sum_p dz[p][c] x[src(p, tap)][c]   (torch layout [C,1,ks,ks]) */
extern "C" int es3_dwconv_wgrad(const void* dz, const void* x, long long ldx, int B, int H, int W, int C, int ks, int stride, float* ws,
                                float* dW, void* stream) {
  ES3_REQUIRE(C % 8 == 0 && ldx % 8 == 0 && (ks == 3 || ks == 5) && (stride == 1 || stride == 2),
              "es3_dwconv_wgrad: unsupported C=%d ks=%d stride=%d", C, ks, stride);
  const int pad = ks / 2;
  const int Ho = (H + 2 * pad - ks) / stride + 1, Wo = (W + 2 * pad - ks) / stride + 1;
  int CPB, nblk, gy;
  long long ppb;
  dw_wgrad_geometry(B, Ho, Wo, C, ks, stride, &CPB, &nblk, &ppb, &gy);
  cudaStream_t st = (cudaStream_t)stream;
  if (stride == 1 && ks == 3)
    dw_wgrad_strip_kernel<3, 8, DWS_P3><<<dim3(nblk, gy), 256, 0, st>>>((const bf16*)dz, (const bf16*)x, ldx, B, H, W, C, CPB, ppb, ws);
  else if (stride == 1)
    dw_wgrad_strip_kernel<5, 4, DWS_P5><<<dim3(nblk, gy), 256, 0, st>>>((const bf16*)dz, (const bf16*)x, ldx, B, H, W, C, CPB, ppb, ws);
  else if (ks == 3)
    dw_wgrad_kernel<3, 8><<<dim3(nblk, gy), 256, 0, st>>>((const bf16*)dz, (const bf16*)x, ldx, B, H, W, C, Ho, Wo, stride, CPB, ppb, ws);
  else
    dw_wgrad_kernel<5, 4><<<dim3(nblk, gy), 256, 0, st>>>((const bf16*)dz, (const bf16*)x, ldx, B, H, W, C, Ho, Wo, stride, CPB, ppb, ws);
  ES3_LAUNCH_CHECK("dw_wgrad_kernel");
  const long long n = (long long)ks * ks * C;
  // part index i = tap * C + c  ->  dW[c * ks*ks + tap]
  sum_partials_kernel<<<(unsigned)ceil_div(n, 32), 256, 0, st>>>(ws, nblk, n, C, 1, (long long)ks * ks, dW);
  ES3_LAUNCH_CHECK("sum_partials_kernel");
  return 0;
}

static int dww_blocks(int B, int Ho, int Wo, int C) {
  const long long ntiles = (long long)B * ceil_div(Ho, DWW_TH) * ceil_div(Wo, DWW_TW);
  long long want = (2LL * 132 + C / DWW_CS - 1) / (C / DWW_CS);      // two resident CTAs per SM over all channel slabs
  if (want > ntiles) want = ntiles;
  if (want < 1) want = 1;
  return (int)want;
}

extern "C" long long es3_dwconv_wgrad_win_ws_floats(int B, int H, int W, int C, int ks, int stride) {
  const int pad = ks / 2;
  const int Ho = (H + 2 * pad - ks) / stride + 1, Wo = (W + 2 * pad - ks) / stride + 1;
  return (long long)dww_blocks(B, Ho, Wo, C) * ks * ks * C;
}

template <int KS, int STRIDE>
static int launch_dw_wgrad_win(const bf16* dz, const bf16* x, long long ldx, int B, int H, int W, int C, int Ho, int Wo, float* ws, cudaStream_t st) {
  using Cfg = DwwCfg<KS, STRIDE>;
  static bool configured = false;
  if (!configured) {
    ES3_CHECK_CUDA(cudaFuncSetAttribute(dw_wgrad_win_kernel<KS, STRIDE>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM));
    configured = true;
  }
  const int nblk = dww_blocks(B, Ho, Wo, C);
  dw_wgrad_win_kernel<KS, STRIDE><<<dim3(nblk, C / DWW_CS), 256, Cfg::SMEM, st>>>(dz, x, ldx, B, H, W, C, Ho, Wo, ceil_div(Wo, DWW_TW),
                                                                                  ceil_div(Ho, DWW_TH), ws);
  ES3_LAUNCH_CHECK("dw_wgrad_win_kernel");
  return 0;
}

/* Same contract as es3_dwconv_wgrad for C % 32 == 0 (stride 1 | 2, ks 3 | 5): register sliding window over shared-memory tiles. */
extern "C" int es3_dwconv_wgrad_win(const void* dz, const void* x, long long ldx, int B, int H, int W, int C, int ks, int stride, float* ws,
                                    float* dW, void* stream) {
  ES3_REQUIRE(C % DWW_CS == 0 && ldx % 8 == 0 && (ks == 3 || ks == 5) && (stride == 1 || stride == 2),
              "es3_dwconv_wgrad_win: need C %% 32 == 0, ks 3|5, stride 1|2 (C=%d ks=%d stride=%d)", C, ks, stride);
  ES3_REQUIRE(((uintptr_t)dz & 15) == 0 && ((uintptr_t)x & 15) == 0, "es3_dwconv_wgrad_win: operands must be 16-byte aligned");
  const int pad = ks / 2;
  const int Ho = (H + 2 * pad - ks) / stride + 1, Wo = (W + 2 * pad - ks) / stride + 1;
  cudaStream_t st = (cudaStream_t)stream;
  const bf16* dzp = (const bf16*)dz;
  const bf16* xp = (const bf16*)x;
  int rc;
  if (ks == 3 && stride == 1) rc = launch_dw_wgrad_win<3, 1>(dzp, xp, ldx, B, H, W, C, Ho, Wo, ws, st);
  else if (ks == 3) rc = launch_dw_wgrad_win<3, 2>(dzp, xp, ldx, B, H, W, C, Ho, Wo, ws, st);
  else if (stride == 1) rc = launch_dw_wgrad_win<5, 1>(dzp, xp, ldx, B, H, W, C, Ho, Wo, ws, st);
  else rc = launch_dw_wgrad_win<5, 2>(dzp, xp, ldx, B, H, W, C, Ho, Wo, ws, st);
  if (rc) return rc;
  const long long n = (long long)ks * ks * C;
  sum_partials_kernel<<<(unsigned)ceil_div(n, 32), 256, 0, st>>>(ws, dww_blocks(B, Ho, Wo, C), n, C, 1, (long long)ks * ks, dW);
  ES3_LAUNCH_CHECK("sum_partials_kernel");
  return 0;
}

static int se_chunks(int HW, int C, int* CVB, int* ppc) {
  const int CV = C / 8;
  *CVB = CV < 256 ? CV : 256;
  const int lanes = 256 / *CVB;
  int nchunk = ceil_div(HW, lanes * 32);                     // >= 32 pixels per lane and chunk
  if (nchunk > 64) nchunk = 64;
  if (nchunk < 1) nchunk = 1;
  *ppc = ceil_div(HW, nchunk);
  return ceil_div(HW, *ppc);
}

extern "C" long long es3_se_bwd_ws_floats(int B, int HW, int C) {
  int CVB, ppc;
  return (long long)se_chunks(HW, C, &CVB, &ppc) * B * C;
}

/* dgate[b][c] += sum_p dy[b][p][c] x[b][p][c]  (dy, x: [B][HW][C] bf16 contiguous) */
extern "C" int es3_se_bwd_dgate(const void* dy, const void* x, int B, int HW, int C, float* ws, float* dgate, void* stream) {
  ES3_REQUIRE(B > 0 && HW > 0 && C % 8 == 0, "es3_se_bwd_dgate: bad shape (C=%d)", C);
  int CVB, ppc;
  const int nchunk = se_chunks(HW, C, &CVB, &ppc);
  cudaStream_t st = (cudaStream_t)stream;
  se_dgate_kernel<<<dim3(nchunk, B), 256, 0, st>>>((const bf16*)dy, (const bf16*)x, HW, C, CVB, ppc, ws);
  ES3_LAUNCH_CHECK("se_dgate_kernel");
  const long long n = (long long)B * C;
  sum_partials_kernel<<<(unsigned)ceil_div(n, 32), 256, 0, st>>>(ws, nchunk, n, (int)n, 0, 1, dgate);
  ES3_LAUNCH_CHECK("sum_partials_kernel");
  return 0;
}

/* dx[b][p][c] = dy[b][p][c] * gate[b][c] + add[b][c] */
extern "C" int es3_se_bwd_apply(const void* dy, const float* gate, const float* add, void* dx, int B, int HW, int C, void* stream) {
  ES3_REQUIRE(B > 0 && HW > 0 && C % 8 == 0, "es3_se_bwd_apply: bad shape (C=%d)", C);
  const long long total = (long long)B * HW * (C / 8);
  se_apply_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)dy, gate, add, (bf16*)dx, HW, C / 8, total);
  ES3_LAUNCH_CHECK("se_apply_kernel");
  return 0;
}

static int stem_wgrad_blocks(int B, int Ho, int Wo, int* chunks_per_block) {
  const long long total = (long long)B * Ho * Wo;
  const long long chunks = (total + SW_PX - 1) / SW_PX;
  long long nblk = chunks < 592 ? chunks : 592;
  *chunks_per_block = (int)((chunks + nblk - 1) / nblk);
  return (int)((chunks + *chunks_per_block - 1) / *chunks_per_block);
}

extern "C" long long es3_stem_wgrad_ws_floats(int B, int H, int W, int Cout) {
  int cpb;
  const int nblk = stem_wgrad_blocks(B, (H - 1) / 2 + 1, (W - 1) / 2 + 1, &cpb);
  return (long long)nblk * Cout * 27;
}

/* dW[n][ci][ky][kx] += sum_p dz[p][n] img[b][ci][2 oy - 1 + ky][2 ox - 1 + kx] */
extern "C" int es3_stem_wgrad(const float* img, const void* dz, int B, int H, int W, int Cout, float* ws, float* dW, void* stream) {
  ES3_REQUIRE(Cout > 0 && Cout <= SW_MAXC && Cout % 8 == 0, "es3_stem_wgrad: Cout=%d not supported (multiple of 8, <= %d)", Cout, SW_MAXC);
  ES3_REQUIRE(((uintptr_t)dz & 15) == 0, "es3_stem_wgrad: dz must be 16-byte aligned");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  int cpb;
  const int nblk = stem_wgrad_blocks(B, Ho, Wo, &cpb);
  cudaStream_t st = (cudaStream_t)stream;
  stem_wgrad_kernel<<<nblk, 256, 0, st>>>(img, (const bf16*)dz, B, H, W, Ho, Wo, Cout, cpb, ws);   // (Cout / 2) * 14 <= 224 compute threads
  ES3_LAUNCH_CHECK("stem_wgrad_kernel");
  const long long n = (long long)Cout * 27;
  sum_partials_kernel<<<(unsigned)ceil_div(n, 32), 256, 0, st>>>(ws, nblk, n, 27, 27, 1, dW);
  ES3_LAUNCH_CHECK("sum_partials_kernel");
  return 0;
}

/* out [C][Mp] = zero-framed, x-shifted transpose of in [B,H,W,C] (see transpose_pad_kernel); Mp = B (H+2) Wp. */
extern "C" int es3_transpose_pad_bf16(const void* in, void* out, int B, int H, int W, int C, int Wp, int dx, void* stream) {
  ES3_REQUIRE(B > 0 && H > 0 && W > 0 && C % 8 == 0, "es3_transpose_pad_bf16: bad shape (C=%d)", C);
  ES3_REQUIRE(Wp % 8 == 0 && Wp >= W + 2 && dx >= -1 && dx <= 1, "es3_transpose_pad_bf16: need Wp %% 8 == 0, Wp >= W + 2, |dx| <= 1");
  const long long Mp = (long long)B * (H + 2) * Wp;
  cudaStream_t st = (cudaStream_t)stream;
  ES3_CHECK_CUDA(cudaMemsetAsync(out, 0, (size_t)C * Mp * sizeof(bf16), st));
  transpose_pad_kernel<<<dim3(ceil_div(C, 64), H, B), 256, 0, st>>>((const bf16*)in, (bf16*)out, H, W, C, Wp, dx, Mp);
  ES3_LAUNCH_CHECK("transpose_pad_kernel");
  return 0;
}

/* dst[(i / inner) ld_outer + (i % inner) ld_inner] += src[i], i < n  (fp32): adds a dense [n / inner][inner] block into a
 * strided parameter-gradient tensor (one tap of a [N][C][3][3] weight). */
extern "C" int es3_accumulate_strided(const float* src, long long n, int inner, long long ld_outer, long long ld_inner, float* dst,
                                      void* stream) {
  ES3_REQUIRE(n > 0 && inner > 0, "es3_accumulate_strided: bad shape");
  sum_partials_kernel<<<(unsigned)ceil_div(n, 32), 256, 0, (cudaStream_t)stream>>>(src, 1, n, inner, ld_outer, ld_inner, dst);
  ES3_LAUNCH_CHECK("sum_partials_kernel");
  return 0;
}

extern "C" int es3_bilinear_bwd(const float* dout, void* din, int B, int Hi, int Wi, int C, int Ho, int Wo, void* stream) {
  ES3_REQUIRE(B > 0 && Hi > 0 && Wi > 0 && Ho > 0 && Wo > 0 && C > 0, "es3_bilinear_bwd: bad shape");
  const int smem = (Wi * (BB_CB + 1) + Wi * BB_MAXT + Wi + BB_MAXT) * (int)sizeof(float);
  ES3_REQUIRE(smem <= 48 * 1024, "es3_bilinear_bwd: Wi=%d too wide for the row tile", Wi);
  // candidates per input pixel and axis: outputs whose 2-tap source interval can contain it, <= 2 * (out / in) + 4
  ES3_REQUIRE(2.f * Ho / Hi + 4.f <= BB_MAXT && 2.f * Wo / Wi + 4.f <= BB_MAXT,
              "es3_bilinear_bwd: up-scaling %dx%d -> %dx%d exceeds the %d-candidate tables", Hi, Wi, Ho, Wo, BB_MAXT);
  bilinear_bwd_kernel<<<dim3(ceil_div(C, BB_CB), Hi, B), 256, smem, (cudaStream_t)stream>>>(dout, (bf16*)din, Hi, Wi, C, Ho, Wo,
                                                                                          (float)Hi / (float)Ho, (float)Wi / (float)Wo);
  ES3_LAUNCH_CHECK("bilinear_bwd_kernel");
  return 0;
}

extern "C" long long es3_litemla_bwd_ws_floats(int B, int HW, int heads2) {
  // dKV partials per 128-pixel chunk + the two chunk-summed tables (KV, dKV)
  return (long long)B * heads2 * (ceil_div(HW, LB_PX) + 2) * 17 * 16;
}

/* kv_part: the [B][heads2][nchunk_f][17][16] partial KV sums es3_litemla_attn_tc left in its workspace
 * (nchunk_f = ceil(HW / 512)). */
extern "C" int es3_litemla_attn_bwd(const void* ms, long long ld, const void* dy, long long lddy, const float* kv_part, int nchunk_f,
                                    float* dkv_ws, void* dms, long long lddms, int B, int HW, int heads2, float eps, void* stream) {
  ES3_REQUIRE(ld >= 48 * heads2 && ld % 8 == 0 && lddy % 8 == 0 && lddms % 8 == 0 && lddy >= 16 * heads2 && lddms >= 48 * heads2,
              "es3_litemla_attn_bwd: bad strides ld=%lld lddy=%lld lddms=%lld heads2=%d", ld, lddy, lddms, heads2);
  ES3_REQUIRE(nchunk_f == ceil_div(HW, 512), "es3_litemla_attn_bwd: kv_part must come from es3_litemla_attn_tc (nchunk %d != %d)", nchunk_f,
              ceil_div(HW, 512));
  cudaStream_t st = (cudaStream_t)stream;
  const int nchunk_b = ceil_div(HW, LB_PX);
  dim3 grid(nchunk_b, heads2, B);
  const int BH = B * heads2;
  float* dkv_part = dkv_ws;
  float* kv_sum = dkv_ws + (long long)BH * nchunk_b * 17 * 16;
  float* dkv_sum = kv_sum + (long long)BH * 17 * 16;
  litemla_sum_partials_kernel<<<BH, 288, 0, st>>>(kv_part, nchunk_f, kv_sum);
  ES3_LAUNCH_CHECK("litemla_sum_partials_kernel");
  litemla_dkv_kernel<<<grid, 288, 0, st>>>((const bf16*)ms, ld, (const bf16*)dy, lddy, kv_sum, nchunk_f, dkv_part, HW, eps);
  ES3_LAUNCH_CHECK("litemla_dkv_kernel");
  litemla_sum_partials_kernel<<<BH, 288, 0, st>>>(dkv_part, nchunk_b, dkv_sum);
  ES3_LAUNCH_CHECK("litemla_sum_partials_kernel");
  litemla_dqkv_kernel<<<grid, 128, 0, st>>>((const bf16*)ms, ld, (const bf16*)dy, lddy, kv_sum, nchunk_f, dkv_sum, nchunk_b, (bf16*)dms,
                                            lddms, HW, eps);
  ES3_LAUNCH_CHECK("litemla_dqkv_kernel");
  return 0;
}
