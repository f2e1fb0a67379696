// MobileCLIP-S0's RepMixerBlock (mobile_clip.py:545-702) with batch-statistics BatchNorm: every BN in train mode, as
// nn.BatchNorm2d trains.  Each BN normalises with the mean and biased variance of its input over all B*L tokens (padding
// included) and updates its running buffers.  BN_ms (mixer.rbr_skip) and BN_ns (norm.rbr_skip) both see x, so their statistics
// are taken once:
//   c = dw(x; w_mc)   r = BN_ms(x) + BN_mc(c) - BN_ns(x)   x1 = x + ls_tm r
//   f = dw(x1; w_f)   u = BN_f(f)   y = fc2(gelu(fc1(u)))   x2 = x1 + ls_blk y
// Forward (es3_repmixer_bn_fwd): statistics of x and c -> finalize (running buffers, folded token-mixer taps) -> statistics of f
// on x1 recomputed with those taps in repmixer_kernel's FMA order (so they describe exactly the x1 the prologue writes) ->
// finalize BN_f -> es3_repmixer_bf16 on the device-folded taps.  Backward: with M = B*L and vhat the normalised input, a BN's
// input gradient is gamma invstd (d - sum(d) / M - vhat sum(d vhat) / M); the two sums are the BN's beta / gamma gradients, so
// each sequence kernel of repmixer_bwd.cu splits into a sums pass and an apply pass with a fixed-order reduction between them.
// Layout as repmixer_bwd.cu: one CTA per (sequence, 32 channels), the sequence plus zero halos in shared memory; per-CTA partials
// in part [B][Q][C] summed over the sequences in index order.  Statistics are fp32 sums shifted by a per-sequence pivot (the
// sequence's first token), combined across sequences in fp64.  No float atomics: every result is bit-reproducible.
#include "repmixer_seq.cuh"

namespace es3 {
namespace {

constexpr int BS_Q_XC = 6, BS_Q_F = 3, BS_Q_FFN = SQ_KS, BS_Q_TM = SQ_KS + 1, BS_Q_MAX = BS_Q_TM, BS_NSUM = 3;
static_assert(BS_Q_MAX * SQ_ROWS <= SQ_PAD, "the partials' reduction reuses a sequence buffer");

// affine rows [9][C]: ls_tm, then (gamma, beta) of BN_ms, BN_mc, BN_ns, BN_f.  stats rows [8][C]: (mean, invstd) of the same four.
enum { A_LS = 0, A_G_MS, A_B_MS, A_G_MC, A_B_MC, A_G_NS, A_B_NS, A_G_F, A_B_F };
enum { S_M_MS = 0, S_I_MS, S_M_MC, S_I_MC, S_M_NS, S_I_NS, S_M_F, S_I_F };

// Shifted sums of one value: (pivot, sum (v - pivot), sum (v - pivot)^2); the pivot is counted by row group 0 only.
__device__ __forceinline__ void shifted(float* v, float piv, float val) {
  const float d = val - piv;
  v[1] += d;
  v[2] = fmaf(d, d, v[2]);
}

// MODE 0: statistics of x and c = dw(x; w_mc) (part Q = 6).  MODE 1: x1 = bm + dw(x; wm) exactly as repmixer_kernel computes
// it, then statistics of f = dw(x1; w_f) (part Q = 3).  taps [2][11][C] raw (w_mc, w_f); fold [24][C] (wm, bm, wf, bf).
template <int MODE>
__global__ void __launch_bounds__(SQ_THREADS) repmixer_bn_stats_kernel(const float* __restrict__ x, const float* __restrict__ taps,
                                                                       const float* __restrict__ fold, float* __restrict__ part,
                                                                       int L, int C) {
  constexpr int Q = MODE == 0 ? BS_Q_XC : BS_Q_F;
  __shared__ float sx[SQ_PAD * SQ_CH];
  __shared__ float sy[SQ_PAD * SQ_CH];
  const int c = threadIdx.x % SQ_CH, r0 = threadIdx.x / SQ_CH;
  const int ch = blockIdx.x * SQ_CH + c;
  const long long base = (long long)blockIdx.y * L * C + ch;
  load_seq(x, sx, base, L, C);
  float w[SQ_KS];
  float v[Q];
#pragma unroll
  for (int q = 0; q < Q; ++q) v[q] = 0.f;
  if constexpr (MODE == 0) {
#pragma unroll
    for (int k = 0; k < SQ_KS; ++k) w[k] = taps[k * C + ch];
    __syncthreads();
    const float px = sx[SQ_HALO * SQ_CH + c], pc = conv_at(w, sx, 0, 0.f);
    if (r0 == 0) { v[0] = px; v[3] = pc; }
    for (int l = r0; l < L; l += SQ_ROWS) {
      shifted(v, px, sx[(l + SQ_HALO) * SQ_CH + c]);
      shifted(v + 3, pc, conv_at(w, sx, l, 0.f));
    }
  } else {
    for (int l = r0; l < L + 2 * SQ_HALO; l += SQ_ROWS)
      if (l < SQ_HALO || l >= L + SQ_HALO) sy[l * SQ_CH + c] = 0.f;
#pragma unroll
    for (int k = 0; k < SQ_KS; ++k) w[k] = fold[k * C + ch];
    const float b = fold[SQ_KS * C + ch];
    __syncthreads();
    for (int l = r0; l < L; l += SQ_ROWS) sy[(l + SQ_HALO) * SQ_CH + c] = conv_at(w, sx, l, b);
#pragma unroll
    for (int k = 0; k < SQ_KS; ++k) w[k] = taps[(SQ_KS + k) * C + ch];
    __syncthreads();
    const float pf = conv_at(w, sy, 0, 0.f);
    if (r0 == 0) v[0] = pf;
    for (int l = r0; l < L; l += SQ_ROWS) shifted(v, pf, conv_at(w, sy, l, 0.f));
  }
  cta_partials<Q>(v, sx, part, blockIdx.y, C, blockIdx.x * SQ_CH);
}

struct BnRun {
  float* rm;
  float* rv;
  long long* nbt;
  float eps, momentum;
};

struct BnFinalize {
  BnRun bn[4];                      // BN_ms, BN_mc, BN_ns, BN_f
  const float* taps;                // [2][11][C] raw w_mc, w_f
  const float* aff;                 // [9][C]
  float* fold;                      // [24][C] wm, bm, wf, bf (repmixer_fold's form)
  float* stats;                     // [8][C]
};

// Mean and biased variance (fp64) of one value from the per-sequence shifted sums at q0 .. q0 + 2 of part [B][Q][C]: Chan's
// combination, sum_b (M2_b + L (mean_b - mean)^2), so no large-magnitude cancellation when |mean| >> std.
__device__ void combine(const float* __restrict__ part, int Q, int q0, int B, int L, int C, int ch, double& mean, double& var) {
  const double n = L, M = (double)B * L;
  double s = 0.0;
  for (int b = 0; b < B; ++b) {
    const float* p = part + ((long long)b * Q + q0) * C + ch;
    s += n * (double)p[0] + (double)p[C];
  }
  mean = s / M;
  double m2 = 0.0;
  for (int b = 0; b < B; ++b) {
    const float* p = part + ((long long)b * Q + q0) * C + ch;
    const double s1 = p[C], mb = (double)p[0] + s1 / n - mean;
    m2 += ((double)p[2 * C] - s1 * s1 / n) + n * mb * mb;
  }
  var = fmax(m2 / M, 0.0);
}

// Running buffers as nn.BatchNorm2d updates them (unbiased variance, momentum); returns invstd with the biased variance.
__device__ float bn_update(const BnRun& r, int ch, double mean, double var, double M) {
  const double mom = r.momentum;
  r.rm[ch] = (float)((1.0 - mom) * (double)r.rm[ch] + mom * mean);
  r.rv[ch] = (float)((1.0 - mom) * (double)r.rv[ch] + mom * var * M / (M - 1.0));
  if (ch == 0) r.nbt[0] += 1;
  return (float)(1.0 / sqrt(var + (double)r.eps));
}

// BN_ms, BN_ns (statistics of x: mx, vx) and BN_mc (of c: mc, vc) over M values: running buffers, stats, folded wm, bm.
__device__ void finalize_xc(const BnFinalize& f, int ch, int C, double mx, double vx, double mc, double vc, double M) {
  const float* aff = f.aff;
  {
    const float i_ms = bn_update(f.bn[0], ch, mx, vx, M), i_mc = bn_update(f.bn[1], ch, mc, vc, M);
    const float i_ns = bn_update(f.bn[2], ch, mx, vx, M);
    const float fmx = (float)mx, fmc = (float)mc;
    float* st = f.stats;
    st[S_M_MS * C + ch] = fmx; st[S_I_MS * C + ch] = i_ms;
    st[S_M_MC * C + ch] = fmc; st[S_I_MC * C + ch] = i_mc;
    st[S_M_NS * C + ch] = fmx; st[S_I_NS * C + ch] = i_ns;
    const float ls = aff[A_LS * C + ch];
    const float s_ms = aff[A_G_MS * C + ch] * i_ms, s_mc = aff[A_G_MC * C + ch] * i_mc, s_ns = aff[A_G_NS * C + ch] * i_ns;
    const float b_ms = aff[A_B_MS * C + ch] - fmx * s_ms, b_mc = aff[A_B_MC * C + ch] - fmc * s_mc;
    const float b_ns = aff[A_B_NS * C + ch] - fmx * s_ns;
    const float sw = ls * s_mc;
#pragma unroll
    for (int k = 0; k < SQ_KS; ++k) {
      float wk = f.taps[k * C + ch] * sw;
      if (k == SQ_HALO) wk += 1.f + ls * (s_ms - s_ns);
      f.fold[k * C + ch] = wk;
    }
    f.fold[SQ_KS * C + ch] = ls * (b_ms + b_mc - b_ns);
  }
}

// BN_f (statistics of f: mf, vf) over M values: running buffers, stats, folded wf, bf.
__device__ void finalize_f(const BnFinalize& f, int ch, int C, double mf, double vf, double M) {
  const float* aff = f.aff;
  {
    const float i_f = bn_update(f.bn[3], ch, mf, vf, M), fmf = (float)mf;
    f.stats[S_M_F * C + ch] = fmf;
    f.stats[S_I_F * C + ch] = i_f;
    const float s_f = aff[A_G_F * C + ch] * i_f;
#pragma unroll
    for (int k = 0; k < SQ_KS; ++k) f.fold[(SQ_KS + 1 + k) * C + ch] = f.taps[(SQ_KS + k) * C + ch] * s_f;
    f.fold[(2 * SQ_KS + 1) * C + ch] = aff[A_B_F * C + ch] - fmf * s_f;
  }
}

// One thread per channel.  MODE 0: BN_ms, BN_ns (statistics of x) and BN_mc (of c); writes wm, bm.  MODE 1: BN_f; writes wf, bf.
template <int MODE>
__global__ void repmixer_bn_finalize_kernel(const float* __restrict__ part, int B, int L, int C, BnFinalize f) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= C) return;
  const double M = (double)B * L;
  if constexpr (MODE == 0) {
    double mx, vx, mc, vc;
    combine(part, BS_Q_XC, 0, B, L, C, ch, mx, vx);
    combine(part, BS_Q_XC, 3, B, L, C, ch, mc, vc);
    finalize_xc(f, ch, C, mx, vx, mc, vc, M);
  } else {
    double mf, vf;
    combine(part, BS_Q_F, 0, B, L, C, ch, mf, vf);
    finalize_f(f, ch, C, mf, vf, M);
  }
}

// Synchronised BatchNorm (SyncBatchNorm over several ranks).  This rank's (count, mean, M2) of each value, fp64 out [NV][3][C]
// (MODE 0: x, c; MODE 1: f), from the per-sequence partials of repmixer_bn_stats_kernel<MODE>.
template <int MODE>
__global__ void repmixer_bn_local_kernel(const float* __restrict__ part, int B, int L, int C, double* __restrict__ out) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= C) return;
  constexpr int NV = MODE == 0 ? 2 : 1, Q = MODE == 0 ? BS_Q_XC : BS_Q_F;
  const double M = (double)B * L;
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    double mean, var;
    combine(part, Q, 3 * v, B, L, C, ch, mean, var);
    out[(v * 3) * C + ch] = M;
    out[(v * 3 + 1) * C + ch] = mean;
    out[(v * 3 + 2) * C + ch] = var * M;
  }
}

// Chan's combination of value v over the W ranks' [W][NV][3][C] partials, in rank order.
__device__ void chan_ranks(const double* __restrict__ parts, int W, int NV, int v, int C, int ch, double& n, double& mean, double& var) {
  n = 0.0; mean = 0.0;
  double m2 = 0.0;
  for (int w = 0; w < W; ++w) {
    const double* p = parts + ((long long)w * NV + v) * 3 * C + ch;
    const double nb = p[0];
    if (nb <= 0.0) continue;
    const double nn = n + nb, d = p[C] - mean;
    mean += d * (nb / nn);
    m2 += p[2 * C] + d * d * (n * nb / nn);
    n = nn;
  }
  var = n > 0.0 ? fmax(m2 / n, 0.0) : 0.0;
}

// The finalize of repmixer_bn_finalize_kernel<MODE> on every rank's partials; total [1] = the count over the group.
template <int MODE>
__global__ void repmixer_bn_finalize_sync_kernel(const double* __restrict__ parts, int W, int C, BnFinalize f, double* __restrict__ total) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= C) return;
  double n;
  if constexpr (MODE == 0) {
    double mx, vx, mc, vc;
    chan_ranks(parts, W, 2, 0, C, ch, n, mx, vx);
    chan_ranks(parts, W, 2, 1, C, ch, n, mc, vc);
    finalize_xc(f, ch, C, mx, vx, mc, vc, n);
  } else {
    double mf, vf;
    chan_ranks(parts, W, 1, 0, C, ch, n, mf, vf);
    finalize_f(f, ch, C, mf, vf, n);
  }
  if (ch == 0 && total != nullptr) total[0] = n;
}

// ConvFFN sums pass: sum du and sum du fhat (BN_f's beta / gamma gradients), fhat = (dw(x1; w_f) - mean_f) invstd_f.
__global__ void __launch_bounds__(SQ_THREADS) repmixer_bn_ffn_sums_kernel(const float* __restrict__ x1, const float* __restrict__ du,
                                                                          const float* __restrict__ taps, const float* __restrict__ stats,
                                                                          float* __restrict__ part, int L, int C) {
  __shared__ float sx1[SQ_PAD * SQ_CH];
  const int c = threadIdx.x % SQ_CH, r0 = threadIdx.x / SQ_CH;
  const int ch = blockIdx.x * SQ_CH + c;
  const long long base = (long long)blockIdx.y * L * C + ch;
  load_seq(x1, sx1, base, L, C);
  float w[SQ_KS];
#pragma unroll
  for (int k = 0; k < SQ_KS; ++k) w[k] = taps[(SQ_KS + k) * C + ch];
  const float mf = stats[S_M_F * C + ch], inv = stats[S_I_F * C + ch];
  float v[2] = {0.f, 0.f};
  __syncthreads();
  for (int l = r0; l < L; l += SQ_ROWS) {
    const float d = du[base + (long long)l * C];
    v[0] += d;
    v[1] = fmaf(d, (conv_at(w, sx1, l, 0.f) - mf) * inv, v[1]);
  }
  cta_partials<2>(v, sx1, part, blockIdx.y, C, blockIdx.x * SQ_CH);
}

// ConvFFN apply pass: df = s_f (du - S0 / M - fhat S1 / M), e = g + dw^T(df; w_f); partials: the taps' sums df[l] x1[l+k-5].
__global__ void __launch_bounds__(SQ_THREADS) repmixer_bn_ffn_apply_kernel(const float* __restrict__ x1, const float* __restrict__ du,
                                                                           const float* __restrict__ g, const float* __restrict__ taps,
                                                                           const float* __restrict__ aff, const float* __restrict__ stats,
                                                                           const float* __restrict__ sums, const double* __restrict__ total,
                                                                           float* __restrict__ e, float* __restrict__ part, int B, int L,
                                                                           int C) {
  __shared__ float sx1[SQ_PAD * SQ_CH];
  __shared__ float sdf[SQ_PAD * SQ_CH];
  const int c = threadIdx.x % SQ_CH, r0 = threadIdx.x / SQ_CH;
  const int ch = blockIdx.x * SQ_CH + c;
  const long long base = (long long)blockIdx.y * L * C + ch;
  load_seq(x1, sx1, base, L, C);
  for (int l = r0; l < L + 2 * SQ_HALO; l += SQ_ROWS)
    if (l < SQ_HALO || l >= L + SQ_HALO) sdf[l * SQ_CH + c] = 0.f;
  float w[SQ_KS];
#pragma unroll
  for (int k = 0; k < SQ_KS; ++k) w[k] = taps[(SQ_KS + k) * C + ch];
  const float mf = stats[S_M_F * C + ch], inv = stats[S_I_F * C + ch], s_f = aff[A_G_F * C + ch] * inv;
  // total: the count over every rank when synchronised, else this batch's B L
  const float rM = total ? (float)(1.0 / total[0]) : 1.f / ((float)B * (float)L), m0 = sums[ch] * rM, m1 = sums[C + ch] * rM;
  float v[BS_Q_FFN];
#pragma unroll
  for (int q = 0; q < BS_Q_FFN; ++q) v[q] = 0.f;
  __syncthreads();
  for (int l = r0; l < L; l += SQ_ROWS) {
    const float fh = (conv_at(w, sx1, l, 0.f) - mf) * inv;
    const float df = s_f * (du[base + (long long)l * C] - m0 - fh * m1);
    sdf[(l + SQ_HALO) * SQ_CH + c] = df;
#pragma unroll
    for (int k = 0; k < SQ_KS; ++k) v[k] = fmaf(df, sx1[(l + k) * SQ_CH + c], v[k]);
  }
  __syncthreads();
  for (int l = r0; l < L; l += SQ_ROWS) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < SQ_KS; ++k) t = fmaf(w[k], sdf[(l + 2 * SQ_HALO - k) * SQ_CH + c], t);   // df[l - k + 5]
    const long long i = base + (long long)l * C;
    e[i] = g[i] + t;
  }
  cta_partials<BS_Q_FFN>(v, sx1, part, blockIdx.y, C, blockIdx.x * SQ_CH);
}

// Token-mixer sums pass, e' = ls e: sum e', sum e' chat, sum e' (x - mean_x).  BN_ms's gamma gradient is invstd_ms times the last,
// BN_ns's is -invstd_ns times it (one xhat up to eps).
__global__ void __launch_bounds__(SQ_THREADS) repmixer_bn_tm_sums_kernel(const float* __restrict__ x, const float* __restrict__ e,
                                                                         const float* __restrict__ taps, const float* __restrict__ aff,
                                                                         const float* __restrict__ stats, float* __restrict__ part,
                                                                         int L, int C) {
  __shared__ float sx[SQ_PAD * SQ_CH];
  const int c = threadIdx.x % SQ_CH, r0 = threadIdx.x / SQ_CH;
  const int ch = blockIdx.x * SQ_CH + c;
  const long long base = (long long)blockIdx.y * L * C + ch;
  load_seq(x, sx, base, L, C);
  float w[SQ_KS];
#pragma unroll
  for (int k = 0; k < SQ_KS; ++k) w[k] = taps[k * C + ch];
  const float ls = aff[A_LS * C + ch], mx = stats[S_M_MS * C + ch], mc = stats[S_M_MC * C + ch], i_mc = stats[S_I_MC * C + ch];
  float v[3] = {0.f, 0.f, 0.f};
  __syncthreads();
  for (int l = r0; l < L; l += SQ_ROWS) {
    const float ep = ls * e[base + (long long)l * C];
    v[0] += ep;
    v[1] = fmaf(ep, (conv_at(w, sx, l, 0.f) - mc) * i_mc, v[1]);
    v[2] = fmaf(ep, sx[(l + SQ_HALO) * SQ_CH + c] - mx, v[2]);
  }
  cta_partials<3>(v, sx, part, blockIdx.y, C, blockIdx.x * SQ_CH);
}

// Token-mixer apply pass: dc = s_mc (e' - S0/M - chat S1/M), dx = e + [s_ms (e' - S0/M - xhat_ms i_ms S2/M) - s_ns (e' - S0/M -
// xhat_ns i_ns S2/M)] + dw^T(dc; w_mc); partials: the taps' sums dc[l] x[l+k-5] and the layer scale's sum e r.
__global__ void __launch_bounds__(SQ_THREADS) repmixer_bn_tm_apply_kernel(const float* __restrict__ x, const float* __restrict__ e,
                                                                          const float* __restrict__ taps, const float* __restrict__ aff,
                                                                          const float* __restrict__ stats, const float* __restrict__ sums,
                                                                          const double* __restrict__ total, float* __restrict__ dx,
                                                                          bf16* __restrict__ dxb,
                                                                          float* __restrict__ part, int B, int L, int C) {
  __shared__ float sx[SQ_PAD * SQ_CH];
  __shared__ float sdc[SQ_PAD * SQ_CH];
  const int c = threadIdx.x % SQ_CH, r0 = threadIdx.x / SQ_CH;
  const int ch = blockIdx.x * SQ_CH + c;
  const long long base = (long long)blockIdx.y * L * C + ch;
  load_seq(x, sx, base, L, C);
  for (int l = r0; l < L + 2 * SQ_HALO; l += SQ_ROWS)
    if (l < SQ_HALO || l >= L + SQ_HALO) sdc[l * SQ_CH + c] = 0.f;
  float w[SQ_KS];
#pragma unroll
  for (int k = 0; k < SQ_KS; ++k) w[k] = taps[k * C + ch];
  const float ls = aff[A_LS * C + ch], mx = stats[S_M_MS * C + ch];
  const float i_ms = stats[S_I_MS * C + ch], mc = stats[S_M_MC * C + ch], i_mc = stats[S_I_MC * C + ch], i_ns = stats[S_I_NS * C + ch];
  const float g_ms = aff[A_G_MS * C + ch], g_mc = aff[A_G_MC * C + ch], g_ns = aff[A_G_NS * C + ch];
  const float s_ms = g_ms * i_ms, s_mc = g_mc * i_mc, s_ns = g_ns * i_ns;
  const float br = aff[A_B_MS * C + ch] + aff[A_B_MC * C + ch] - aff[A_B_NS * C + ch];
  const float rM = total ? (float)(1.0 / total[0]) : 1.f / ((float)B * (float)L);
  const float m0 = sums[ch] * rM, m1 = sums[C + ch] * rM, m2 = sums[2 * C + ch] * rM;
  const float k_ms = s_ms * i_ms * i_ms * m2, k_ns = s_ns * i_ns * i_ns * m2;     // xhat i S2 / M, per unit (x - mean)
  float v[BS_Q_TM];
#pragma unroll
  for (int q = 0; q < BS_Q_TM; ++q) v[q] = 0.f;
  __syncthreads();
  for (int l = r0; l < L; l += SQ_ROWS) {
    const float ev = e[base + (long long)l * C], ep = ls * ev;
    const float ch_ = (conv_at(w, sx, l, 0.f) - mc) * i_mc, xc = sx[(l + SQ_HALO) * SQ_CH + c] - mx;
    const float dc = s_mc * (ep - m0 - ch_ * m1);
    sdc[(l + SQ_HALO) * SQ_CH + c] = dc;
#pragma unroll
    for (int k = 0; k < SQ_KS; ++k) v[k] = fmaf(dc, sx[(l + k) * SQ_CH + c], v[k]);
    const float r = fmaf(g_ms * i_ms - g_ns * i_ns, xc, fmaf(g_mc, ch_, br));
    v[SQ_KS] = fmaf(ev, r, v[SQ_KS]);
  }
  __syncthreads();
  for (int l = r0; l < L; l += SQ_ROWS) {
    const long long i = base + (long long)l * C;
    const float ev = e[i], ep = ls * ev, xc = sx[(l + SQ_HALO) * SQ_CH + c] - mx;
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < SQ_KS; ++k) t = fmaf(w[k], sdc[(l + 2 * SQ_HALO - k) * SQ_CH + c], t);   // dc[l - k + 5]
    const float d0 = ep - m0;
    const float out = ev + ((s_ms - s_ns) * d0 - (k_ms - k_ns) * xc) + t;
    dx[i] = out;
    if (dxb != nullptr) dxb[i] = __float2bfloat16_rn(out);
  }
  cta_partials<BS_Q_TM>(v, sx, part, blockIdx.y, C, blockIdx.x * SQ_CH);
}

// Sums of the sums passes: sums[q][c] = sum_b part[b][q][c] (index order); then dst[j][c] += sign[j] (scale[j][c]) sums[src[j]][c].
constexpr int BS_MAXDST = 6;
struct BnGradDst {
  int n;
  int src[BS_MAXDST];
  float sign[BS_MAXDST];
  const float* scale[BS_MAXDST];
  float* dst[BS_MAXDST];
};

template <int Q>
__global__ void repmixer_bn_sums_kernel(const float* __restrict__ part, int nseq, int C, float* __restrict__ sums, BnGradDst d) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float acc[Q];
#pragma unroll
  for (int q = 0; q < Q; ++q) acc[q] = 0.f;
  for (int b = 0; b < nseq; ++b) {
#pragma unroll
    for (int q = 0; q < Q; ++q) acc[q] += part[((long long)b * Q + q) * C + c];
  }
#pragma unroll
  for (int q = 0; q < Q; ++q) sums[q * C + c] = acc[q];
  for (int j = 0; j < d.n; ++j) {
    float a = 0.f;
#pragma unroll
    for (int q = 0; q < Q; ++q) if (q == d.src[j]) a = acc[q];
    if (d.scale[j] != nullptr) a *= d.scale[j][c];
    d.dst[j][c] += d.sign[j] * a;
  }
}

struct DstBuilder {
  BnGradDst d;
  DstBuilder() { d.n = 0; }
  void add(int src, float* dst, float sign = 1.f, const float* scale = nullptr) {
    if (dst == nullptr) return;
    d.src[d.n] = src; d.dst[d.n] = dst; d.sign[d.n] = sign; d.scale[d.n] = scale;
    ++d.n;
  }
};

// ------------------------------------------------------------------------------------------ the passes
// Each pass's launches, once for the per-rank entries and the synchronised ones (which split the forward at its two finalize
// points and the backward at its two sums).  ws: the CTA partials [B][BS_Q_MAX][C], then the BS_NSUM rows [C] a per-rank backward
// and the rank reductions keep their sums in.
float* ws_sums(float* ws, int B, int C) { return ws + (long long)B * BS_Q_MAX * C; }

// mode 0: the shifted sums of x and c = dw(x; w_mc); mode 1: of f = dw(x1; w_f), x1 from fold's wm, bm.
int stats_pass(int mode, const float* x, const float* taps, const float* fold, float* ws, int B, int L, int C, cudaStream_t st) {
  const dim3 grid(C / SQ_CH, B);
  if (mode == 0)
    repmixer_bn_stats_kernel<0><<<grid, SQ_THREADS, 0, st>>>(x, taps, fold, ws, L, C);
  else
    repmixer_bn_stats_kernel<1><<<grid, SQ_THREADS, 0, st>>>(x, taps, fold, ws, L, C);
  ES3_LAUNCH_CHECK(mode == 0 ? "repmixer_bn_stats_kernel<xc>" : "repmixer_bn_stats_kernel<f>");
  return 0;
}

BnFinalize make_finalize(const float* taps, const float* aff, float* rm_ms, float* rv_ms, long long* nbt_ms, float* rm_mc, float* rv_mc,
                         long long* nbt_mc, float* rm_ns, float* rv_ns, long long* nbt_ns, float* rm_f, float* rv_f, long long* nbt_f,
                         float eps_ms, float eps_mc, float eps_ns, float eps_f, float mom_ms, float mom_mc, float mom_ns, float mom_f,
                         float* fold, float* stats) {
  BnFinalize f;
  f.bn[0] = BnRun{rm_ms, rv_ms, nbt_ms, eps_ms, mom_ms};
  f.bn[1] = BnRun{rm_mc, rv_mc, nbt_mc, eps_mc, mom_mc};
  f.bn[2] = BnRun{rm_ns, rv_ns, nbt_ns, eps_ns, mom_ns};
  f.bn[3] = BnRun{rm_f, rv_f, nbt_f, eps_f, mom_f};
  f.taps = taps; f.aff = aff; f.fold = fold; f.stats = stats;
  return f;
}

// sums [2][C] = this batch's (sum du, sum du fhat); BN_f's dbeta / dgamma += them.
int ffn_sums_pass(const float* x1, const float* du, const float* taps, const float* stats, float* ws, float* sums, float* dgamma,
                  float* dbeta, int B, int L, int C, cudaStream_t st) {
  repmixer_bn_ffn_sums_kernel<<<dim3(C / SQ_CH, B), SQ_THREADS, 0, st>>>(x1, du, taps, stats, ws, L, C);
  ES3_LAUNCH_CHECK("repmixer_bn_ffn_sums_kernel");
  DstBuilder db;
  db.add(0, dbeta);
  db.add(1, dgamma);
  repmixer_bn_sums_kernel<2><<<ceil_div(C, 128), 128, 0, st>>>(ws, B, C, sums, db.d);
  ES3_LAUNCH_CHECK("repmixer_bn_sums_kernel<ffn>");
  return 0;
}

// sums [3][C] = this batch's (sum e', sum e' chat, sum e' (x - mean_x)); the gamma / beta gradients of BN_ms, BN_mc, BN_ns += theirs.
int tm_sums_pass(const float* x, const float* e, const float* taps, const float* aff, const float* stats, float* ws, float* sums,
                 float* dg_ms, float* db_ms, float* dg_mc, float* db_mc, float* dg_ns, float* db_ns, int B, int L, int C,
                 cudaStream_t st) {
  repmixer_bn_tm_sums_kernel<<<dim3(C / SQ_CH, B), SQ_THREADS, 0, st>>>(x, e, taps, aff, stats, ws, L, C);
  ES3_LAUNCH_CHECK("repmixer_bn_tm_sums_kernel");
  DstBuilder db;
  db.add(0, db_ms);
  db.add(0, db_mc);
  db.add(0, db_ns, -1.f);
  db.add(1, dg_mc);
  db.add(2, dg_ms, 1.f, stats + S_I_MS * C);
  db.add(2, dg_ns, -1.f, stats + S_I_NS * C);
  repmixer_bn_sums_kernel<3><<<ceil_div(C, 128), 128, 0, st>>>(ws, B, C, sums, db.d);
  ES3_LAUNCH_CHECK("repmixer_bn_sums_kernel<tm>");
  return 0;
}

// sums [2][C] over every token the statistics were taken on; total: their count when that spans several ranks, else null (B L).
int ffn_apply_pass(const float* x1, const float* du, const float* g, const float* taps, const float* aff, const float* stats,
                   const float* sums, const double* total, float* e, float* ws, float* dwf, int B, int L, int C, cudaStream_t st) {
  repmixer_bn_ffn_apply_kernel<<<dim3(C / SQ_CH, B), SQ_THREADS, 0, st>>>(x1, du, g, taps, aff, stats, sums, total, e, ws, B, L, C);
  ES3_LAUNCH_CHECK("repmixer_bn_ffn_apply_kernel");
  SumBuilder sb(BS_Q_FFN);
  sb.taps(dwf);
  return launch_sums(sb, ws, B, C, st);
}

// sums [3][C] and total as ffn_apply_pass.
int tm_apply_pass(const float* x, const float* e, const float* taps, const float* aff, const float* stats, const float* sums,
                  const double* total, float* dx, void* dxb, float* ws, float* dwmc, float* dls, int B, int L, int C, cudaStream_t st) {
  repmixer_bn_tm_apply_kernel<<<dim3(C / SQ_CH, B), SQ_THREADS, 0, st>>>(x, e, taps, aff, stats, sums, total, dx, (bf16*)dxb, ws, B, L, C);
  ES3_LAUNCH_CHECK("repmixer_bn_tm_apply_kernel");
  SumBuilder sb(BS_Q_TM);
  sb.taps(dwmc);
  sb.add(SQ_KS, dls);
  return launch_sums(sb, ws, B, C, st);
}

}  // namespace
}  // namespace es3

using namespace es3;

extern "C" int es3_repmixer_bf16(const float* x, float* x1, void* u, const float* wm, const float* bm, const float* wf,
                                 const float* bf, int B, int L, int C, void* stream);

// min_tokens: 2 where the statistics are this batch's own (a batch statistic needs more than one value per channel), 1 for the
// synchronised entries: one rank's batch may hold a single token, only the count over the group matters, and with two or more
// ranks it is >= 2.
#define BS_CHECK_SHAPE(fn, min_tokens)                                                                                         \
  ES3_REQUIRE(L >= 1 && L <= SQ_MAXL, fn ": sequence length %d outside 1..%d (the sequence is kept in shared memory)", L,  \
              SQ_MAXL);                                                                                                        \
  ES3_REQUIRE(B >= 1 && C >= SQ_CH && C % SQ_CH == 0, fn ": need B >= 1 and C %% %d == 0 (B=%d C=%d)", SQ_CH, B, C);          \
  ES3_REQUIRE((long long)B * L >= min_tokens, fn ": batch statistics need more than one value per channel (B*L=%d)", B * L)

extern "C" long long es3_repmixer_bn_ws_floats(int B, int C) { return ((long long)B * BS_Q_MAX + BS_NSUM) * C; }

/* Batch-statistics forward: x [B*L, C] fp32 -> x1 fp32, u bf16 (as es3_repmixer_bf16); updates the four BNs' running buffers and
 * num_batches_tracked; writes fold [24][C] (wm, bm, wf, bf) and stats [8][C] ((mean, invstd) of BN_ms, BN_mc, BN_ns, BN_f). */
extern "C" int es3_repmixer_bn_fwd(const float* x, float* x1, void* u, const float* taps, const float* aff, float* rm_ms, float* rv_ms,
                                   long long* nbt_ms, float* rm_mc, float* rv_mc, long long* nbt_mc, float* rm_ns, float* rv_ns,
                                   long long* nbt_ns, float* rm_f, float* rv_f, long long* nbt_f, float eps_ms, float eps_mc,
                                   float eps_ns, float eps_f, float mom_ms, float mom_mc, float mom_ns, float mom_f, float* fold,
                                   float* stats, float* ws, int B, int L, int C, void* stream) {
  BS_CHECK_SHAPE("es3_repmixer_bn_fwd", 2);
  cudaStream_t st = (cudaStream_t)stream;
  const BnFinalize f = make_finalize(taps, aff, rm_ms, rv_ms, nbt_ms, rm_mc, rv_mc, nbt_mc, rm_ns, rv_ns, nbt_ns, rm_f, rv_f, nbt_f,
                                     eps_ms, eps_mc, eps_ns, eps_f, mom_ms, mom_mc, mom_ns, mom_f, fold, stats);
  if (int rc = stats_pass(0, x, taps, fold, ws, B, L, C, st)) return rc;
  repmixer_bn_finalize_kernel<0><<<ceil_div(C, 128), 128, 0, st>>>(ws, B, L, C, f);
  ES3_LAUNCH_CHECK("repmixer_bn_finalize_kernel<xc>");
  if (int rc = stats_pass(1, x, taps, fold, ws, B, L, C, st)) return rc;
  repmixer_bn_finalize_kernel<1><<<ceil_div(C, 128), 128, 0, st>>>(ws, B, L, C, f);
  ES3_LAUNCH_CHECK("repmixer_bn_finalize_kernel<f>");
  return es3_repmixer_bf16(x, x1, u, fold, fold + SQ_KS * C, fold + (SQ_KS + 1) * C, fold + (2 * SQ_KS + 1) * C, B, L, C, stream);
}

/* ConvFFN.conv + BN_f backward with batch statistics: e = g + dw^T(df; w_f); dwf [C,1,1,11], dgamma, dbeta [C] += (may be null). */
extern "C" int es3_repmixer_bn_ffn_bwd(const float* x1, const float* du, const float* g, const float* taps, const float* aff,
                                       const float* stats, float* e, float* ws, float* dwf, float* dgamma, float* dbeta, int B, int L,
                                       int C, void* stream) {
  BS_CHECK_SHAPE("es3_repmixer_bn_ffn_bwd", 2);
  cudaStream_t st = (cudaStream_t)stream;
  float* sums = ws_sums(ws, B, C);
  if (int rc = ffn_sums_pass(x1, du, taps, stats, ws, sums, dgamma, dbeta, B, L, C, st)) return rc;
  return ffn_apply_pass(x1, du, g, taps, aff, stats, sums, nullptr, e, ws, dwf, B, L, C, st);
}

/* Token-mixer backward with batch statistics: dx fp32 (+ bf16 copy dxb, may be null); dwmc [C,1,1,11], dls [C,1,1] and the gamma /
 * beta gradients [C] of BN_ms, BN_mc, BN_ns += theirs (each may be null). */
extern "C" int es3_repmixer_bn_tm_bwd(const float* x, const float* e, const float* taps, const float* aff, const float* stats, float* dx,
                                      void* dxb, float* ws, float* dwmc, float* dls, float* dg_ms, float* db_ms, float* dg_mc,
                                      float* db_mc, float* dg_ns, float* db_ns, int B, int L, int C, void* stream) {
  BS_CHECK_SHAPE("es3_repmixer_bn_tm_bwd", 2);
  cudaStream_t st = (cudaStream_t)stream;
  float* sums = ws_sums(ws, B, C);
  if (int rc = tm_sums_pass(x, e, taps, aff, stats, ws, sums, dg_ms, db_ms, dg_mc, db_mc, dg_ns, db_ns, B, L, C, st)) return rc;
  return tm_apply_pass(x, e, taps, aff, stats, sums, nullptr, dx, dxb, ws, dwmc, dls, B, L, C, st);
}

// ------------------------------------------------------------------------------------------ synchronised BatchNorm
// nn.SyncBatchNorm over several ranks: the forward above split at its two finalize points, the backward at its two sums.  Every
// rank all-gathers the partials (fp64 (count, mean, M2) forward, fp32 sums backward) and combines them in rank order, so the
// statistics and running buffers are bit-identical on every rank.

/* mode 0: part [2][3][C] = (count, mean, M2) of x and c = dw(x; w_mc); mode 1: part [1][3][C] of f = dw(x1; w_f), x1 from
 * fold's wm, bm (es3_repmixer_bn_finalize_sync mode 0).  ws: es3_repmixer_bn_ws_floats(B, C). */
extern "C" int es3_repmixer_bn_stats_partial(const float* x, const float* taps, const float* fold, int mode, float* ws, double* part,
                                             int B, int L, int C, void* stream) {
  BS_CHECK_SHAPE("es3_repmixer_bn_stats_partial", 1);
  ES3_REQUIRE(mode == 0 || mode == 1, "es3_repmixer_bn_stats_partial: mode %d", mode);
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = stats_pass(mode, x, taps, fold, ws, B, L, C, st)) return rc;
  if (mode == 0)
    repmixer_bn_local_kernel<0><<<ceil_div(C, 128), 128, 0, st>>>(ws, B, L, C, part);
  else
    repmixer_bn_local_kernel<1><<<ceil_div(C, 128), 128, 0, st>>>(ws, B, L, C, part);
  ES3_LAUNCH_CHECK("repmixer_bn_local_kernel");
  return 0;
}

/* parts [W][2 | 1][3][C] (every rank's es3_repmixer_bn_stats_partial, rank order) -> as es3_repmixer_bn_fwd's finalize mode 0 | 1:
 * running buffers over the total count, num_batches_tracked, stats and fold rows; total [1] = the count over the group. */
extern "C" int es3_repmixer_bn_finalize_sync(const double* parts, int W, int mode, const float* taps, const float* aff, float* rm_ms,
                                             float* rv_ms, long long* nbt_ms, float* rm_mc, float* rv_mc, long long* nbt_mc, float* rm_ns,
                                             float* rv_ns, long long* nbt_ns, float* rm_f, float* rv_f, long long* nbt_f, float eps_ms,
                                             float eps_mc, float eps_ns, float eps_f, float mom_ms, float mom_mc, float mom_ns,
                                             float mom_f, float* fold, float* stats, double* total, int C, void* stream) {
  ES3_REQUIRE(W >= 1 && C >= SQ_CH && C % SQ_CH == 0, "es3_repmixer_bn_finalize_sync: need W >= 1 and C %% %d == 0", SQ_CH);
  ES3_REQUIRE(mode == 0 || mode == 1, "es3_repmixer_bn_finalize_sync: mode %d", mode);
  cudaStream_t st = (cudaStream_t)stream;
  const BnFinalize f = make_finalize(taps, aff, rm_ms, rv_ms, nbt_ms, rm_mc, rv_mc, nbt_mc, rm_ns, rv_ns, nbt_ns, rm_f, rv_f, nbt_f,
                                     eps_ms, eps_mc, eps_ns, eps_f, mom_ms, mom_mc, mom_ns, mom_f, fold, stats);
  if (mode == 0)
    repmixer_bn_finalize_sync_kernel<0><<<ceil_div(C, 128), 128, 0, st>>>(parts, W, C, f, total);
  else
    repmixer_bn_finalize_sync_kernel<1><<<ceil_div(C, 128), 128, 0, st>>>(parts, W, C, f, total);
  ES3_LAUNCH_CHECK("repmixer_bn_finalize_sync_kernel");
  return 0;
}

/* ConvFFN backward, first half: this rank's sums [2][C] (sum du, sum du fhat) and its BN_f dgamma / dbeta (+=, may be null). */
extern "C" int es3_repmixer_bn_ffn_sums(const float* x1, const float* du, const float* taps, const float* stats, float* ws, float* sums,
                                        float* dgamma, float* dbeta, int B, int L, int C, void* stream) {
  BS_CHECK_SHAPE("es3_repmixer_bn_ffn_sums", 1);
  return ffn_sums_pass(x1, du, taps, stats, ws, sums, dgamma, dbeta, B, L, C, (cudaStream_t)stream);
}

/* ConvFFN backward, second half: parts [W][2][C] (every rank's sums, rank order) and the total count -> e, dwf (+=). */
extern "C" int es3_repmixer_bn_ffn_apply(const float* x1, const float* du, const float* g, const float* taps, const float* aff,
                                         const float* stats, const float* parts, int W, const double* total, float* e, float* ws,
                                         float* dwf, int B, int L, int C, void* stream) {
  BS_CHECK_SHAPE("es3_repmixer_bn_ffn_apply", 1);
  ES3_REQUIRE(W >= 1 && parts && total, "es3_repmixer_bn_ffn_apply: need W >= 1, parts and total");
  cudaStream_t st = (cudaStream_t)stream;
  float* sums = ws_sums(ws, B, C);
  repmixer_bn_sums_kernel<2><<<ceil_div(C, 128), 128, 0, st>>>(parts, W, C, sums, DstBuilder().d);
  ES3_LAUNCH_CHECK("repmixer_bn_sums_kernel<ffn ranks>");
  return ffn_apply_pass(x1, du, g, taps, aff, stats, sums, total, e, ws, dwf, B, L, C, st);
}

/* Token-mixer backward, first half: this rank's sums [3][C] and the gamma / beta gradients of BN_ms, BN_mc, BN_ns (+=, may be null). */
extern "C" int es3_repmixer_bn_tm_sums(const float* x, const float* e, const float* taps, const float* aff, const float* stats, float* ws,
                                       float* sums, float* dg_ms, float* db_ms, float* dg_mc, float* db_mc, float* dg_ns, float* db_ns,
                                       int B, int L, int C, void* stream) {
  BS_CHECK_SHAPE("es3_repmixer_bn_tm_sums", 1);
  return tm_sums_pass(x, e, taps, aff, stats, ws, sums, dg_ms, db_ms, dg_mc, db_mc, dg_ns, db_ns, B, L, C, (cudaStream_t)stream);
}

/* Token-mixer backward, second half: parts [W][3][C] and the total count -> dx (+ bf16 copy dxb, may be null), dwmc, dls (+=). */
extern "C" int es3_repmixer_bn_tm_apply(const float* x, const float* e, const float* taps, const float* aff, const float* stats,
                                        const float* parts, int W, const double* total, float* dx, void* dxb, float* ws, float* dwmc,
                                        float* dls, int B, int L, int C, void* stream) {
  BS_CHECK_SHAPE("es3_repmixer_bn_tm_apply", 1);
  ES3_REQUIRE(W >= 1 && parts && total, "es3_repmixer_bn_tm_apply: need W >= 1, parts and total");
  cudaStream_t st = (cudaStream_t)stream;
  float* sums = ws_sums(ws, B, C);
  repmixer_bn_sums_kernel<3><<<ceil_div(C, 128), 128, 0, st>>>(parts, W, C, sums, DstBuilder().d);
  ES3_LAUNCH_CHECK("repmixer_bn_sums_kernel<tm ranks>");
  return tm_apply_pass(x, e, taps, aff, stats, sums, total, dx, dxb, ws, dwmc, dls, B, L, C, st);
}
