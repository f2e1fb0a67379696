// Backward of MobileCLIP-S0's RepMixerBlock (mobile_clip.py:545-702) with frozen BatchNorm.  With its running statistics each
// BatchNorm is the per-channel affine map BN(v) = s v + b (s = gamma / sqrt(rv + eps), b = beta - rm s, vhat = (v - rm) / sqrt(rv +
// eps)), so the block is exactly its eval function (the forward is es3_repmixer_bf16 on folded taps):
//   c = dw(x; w_mc)   r = BN_ms(x) + BN_mc(c) - BN_ns(x)   x1 = x + ls_tm r
//   f = dw(x1; w_f)   u = BN_f(f)   y = fc2(gelu(fc1(u)))   x2 = x1 + ls_blk y
// dw = the depthwise (1, 11) conv along one sequence, zero padding 5.  Given g = dL/dx2 (fp32):
//   es3_repmixer_ls_bwd   dy = ls_blk g (bf16, the operand of fc2's backward); sums of g y (d ls_blk) and of dy (fc2's bias)
//   es3_repmixer_ffn_bwd  e = g + dw^T(s_f du; w_f); sums of du fhat, du (BN_f's gamma / beta) and s_f du[l] x1[l+k-5] (w_f)
//   es3_repmixer_tm_bwd   e' = ls_tm e, dc = s_mc e', dx = e + (s_ms - s_ns) e' + dw^T(dc; w_mc); sums of e r (ls_tm),
//                         e' xhat_ms, e' xhat_ns, e' chat, e' (the three BNs' gamma / beta) and dc[l] x[l+k-5] (w_mc)
// The CTA layout, the per-CTA partials part [B][Q][C] and their fixed-order reduction (repmixer_sum_kernel) are repmixer_seq.cuh's.
#include "repmixer_seq.cuh"

namespace es3 {
namespace {

constexpr int RB_Q_LS = 2, RB_Q_FFN = SQ_KS + 2, RB_Q_TM = SQ_KS + 5;
static_assert(RB_Q_TM * SQ_ROWS <= SQ_PAD, "the partials' reduction reuses a sequence buffer");

// dy = bf16(ls g); sums of g y and of ls g.
__global__ void __launch_bounds__(SQ_THREADS) repmixer_ls_bwd_kernel(const float* __restrict__ g, const float* __restrict__ y,
                                                                     const float* __restrict__ ls, bf16* __restrict__ dy,
                                                                     float* __restrict__ part, int L, int C) {
  __shared__ float red[RB_Q_LS * SQ_ROWS * SQ_CH];
  const int c = threadIdx.x % SQ_CH, r0 = threadIdx.x / SQ_CH;
  const int ch = blockIdx.x * SQ_CH + c;
  const long long base = (long long)blockIdx.y * L * C + ch;
  const float s = ls[ch];
  float v[RB_Q_LS] = {0.f, 0.f};
  for (int l = r0; l < L; l += SQ_ROWS) {
    const long long i = base + (long long)l * C;
    const float gg = g[i], d = s * gg;
    v[0] = fmaf(gg, y[i], v[0]);
    v[1] += d;
    dy[i] = __float2bfloat16_rn(d);
  }
  cta_partials<RB_Q_LS>(v, red, part, blockIdx.y, C, blockIdx.x * SQ_CH);
}

// bnf: [4][C] = (s_f, b_f, rm_f, 1 / sqrt(rv_f + eps)); wf: raw taps [11][C].
__global__ void __launch_bounds__(SQ_THREADS) repmixer_ffn_bwd_kernel(const float* __restrict__ x1, const float* __restrict__ du,
                                                                      const float* __restrict__ g, const float* __restrict__ wf,
                                                                      const float* __restrict__ bnf, float* __restrict__ e,
                                                                      float* __restrict__ part, int L, int C) {
  __shared__ float sx1[SQ_PAD * SQ_CH];
  __shared__ float sdu[SQ_PAD * SQ_CH];
  const int c = threadIdx.x % SQ_CH, r0 = threadIdx.x / SQ_CH;
  const int ch = blockIdx.x * SQ_CH + c;
  const long long base = (long long)blockIdx.y * L * C + ch;
  for (int l = r0; l < L + 2 * SQ_HALO; l += SQ_ROWS) {
    const int t = l - SQ_HALO;
    const bool in = t >= 0 && t < L;
    sx1[l * SQ_CH + c] = in ? x1[base + (long long)t * C] : 0.f;
    sdu[l * SQ_CH + c] = in ? du[base + (long long)t * C] : 0.f;
  }
  float w[SQ_KS];
#pragma unroll
  for (int k = 0; k < SQ_KS; ++k) w[k] = wf[k * C + ch];
  const float s = bnf[ch], rm = bnf[2 * C + ch], inv = bnf[3 * C + ch];
  float v[RB_Q_FFN];
#pragma unroll
  for (int q = 0; q < RB_Q_FFN; ++q) v[q] = 0.f;
  __syncthreads();
  for (int l = r0; l < L; l += SQ_ROWS) {
    const float d = sdu[(l + SQ_HALO) * SQ_CH + c];
    float f = 0.f, t = 0.f;
#pragma unroll
    for (int k = 0; k < SQ_KS; ++k) {
      const float xv = sx1[(l + k) * SQ_CH + c];                          // x1[l + k - 5]
      f = fmaf(w[k], xv, f);
      v[k] = fmaf(d, xv, v[k]);
      t = fmaf(w[k], sdu[(l + 2 * SQ_HALO - k) * SQ_CH + c], t);           // du[l - k + 5]
    }
    v[SQ_KS] = fmaf(d, (f - rm) * inv, v[SQ_KS]);
    v[SQ_KS + 1] += d;
    const long long i = base + (long long)l * C;
    e[i] = fmaf(s, t, g[i]);
  }
#pragma unroll
  for (int k = 0; k < SQ_KS; ++k) v[k] *= s;
  cta_partials<RB_Q_FFN>(v, sx1, part, blockIdx.y, C, blockIdx.x * SQ_CH);
}

// bnp: [13][C] = (s, b, rm, invstd) of BN_ms, BN_mc, BN_ns, then ls_tm; wmc: raw taps [11][C].
__global__ void __launch_bounds__(SQ_THREADS) repmixer_tm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ e,
                                                                     const float* __restrict__ wmc, const float* __restrict__ bnp,
                                                                     float* __restrict__ dx, bf16* __restrict__ dxb,
                                                                     float* __restrict__ part, int L, int C) {
  __shared__ float sx[SQ_PAD * SQ_CH];
  __shared__ float sdc[SQ_PAD * SQ_CH];
  const int c = threadIdx.x % SQ_CH, r0 = threadIdx.x / SQ_CH;
  const int ch = blockIdx.x * SQ_CH + c;
  const long long base = (long long)blockIdx.y * L * C + ch;
  for (int l = r0; l < L + 2 * SQ_HALO; l += SQ_ROWS) {
    const int t = l - SQ_HALO;
    const bool in = t >= 0 && t < L;
    sx[l * SQ_CH + c] = in ? x[base + (long long)t * C] : 0.f;
    if (!in) sdc[l * SQ_CH + c] = 0.f;
  }
  float w[SQ_KS];
#pragma unroll
  for (int k = 0; k < SQ_KS; ++k) w[k] = wmc[k * C + ch];
  const float s_ms = bnp[ch], b_ms = bnp[C + ch], rm_ms = bnp[2 * C + ch], inv_ms = bnp[3 * C + ch];
  const float s_mc = bnp[4 * C + ch], b_mc = bnp[5 * C + ch], rm_mc = bnp[6 * C + ch], inv_mc = bnp[7 * C + ch];
  const float s_ns = bnp[8 * C + ch], b_ns = bnp[9 * C + ch], rm_ns = bnp[10 * C + ch], inv_ns = bnp[11 * C + ch];
  const float ls = bnp[12 * C + ch];
  const float sd = s_ms - s_ns, br = b_ms + b_mc - b_ns;
  float v[RB_Q_TM];
#pragma unroll
  for (int q = 0; q < RB_Q_TM; ++q) v[q] = 0.f;
  __syncthreads();
  for (int l = r0; l < L; l += SQ_ROWS) {
    const float xv = sx[(l + SQ_HALO) * SQ_CH + c], ev = e[base + (long long)l * C];
    float cv = 0.f;
#pragma unroll
    for (int k = 0; k < SQ_KS; ++k) cv = fmaf(w[k], sx[(l + k) * SQ_CH + c], cv);
    const float r = fmaf(sd, xv, fmaf(s_mc, cv, br));
    const float ep = ls * ev, dc = s_mc * ep;
    sdc[(l + SQ_HALO) * SQ_CH + c] = dc;
#pragma unroll
    for (int k = 0; k < SQ_KS; ++k) v[k] = fmaf(dc, sx[(l + k) * SQ_CH + c], v[k]);
    v[SQ_KS] = fmaf(ev, r, v[SQ_KS]);
    v[SQ_KS + 1] = fmaf(ep, (xv - rm_ms) * inv_ms, v[SQ_KS + 1]);
    v[SQ_KS + 2] = fmaf(ep, (xv - rm_ns) * inv_ns, v[SQ_KS + 2]);
    v[SQ_KS + 3] = fmaf(ep, (cv - rm_mc) * inv_mc, v[SQ_KS + 3]);
    v[SQ_KS + 4] += ep;
  }
  __syncthreads();
  for (int l = r0; l < L; l += SQ_ROWS) {
    const long long i = base + (long long)l * C;
    const float ev = e[i];
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < SQ_KS; ++k) t = fmaf(w[k], sdc[(l + 2 * SQ_HALO - k) * SQ_CH + c], t);   // dc[l - k + 5]
    const float out = fmaf(sd, ls * ev, ev) + t;
    dx[i] = out;
    if (dxb != nullptr) dxb[i] = __float2bfloat16_rn(out);
  }
  cta_partials<RB_Q_TM>(v, sx, part, blockIdx.y, C, blockIdx.x * SQ_CH);
}

}  // namespace
}  // namespace es3

using namespace es3;

#define RB_CHECK_SHAPE(fn)                                                                                                     \
  ES3_REQUIRE(L >= 1 && L <= SQ_MAXL, fn ": sequence length %d outside 1..%d (the sequence is kept in shared memory)", L,  \
              SQ_MAXL);                                                                                                        \
  ES3_REQUIRE(B >= 1 && C >= SQ_CH && C % SQ_CH == 0, fn ": need B >= 1 and C %% %d == 0 (B=%d C=%d)", SQ_CH, B, C)

extern "C" long long es3_repmixer_bwd_ws_floats(int B, int C) { return (long long)B * RB_Q_TM * C; }

/* dy [B*L, C] bf16 = ls * g; dls [C] += sum g y, dbias [C] += sum ls g (either may be null).  g, y fp32 [B*L, C]. */
extern "C" int es3_repmixer_ls_bwd(const float* g, const float* y, const float* ls, void* dy, float* ws, float* dls, float* dbias,
                                   int B, int L, int C, void* stream) {
  RB_CHECK_SHAPE("es3_repmixer_ls_bwd");
  cudaStream_t st = (cudaStream_t)stream;
  repmixer_ls_bwd_kernel<<<dim3(C / SQ_CH, B), SQ_THREADS, 0, st>>>(g, y, ls, (bf16*)dy, ws, L, C);
  ES3_LAUNCH_CHECK("repmixer_ls_bwd_kernel");
  SumBuilder sb(RB_Q_LS);
  sb.add(0, dls);
  sb.add(1, dbias);
  return launch_sums(sb, ws, B, C, st);
}

/* e [B*L, C] fp32 = g + dw^T(s_f du; w_f); dwf [C,1,1,11] += the tap gradient, dgamma / dbeta [C] += BN_f's (each may be null). */
extern "C" int es3_repmixer_ffn_bwd(const float* x1, const float* du, const float* g, const float* wf, const float* bnf, float* e,
                                    float* ws, float* dwf, float* dgamma, float* dbeta, int B, int L, int C, void* stream) {
  RB_CHECK_SHAPE("es3_repmixer_ffn_bwd");
  cudaStream_t st = (cudaStream_t)stream;
  repmixer_ffn_bwd_kernel<<<dim3(C / SQ_CH, B), SQ_THREADS, 0, st>>>(x1, du, g, wf, bnf, e, ws, L, C);
  ES3_LAUNCH_CHECK("repmixer_ffn_bwd_kernel");
  SumBuilder sb(RB_Q_FFN);
  sb.taps(dwf);
  sb.add(SQ_KS, dgamma);
  sb.add(SQ_KS + 1, dbeta);
  return launch_sums(sb, ws, B, C, st);
}

/* dx [B*L, C] fp32 (+ bf16 copy dxb, may be null) = the token mixer's input gradient; dwmc [C,1,1,11], dls [C,1,1] and the
 * gamma / beta gradients [C] of BN_ms (mixer.rbr_skip), BN_mc (mixer.rbr_conv.0.bn), BN_ns (norm.rbr_skip) += theirs. */
extern "C" int es3_repmixer_tm_bwd(const float* x, const float* e, const float* wmc, const float* bnp, float* dx, void* dxb, float* ws,
                                   float* dwmc, float* dls, float* dg_ms, float* db_ms, float* dg_mc, float* db_mc, float* dg_ns,
                                   float* db_ns, int B, int L, int C, void* stream) {
  RB_CHECK_SHAPE("es3_repmixer_tm_bwd");
  cudaStream_t st = (cudaStream_t)stream;
  repmixer_tm_bwd_kernel<<<dim3(C / SQ_CH, B), SQ_THREADS, 0, st>>>(x, e, wmc, bnp, dx, (bf16*)dxb, ws, L, C);
  ES3_LAUNCH_CHECK("repmixer_tm_bwd_kernel");
  SumBuilder sb(RB_Q_TM);
  sb.taps(dwmc);
  sb.add(SQ_KS, dls);
  sb.add(SQ_KS + 1, dg_ms);
  sb.add(SQ_KS + 2, dg_ns, 1, -1.f);
  sb.add(SQ_KS + 3, dg_mc);
  sb.add(SQ_KS + 4, db_ms);
  sb.add(SQ_KS + 4, db_mc);
  sb.add(SQ_KS + 4, db_ns, 1, -1.f);
  return launch_sums(sb, ws, B, C, st);
}
