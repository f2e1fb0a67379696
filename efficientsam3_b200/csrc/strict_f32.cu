// Strict (fp32-class) precision mode: the same graphs on fp32 activations, fp32 weights and fp32 FMA accumulation on the CUDA
// cores.  north_star asks embeddings rtol 1e-4, mask logits rtol 1e-3 and bit-exact binary masks against the reference's
// PyTorch fp32 path; the bf16-operand tensor-core mode is 3e-3 .. 1.5e-2 from it by construction (operand rounding), and the
// reference itself forces its LiteMLA to fp32 (efficientvit/nn/ops.py:586-589).  These kernels are the parity mode, not the fast
// path: one tiled SGEMM with the full epilogue contract of gemm_tc.cu, an im2col that turns every dense / strided / NCHW-image
// convolution into that SGEMM, a depthwise stencil, the ReLU linear attention of LiteMLA in two passes, and the bilinear / layout
// change of the student head.  Reductions run in a fixed order (no atomics): results are bit-reproducible run to run.
#include "common.cuh"

namespace es3 {
namespace {

constexpr int SG_BM = 64, SG_BN = 64, SG_BK = 16;

// out[m,n] = act(scale[n] * sum_k A[m,k] W[n,k] + bias[n]) (+ residual[m,n]) [act after the residual when act_after_res].
// 256 threads, 64 x 64 tile, 4 x 4 outputs per thread, K staged through shared memory 16 at a time (k-major tiles: conflict-free
// float4 reads of 4 consecutive rows / columns).
__global__ void __launch_bounds__(256) sgemm_f32_kernel(const float* __restrict__ A, long long lda, const float* __restrict__ W,
                                                        long long ldw, float* __restrict__ out, long long ldo, int M, int N, int K,
                                                        const float* __restrict__ scale, const float* __restrict__ bias, int act,
                                                        const float* __restrict__ residual, long long ldr, int act_after_res) {
  __shared__ __align__(16) float sA[SG_BK][SG_BM + 4];
  __shared__ __align__(16) float sW[SG_BK][SG_BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;          // thread -> rows ty*4.., cols tx*4..
  const long long m0 = (long long)blockIdx.x * SG_BM;      // M on grid.x (2^31 - 1 blocks): B * H * W rows of a 1024^2 batch
  const int n0 = blockIdx.y * SG_BN;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < K; k0 += SG_BK) {
    // 64 x 16 elements each: thread loads 4 consecutive k of one row
    {
      const int r = tid >> 2, kc = (tid & 3) * 4;
      const long long m = m0 + r;
      const int n = n0 + r;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int k = k0 + kc + e;
        sA[kc + e][r] = (m < M && k < K) ? A[m * lda + k] : 0.f;
        sW[kc + e][r] = (n < N && k < K) ? W[(long long)n * ldw + k] : 0.f;
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < SG_BK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&sA[k][ty * 4]);
      const float4 w = *reinterpret_cast<const float4*>(&sW[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      float v = acc[i][j];
      if (scale) v *= scale[n];
      if (bias) v += bias[n];
      if (!act_after_res) v = es3_act(v, act);
      if (residual) v += residual[m * ldr + n];
      if (act_after_res) v = es3_act(v, act);
      out[m * ldo + n] = v;
    }
  }
}

// cols[(b, oy, ox)][(ky*kw + kx) * C + c] = x[b, oy*s - pad + ky, ox*s - pad + kx, c] (0 outside).  x is NHWC fp32, or the NCHW
// fp32 image when nchw != 0 (the stem reads the loader's tensor directly).
__global__ void im2col_f32_kernel(const float* __restrict__ x, float* __restrict__ cols, int B, int H, int W, int C, int ks, int stride,
                                  int pad, int Ho, int Wo, int nchw, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int Kc = ks * ks * C;
  const long long row = i / Kc;
  const int kk = (int)(i - row * Kc);
  const int tap = kk / C, c = kk - tap * C;
  const int ky = tap / ks, kx = tap - ky * ks;
  const int ox = (int)(row % Wo);
  const long long t = row / Wo;
  const int oy = (int)(t % Ho), b = (int)(t / Ho);
  const int iy = oy * stride - pad + ky, ix = ox * stride - pad + kx;
  float v = 0.f;
  if (iy >= 0 && iy < H && ix >= 0 && ix < W)
    v = nchw ? x[(((long long)b * C + c) * H + iy) * W + ix] : x[(((long long)b * H + iy) * W + ix) * C + c];
  cols[i] = v;
}

// depthwise k x k, stride s, same padding; w [k*k][C] tap-major; y = act(scale[c] * conv + bias[c])
__global__ void dwconv_f32_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ w, const float* __restrict__ scale,
                                  const float* __restrict__ bias, float* __restrict__ y, long long ldy, int B, int H, int W, int C, int ks,
                                  int stride, int Ho, int Wo, int act, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % C);
  const long long p = i / C;
  const int ox = (int)(p % Wo);
  const long long t = p / Wo;
  const int oy = (int)(t % Ho), b = (int)(t / Ho);
  const int pad = ks / 2;
  float acc = 0.f;
  for (int ky = 0; ky < ks; ++ky) {
    const int iy = oy * stride - pad + ky;
    if (iy < 0 || iy >= H) continue;
    for (int kx = 0; kx < ks; ++kx) {
      const int ix = ox * stride - pad + kx;
      if (ix < 0 || ix >= W) continue;
      acc = fmaf(x[(((long long)b * H + iy) * W + ix) * ldx + c], w[(ky * ks + kx) * C + c], acc);
    }
  }
  if (scale) acc *= scale[c];
  if (bias) acc += bias[c];
  y[p * ldy + c] = es3_act(acc, act);
}

// LiteMLA ReLU linear attention (efficientvit/nn/ops.py:584-621), head dim D: ms [B][HW][ld] fp32 with head h at columns
// [3 D h, 3 D (h+1)) = q | k | v.  Pass 1: kv[b][h][i][j] = sum_p v1[p][i] relu(k[p][j]), v1 = (v, 1): i < D + 1, j < D.
// One CTA per (b, head, pixel chunk); thread = one (i, j) entry; partial sums per chunk, then a fixed-order sum.
template <int D>
__global__ void litemla_kv_f32_kernel(const float* __restrict__ ms, long long ld, int HW, int heads, int chunk, float* __restrict__ part) {
  const int b = blockIdx.z, h = blockIdx.y, ch = blockIdx.x;
  const int tid = threadIdx.x;
  constexpr int NE = (D + 1) * D;
  __shared__ float s_k[32][D], s_v[32][D + 1];
  const int p0 = ch * chunk, p1 = min(HW, p0 + chunk);
  float acc[(NE + 255) / 256];
#pragma unroll
  for (int e = 0; e < (NE + 255) / 256; ++e) acc[e] = 0.f;
  for (int pb = p0; pb < p1; pb += 32) {
    for (int t = tid; t < 32 * 2 * D; t += 256) {
      const int r = t / (2 * D), c = t % (2 * D);
      const int p = pb + r;
      float v = 0.f;
      if (p < p1) v = ms[((long long)b * HW + p) * ld + 3 * D * h + D + c];
      if (c < D) s_k[r][c] = fmaxf(v, 0.f);
      else s_v[r][c - D] = v;
    }
    if (tid < 32) s_v[tid][D] = (pb + tid < p1) ? 1.f : 0.f;
    __syncthreads();
#pragma unroll
    for (int e = 0; e < (NE + 255) / 256; ++e) {
      const int idx = tid + e * 256;
      if (idx < NE) {
        const int i = idx / D, j = idx % D;
        float a = acc[e];
#pragma unroll 8
        for (int r = 0; r < 32; ++r) a = fmaf(s_v[r][i], s_k[r][j], a);
        acc[e] = a;
      }
    }
    __syncthreads();
  }
  float* dst = part + (((long long)b * heads + h) * gridDim.x + ch) * NE;
#pragma unroll
  for (int e = 0; e < (NE + 255) / 256; ++e) {
    const int idx = tid + e * 256;
    if (idx < NE) dst[idx] = acc[e];
  }
}

// Pass 2: out[p][h*D + i] = (sum_j kv[i][j] relu(q[p][j])) / (sum_j kv[D][j] relu(q[p][j]) + eps).  Thread = (pixel, head).
template <int D>
__global__ void litemla_apply_f32_kernel(const float* __restrict__ ms, long long ld, int HW, int heads, int nchunk,
                                         const float* __restrict__ part, float eps, float* __restrict__ out, long long ldo) {
  constexpr int NE = (D + 1) * D;
  __shared__ float s_kv[NE];
  const int b = blockIdx.z, h = blockIdx.y;
  const float* src = part + ((long long)b * heads + h) * nchunk * NE;
  for (int idx = threadIdx.x; idx < NE; idx += blockDim.x) {
    float a = 0.f;
    for (int c = 0; c < nchunk; ++c) a += src[(long long)c * NE + idx];
    s_kv[idx] = a;
  }
  __syncthreads();
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const float* qp = ms + ((long long)b * HW + p) * ld + 3 * D * h;
  float q[D];
#pragma unroll
  for (int j = 0; j < D; ++j) q[j] = fmaxf(qp[j], 0.f);
  float den = 0.f;
#pragma unroll
  for (int j = 0; j < D; ++j) den = fmaf(s_kv[D * D + j], q[j], den);
  const float inv = 1.f / (den + eps);
  float* op = out + ((long long)b * HW + p) * ldo + D * h;
#pragma unroll 4
  for (int i = 0; i < D; ++i) {
    float a = 0.f;
#pragma unroll
    for (int j = 0; j < D; ++j) a = fmaf(s_kv[i * D + j], q[j], a);
    op[i] = a * inv;
  }
}

// F.interpolate(mode="bilinear", align_corners=False) from NHWC fp32 [B,Hi,Wi,C] to NCHW fp32 [B,C,Ho,Wo]; equal sizes make it
// the pure layout change (the source index lands on the pixel centre, weights 1 / 0).
__global__ void bilinear_nhwc_f32_to_nchw_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int Hi, int Wi, int C, int Ho,
                                                 int Wo, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int ox = (int)(i % Wo);
  long long t = i / Wo;
  const int oy = (int)(t % Ho);
  t /= Ho;
  const int c = (int)(t % C), b = (int)(t / C);
  const float sy = (float)Hi / (float)Ho, sx = (float)Wi / (float)Wo;
  float fy = ((float)oy + 0.5f) * sy - 0.5f, fx = ((float)ox + 0.5f) * sx - 0.5f;
  fy = fmaxf(fy, 0.f); fx = fmaxf(fx, 0.f);
  const int y0 = min((int)fy, Hi - 1), x0 = min((int)fx, Wi - 1);
  const int y1 = min(y0 + 1, Hi - 1), x1 = min(x0 + 1, Wi - 1);
  const float ly = fy - (float)y0, lx = fx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
  const float* base = x + (long long)b * Hi * Wi * C + c;
  const float v00 = base[((long long)y0 * Wi + x0) * C], v01 = base[((long long)y0 * Wi + x1) * C];
  const float v10 = base[((long long)y1 * Wi + x0) * C], v11 = base[((long long)y1 * Wi + x1) * C];
  y[i] = hy * (hx * v00 + lx * v01) + ly * (hx * v10 + lx * v11);
}


// image -> token attention with few keys (TwoWayAttentionBlock.cross_attn_image_to_token, sam/transformer.py:168-176), fp32 in / out,
// libm expf (the bf16-mode kernel in decoder.cu uses ex2.approx).  Thread = (query row, head).  Keys / values stream through smem
// in tiles of FEW_KEYS_TILE tokens, once per pass of the two-pass softmax (max, then the sum of the exponentials) and once more for
// P V; each pass recomputes the scores with the same fmaf chain, so every pass sees the same fp32 score.
template <int HD>
__global__ void attn_few_keys_f32_kernel(const float* __restrict__ q, long long ldq, const float* __restrict__ k,
                                         const float* __restrict__ v, long long ldkv, float* __restrict__ out, long long ldo, int Nq,
                                         int Tk, int H, float scale) {
  extern __shared__ float skv[];  // [2][cap][H*HD], cap = min(Tk, FEW_KEYS_TILE)
  const int b = blockIdx.y;
  const int D = H * HD, cap = min(Tk, FEW_KEYS_TILE), ntile = (Tk + FEW_KEYS_TILE - 1) / FEW_KEYS_TILE;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const bool active = idx < Nq * H;   // inactive threads still take part in the tile loads and barriers
  const int h = idx % H, n = idx / H;
  const float* qp = q + ((long long)b * Nq + n) * ldq + h * HD;
  float qr[HD], o[HD];
#pragma unroll
  for (int d = 0; d < HD; ++d) { qr[d] = active ? qp[d] : 0.f; o[d] = 0.f; }
  float mx = -INFINITY, l = 0.f, inv = 0.f;
  for (int pass = 0; pass < 3; ++pass) {   // 0: row max; 1: l = sum of exp; 2: o = sum of (exp / l) v
    if (pass == 2) inv = 1.f / l;
    for (int tile = 0; tile < ntile; ++tile) {
      const int t0 = tile * FEW_KEYS_TILE, nt = min(FEW_KEYS_TILE, Tk - t0);
      if (pass == 0 || ntile > 1) few_keys_load_tile(skv, k, v, ldkv, (long long)b * Tk + t0, nt, cap, D);
      if (!active) continue;
      for (int t = 0; t < nt; ++t) {
        const float* kp = skv + t * D + h * HD;
        float a = 0.f;
#pragma unroll
        for (int d = 0; d < HD; ++d) a = fmaf(qr[d], kp[d], a);
        const float s = __fmul_rn(a, scale);   // rounded before the max and the subtraction: no contraction into an fma
        if (pass == 0) { mx = fmaxf(mx, s); continue; }
        const float p = expf(s - mx);
        if (pass == 1) { l += p; continue; }
        const float w = p * inv;
        const float* vp = skv + cap * D + t * D + h * HD;
#pragma unroll
        for (int d = 0; d < HD; ++d) o[d] = fmaf(w, vp[d], o[d]);
      }
    }
  }
  if (!active) return;
  float* op = out + ((long long)b * Nq + n) * ldo + h * HD;
#pragma unroll
  for (int d = 0; d < HD; ++d) op[d] = o[d];
}

// y = gelu_erf(LayerNorm(x) * w + b) over rows of C <= 128 channels, fp32 out (MaskDecoder.output_upscaling, mask_decoder.py:59-70).
__global__ void ln_rows_gelu_f32_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                        float eps, float* __restrict__ y, long long M, int C) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  const int per = C >> 5;
  float v[4];
  float s = 0.f;
  for (int i = 0; i < per; ++i) { v[i] = x[row * C + lane + i * 32]; s += v[i]; }
  const float mean = warp_sum(s) / C;
  float qv = 0.f;
  for (int i = 0; i < per; ++i) { const float d = v[i] - mean; qv += d * d; }
  const float rstd = 1.f / sqrtf(warp_sum(qv) / C + eps);
  for (int i = 0; i < per; ++i) {
    const int c = lane + i * 32;
    y[row * C + c] = es3_act((v[i] - mean) * rstd * w[c] + bias[c], ACT_GELU);
  }
}

// y = LayerNorm(x) * w + b over rows of any width C, fp32 in / out, two-pass (mean, then centred variance) per row: warp = row.
// nn.LayerNorm of the strict TinyViT walk (tiny_vit.py:235, 259: C = 64 .. 576, not multiples of 128).
__global__ void ln_rows_f32_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias, float eps,
                                   float* __restrict__ y, long long M, int C) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  const float* xr = x + row * C;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += xr[c];
  const float mean = warp_sum(s) / C;
  float qv = 0.f;
  for (int c = lane; c < C; c += 32) { const float d = xr[c] - mean; qv = fmaf(d, d, qv); }
  const float rstd = 1.f / sqrtf(warp_sum(qv) / C + eps);
  float* yr = y + row * C;
  for (int c = lane; c < C; c += 32) yr[c] = (xr[c] - mean) * rstd * w[c] + bias[c];
}

// y[m][c] = act(x[m][c] + bias[c]) + residual  |  act(x + bias + residual)   (elementwise tail of the strict ConvTranspose path)
__global__ void bias_act_res_f32_kernel(const float* __restrict__ x, const float* __restrict__ bias, const float* __restrict__ residual,
                                        float* __restrict__ y, long long total, int C, int act, int act_after_res) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  float v = x[i];
  if (bias) v += bias[i % C];
  if (!act_after_res) v = es3_act(v, act);
  if (residual) v += residual[i];
  if (act_after_res) v = es3_act(v, act);
  y[i] = v;
}

// 2-D axial RoPE of the q and k heads, in place on fp32 qkv rows (vitdet.py:68-90 apply_rotary_enc): columns [0, rope_cols) are heads
// of 64 dims = 32 complex pairs (2 i, 2 i + 1); table [positions][32] (cos, sin); position = window-local index when win > 0.
__global__ void rope_f32_kernel(float* __restrict__ qkv, long long ld, const float2* __restrict__ table, int rope_cols, int H, int W,
                                int win, long long total_pairs) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total_pairs) return;
  const int ppr = rope_cols >> 1;                    // pairs per row
  const long long row = i / ppr;
  const int pr = (int)(i - row * ppr);
  const int t = (int)(row % ((long long)H * W));
  const int h = t / W, w = t - h * W;
  const int pidx = win ? (h % win) * win + (w % win) : t;
  const float2 cs = table[(long long)pidx * 32 + (pr & 31)];
  float* p = qkv + row * ld + 2 * pr;
  const float x0 = p[0], x1 = p[1];
  p[0] = x0 * cs.x - x1 * cs.y;
  p[1] = x0 * cs.y + x1 * cs.x;
}

// softmax(q k^T scale + bias) v in fp32 over (optionally windowed) token grids.  Rows of `qkv` are tokens [B*H*W][ld]; head h reads
// q / k / v at columns q_off + h * head_stride (k_off, v_off alike) -- the ViT trunk's q | k | v blocks (head_stride = D) and TinyViT's
// per-head (q, k, v) triples (head_stride = 3 D) are both this.  win > 0: win x win windows gathered in place; a window that
// overhangs the grid takes `pad_row` (one qkv row, the projection of a zero-padded token) for the missing tokens, whose outputs are
// dropped (tiny_vit.py:352-372).  bias [heads][L][L] optional.  Thread = one query: q and the running output in registers, keys /
// values staged 64 at a time in shared memory, online softmax with libm expf.
template <int D>
__global__ void __launch_bounds__(128) attn_f32_kernel(const float* __restrict__ qkv, float* __restrict__ out, const float* __restrict__ bias,
                                                       const float* __restrict__ pad_row, int H, int W, int ld, int ldo, int q_off, int k_off,
                                                       int v_off, int head_stride, int win, int nwx, int nwin, int L, float scale) {
  __shared__ __align__(16) float s_k[64][D];
  __shared__ __align__(16) float s_v[64][D];
  const int head = blockIdx.y;
  const int b = blockIdx.z / nwin, wi = blockIdx.z % nwin;
  auto token_row = [&](int l) -> long long {          // -1: a padded position of an overhanging window
    if (win == 0) return (long long)b * H * W + l;
    const int wy = wi / nwx, wx = wi % nwx;
    const int y = wy * win + l / win, x = wx * win + l % win;
    if (y >= H || x >= W) return -1;
    return (long long)b * H * W + (long long)y * W + x;
  };
  const int lq = blockIdx.x * 128 + threadIdx.x;
  const long long row_q = lq < L ? token_row(lq) : -1;
  const bool live = row_q >= 0;
  float q[D], o[D];
  {
    const float* qp = live ? qkv + row_q * ld + q_off + head * head_stride : nullptr;
#pragma unroll
    for (int d = 0; d < D; ++d) q[d] = live ? qp[d] * scale : 0.f;
  }
#pragma unroll
  for (int d = 0; d < D; ++d) o[d] = 0.f;
  float m = -INFINITY, lsum = 0.f;
  const float* brow = (bias && lq < L) ? bias + ((long long)head * L + lq) * L : nullptr;
  for (int k0 = 0; k0 < L; k0 += 64) {
    __syncthreads();
    for (int i = threadIdx.x; i < 64 * (D / 4); i += 128) {
      const int r = i / (D / 4), c4 = i % (D / 4);
      float4 kk = make_float4(0.f, 0.f, 0.f, 0.f), vv = kk;
      if (k0 + r < L) {
        const long long tr = token_row(k0 + r);
        const float* base = (tr >= 0 ? qkv + tr * ld : pad_row) + head * head_stride + c4 * 4;
        kk = *reinterpret_cast<const float4*>(base + k_off);
        vv = *reinterpret_cast<const float4*>(base + v_off);
      }
      *reinterpret_cast<float4*>(&s_k[r][c4 * 4]) = kk;
      *reinterpret_cast<float4*>(&s_v[r][c4 * 4]) = vv;
    }
    __syncthreads();
    const int nk = min(64, L - k0);
    for (int j = 0; j < nk; ++j) {
      float sc = 0.f;
#pragma unroll
      for (int d4 = 0; d4 < D / 4; ++d4) {
        const float4 kk = *reinterpret_cast<const float4*>(&s_k[j][d4 * 4]);
        sc = fmaf(q[d4 * 4], kk.x, sc); sc = fmaf(q[d4 * 4 + 1], kk.y, sc); sc = fmaf(q[d4 * 4 + 2], kk.z, sc); sc = fmaf(q[d4 * 4 + 3], kk.w, sc);
      }
      if (brow) sc += brow[k0 + j];
      if (sc > m) {                                   // new running maximum: rescale what has been accumulated
        const float corr = expf(m - sc);
        lsum *= corr;
#pragma unroll
        for (int d = 0; d < D; ++d) o[d] *= corr;
        m = sc;
      }
      const float p = expf(sc - m);
      lsum += p;
#pragma unroll
      for (int d4 = 0; d4 < D / 4; ++d4) {
        const float4 vv = *reinterpret_cast<const float4*>(&s_v[j][d4 * 4]);
        o[d4 * 4] = fmaf(p, vv.x, o[d4 * 4]); o[d4 * 4 + 1] = fmaf(p, vv.y, o[d4 * 4 + 1]);
        o[d4 * 4 + 2] = fmaf(p, vv.z, o[d4 * 4 + 2]); o[d4 * 4 + 3] = fmaf(p, vv.w, o[d4 * 4 + 3]);
      }
    }
  }
  if (live) {
    const float inv = 1.f / lsum;
    float* op = out + row_q * ldo + head * D;
#pragma unroll
    for (int d = 0; d < D; ++d) op[d] = o[d] * inv;
  }
}

// per-(image, channel) gate: y[b][p][c] = x[b][p][c] * gate[b][c]   (SqueezeExcite excitation, fp32)
__global__ void scale_channels_f32_kernel(const float* __restrict__ x, const float* __restrict__ gate, float* __restrict__ y, long long HW,
                                          int C, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % C);
  const long long b = i / ((long long)HW * C);
  y[i] = x[i] * gate[b * C + c];
}
}  // namespace
}  // namespace es3

using namespace es3;

extern "C" int es3_sgemm_f32(const float* A, long long lda, const float* W, long long ldw, float* out, long long ldo, long long M, int N,
                             int K, const float* scale, const float* bias, int act, const float* residual, long long ldr,
                             int act_after_res, void* stream) {
  ES3_REQUIRE(M > 0 && N > 0 && K > 0 && M < (1LL << 31), "es3_sgemm_f32: bad shape M=%lld N=%d K=%d", M, N, K);
  dim3 grid((unsigned)ceil_div(M, SG_BM), ceil_div(N, SG_BN));
  sgemm_f32_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(A, lda, W, ldw, out, ldo, (int)M, N, K, scale, bias, act, residual, ldr,
                                                          act_after_res);
  ES3_LAUNCH_CHECK("sgemm_f32_kernel");
  return 0;
}

extern "C" int es3_im2col_f32(const float* x, float* cols, int B, int H, int W, int C, int ks, int stride, int pad, int nchw,
                              void* stream) {
  ES3_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && ks > 0 && stride > 0, "es3_im2col_f32: bad shape");
  const int Ho = (H + 2 * pad - ks) / stride + 1, Wo = (W + 2 * pad - ks) / stride + 1;
  const long long total = (long long)B * Ho * Wo * ks * ks * C;
  im2col_f32_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, cols, B, H, W, C, ks, stride, pad, Ho, Wo, nchw,
                                                                                      total);
  ES3_LAUNCH_CHECK("im2col_f32_kernel");
  return 0;
}

extern "C" int es3_dwconv_f32(const float* x, long long ldx, const float* w, const float* scale, const float* bias, float* y, long long ldy,
                              int B, int H, int W, int C, int ks, int stride, int act, void* stream) {
  ES3_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && (ks & 1) && stride > 0, "es3_dwconv_f32: bad shape");
  const int pad = ks / 2;
  const int Ho = (H + 2 * pad - ks) / stride + 1, Wo = (W + 2 * pad - ks) / stride + 1;
  const long long total = (long long)B * Ho * Wo * C;
  ES3_REQUIRE(ldx >= C && ldy >= C, "es3_dwconv_f32: pixel strides (%lld, %lld) below C=%d", ldx, ldy, C);
  dwconv_f32_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, ldx, w, scale, bias, y, ldy, B, H, W, C, ks,
                                                                                      stride, Ho, Wo, act, total);
  ES3_LAUNCH_CHECK("dwconv_f32_kernel");
  return 0;
}

static int litemla_f32_chunks(int HW, int* chunk) {
  int n = ceil_div(HW, 2048);
  if (n < 1) n = 1;
  *chunk = ceil_div(ceil_div(HW, n), 32) * 32;
  return ceil_div(HW, *chunk);
}

extern "C" long long es3_litemla_attn_f32_ws_floats(int B, int HW, int heads, int dim) {
  int chunk;
  return (long long)B * heads * litemla_f32_chunks(HW, &chunk) * (dim + 1) * dim;
}

/* ms [B][HW][ld] fp32 (head h: q | k | v at columns 3 dim h ...), out [B][HW][ldo] fp32 (head h at columns dim h). */
extern "C" int es3_litemla_attn_f32(const float* ms, long long ld, float* ws, float* out, long long ldo, int B, int HW, int heads, int dim,
                                    float eps, void* stream) {
  ES3_REQUIRE(dim == 16 || dim == 32, "es3_litemla_attn_f32: head dim %d not instantiated (16, 32)", dim);
  ES3_REQUIRE(B > 0 && HW > 0 && heads > 0 && ld >= 3LL * dim * heads && ldo >= (long long)dim * heads, "es3_litemla_attn_f32: bad shape");
  int chunk;
  const int nchunk = litemla_f32_chunks(HW, &chunk);
  cudaStream_t st = (cudaStream_t)stream;
  dim3 g1(nchunk, heads, B), g2(ceil_div(HW, 128), heads, B);
  if (dim == 16) {
    litemla_kv_f32_kernel<16><<<g1, 256, 0, st>>>(ms, ld, HW, heads, chunk, ws);
    ES3_LAUNCH_CHECK("litemla_kv_f32_kernel");
    litemla_apply_f32_kernel<16><<<g2, 128, 0, st>>>(ms, ld, HW, heads, nchunk, ws, eps, out, ldo);
  } else {
    litemla_kv_f32_kernel<32><<<g1, 256, 0, st>>>(ms, ld, HW, heads, chunk, ws);
    ES3_LAUNCH_CHECK("litemla_kv_f32_kernel");
    litemla_apply_f32_kernel<32><<<g2, 128, 0, st>>>(ms, ld, HW, heads, nchunk, ws, eps, out, ldo);
  }
  ES3_LAUNCH_CHECK("litemla_apply_f32_kernel");
  return 0;
}

extern "C" int es3_bilinear_nhwc_f32_to_nchw(const float* x, float* y, int B, int Hi, int Wi, int C, int Ho, int Wo, void* stream) {
  ES3_REQUIRE(B > 0 && Hi > 0 && Wi > 0 && C > 0 && Ho > 0 && Wo > 0, "es3_bilinear_nhwc_f32_to_nchw: bad shape");
  const long long total = (long long)B * C * Ho * Wo;
  bilinear_nhwc_f32_to_nchw_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, y, B, Hi, Wi, C, Ho, Wo, total);
  ES3_LAUNCH_CHECK("bilinear_nhwc_f32_to_nchw_kernel");
  return 0;
}

extern "C" int es3_attn_few_keys_f32(const float* q, long long ldq, const float* k, const float* v, long long ldkv, float* out,
                                     long long ldo, int B, int H, int head_dim, int Nq, int Tk, float scale, void* stream) {
  ES3_REQUIRE(head_dim == 16 && Tk > 0, "es3_attn_few_keys_f32: head_dim must be 16 and Tk > 0 (got %d, %d)", head_dim, Tk);
  const int smem = 2 * std::min(Tk, FEW_KEYS_TILE) * H * head_dim * (int)sizeof(float);
  dim3 grid(ceil_div((long long)Nq * H, 256), B);
  attn_few_keys_f32_kernel<16><<<grid, 256, smem, (cudaStream_t)stream>>>(q, ldq, k, v, ldkv, out, ldo, Nq, Tk, H, scale);
  ES3_LAUNCH_CHECK("attn_few_keys_f32_kernel");
  return 0;
}

extern "C" int es3_ln_rows_gelu_f32(const float* x, const float* w, const float* bias, float eps, float* y, long long M, int C,
                                    void* stream) {
  ES3_REQUIRE(C % 32 == 0 && C <= 128, "es3_ln_rows_gelu_f32: C=%d must be a multiple of 32 and <= 128", C);
  ln_rows_gelu_f32_kernel<<<(unsigned)ceil_div(M, 8), 256, 0, (cudaStream_t)stream>>>(x, w, bias, eps, y, M, C);
  ES3_LAUNCH_CHECK("ln_rows_gelu_f32_kernel");
  return 0;
}

extern "C" int es3_ln_rows_f32(const float* x, const float* w, const float* bias, float eps, float* y, long long M, int C, void* stream) {
  ES3_REQUIRE(M > 0 && C > 0, "es3_ln_rows_f32: bad shape");
  ln_rows_f32_kernel<<<(unsigned)ceil_div(M, 8), 256, 0, (cudaStream_t)stream>>>(x, w, bias, eps, y, M, C);
  ES3_LAUNCH_CHECK("ln_rows_f32_kernel");
  return 0;
}

extern "C" int es3_bias_act_res_f32(const float* x, const float* bias, const float* residual, float* y, long long total, int C, int act,
                                    int act_after_res, void* stream) {
  ES3_REQUIRE(total > 0 && C > 0, "es3_bias_act_res_f32: bad shape");
  bias_act_res_f32_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, bias, residual, y, total, C, act,
                                                                                            act_after_res);
  ES3_LAUNCH_CHECK("bias_act_res_f32_kernel");
  return 0;
}

/* In-place 2-D axial RoPE on columns [0, rope_cols) of fp32 rows (q | k heads of 64 dims); table [positions][32][2] = (cos, sin). */
extern "C" int es3_rope_f32(float* qkv, long long ld, long long rows, const float* table, int rope_cols, int H, int W, int win, void* stream) {
  ES3_REQUIRE(rows > 0 && rope_cols % 64 == 0 && H > 0 && W > 0 && rows % ((long long)H * W) == 0, "es3_rope_f32: bad arguments");
  const long long total = rows * (rope_cols / 2);
  rope_f32_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(qkv, ld, reinterpret_cast<const float2*>(table),
                                                                                    rope_cols, H, W, win, total);
  ES3_LAUNCH_CHECK("rope_f32_kernel");
  return 0;
}

/* fp32 softmax attention over token rows (see attn_f32_kernel): ViT trunk = (q_off 0, k_off C, v_off 2C, head_stride D),
 * TinyViT = (0, D, 2D, 3D) with bias [heads][win^2][win^2] and pad_row; out [B*H*W][heads*D]. */
extern "C" int es3_attention_f32(const float* qkv, float* out, const float* bias, const float* pad_row, int B, int H, int W, int ld,
                                 int num_heads, int head_dim, int q_off, int k_off, int v_off, int head_stride, int win, float scale,
                                 void* stream) {
  ES3_REQUIRE(head_dim == 32 || head_dim == 64, "es3_attention_f32: head_dim must be 32 or 64 (got %d)", head_dim);
  ES3_REQUIRE(B > 0 && H > 0 && W > 0 && ld % 4 == 0 && q_off % 4 == 0 && k_off % 4 == 0 && v_off % 4 == 0 && head_stride % 4 == 0,
              "es3_attention_f32: bad layout");
  // keys and values are read as float4 from qkv rows and from pad_row
  ES3_REQUIRE(((uintptr_t)qkv & 15) == 0 && ((uintptr_t)pad_row & 15) == 0, "es3_attention_f32: qkv and pad_row must be 16-byte aligned");
  ES3_REQUIRE(win >= 0 && (win == 0 || (H % win == 0 && W % win == 0) || pad_row != nullptr),
              "es3_attention_f32: windows overhang the %dx%d grid and no pad_row was given", H, W);
  const int nwx = win ? ceil_div(W, win) : 1, nwin = win ? ceil_div(H, win) * nwx : 1;
  const int L = win ? win * win : H * W;
  const dim3 grid(ceil_div(L, 128), num_heads, B * nwin);
  const int ldo = num_heads * head_dim;
  if (head_dim == 64)
    attn_f32_kernel<64><<<grid, 128, 0, (cudaStream_t)stream>>>(qkv, out, bias, pad_row, H, W, ld, ldo, q_off, k_off, v_off, head_stride,
                                                                 win, nwx, nwin, L, scale);
  else
    attn_f32_kernel<32><<<grid, 128, 0, (cudaStream_t)stream>>>(qkv, out, bias, pad_row, H, W, ld, ldo, q_off, k_off, v_off, head_stride,
                                                                 win, nwx, nwin, L, scale);
  ES3_LAUNCH_CHECK("attn_f32_kernel");
  return 0;
}

extern "C" int es3_scale_channels_f32(const float* x, const float* gate, float* y, int B, long long HW, int C, void* stream) {
  ES3_REQUIRE(B > 0 && HW > 0 && C > 0, "es3_scale_channels_f32: bad shape");
  const long long total = (long long)B * HW * C;
  scale_channels_f32_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, gate, y, HW, C, total);
  ES3_LAUNCH_CHECK("scale_channels_f32_kernel");
  return 0;
}
