// Backward kernels of the MobileCLIP text students (base trunk of TransformerEncoder layers, mobile_clip.py:345-491, 815-823)
// and the stage-1 text KD loss (train_text_encoder_stage1.py:244-270, 336-370):
//   es3_text_attn_bwd        attention backward, head_dim 64, L <= 128, causal or not: dqkv in the forward's qkv layout
//   es3_layernorm_bwd_f32    LayerNorm backward over the fp32 residual stream: fp32 dx (+ fp32 residual gradient, + bf16 copy)
//   es3_text_embed_grad      nn.Embedding weight gradient: chunked segmented sum over tokens sorted by id (host permutation)
//   es3_text_pos_grad        positional-table gradient: batch sum, then the transpose of the 1-D linear resize N -> L
//   es3_text_kd_loss_fwd/bwd text MSE + cosine (masked or not) with per-sample partials and a fixed-order final reduction
//   es3_text_consistency_fwd/bwd  mse(mean_L(p), mean_L(q)) and its gradient into both inputs
//   es3_cast_f32_to_bf16     GEMM operand copy of an fp32 gradient
// Every reduction runs in a fixed order (no float atomics), so a backward pass is bit-reproducible.
#include "common.cuh"

namespace es3 {
namespace {

// ------------------------------------------------------------------------------------------ attention backward
// One CTA per (sequence, head).  q, k, v, dO of the sequence are staged in shared memory as bf16 (exactly the values of the
// forward's operands) with a row pitch of 66 elements (33 words: row-strided reads by consecutive lanes hit distinct banks);
// P and dS are fp32 [L][L + 1].  Forward: S = scale q k^T (+ causal -inf above the diagonal), P = softmax_row(S), O = P v.
// Backward: D_i = sum_c dO_ic O_ic, dP = dO v^T, dS = P (dP - D), dQ = scale dS k, dK = scale dS^T q, dV = P^T dO.
// fp32 FMA on the CUDA cores: at L <= 128 and head_dim 64 a CTA does 5 L^2 64 multiply-adds on operands that already sit in
// shared memory.  Each output element is one thread's sum over a fixed index order.
constexpr int TA_D = 64, TA_LD = 66, TA_THREADS = 256, TA_MAXL = 128;

__device__ __forceinline__ float dot64(const bf16* a, const bf16* b) {
  const __nv_bfloat162* a2 = reinterpret_cast<const __nv_bfloat162*>(a);
  const __nv_bfloat162* b2 = reinterpret_cast<const __nv_bfloat162*>(b);
  float s0 = 0.f, s1 = 0.f;
#pragma unroll
  for (int c = 0; c < TA_D / 2; ++c) {
    const float2 x = __bfloat1622float2(a2[c]), y = __bfloat1622float2(b2[c]);
    s0 = fmaf(x.x, y.x, s0);
    s1 = fmaf(x.y, y.y, s1);
  }
  return s0 + s1;
}

template <bool CAUSAL>
__global__ void __launch_bounds__(TA_THREADS) text_attn_bwd_kernel(const bf16* __restrict__ qkv, const bf16* __restrict__ o,
                                                                   const bf16* __restrict__ dout, bf16* __restrict__ dqkv, int L, int C,
                                                                   float scale) {
  extern __shared__ __align__(16) uint8_t ta_smem[];
  bf16* s_q = reinterpret_cast<bf16*>(ta_smem);
  bf16* s_k = s_q + L * TA_LD;
  bf16* s_v = s_k + L * TA_LD;
  bf16* s_do = s_v + L * TA_LD;
  float* s_p = reinterpret_cast<float*>(s_do + L * TA_LD);      // 4 L 66 bf16 = 528 L bytes: 16-byte aligned
  float* s_ds = s_p + L * (L + 1);
  float* s_D = s_ds + L * (L + 1);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.x, head = blockIdx.y;
  const long long ld = 3LL * C;
  const long long tok0 = (long long)b * L;

  // stage q, k, v, dO (32-bit words: 32 per 64-channel row) and D_i = sum_c dO_ic O_ic
  for (int i = tid; i < L * 32; i += TA_THREADS) {
    const int r = i >> 5, w = i & 31;
    const uint32_t* row = reinterpret_cast<const uint32_t*>(qkv + (tok0 + r) * ld + head * TA_D);
    reinterpret_cast<uint32_t*>(s_q + r * TA_LD)[w] = row[w];
    reinterpret_cast<uint32_t*>(s_k + r * TA_LD)[w] = row[C / 2 + w];
    reinterpret_cast<uint32_t*>(s_v + r * TA_LD)[w] = row[C + w];
    reinterpret_cast<uint32_t*>(s_do + r * TA_LD)[w] =
        reinterpret_cast<const uint32_t*>(dout + (tok0 + r) * C + head * TA_D)[w];
  }
  for (int r = warp; r < L; r += TA_THREADS / 32) {
    const float2 d = unpack_bf16x2(reinterpret_cast<const uint32_t*>(dout + (tok0 + r) * C + head * TA_D)[lane]);
    const float2 y = unpack_bf16x2(reinterpret_cast<const uint32_t*>(o + (tok0 + r) * C + head * TA_D)[lane]);
    const float s = warp_sum(fmaf(d.x, y.x, d.y * y.y));
    if (lane == 0) s_D[r] = s;
  }
  __syncthreads();
  // S and dP
  for (int idx = tid; idx < L * L; idx += TA_THREADS) {
    const int i = idx / L, j = idx - i * L;
    float s = -INFINITY, dp = 0.f;
    if (!CAUSAL || j <= i) {
      s = dot64(s_q + i * TA_LD, s_k + j * TA_LD) * scale;
      dp = dot64(s_do + i * TA_LD, s_v + j * TA_LD);
    }
    s_p[i * (L + 1) + j] = s;
    s_ds[i * (L + 1) + j] = dp;
  }
  __syncthreads();
  // row softmax (a warp per row), then dS = P (dP - D)
  for (int i = warp; i < L; i += TA_THREADS / 32) {
    float* pr = s_p + i * (L + 1);
    float* dr = s_ds + i * (L + 1);
    float mx = -INFINITY;
    for (int j = lane; j < L; j += 32) mx = fmaxf(mx, pr[j]);
    mx = warp_max(mx);
    float sum = 0.f;
    for (int j = lane; j < L; j += 32) {
      const float e = expf(pr[j] - mx);          // exp(-inf) = 0 above the diagonal
      pr[j] = e;
      sum += e;
    }
    const float inv = 1.f / warp_sum(sum);
    const float Di = s_D[i];
    for (int j = lane; j < L; j += 32) {
      const float p = pr[j] * inv;
      pr[j] = p;
      dr[j] = p * (dr[j] - Di);
    }
  }
  __syncthreads();
  // dQ_i = scale sum_j dS_ij k_j ; dK_j = scale sum_i dS_ij q_i ; dV_j = sum_i P_ij dO_i   (thread = row x channel pair)
  for (int idx = tid; idx < L * 32; idx += TA_THREADS) {
    const int r = idx >> 5, w = idx & 31;
    float2 dq = make_float2(0.f, 0.f), dk = dq, dv = dq;
    const int j_end = CAUSAL ? r + 1 : L;
    for (int j = 0; j < j_end; ++j) {
      const float ds = s_ds[r * (L + 1) + j];
      const float2 kk = unpack_bf16x2(reinterpret_cast<const uint32_t*>(s_k + j * TA_LD)[w]);
      dq.x = fmaf(ds, kk.x, dq.x); dq.y = fmaf(ds, kk.y, dq.y);
    }
    for (int i = CAUSAL ? r : 0; i < L; ++i) {
      const float ds = s_ds[i * (L + 1) + r], p = s_p[i * (L + 1) + r];
      const float2 qq = unpack_bf16x2(reinterpret_cast<const uint32_t*>(s_q + i * TA_LD)[w]);
      const float2 gg = unpack_bf16x2(reinterpret_cast<const uint32_t*>(s_do + i * TA_LD)[w]);
      dk.x = fmaf(ds, qq.x, dk.x); dk.y = fmaf(ds, qq.y, dk.y);
      dv.x = fmaf(p, gg.x, dv.x); dv.y = fmaf(p, gg.y, dv.y);
    }
    uint32_t* out = reinterpret_cast<uint32_t*>(dqkv + (tok0 + r) * ld + head * TA_D);
    out[w] = pack_bf16x2(dq.x * scale, dq.y * scale);
    out[C / 2 + w] = pack_bf16x2(dk.x * scale, dk.y * scale);
    out[C + w] = pack_bf16x2(dv.x, dv.y);
  }
}

// ------------------------------------------------------------------------------------------ LayerNorm backward (fp32 rows)
// Same scheme as es3_layernorm_bwd (a warp per row, per-lane dgamma / dbeta partials over the block's rows, cross-warp sums in
// shared memory, per-block partials summed by a finalize kernel in block order) on fp32 x / dy / dres, float4 per lane-vector.
constexpr int LNF_MAXV = 6;    // C <= 6 * 4 * 32 = 768
__global__ void __launch_bounds__(256) layernorm_bwd_f32_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                                const float* __restrict__ gamma, const float* __restrict__ dres,
                                                                float eps, float* __restrict__ dx, bf16* __restrict__ dxb, long long M,
                                                                int C, long long rows_per_block, float* __restrict__ part) {
  __shared__ float red[8][LNF_MAXV * 128];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int CV = C >> 2;
  float dg[LNF_MAXV][4], db[LNF_MAXV][4];
#pragma unroll
  for (int v = 0; v < LNF_MAXV; ++v)
#pragma unroll
    for (int k = 0; k < 4; ++k) dg[v][k] = db[v][k] = 0.f;
  const long long r0 = (long long)blockIdx.x * rows_per_block, r1 = min(M, r0 + rows_per_block);
  const float inv_c = 1.f / (float)C;
  for (long long r = r0 + warp; r < r1; r += 8) {
    float xv[LNF_MAXV][4], gv[LNF_MAXV][4];
    float s = 0.f;
#pragma unroll
    for (int v = 0; v < LNF_MAXV; ++v) {
      const int cv = lane + 32 * v;
      if (cv < CV) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(x + r * C) + cv);
        xv[v][0] = t.x; xv[v][1] = t.y; xv[v][2] = t.z; xv[v][3] = t.w;
        s += (t.x + t.y) + (t.z + t.w);
      }
    }
    const float mu = warp_sum(s) * inv_c;
    float q = 0.f;
#pragma unroll
    for (int v = 0; v < LNF_MAXV; ++v) {
      if (lane + 32 * v < CV) {
#pragma unroll
        for (int k = 0; k < 4; ++k) { const float d = xv[v][k] - mu; q = fmaf(d, d, q); }
      }
    }
    const float rstd = rsqrtf(warp_sum(q) * inv_c + eps);
    float sg = 0.f, sgx = 0.f;
#pragma unroll
    for (int v = 0; v < LNF_MAXV; ++v) {
      const int cv = lane + 32 * v;
      if (cv < CV) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(dy + r * C) + cv);
        const float4 gm = __ldg(reinterpret_cast<const float4*>(gamma) + cv);
        const float d[4] = {t.x, t.y, t.z, t.w}, gk[4] = {gm.x, gm.y, gm.z, gm.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float xh = (xv[v][k] - mu) * rstd;
          xv[v][k] = xh;
          dg[v][k] = fmaf(d[k], xh, dg[v][k]);
          db[v][k] += d[k];
          const float g = d[k] * gk[k];
          gv[v][k] = g;
          sg += g;
          sgx = fmaf(g, xh, sgx);
        }
      }
    }
    const float c1 = warp_sum(sg) * inv_c, c2 = warp_sum(sgx) * inv_c;
#pragma unroll
    for (int v = 0; v < LNF_MAXV; ++v) {
      const int cv = lane + 32 * v;
      if (cv < CV) {
        float out[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) out[k] = rstd * (gv[v][k] - c1 - xv[v][k] * c2);
        if (dres) {
          const float4 rr = __ldg(reinterpret_cast<const float4*>(dres + r * C) + cv);
          out[0] += rr.x; out[1] += rr.y; out[2] += rr.z; out[3] += rr.w;
        }
        reinterpret_cast<float4*>(dx + r * C)[cv] = make_float4(out[0], out[1], out[2], out[3]);
        if (dxb) {
          uint2 u;
          u.x = pack_bf16x2(out[0], out[1]);
          u.y = pack_bf16x2(out[2], out[3]);
          reinterpret_cast<uint2*>(dxb + r * C)[cv] = u;
        }
      }
    }
  }
#pragma unroll
  for (int which = 0; which < 2; ++which) {
    __syncthreads();
#pragma unroll
    for (int v = 0; v < LNF_MAXV; ++v) {
      const int cv = lane + 32 * v;
      if (cv < CV) {
#pragma unroll
        for (int k = 0; k < 4; ++k) red[warp][cv * 4 + k] = which ? db[v][k] : dg[v][k];
      }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += 256) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) t += red[w][c];
      part[((long long)blockIdx.x * 2 + which) * C + c] = t;
    }
  }
}

__global__ void layernorm_bwd_f32_finalize_kernel(const float* __restrict__ part, int nblk, int C, float* __restrict__ dgamma,
                                                  float* __restrict__ dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float a = 0.f, b = 0.f;
  for (int k = 0; k < nblk; ++k) {
    a += part[((long long)k * 2) * C + c];
    b += part[((long long)k * 2 + 1) * C + c];
  }
  if (dgamma) dgamma[c] += a;
  if (dbeta) dbeta[c] += b;
}

// ------------------------------------------------------------------------------------------ embedding gradients
// Tokens sorted by id (host permutation perm, stable) are cut into chunks of at most TE_CHUNK tokens that never straddle two ids,
// so a frequent id (the padding id 0 holds most tokens of a batch) is spread over many CTAs instead of one long serial loop.
// Pass 1: part[k] = sum of dx over the tokens of chunk k, in perm order.  Pass 2: grad[uid[u]] += sum of the chunks of id u, in
// chunk order.  One thread per 4 channels; rows of ids that do not occur are not touched.
__global__ void text_embed_grad_chunk_kernel(const float* __restrict__ dx, const int* __restrict__ perm,
                                             const int* __restrict__ chunk_start, int C4, float* __restrict__ part) {
  const int k = blockIdx.x;
  const int s0 = chunk_start[k], s1 = chunk_start[k + 1];
  for (int c4 = threadIdx.x; c4 < C4; c4 += blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = s0; s < s1; ++s) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(dx) + (long long)perm[s] * C4 + c4);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    reinterpret_cast<float4*>(part)[(long long)k * C4 + c4] = acc;
  }
}

__global__ void text_embed_grad_sum_kernel(const float* __restrict__ part, const int* __restrict__ seg, const long long* __restrict__ uid,
                                           int C4, float* __restrict__ grad) {
  const int u = blockIdx.x;
  const int k0 = seg[u], k1 = seg[u + 1];
  float4* g = reinterpret_cast<float4*>(grad) + uid[u] * C4;
  for (int c4 = threadIdx.x; c4 < C4; c4 += blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int k = k0; k < k1; ++k) {
      const float4 v = reinterpret_cast<const float4*>(part)[(long long)k * C4 + c4];
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    float4 t = g[c4];
    t.x += acc.x; t.y += acc.y; t.z += acc.z; t.w += acc.w;
    g[c4] = t;
  }
}

// The N -> L resize of F.interpolate(mode="bilinear", align_corners=False) on [1, 1, N, C] along N (upsample_bilinear2d's
// area_pixel_compute_source_index): row l reads rows i0 = (int)src and i0 + (i0 < N - 1) with weights 1 - lambda, lambda.
__device__ __forceinline__ void resize_src(int l, int L, int N, int& i0, int& i1, float& l0, float& l1) {
  float src = (float)N / (float)L * ((float)l + 0.5f) - 0.5f;
  if (src < 0.f) src = 0.f;
  i0 = (int)src;
  i1 = i0 + (i0 < N - 1 ? 1 : 0);
  l1 = src - (float)i0;
  l0 = 1.f - l1;
}

// Forward of the training graph's positional table: out [L][C] = the resized table (one thread per 4 channels of a row).
__global__ void text_pos_resize_kernel(const float* __restrict__ tab, int N, int L, int C4, float* __restrict__ out) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)L * C4) return;
  const int l = (int)(i / C4), c4 = (int)(i - (long long)l * C4);
  int i0, i1;
  float l0, l1;
  resize_src(l, L, N, i0, i1, l0, l1);
  const float4 a = __ldg(reinterpret_cast<const float4*>(tab) + (long long)i0 * C4 + c4);
  const float4 b = __ldg(reinterpret_cast<const float4*>(tab) + (long long)i1 * C4 + c4);
  reinterpret_cast<float4*>(out)[i] = make_float4(fmaf(l0, a.x, l1 * b.x), fmaf(l0, a.y, l1 * b.y), fmaf(l0, a.z, l1 * b.z),
                                                  fmaf(l0, a.w, l1 * b.w));
}

// grad[n][c] += sum_l w(l, n) sum_b dx[b][l][c], w = the weights of F.interpolate(mode="bilinear", align_corners=False) that map
// a table of N rows to L rows (upsample_bilinear2d's area_pixel_compute_source_index; the D axis is resized to itself, which is
// the identity).  N == L gives w = identity.  One thread per (n, 4 channels); b summed in ascending order inside each l.
__global__ void text_pos_grad_kernel(const float* __restrict__ dx, int B, int L, int N, int C4, float* __restrict__ grad) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)N * C4) return;
  const int n = (int)(i / C4), c4 = (int)(i - (long long)n * C4);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int l = 0; l < L; ++l) {
    float w;
    if (N == L) {
      w = (l == n) ? 1.f : 0.f;
    } else {
      int i0, i1;
      float l0, l1;
      resize_src(l, L, N, i0, i1, l0, l1);
      w = (i0 == n ? l0 : 0.f) + (i1 == n ? l1 : 0.f);
    }
    if (w == 0.f) continue;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int b = 0; b < B; ++b) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(dx) + ((long long)b * L + l) * C4 + c4);
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    acc.x = fmaf(w, s.x, acc.x); acc.y = fmaf(w, s.y, acc.y); acc.z = fmaf(w, s.z, acc.z); acc.w = fmaf(w, s.w, acc.w);
  }
  float4* g = reinterpret_cast<float4*>(grad) + i;
  float4 t = *g;
  t.x += acc.x; t.y += acc.y; t.z += acc.z; t.w += acc.w;
  *g = t;
}

// ------------------------------------------------------------------------------------------ text KD loss
// Per token (b, l) over D channels: d2 = |p - t|^2, cos = p.t / (max(|p|, eps) max(|t|, eps)) (torch's cosine_similarity,
// eps 1e-8: the norms are clamped without a gradient path of their own).  valid = !pad[b, l] when masked (pad != null).
// part[b] = (sum valid d2, sum valid (1 - cos), sum valid); a warp per token, warps summed in index order.
constexpr float TXT_COS_EPS = 1e-8f;

__device__ __forceinline__ void token_stats(const float* p, const float* t, int D, int lane, float& d2, float& dot, float& np2,
                                            float& nt2) {
  d2 = dot = np2 = nt2 = 0.f;
  for (int c = lane; c < D; c += 32) {
    const float a = __ldg(p + c), b = __ldg(t + c), d = a - b;
    d2 = fmaf(d, d, d2); dot = fmaf(a, b, dot); np2 = fmaf(a, a, np2); nt2 = fmaf(b, b, nt2);
  }
  d2 = warp_sum(d2); dot = warp_sum(dot); np2 = warp_sum(np2); nt2 = warp_sum(nt2);
}

__global__ void __launch_bounds__(256) text_kd_partial_kernel(const float* __restrict__ p, const float* __restrict__ t,
                                                              const unsigned char* __restrict__ pad, int L, int D, float* __restrict__ part) {
  __shared__ float red[3][8];
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float sq = 0.f, cl = 0.f, cnt = 0.f;
  for (int l = warp; l < L; l += 8) {
    const long long off = ((long long)b * L + l) * D;
    float d2, dot, np2, nt2;
    token_stats(p + off, t + off, D, lane, d2, dot, np2, nt2);
    const float v = (pad == nullptr || pad[(long long)b * L + l] == 0) ? 1.f : 0.f;
    const float cosv = dot / (fmaxf(sqrtf(np2), TXT_COS_EPS) * fmaxf(sqrtf(nt2), TXT_COS_EPS));
    sq += v * d2; cl += v * (1.f - cosv); cnt += v;
  }
  if (lane == 0) { red[0][warp] = sq; red[1][warp] = cl; red[2][warp] = cnt; }
  __syncthreads();
  if (threadIdx.x < 3) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += red[threadIdx.x][w];
    part[b * 3 + threadIdx.x] = s;
  }
}

// out = (loss, mse, cos).  masked: mse = mean_b sum_sq_b / (max(n_b, 1) D), cos = mean_b sum_cl_b / max(n_b, 1)
// (masked_text_mse / masked_text_cosine_loss); plain: mse = sum sq / (B L D), cos = sum cl / (B L) (text_mse / text_cosine_loss).
__global__ void text_kd_final_kernel(const float* __restrict__ part, int B, int L, int D, int masked, float cosine_w,
                                     float* __restrict__ out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float mse = 0.f, cosl = 0.f;
  for (int b = 0; b < B; ++b) {
    if (masked) {
      const float den = fmaxf(part[b * 3 + 2], 1.f);
      mse += part[b * 3] / (den * (float)D);
      cosl += part[b * 3 + 1] / den;
    } else {
      mse += part[b * 3];
      cosl += part[b * 3 + 1];
    }
  }
  if (masked) { mse /= (float)B; cosl /= (float)B; }
  else { mse /= (float)B * (float)L * (float)D; cosl /= (float)B * (float)L; }
  out[0] = mse + cosine_w * cosl; out[1] = mse; out[2] = cosl;
}

// dp = g * (a_mse 2 (p - t) - a_cos dcos/dp) on valid tokens, 0 elsewhere;  g = grad_scale * scale_dev[0] (* gout[0]).
// dcos/dp = t / (np' nt') - (p.t) / (np'^2 nt') * p / |p|   (np' = max(|p|, eps); p / |p| := 0 at p = 0, as the norm's backward).
__global__ void __launch_bounds__(256) text_kd_bwd_kernel(const float* __restrict__ p, const float* __restrict__ t,
                                                          const unsigned char* __restrict__ pad, const float* __restrict__ part, int B,
                                                          int L, int D, float cosine_w, float grad_scale,
                                                          const float* __restrict__ scale_dev, const float* __restrict__ gout,
                                                          float* __restrict__ dp) {
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float g = grad_scale;
  if (scale_dev) g *= scale_dev[0];
  if (gout) g *= gout[0];
  float a_mse, a_cos;
  if (pad != nullptr) {
    const float den = fmaxf(part[b * 3 + 2], 1.f);
    a_mse = 2.f / (den * (float)D * (float)B);
    a_cos = cosine_w / (den * (float)B);
  } else {
    a_mse = 2.f / ((float)B * (float)L * (float)D);
    a_cos = cosine_w / ((float)B * (float)L);
  }
  for (int l = warp; l < L; l += 8) {
    const long long off = ((long long)b * L + l) * D;
    const bool v = pad == nullptr || pad[(long long)b * L + l] == 0;
    if (!v) {
      for (int c = lane; c < D; c += 32) dp[off + c] = 0.f;
      continue;
    }
    float d2, dot, np2, nt2;
    token_stats(p + off, t + off, D, lane, d2, dot, np2, nt2);
    const float np = sqrtf(np2), nt = sqrtf(nt2);
    const float npc = fmaxf(np, TXT_COS_EPS), ntc = fmaxf(nt, TXT_COS_EPS);
    const float ct = 1.f / (npc * ntc);
    const float cp = np > 0.f ? dot / (npc * npc * ntc * np) : 0.f;
    for (int c = lane; c < D; c += 32) {
      const float a = p[off + c], tt = t[off + c];
      const float dcos = tt * ct - a * cp;
      dp[off + c] = g * (a_mse * (a - tt) - a_cos * dcos);
    }
  }
}

// Consistency: mp = mean_l p[b, l, :], mq likewise; part[b] = sum_c (mp - mq)^2.  Block = one sample, thread = channels.
__global__ void __launch_bounds__(256) text_consistency_partial_kernel(const float* __restrict__ p, const float* __restrict__ q, int L,
                                                                       int D, float* __restrict__ mdiff, float* __restrict__ part) {
  __shared__ float red[8];
  const int b = blockIdx.x;
  float acc = 0.f;
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    float sp = 0.f, sq = 0.f;
    for (int l = 0; l < L; ++l) {
      sp += p[((long long)b * L + l) * D + c];
      sq += q[((long long)b * L + l) * D + c];
    }
    const float d = sp / (float)L - sq / (float)L;
    mdiff[(long long)b * D + c] = d;
    acc = fmaf(d, d, acc);
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
    part[b] = s;
  }
}

// out2[1] = mse over [B, D]; out2[0] += weight * out2[1] (the running loss of the caller's composition).
__global__ void text_consistency_final_kernel(const float* __restrict__ part, int B, int D, float weight, float* __restrict__ loss,
                                              float* __restrict__ value) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float s = 0.f;
  for (int b = 0; b < B; ++b) s += part[b];
  s /= (float)B * (float)D;
  *value = s;
  if (loss) *loss += weight * s;
}

// dp[b, l, c] += k (mp - mq)[b, c], dq[b, l, c] = -k (mp - mq)[b, c],  k = 2 weight g / (B D L).
__global__ void text_consistency_bwd_kernel(const float* __restrict__ mdiff, int B, int L, int D, float weight, float grad_scale,
                                            const float* __restrict__ scale_dev, const float* __restrict__ gout, float* __restrict__ dp,
                                            float* __restrict__ dq) {
  const long long n = (long long)B * L * D;
  float g = grad_scale;
  if (scale_dev) g *= scale_dev[0];
  if (gout) g *= gout[0];
  const float k = 2.f * weight * g / ((float)B * (float)D * (float)L);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % D);
    const long long b = i / ((long long)L * D);
    const float v = k * mdiff[b * D + c];
    dp[i] += v;
    dq[i] = -v;
  }
}

__global__ void cast_f32_to_bf16_kernel(const float* __restrict__ x, bf16* __restrict__ y, long long n4) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
    uint2 u;
    u.x = pack_bf16x2(v.x, v.y);
    u.y = pack_bf16x2(v.z, v.w);
    reinterpret_cast<uint2*>(y)[i] = u;
  }
}

}  // namespace
}  // namespace es3

using namespace es3;

static int grid_for(long long n, int block) {
  const long long g = (n + block - 1) / block;
  return (int)(g < 132 * 16 ? (g > 0 ? g : 1) : 132 * 16);
}

/* Attention backward of es3_attention_bf16 (H = 1, W = L, no window) / es3_attention_causal_bf16 on head_dim 64 and L <= 128.
 * qkv [B*L, 3C] bf16 ([q | k | v], head h at columns 64 h of each third), o = the forward output [B*L, C], dout like o;
 * dqkv [B*L, 3C] bf16 in qkv's layout.  The softmax is recomputed from q and k. */
extern "C" int es3_text_attn_bwd(const void* qkv, const void* o, const void* dout, void* dqkv, int B, int L, int C, int num_heads,
                                 int causal, float scale, void* stream) {
  ES3_REQUIRE(L >= 1 && L <= TA_MAXL, "es3_text_attn_bwd: sequence length %d outside 1..%d", L, TA_MAXL);
  ES3_REQUIRE(B >= 1 && num_heads >= 1 && C == num_heads * TA_D, "es3_text_attn_bwd: head_dim must be 64 (C=%d heads=%d)", C,
              num_heads);
  const int smem = 4 * L * TA_LD * (int)sizeof(bf16) + (2 * L * (L + 1) + L) * (int)sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
  if (causal) {
    ES3_CHECK_CUDA(cudaFuncSetAttribute(text_attn_bwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    text_attn_bwd_kernel<true><<<dim3(B, num_heads), TA_THREADS, smem, st>>>((const bf16*)qkv, (const bf16*)o, (const bf16*)dout,
                                                                              (bf16*)dqkv, L, C, scale);
  } else {
    ES3_CHECK_CUDA(cudaFuncSetAttribute(text_attn_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    text_attn_bwd_kernel<false><<<dim3(B, num_heads), TA_THREADS, smem, st>>>((const bf16*)qkv, (const bf16*)o, (const bf16*)dout,
                                                                               (bf16*)dqkv, L, C, scale);
  }
  ES3_LAUNCH_CHECK("text_attn_bwd_kernel");
  return 0;
}

static int lnf_blocks(long long M, long long* rpb) {
  long long nblk = (M + 63) / 64;
  if (nblk > 592) nblk = 592;
  if (nblk < 1) nblk = 1;
  *rpb = (M + nblk - 1) / nblk;
  return (int)((M + *rpb - 1) / *rpb);
}

extern "C" long long es3_layernorm_bwd_f32_ws_floats(long long M, int C) {
  long long rpb;
  return (long long)lnf_blocks(M, &rpb) * 2 * C;
}

/* dx = d LayerNorm(x) (+ dres) in fp32, optionally also rounded to bf16 into dxb; dgamma += sum dy xhat, dbeta += sum dy.
 * x, dy, dres, dx: [M][C] fp32 contiguous, C % 4 == 0, C <= 768. */
extern "C" int es3_layernorm_bwd_f32(const float* x, const float* dy, const float* gamma, const float* dres, float eps, float* dx,
                                     void* dxb, long long M, int C, float* ws, float* dgamma, float* dbeta, void* stream) {
  ES3_REQUIRE(M > 0 && C % 4 == 0 && C <= LNF_MAXV * 128, "es3_layernorm_bwd_f32: C=%d must be a multiple of 4 and <= %d", C,
              LNF_MAXV * 128);
  long long rpb;
  const int nblk = lnf_blocks(M, &rpb);
  cudaStream_t st = (cudaStream_t)stream;
  layernorm_bwd_f32_kernel<<<nblk, 256, 0, st>>>(x, dy, gamma, dres, eps, dx, (bf16*)dxb, M, C, rpb, ws);
  ES3_LAUNCH_CHECK("layernorm_bwd_f32_kernel");
  layernorm_bwd_f32_finalize_kernel<<<ceil_div(C, 128), 128, 0, st>>>(ws, nblk, C, dgamma, dbeta);
  ES3_LAUNCH_CHECK("layernorm_bwd_f32_finalize_kernel");
  return 0;
}

/* grad [V][C] fp32 += the embedding gradient of dx [M][C]: perm [M] int32 = token indices sorted by id (stable), chunk_start
 * [nchunk + 1] int32 = chunk bounds in perm (a chunk holds tokens of one id), seg [U + 1] int32 = the first chunk of each distinct
 * id, uid [U] int64 = the distinct ids (checked in [0, V) on the host); ws: nchunk * C floats. */
extern "C" int es3_text_embed_grad(const float* dx, const int* perm, const int* chunk_start, int nchunk, const int* seg,
                                   const long long* uid, int U, int C, float* ws, float* grad, void* stream) {
  ES3_REQUIRE(U >= 1 && nchunk >= U && C >= 4 && C % 4 == 0, "es3_text_embed_grad: need nchunk >= U >= 1 and C %% 4 == 0 "
              "(U=%d nchunk=%d C=%d)", U, nchunk, C);
  const int C4 = C / 4, threads = C4 < 256 ? C4 : 256;
  cudaStream_t st = (cudaStream_t)stream;
  text_embed_grad_chunk_kernel<<<nchunk, threads, 0, st>>>(dx, perm, chunk_start, C4, ws);
  ES3_LAUNCH_CHECK("text_embed_grad_chunk_kernel");
  text_embed_grad_sum_kernel<<<U, threads, 0, st>>>(ws, seg, uid, C4, grad);
  ES3_LAUNCH_CHECK("text_embed_grad_sum_kernel");
  return 0;
}

/* grad [N][C] fp32 += positional-table gradient of dx [B][L][C] (table resized N -> L in the forward when N != L). */
extern "C" int es3_text_pos_grad(const float* dx, int B, int L, int N, int C, float* grad, void* stream) {
  ES3_REQUIRE(B >= 1 && L >= 1 && N >= 1 && C % 4 == 0, "es3_text_pos_grad: bad shape B=%d L=%d N=%d C=%d", B, L, N, C);
  const long long n = (long long)N * (C / 4);
  text_pos_grad_kernel<<<(int)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(dx, B, L, N, C / 4, grad);
  ES3_LAUNCH_CHECK("text_pos_grad_kernel");
  return 0;
}

/* out [L][C] = the table [N][C] resized to L rows as the forward of LearnablePositionalEmbedding does (N != L). */
extern "C" int es3_text_pos_resize(const float* table, int N, int L, int C, float* out, void* stream) {
  ES3_REQUIRE(L >= 1 && N >= 1 && C % 4 == 0, "es3_text_pos_resize: bad shape N=%d L=%d C=%d", N, L, C);
  const long long n = (long long)L * (C / 4);
  text_pos_resize_kernel<<<(int)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(table, N, L, C / 4, out);
  ES3_LAUNCH_CHECK("text_pos_resize_kernel");
  return 0;
}

/* Text KD loss on preds / teacher [B][L][D] fp32.  pad [B][L] bytes (masked loss, valid = pad == 0, i.e. id != 0) or null
 * (plain loss).
 * ws: B * 3 floats (per-sample partials, kept for the backward); out3 = (loss, mse, cos). */
extern "C" int es3_text_kd_loss_fwd(const float* preds, const float* teacher, const unsigned char* pad, int B, int L, int D,
                                    float cosine_weight, float* ws, float* out3, void* stream) {
  ES3_REQUIRE(B >= 1 && L >= 1 && D >= 1, "es3_text_kd_loss_fwd: bad shape B=%d L=%d D=%d", B, L, D);
  cudaStream_t st = (cudaStream_t)stream;
  text_kd_partial_kernel<<<B, 256, 0, st>>>(preds, teacher, pad, L, D, ws);
  ES3_LAUNCH_CHECK("text_kd_partial_kernel");
  text_kd_final_kernel<<<1, 32, 0, st>>>(ws, B, L, D, pad != nullptr, cosine_weight, out3);
  ES3_LAUNCH_CHECK("text_kd_final_kernel");
  return 0;
}

/* d loss / d preds times grad_scale, scale_dev[0] and gout[0] (each pointer may be null); ws from es3_text_kd_loss_fwd. */
extern "C" int es3_text_kd_loss_bwd(const float* preds, const float* teacher, const unsigned char* pad, const float* ws, int B, int L,
                                    int D, float cosine_weight, float grad_scale, const float* scale_dev, const float* gout,
                                    float* dpreds, void* stream) {
  ES3_REQUIRE(B >= 1 && L >= 1 && D >= 1, "es3_text_kd_loss_bwd: bad shape B=%d L=%d D=%d", B, L, D);
  text_kd_bwd_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(preds, teacher, pad, ws, B, L, D, cosine_weight, grad_scale, scale_dev,
                                                          gout, dpreds);
  ES3_LAUNCH_CHECK("text_kd_bwd_kernel");
  return 0;
}

/* value[0] = mse(mean_L(p), mean_L(q)); loss[0] += weight * value[0] (loss may be null).  mdiff: [B][D] fp32 out (kept for the
 * backward); ws: B floats. */
extern "C" int es3_text_consistency_fwd(const float* p, const float* q, int B, int L, int D, float weight, float* mdiff, float* ws,
                                        float* loss, float* value, void* stream) {
  ES3_REQUIRE(B >= 1 && L >= 1 && D >= 1, "es3_text_consistency_fwd: bad shape B=%d L=%d D=%d", B, L, D);
  cudaStream_t st = (cudaStream_t)stream;
  text_consistency_partial_kernel<<<B, 256, 0, st>>>(p, q, L, D, mdiff, ws);
  ES3_LAUNCH_CHECK("text_consistency_partial_kernel");
  text_consistency_final_kernel<<<1, 32, 0, st>>>(ws, B, D, weight, loss, value);
  ES3_LAUNCH_CHECK("text_consistency_final_kernel");
  return 0;
}

/* dp += gradient of weight * consistency w.r.t. p, dq = the gradient w.r.t. q (both [B][L][D] fp32). */
extern "C" int es3_text_consistency_bwd(const float* mdiff, int B, int L, int D, float weight, float grad_scale, const float* scale_dev,
                                        const float* gout, float* dp, float* dq, void* stream) {
  ES3_REQUIRE(B >= 1 && L >= 1 && D >= 1, "es3_text_consistency_bwd: bad shape B=%d L=%d D=%d", B, L, D);
  text_consistency_bwd_kernel<<<grid_for((long long)B * L * D, 256), 256, 0, (cudaStream_t)stream>>>(mdiff, B, L, D, weight, grad_scale,
                                                                                                    scale_dev, gout, dp, dq);
  ES3_LAUNCH_CHECK("text_consistency_bwd_kernel");
  return 0;
}

/* y = bf16(x), n % 4 == 0 (both contiguous). */
extern "C" int es3_cast_f32_to_bf16(const float* x, void* y, long long n, void* stream) {
  ES3_REQUIRE(n > 0 && n % 4 == 0, "es3_cast_f32_to_bf16: n=%lld must be a positive multiple of 4", n);
  cast_f32_to_bf16_kernel<<<grid_for(n / 4, 256), 256, 0, (cudaStream_t)stream>>>(x, (bf16*)y, n / 4);
  ES3_LAUNCH_CHECK("cast_f32_to_bf16_kernel");
  return 0;
}
