// Small kernels of the SAM-style prompt encoder / TwoWayTransformer / MaskDecoder path
// (sam3/sam3/sam/{prompt_encoder,transformer,mask_decoder}.py, glue sam3_tracker_base.py:220-389).
// The dense contractions over the 5184 image tokens run on gemm_tc.cu; everything here is either tiny
// (8 prompt/output tokens per image: latency-bound) or a streaming pass over the image tokens / masks.
// Token-side math is fp32 end to end (it feeds the mask logits through the hypernetwork).
#include "bilinear.cuh"

namespace es3 {

// ------------------------------------------------------------------------------------ positional enc.
// PositionEmbeddingRandom (prompt_encoder.py:200-243): c = 2*coords01 - 1; c @ G[2,F]; *2pi; [sin | cos].
__device__ __forceinline__ void pe_pair(const float* __restrict__ gauss, int F, float x01, float y01, int f, float* s,
                                        float* c) {
  const float cx = 2.f * x01 - 1.f, cy = 2.f * y01 - 1.f;
  const float a = 6.283185307179586f * (cx * gauss[f] + cy * gauss[F + f]);
  sincosf(a, s, c);
}

// Dense PE for an h x w grid, token-major: out [h*w][2F] fp32 (get_dense_pe, prompt_encoder.py:61-69).
__global__ void dense_pe_kernel(const float* __restrict__ gauss, int F, int h, int w, float* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= h * w * F) return;
  const int f = idx % F, p = idx / F;
  const int y = p / w, x = p % w;
  float s, c;
  pe_pair(gauss, F, (x + 0.5f) / w, (y + 0.5f) / h, f, &s, &c);
  out[(long long)p * 2 * F + f] = s;
  out[(long long)p * 2 * F + F + f] = c;
}

// Sparse point embeddings, optionally with the trailing padding point (_embed_points, pad = boxes is None, :71-117).
// coords [B,P,2] (x,y) pixels, labels [B,P] int32.  out [B,P+pad,2F] fp32.
// tables: not_a_point [2F], point_emb [4][2F].
__global__ void point_embed_kernel(const float* __restrict__ coords, const int* __restrict__ labels,
                                   const float* __restrict__ gauss, const float* __restrict__ not_a_point,
                                   const float* __restrict__ point_emb, int F, int P, int pad, float img_w, float img_h,
                                   float* __restrict__ out) {
  const int bp = blockIdx.x;  // b*(P+pad) + p
  const int b = bp / (P + pad), p = bp % (P + pad);
  float x = 0.f, y = 0.f;
  int lab = -1;
  if (p < P) {
    x = coords[((long long)b * P + p) * 2 + 0];
    y = coords[((long long)b * P + p) * 2 + 1];
    lab = labels[(long long)b * P + p];
  }
  x = (x + 0.5f) / img_w;
  y = (y + 0.5f) / img_h;
  for (int f = threadIdx.x; f < F; f += blockDim.x) {
    float s, c;
    pe_pair(gauss, F, x, y, f, &s, &c);
    if (lab == -1) { s = not_a_point[f]; c = not_a_point[F + f]; }
    else if (lab >= 0 && lab < 4) { s += point_emb[lab * 2 * F + f]; c += point_emb[lab * 2 * F + F + f]; }
    out[(long long)bp * 2 * F + f] = s;
    out[(long long)bp * 2 * F + F + f] = c;
  }
}

// ------------------------------------------------------------------------------------ elementwise
// y[m][c] = x[m][c] + add[(m % R)][c]; writes bf16 and/or fp32.  C % 4 == 0.
__global__ void add_rows_kernel(const float* __restrict__ x, const float* __restrict__ add, long long M, int C, int R,
                                bf16* __restrict__ y_bf16, float* __restrict__ y_f32) {
  const long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int c4 = C >> 2;
  if (i4 >= M * c4) return;
  const long long m = i4 / c4;
  const int c = (int)(i4 % c4);
  float4 v = reinterpret_cast<const float4*>(x)[i4];
  if (add != nullptr) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(add) + (m % R) * c4 + c);
    v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
  }
  if (y_f32) reinterpret_cast<float4*>(y_f32)[i4] = v;
  if (y_bf16) {
    uint2 u;
    u.x = pack_bf16x2(v.x, v.y);
    u.y = pack_bf16x2(v.z, v.w);
    reinterpret_cast<uint2*>(y_bf16)[i4] = u;
  }
}

// [B,C,HW] fp32 -> [B,HW,C] fp32 and / or its bf16 copy.
__global__ void nchw_to_tokens_kernel(const float* __restrict__ in, float* __restrict__ out_f32, bf16* __restrict__ out_bf16, int HW,
                                      int C) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i, p = p0 + tx;
    tile[i][tx] = (p < HW && c < C) ? in[((long long)b * C + c) * HW + p] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int p = p0 + i, c = c0 + tx;
    if (p < HW && c < C) {
      const float v = tile[tx][i];
      if (out_f32) out_f32[((long long)b * HW + p) * C + c] = v;
      if (out_bf16) out_bf16[((long long)b * HW + p) * C + c] = __float2bfloat16(v);
    }
  }
}

// ------------------------------------------------------------------------------------ attention
__device__ __forceinline__ float ld_f(const float* p) { return *p; }
__device__ __forceinline__ float ld_f(const bf16* p) { return __bfloat162float(*p); }

// Few queries (<= 32 per image), many keys: one warp per (query, head, image); lanes stride the keys with a
// private online-softmax state that is merged by shuffles.  q [B,Tq,ldq] fp32, k/v [B,Tk,ld] (bf16|fp32),
// out [B,Tq,ldo] fp32, heads laid out [h*HD, (h+1)*HD).   Attention(transformer.py:185-264) core.
template <int HD, typename TKV>
__global__ void attn_few_queries_kernel(const float* __restrict__ q, long long ldq, const TKV* __restrict__ k,
                                        const TKV* __restrict__ v, long long ldkv, float* __restrict__ out, long long ldo,
                                        int Tq, int Tk, float scale) {
  const int lane = threadIdx.x & 31;
  const int qi = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int h = blockIdx.y, b = blockIdx.z;
  if (qi >= Tq) return;
  float qr[HD];
  const float* qp = q + ((long long)b * Tq + qi) * ldq + h * HD;
#pragma unroll
  for (int d = 0; d < HD; ++d) qr[d] = qp[d] * scale;
  float m = -INFINITY, l = 0.f, acc[HD];
#pragma unroll
  for (int d = 0; d < HD; ++d) acc[d] = 0.f;
  const TKV* kb = k + (long long)b * Tk * ldkv + h * HD;
  const TKV* vb = v + (long long)b * Tk * ldkv + h * HD;
  for (int j = lane; j < Tk; j += 32) {
    const TKV* kp = kb + (long long)j * ldkv;
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < HD; ++d) s = fmaf(qr[d], ld_f(kp + d), s);
    const float mn = fmaxf(m, s);
    const float corr = __expf(m - mn), p = __expf(s - mn);
    l = l * corr + p;
    const TKV* vp = vb + (long long)j * ldkv;
#pragma unroll
    for (int d = 0; d < HD; ++d) acc[d] = fmaf(p, ld_f(vp + d), acc[d] * corr);
    m = mn;
  }
  // merge the 32 partial states
  float mw = warp_max(m);
  const float f = (m == -INFINITY) ? 0.f : __expf(m - mw);
  l = warp_sum(l * f);
#pragma unroll
  for (int d = 0; d < HD; ++d) acc[d] = warp_sum(acc[d] * f);
  if (lane == 0) {
    float* op = out + ((long long)b * Tq + qi) * ldo + h * HD;
    const float inv = 1.f / l;
#pragma unroll
    for (int d = 0; d < HD; ++d) op[d] = acc[d] * inv;
  }
}

// Many queries (image tokens), few keys (the decoder's output and prompt tokens, any number): one thread per (query, head).
// q [B,Nq,ldq] bf16, k/v [B,Tk,ldkv] fp32, out [B,Nq,ldo] bf16.  cross_attn_image_to_token core.  K/V stream through shared
// memory in tiles of FEW_KEYS_TILE tokens; the softmax is sequential per thread, so the tiling does not change the arithmetic.
template <int HD>
__global__ void attn_few_keys_kernel(const bf16* __restrict__ q, long long ldq, const float* __restrict__ k,
                                     const float* __restrict__ v, long long ldkv, bf16* __restrict__ out, long long ldo,
                                     int Nq, int Tk, int H, float scale) {
  extern __shared__ float skv[];  // [2][cap][H*HD], cap = min(Tk, FEW_KEYS_TILE)
  const int b = blockIdx.y;
  const int D = H * HD, cap = min(Tk, FEW_KEYS_TILE);
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const bool active = idx < Nq * H;   // inactive threads still take part in the tile loads and barriers
  const int h = idx % H, n = idx / H;
  float qr[HD];
  const bf16* qp = q + ((long long)b * Nq + n) * ldq + h * HD;
  if (active) {
#pragma unroll
    for (int d = 0; d < HD; d += 8) {
      float f[8];
      unpack8(*reinterpret_cast<const uint4*>(qp + d), f);
#pragma unroll
      for (int e = 0; e < 8; ++e) qr[d + e] = f[e] * scale;
    }
  }
  float mx = -INFINITY, l = 0.f, o[HD];
#pragma unroll
  for (int d = 0; d < HD; ++d) o[d] = 0.f;
  for (int t0 = 0; t0 < Tk; t0 += FEW_KEYS_TILE) {
    const int nt = min(FEW_KEYS_TILE, Tk - t0);
    few_keys_load_tile(skv, k, v, ldkv, (long long)b * Tk + t0, nt, cap, D);
    if (active) {
      for (int t = 0; t < nt; ++t) {   // online softmax over the few keys
        const float* kp = skv + t * D + h * HD;
        float a = 0.f;
#pragma unroll
        for (int d = 0; d < HD; ++d) a = fmaf(qr[d], kp[d], a);
        const float mn = fmaxf(mx, a);
        const float corr = __expf(mx - mn), p = __expf(a - mn);
        l = l * corr + p;
        const float* vp = skv + cap * D + t * D + h * HD;
#pragma unroll
        for (int d = 0; d < HD; ++d) o[d] = fmaf(p, vp[d], o[d] * corr);
        mx = mn;
      }
    }
  }
  if (!active) return;
  const float inv = 1.f / l;
  bf16* op = out + ((long long)b * Nq + n) * ldo + h * HD;
#pragma unroll
  for (int d = 0; d < HD; d += 8) {
    float f[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = o[d + e] * inv;
    *reinterpret_cast<uint4*>(op + d) = pack8(f);
  }
}

// ------------------------------------------------------------------------------------ LayerNorm2d + GELU
// Rows of C <= 128 channels (C % 32 == 0): y = gelu(LN(x) * w + b) -> bf16.  One warp per row.
// LayerNorm2d (sam/common.py:27-39, eps 1e-6) over the channel dim of an NHWC map, fused with the activation of
// MaskDecoder.output_upscaling (mask_decoder.py:59-70, 213-216).
__global__ void ln_rows_gelu_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                    float eps, bf16* __restrict__ y, long long M, int C) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  const int per = C >> 5;  // 1..4
  float v[4];
  float s = 0.f;
  for (int i = 0; i < per; ++i) { v[i] = x[row * C + lane + i * 32]; s += v[i]; }
  const float mean = warp_sum(s) / C;
  float qv = 0.f;
  for (int i = 0; i < per; ++i) { const float d = v[i] - mean; qv += d * d; }
  const float rstd = rsqrtf(warp_sum(qv) / C + eps);
  for (int i = 0; i < per; ++i) {
    const int c = lane + i * 32;
    const float o = (v[i] - mean) * rstd * w[c] + bias[c];
    y[row * C + c] = __float2bfloat16(es3_act_t<ACT_GELU>(o));
  }
}

// ------------------------------------------------------------------------------------ mask tail
// masks[b][k][p] = sum_c hyper[b][k][c] * up[b][p][c]   (mask_decoder.py:225-226), optional object gating
// (sam3_tracker_base.py:344-353: where(obj_logit > 0, masks, NO_OBJ_SCORE)).  up fp32 [B,HW,CU], CU == 32.
__global__ void hyper_masks_kernel(const float* __restrict__ up, const float* __restrict__ hyper,
                                   const float* __restrict__ obj_logits, float no_obj, float* __restrict__ masks, int HW,
                                   int Ktot, int K, int k_off) {
  __shared__ float sh[8 * 32];
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < K * 32; i += blockDim.x) sh[i] = hyper[((long long)b * Ktot + k_off) * 32 + i];
  __syncthreads();
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const float4* u4 = reinterpret_cast<const float4*>(up + ((long long)b * HW + p) * 32);
  float u[32];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 t = u4[j];
    u[4 * j] = t.x; u[4 * j + 1] = t.y; u[4 * j + 2] = t.z; u[4 * j + 3] = t.w;
  }
  const bool gated = obj_logits != nullptr && !(obj_logits[b] > 0.f);
  for (int k = 0; k < K; ++k) {
    float a = 0.f;
#pragma unroll
    for (int c = 0; c < 32; ++c) a = fmaf(sh[k * 32 + c], u[c], a);
    masks[((long long)b * K + k) * HW + p] = gated ? no_obj : a;
  }
}

// Bilinear (align_corners=False) NCHW fp32 -> NCHW fp32; optional uint8 binarisation (x > thr).
__global__ void bilinear_nchw_kernel(const float* __restrict__ in, float* __restrict__ out, uint8_t* __restrict__ bin,
                                     float thr, int Hi, int Wi, int Ho, int Wo, float sy, float sx, long long planes) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = planes * Ho * Wo;
  if (idx >= total) return;
  const int ox = (int)(idx % Wo);
  const int oy = (int)((idx / Wo) % Ho);
  const long long pl = idx / ((long long)Wo * Ho);
  const BilinearTap ty = bilinear_tap(oy, sy, Hi), tx = bilinear_tap(ox, sx, Wi);
  const float* p = in + pl * Hi * Wi;
  const float v = bilinear_mix(ty, tx, __ldg(p + ty.i0 * Wi + tx.i0), __ldg(p + ty.i0 * Wi + tx.i1), __ldg(p + ty.i1 * Wi + tx.i0),
                               __ldg(p + ty.i1 * Wi + tx.i1));
  if (out) out[idx] = v;
  if (bin) bin[idx] = v > thr ? 1 : 0;
}


// ------------------------------------------------------------------------------------ mask prompt
// PromptEncoder.mask_downscaling (prompt_encoder.py:45-63): Conv2d(1,4,k2,s2) -> LayerNorm2d -> GELU -> Conv2d(4,16,k2,s2)
// -> LayerNorm2d -> GELU -> Conv2d(16,C,1), fused with `src = image_embeddings + dense` (mask_decoder.py:189) and emitted
// token-major: keys[row][c] = base[row % base_rows][c] + dense[row][c].  One block = 16 output pixels: 16 threads run the
// two tiny convs for their pixel (a 4x4 input patch), then thread c owns output channel c for all 16 pixels.
struct MaskDsW {
  const float *w0, *b0, *g1, *be1;   // [4][2][2], [4], LN 4
  const float *w1, *b1, *g2, *be2;   // [16][4][2][2], [16], LN 16
  const float *w2, *b2;              // [C][16], [C]
};
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }

__global__ void __launch_bounds__(256) mask_downscale_kernel(const float* __restrict__ mask, MaskDsW wt, const float* __restrict__ base,
                                                             long long base_rows, float* __restrict__ out_f32,
                                                             bf16* __restrict__ out_bf16, int B, int h, int w, int C, float eps) {
  __shared__ float s_v[16][17];
  const long long row0 = (long long)blockIdx.x * 16;
  const long long rows = (long long)B * h * w;
  if (threadIdx.x < 16 && row0 + threadIdx.x < rows) {
    const long long row = row0 + threadIdx.x;
    const int b = (int)(row / (h * w)), p = (int)(row % (h * w));
    const int y = p / w, x = p % w;
    const float* mp = mask + ((long long)b * 4 * h + 4 * y) * (4 * w) + 4 * x;   // 4x4 input patch
    float a[4][4];   // [position (py*2+px)][channel] after conv0 + LN + GELU
#pragma unroll
    for (int py = 0; py < 2; ++py)
#pragma unroll
      for (int px = 0; px < 2; ++px) {
        float t[4], mu = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          float acc = wt.b0[c];
#pragma unroll
          for (int ky = 0; ky < 2; ++ky)
#pragma unroll
            for (int kx = 0; kx < 2; ++kx) acc = fmaf(wt.w0[c * 4 + ky * 2 + kx], mp[(2 * py + ky) * (4 * w) + 2 * px + kx], acc);
          t[c] = acc; mu += acc;
        }
        mu *= 0.25f;
        float var = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) var += (t[c] - mu) * (t[c] - mu);
        const float rs = rsqrtf(var * 0.25f + eps);
#pragma unroll
        for (int c = 0; c < 4; ++c) a[py * 2 + px][c] = gelu_erf(wt.g1[c] * ((t[c] - mu) * rs) + wt.be1[c]);
      }
    float u[16], mu = 0.f;
#pragma unroll
    for (int n = 0; n < 16; ++n) {
      float acc = wt.b1[n];
#pragma unroll
      for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int pos = 0; pos < 4; ++pos) acc = fmaf(wt.w1[(n * 4 + c) * 4 + pos], a[pos][c], acc);
      u[n] = acc; mu += acc;
    }
    mu *= (1.f / 16.f);
    float var = 0.f;
#pragma unroll
    for (int n = 0; n < 16; ++n) var += (u[n] - mu) * (u[n] - mu);
    const float rs = rsqrtf(var * (1.f / 16.f) + eps);
#pragma unroll
    for (int n = 0; n < 16; ++n) s_v[threadIdx.x][n] = gelu_erf(wt.g2[n] * ((u[n] - mu) * rs) + wt.be2[n]);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += 256) {
    float wr[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) wr[k] = wt.w2[c * 16 + k];
    const float bc = wt.b2[c];
    for (int i = 0; i < 16 && row0 + i < rows; ++i) {
      float acc = bc;
#pragma unroll
      for (int k = 0; k < 16; ++k) acc = fmaf(wr[k], s_v[i][k], acc);
      const long long row = row0 + i;
      if (base != nullptr) acc += base[(row % base_rows) * C + c];
      if (out_f32) out_f32[row * C + c] = acc;
      if (out_bf16) out_bf16[row * C + c] = __float2bfloat16(acc);
    }
  }
}

// ------------------------------------------------------------------------------------ small-component filling
// SAM2Transforms.postprocess_masks before the resize (sam1_utils.py:77-105): connected components (8-connectivity, as
// skimage.measure.label / cc_torch / the Triton kernel in perflib/) of the background (score <= thr) with area <= max_hole
// become thr + 10; components of the foreground (score > thr, judged on the ORIGINAL scores) with area <= max_sprinkle
// become thr - 10.  Labels: lock-free union-find on global memory (root = smallest pixel index of the component, so the
// result is deterministic), areas by integer atomics on the roots.
__device__ __forceinline__ int cc_find(const int* L, int i) {
  int p = L[i];
  while (p != i) { i = p; p = L[i]; }
  return i;
}
__device__ __forceinline__ void cc_union(int* L, int a, int b) {
  bool done;
  do {
    a = cc_find(L, a);
    b = cc_find(L, b);
    if (a < b) { const int old = atomicMin(&L[b], a); done = (old == b); b = old; }
    else if (b < a) { const int old = atomicMin(&L[a], b); done = (old == a); a = old; }
    else done = true;
  } while (!done);
}
// sel > 0: component class = (score > thr); sel == 0: class = (score <= thr).
__device__ __forceinline__ bool cc_in_class(float v, float thr, int fg) { return fg ? (v > thr) : (v <= thr); }

__global__ void cc_init_kernel(const float* __restrict__ in, int* __restrict__ L, int* __restrict__ area, long long total, float thr, int fg) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  L[i] = cc_in_class(in[i], thr, fg) ? (int)i : -1;
  area[i] = 0;
}
__global__ void cc_merge_kernel(const float* __restrict__ in, int* __restrict__ L, int N, int H, int W) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * H * W) return;
  if (L[i] < 0) return;
  const int x = (int)(i % W), y = (int)((i / W) % H);
  // half of the 8-neighbourhood is enough: W, NW, N, NE
  if (x > 0 && L[i - 1] >= 0) cc_union(L, (int)i, (int)i - 1);
  if (y > 0) {
    if (L[i - W] >= 0) cc_union(L, (int)i, (int)i - W);
    if (x > 0 && L[i - W - 1] >= 0) cc_union(L, (int)i, (int)i - W - 1);
    if (x + 1 < W && L[i - W + 1] >= 0) cc_union(L, (int)i, (int)i - W + 1);
  }
}
__global__ void cc_count_kernel(int* __restrict__ L, int* __restrict__ area, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total || L[i] < 0) return;
  const int r = cc_find(L, (int)i);
  L[i] = r;                     // roots are fixed points, so compressing while others still read is safe
  atomicAdd(&area[r], 1);
}
__global__ void cc_apply_kernel(const int* __restrict__ L, const int* __restrict__ area, float* __restrict__ out, long long total,
                                float max_area, float value) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total || L[i] < 0) return;
  if ((float)area[cc_find(L, (int)i)] <= max_area) out[i] = value;
}

}  // namespace es3

using namespace es3;

extern "C" int es3_dense_pe(const float* gauss, int F, int h, int w, float* out, void* stream) {
  const int total = h * w * F;
  dense_pe_kernel<<<ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(gauss, F, h, w, out);
  ES3_LAUNCH_CHECK("dense_pe_kernel");
  return 0;
}

extern "C" int es3_point_embed(const float* coords, const int* labels, const float* gauss, const float* not_a_point,
                               const float* point_emb, int F, int B, int P, int pad, float img_w, float img_h, float* out,
                               void* stream) {
  ES3_REQUIRE(B > 0 && P + (pad != 0) > 0, "es3_point_embed: empty prompt batch");
  point_embed_kernel<<<B * (P + (pad != 0)), 128, 0, (cudaStream_t)stream>>>(coords, labels, gauss, not_a_point, point_emb, F, P,
                                                                           pad != 0, img_w, img_h, out);
  ES3_LAUNCH_CHECK("point_embed_kernel");
  return 0;
}

extern "C" int es3_add_rows(const float* x, const float* add, long long M, int C, int R, void* y_bf16, float* y_f32,
                            void* stream) {
  ES3_REQUIRE(C % 4 == 0 && (add == nullptr || R > 0), "es3_add_rows: bad C=%d R=%d", C, R);
  const long long n4 = M * (C / 4);
  add_rows_kernel<<<(unsigned)ceil_div(n4, 256), 256, 0, (cudaStream_t)stream>>>(x, add, M, C, R > 0 ? R : 1, (bf16*)y_bf16, y_f32);
  ES3_LAUNCH_CHECK("add_rows_kernel");
  return 0;
}

extern "C" int es3_nchw_f32_to_tokens(const float* in, float* out_f32, void* out_bf16, int B, int HW, int C, void* stream) {
  dim3 grid(ceil_div(HW, 32), ceil_div(C, 32), B);
  nchw_to_tokens_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in, out_f32, (bf16*)out_bf16, HW, C);
  ES3_LAUNCH_CHECK("nchw_to_tokens_kernel");
  return 0;
}

extern "C" int es3_attn_few_queries(const float* q, long long ldq, const void* k, const void* v, long long ldkv, int kv_f32,
                                    float* out, long long ldo, int B, int H, int head_dim, int Tq, int Tk, float scale,
                                    void* stream) {
  // head_dim 32 is self-attention over the tokens, whose K/V are fp32; token-to-image attention (bf16 or fp32 K/V) has head_dim 16
  ES3_REQUIRE(head_dim == 16 || (head_dim == 32 && kv_f32), "es3_attn_few_queries: head_dim %d with %s K/V not supported", head_dim,
              kv_f32 ? "fp32" : "bf16");
  dim3 grid(ceil_div(Tq, 4), H, B);
  cudaStream_t st = (cudaStream_t)stream;
  if (head_dim == 16) {
    if (kv_f32) attn_few_queries_kernel<16, float><<<grid, 128, 0, st>>>(q, ldq, (const float*)k, (const float*)v, ldkv, out, ldo, Tq, Tk, scale);
    else attn_few_queries_kernel<16, bf16><<<grid, 128, 0, st>>>(q, ldq, (const bf16*)k, (const bf16*)v, ldkv, out, ldo, Tq, Tk, scale);
  } else {
    attn_few_queries_kernel<32, float><<<grid, 128, 0, st>>>(q, ldq, (const float*)k, (const float*)v, ldkv, out, ldo, Tq, Tk, scale);
  }
  ES3_LAUNCH_CHECK("attn_few_queries_kernel");
  return 0;
}

extern "C" int es3_attn_few_keys(const void* q, long long ldq, const float* k, const float* v, long long ldkv, void* out,
                                 long long ldo, int B, int H, int head_dim, int Nq, int Tk, float scale, void* stream) {
  ES3_REQUIRE(head_dim == 16 && Tk > 0, "es3_attn_few_keys: head_dim must be 16 and Tk > 0 (got %d, %d)", head_dim, Tk);
  const size_t smem = (size_t)2 * std::min(Tk, FEW_KEYS_TILE) * H * head_dim * sizeof(float);
  dim3 grid(ceil_div((long long)Nq * H, 256), B);
  attn_few_keys_kernel<16><<<grid, 256, smem, (cudaStream_t)stream>>>((const bf16*)q, ldq, k, v, ldkv, (bf16*)out, ldo, Nq, Tk, H, scale);
  ES3_LAUNCH_CHECK("attn_few_keys_kernel");
  return 0;
}

extern "C" int es3_ln_rows_gelu(const float* x, const float* w, const float* bias, float eps, void* y, long long M, int C,
                                void* stream) {
  ES3_REQUIRE(C % 32 == 0 && C <= 128, "es3_ln_rows_gelu: C=%d must be a multiple of 32 and <= 128", C);
  ln_rows_gelu_kernel<<<(unsigned)ceil_div(M, 8), 256, 0, (cudaStream_t)stream>>>(x, w, bias, eps, (bf16*)y, M, C);
  ES3_LAUNCH_CHECK("ln_rows_gelu_kernel");
  return 0;
}

extern "C" int es3_hyper_masks(const float* up, const float* hyper, const float* obj_logits, float no_obj, float* masks,
                               int B, int HW, int CU, int Ktot, int K, int k_off, void* stream) {
  ES3_REQUIRE(CU == 32 && K <= 8 && k_off + K <= Ktot, "es3_hyper_masks: CU must be 32, K <= 8, k_off + K <= Ktot");
  dim3 grid(ceil_div(HW, 256), B);
  hyper_masks_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(up, hyper, obj_logits, no_obj, masks, HW, Ktot, K, k_off);
  ES3_LAUNCH_CHECK("hyper_masks_kernel");
  return 0;
}

extern "C" int es3_bilinear_nchw_f32(const float* in, float* out, void* bin, float thr, long long planes, int Hi, int Wi,
                                     int Ho, int Wo, void* stream) {
  const long long total = planes * Ho * Wo;
  bilinear_nchw_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(
      in, out, (uint8_t*)bin, thr, Hi, Wi, Ho, Wo, (float)Hi / Ho, (float)Wi / Wo, planes);
  ES3_LAUNCH_CHECK("bilinear_nchw_kernel");
  return 0;
}

extern "C" int es3_mask_downscale_tokens(const float* mask, const float* w0, const float* b0, const float* g1, const float* be1,
                                         const float* w1, const float* b1, const float* g2, const float* be2, const float* w2,
                                         const float* b2, const float* base, long long base_rows, float* out_f32, void* out_bf16,
                                         int B, int h, int w, int C, float eps, void* stream) {
  ES3_REQUIRE(B > 0 && h > 0 && w > 0 && C > 0 && (base == nullptr || base_rows > 0), "es3_mask_downscale_tokens: bad shape");
  MaskDsW wt{w0, b0, g1, be1, w1, b1, g2, be2, w2, b2};
  const long long rows = (long long)B * h * w;
  mask_downscale_kernel<<<(unsigned)ceil_div(rows, 16), 256, 0, (cudaStream_t)stream>>>(mask, wt, base, base_rows, out_f32,
                                                                                       (bf16*)out_bf16, B, h, w, C, eps);
  ES3_LAUNCH_CHECK("mask_downscale_kernel");
  return 0;
}

// in/out [N,H,W] fp32 (out may not alias in); labels_ws / area_ws: N*H*W ints each.
extern "C" int es3_fill_small_components(const float* in, float* out, int* labels_ws, int* area_ws, int N, int H, int W, float thr,
                                         float max_hole_area, float max_sprinkle_area, void* stream) {
  ES3_REQUIRE(N > 0 && H > 0 && W > 0 && (long long)N * H * W < 2147483647LL, "es3_fill_small_components: bad shape");
  ES3_REQUIRE(in != out, "es3_fill_small_components: in-place operation is not supported");
  cudaStream_t st = (cudaStream_t)stream;
  const long long total = (long long)N * H * W;
  const unsigned blocks = (unsigned)ceil_div(total, 256);
  ES3_CHECK_CUDA(cudaMemcpyAsync(out, in, total * sizeof(float), cudaMemcpyDeviceToDevice, st));
  for (int fg = 0; fg < 2; ++fg) {
    const float max_area = fg ? max_sprinkle_area : max_hole_area;
    if (!(max_area > 0.f)) continue;
    cc_init_kernel<<<blocks, 256, 0, st>>>(in, labels_ws, area_ws, total, thr, fg);
    cc_merge_kernel<<<blocks, 256, 0, st>>>(in, labels_ws, N, H, W);
    cc_count_kernel<<<blocks, 256, 0, st>>>(labels_ws, area_ws, total);
    cc_apply_kernel<<<blocks, 256, 0, st>>>(labels_ws, area_ws, out, total, max_area, fg ? thr - 10.f : thr + 10.f);
  }
  ES3_LAUNCH_CHECK("cc kernels");
  return 0;
}
