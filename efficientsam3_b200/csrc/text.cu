// Text-encoder pieces that are not GEMMs, LayerNorms or attention (those reuse the ViT kernels):
//   es3_text_embed     nn.Embedding lookup + positional add (mobile_clip.py:815-823, text_encoder_ve.py:232-238)
//   es3_repmixer_bf16  the RepMixerBlock prologue in eval mode (mobile_clip.py:545-702): folded token mixer, then the
//                      ConvFFN's folded depthwise 1x11 + BatchNorm, written as the bf16 A operand of fc1
#include "common.cuh"

namespace es3 {

// One thread per 4 channels of one token.  ids are validated on the host before they reach the device; an id outside
// [0, vocab) still never reads outside the table here (its row is written as zeros).
__global__ void text_embed_kernel(const long long* __restrict__ ids, const float* __restrict__ table, int vocab,
                                  const float* __restrict__ pos, float* __restrict__ x, float* __restrict__ emb,
                                  int L, int C4, long long n4) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const long long tok = i / C4;
    const int c4 = (int)(i - tok * C4);
    const long long id = ids[tok];
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
    if (id >= 0 && id < vocab) t = reinterpret_cast<const float4*>(table)[id * C4 + c4];
    float4 y = t;
    if (pos != nullptr) {
      const float4 p = reinterpret_cast<const float4*>(pos)[(tok % L) * C4 + c4];
      y = make_float4(t.x + p.x, t.y + p.y, t.z + p.z, t.w + p.w);
    }
    reinterpret_cast<float4*>(x)[i] = y;
    if (emb != nullptr) reinterpret_cast<float4*>(emb)[i] = t;
  }
}

constexpr int RM_KS = 11, RM_HALO = RM_KS / 2, RM_CH = 32, RM_MAXL = 128, RM_THREADS = 256;

// One CTA = one sequence x 32 channels; the whole sequence (plus zero halos) stays in shared memory for both convs.
//   x1[l] = bm + sum_k wm[k] x[l + k - 5]      (RepMixer: identity, BN_skip difference, BN(conv) and layer scale folded)
//   u[l]  = bf + sum_k wf[k] x1[l + k - 5]     (ConvFFN.conv: depthwise 1x11 + BN folded), rounded to bf16
__global__ void __launch_bounds__(RM_THREADS) repmixer_kernel(const float* __restrict__ x, float* __restrict__ x1,
                                                              bf16* __restrict__ u, const float* __restrict__ wm,
                                                              const float* __restrict__ bm, const float* __restrict__ wf,
                                                              const float* __restrict__ bfb, int L, int C) {
  __shared__ float sx[(RM_MAXL + 2 * RM_HALO) * RM_CH];
  __shared__ float sx1[(RM_MAXL + 2 * RM_HALO) * RM_CH];
  const int c = threadIdx.x % RM_CH, r0 = threadIdx.x / RM_CH, rstep = RM_THREADS / RM_CH;
  const int ch = blockIdx.x * RM_CH + c;
  const long long base = (long long)blockIdx.y * L * C + ch;
  for (int l = r0; l < L + 2 * RM_HALO; l += rstep) {
    const int t = l - RM_HALO;
    sx[l * RM_CH + c] = (t >= 0 && t < L) ? x[base + (long long)t * C] : 0.f;
    if (t < 0 || t >= L) sx1[l * RM_CH + c] = 0.f;
  }
  float w[RM_KS];
#pragma unroll
  for (int k = 0; k < RM_KS; ++k) w[k] = wm[k * C + ch];
  float b = bm[ch];
  __syncthreads();
  for (int l = r0; l < L; l += rstep) {
    float acc = b;
#pragma unroll
    for (int k = 0; k < RM_KS; ++k) acc = fmaf(w[k], sx[(l + k) * RM_CH + c], acc);
    sx1[(l + RM_HALO) * RM_CH + c] = acc;
    x1[base + (long long)l * C] = acc;
  }
#pragma unroll
  for (int k = 0; k < RM_KS; ++k) w[k] = wf[k * C + ch];
  b = bfb[ch];
  __syncthreads();
  for (int l = r0; l < L; l += rstep) {
    float acc = b;
#pragma unroll
    for (int k = 0; k < RM_KS; ++k) acc = fmaf(w[k], sx1[(l + k) * RM_CH + c], acc);
    u[base + (long long)l * C] = __float2bfloat16_rn(acc);
  }
}

}  // namespace es3

using namespace es3;

extern "C" int es3_text_embed(const long long* ids, const float* table, int vocab, const float* pos, float* x, float* emb, int B,
                              int L, int C, void* stream) {
  ES3_REQUIRE(B >= 1 && L >= 1 && C >= 4 && C % 4 == 0, "es3_text_embed: need B, L >= 1 and C %% 4 == 0 (B=%d L=%d C=%d)", B, L, C);
  ES3_REQUIRE(vocab >= 1, "es3_text_embed: empty table");
  const long long n4 = (long long)B * L * (C / 4);
  const int grid = (int)((n4 + 255) / 256 < 132 * 16 ? (n4 + 255) / 256 : 132 * 16);
  text_embed_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(ids, table, vocab, pos, x, emb, L, C / 4, n4);
  ES3_LAUNCH_CHECK("text_embed_kernel");
  return 0;
}

extern "C" int es3_repmixer_bf16(const float* x, float* x1, void* u, const float* wm, const float* bm, const float* wf,
                                 const float* bf, int B, int L, int C, void* stream) {
  ES3_REQUIRE(L >= 1 && L <= RM_MAXL, "es3_repmixer_bf16: sequence length %d outside 1..%d (the sequence is kept in shared memory)",
              L, RM_MAXL);
  ES3_REQUIRE(B >= 1 && C % RM_CH == 0, "es3_repmixer_bf16: need B >= 1 and C %% %d == 0 (B=%d C=%d)", RM_CH, B, C);
  repmixer_kernel<<<dim3(C / RM_CH, B), RM_THREADS, 0, (cudaStream_t)stream>>>(x, x1, (bf16*)u, wm, bm, wf, bf, L, C);
  ES3_LAUNCH_CHECK("repmixer_kernel");
  return 0;
}
