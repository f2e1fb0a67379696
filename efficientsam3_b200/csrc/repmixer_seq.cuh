// The sequence layout of the RepMixerBlock training kernels, shared by repmixer_bwd.cu (frozen BatchNorm) and repmixer_bn_train.cu
// (batch statistics): one CTA per (sequence, 32 channels) holds the sequence plus zero halos in shared memory, as repmixer_kernel
// does.  Each CTA writes its per-channel sums (the 8 row groups added in order) to part [B][Q][C]; repmixer_sum_kernel then adds
// the sequences in index order and accumulates (+=) into the gradients in torch layouts (taps [C,1,1,11], layer scales [C,1,1]).
// No float atomics: a backward pass is bit-reproducible.
#pragma once
#include "common.cuh"

namespace es3 {

constexpr int SQ_KS = 11, SQ_HALO = SQ_KS / 2, SQ_CH = 32, SQ_MAXL = 128, SQ_THREADS = 256, SQ_ROWS = SQ_THREADS / SQ_CH;
constexpr int SQ_PAD = SQ_MAXL + 2 * SQ_HALO;

// part[(b Q + q) C + ch0 + c] = sum over the CTA's row groups (in order) of v[q].  red: Q * SQ_ROWS * SQ_CH floats of shared
// memory, which may alias a buffer the caller has finished reading (the first barrier orders that).
template <int Q>
__device__ __forceinline__ void cta_partials(const float (&v)[Q], float* red, float* __restrict__ part, int b, int C, int ch0) {
  const int c = threadIdx.x % SQ_CH, r = threadIdx.x / SQ_CH;
  __syncthreads();
#pragma unroll
  for (int q = 0; q < Q; ++q) red[(q * SQ_ROWS + r) * SQ_CH + c] = v[q];
  __syncthreads();
  for (int i = threadIdx.x; i < Q * SQ_CH; i += SQ_THREADS) {
    const int q = i / SQ_CH, cc = i % SQ_CH;
    float s = 0.f;
#pragma unroll
    for (int rr = 0; rr < SQ_ROWS; ++rr) s += red[(q * SQ_ROWS + rr) * SQ_CH + cc];
    part[((long long)b * Q + q) * C + ch0 + cc] = s;
  }
}

// s[l + 5] = the sequence's rows, zero halos.
__device__ __forceinline__ void load_seq(const float* __restrict__ src, float* s, long long base, int L, int C) {
  const int c = threadIdx.x % SQ_CH;
  for (int l = threadIdx.x / SQ_CH; l < L + 2 * SQ_HALO; l += SQ_ROWS) {
    const int t = l - SQ_HALO;
    s[l * SQ_CH + c] = (t >= 0 && t < L) ? src[base + (long long)t * C] : 0.f;
  }
}

__device__ __forceinline__ float conv_at(const float (&w)[SQ_KS], const float* s, int l, float acc) {
  const int c = threadIdx.x % SQ_CH;
#pragma unroll
  for (int k = 0; k < SQ_KS; ++k) acc = fmaf(w[k], s[(l + k) * SQ_CH + c], acc);
  return acc;
}

namespace {   // a kernel and its launcher: one copy per translation unit

// Destinations of the summed partials: dst[j][c * stride[j]] += sign[j] * sum_b part[b][src[j]][c].
constexpr int SQ_MAXSUM = 20;
struct RbSums {
  int n, Q;
  int src[SQ_MAXSUM], stride[SQ_MAXSUM];
  float sign[SQ_MAXSUM];
  float* dst[SQ_MAXSUM];
};

__global__ void repmixer_sum_kernel(const float* __restrict__ part, int nseq, int C, RbSums s) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y;
  if (c >= C) return;
  const int q = s.src[j];
  float acc = 0.f;
  for (int b = 0; b < nseq; ++b) acc += part[((long long)b * s.Q + q) * C + c];
  float* d = s.dst[j] + (long long)c * s.stride[j];
  *d += s.sign[j] * acc;
}

struct SumBuilder {
  RbSums s;
  explicit SumBuilder(int Q) { s.n = 0; s.Q = Q; }
  void add(int src, float* dst, int stride = 1, float sign = 1.f) {
    if (dst == nullptr) return;
    s.src[s.n] = src; s.dst[s.n] = dst; s.stride[s.n] = stride; s.sign[s.n] = sign;
    ++s.n;
  }
  void taps(float* dw) {                      // tap k of a [C,1,1,11] weight gradient: dw[c * 11 + k]
    if (dw == nullptr) return;
    for (int k = 0; k < SQ_KS; ++k) add(k, dw + k, SQ_KS);
  }
};

int launch_sums(const SumBuilder& sb, const float* part, int B, int C, cudaStream_t st) {
  if (sb.s.n == 0) return 0;
  repmixer_sum_kernel<<<dim3(ceil_div(C, 128), sb.s.n), 128, 0, st>>>(part, B, C, sb.s);
  ES3_LAUNCH_CHECK("repmixer_sum_kernel");
  return 0;
}

}  // namespace
}  // namespace es3
