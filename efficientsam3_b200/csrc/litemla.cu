// EfficientViT LiteMLA ReLU linear attention for any head dim DIM <= 32 -- reference efficientvit/nn/ops.py:592-621.
// efficientvit_b2 / b3 use dim = 32; the tensor-core kernels in litemla_tc.cu are specialised for dim = 16 (b0 / b1, the
// benchmarked student).  CUDA-core formulation, all arithmetic fp32 (the reference forces fp32 here, ops.py:586-589).
//
// Head h owns channels [h*3*dim, (h+1)*3*dim) of the NHWC bf16 input as q | k | v (ops.py:590-606).
//   kv kernel   : KV[b,h] ((dim+1) x dim) = sum_p [v_p ; 1] relu(k_p)^T       (ops.py:609-616, the padded ones row)
//                 two-stage, fixed summation order -> bit-reproducible (no atomics)
//   apply kernel: out_p = KV[:dim] relu(q_p) / (KV[dim] . relu(q_p) + eps)   (ops.py:617-620)
#include "common.cuh"

namespace es3 {
constexpr int GA_PX = 128;

// part: [B][heads2][nchunk][DIM+1][DIM] fp32 partial sums of v^T relu(k) (+ ones row) over a chunk of GA_PX pixels.
template <int DIM>
__global__ void __launch_bounds__(256) litemla_kv_generic_kernel(const bf16* __restrict__ ms, long long ld,
                                                                 float* __restrict__ part, int HW) {
  __shared__ float s_k[GA_PX][DIM + 1];
  __shared__ float s_v[GA_PX][DIM + 1];
  const int h = blockIdx.y, b = blockIdx.z, heads2 = gridDim.y, nchunk = gridDim.x;
  const int p0 = blockIdx.x * GA_PX;
  const bf16* src = ms + (long long)b * HW * ld + h * 3 * DIM;
  for (int i = threadIdx.x; i < GA_PX * DIM; i += 256) {
    const int c = i % DIM, pl = i / DIM;
    const bool ok = p0 + pl < HW;
    const bf16* r = src + (long long)(p0 + pl) * ld;
    s_k[pl][c] = ok ? fmaxf(__bfloat162float(r[DIM + c]), 0.f) : 0.f;
    s_v[pl][c] = ok ? __bfloat162float(r[2 * DIM + c]) : 0.f;
  }
  __syncthreads();
  const int np = min(GA_PX, HW - p0);
  float* dst = part + (((long long)b * heads2 + h) * nchunk + blockIdx.x) * (DIM + 1) * DIM;
  for (int e = threadIdx.x; e < (DIM + 1) * DIM; e += 256) {
    const int i = e / DIM, j = e % DIM;   // i = DIM is the ones row (F.pad(v, value=1), ops.py:613)
    float s = 0.f;
    if (i < DIM) {
      for (int p = 0; p < np; ++p) s = fmaf(s_v[p][i], s_k[p][j], s);
    } else {
      for (int p = 0; p < np; ++p) s += s_k[p][j];
    }
    dst[e] = s;
  }
}

// att[b,p,h*DIM+d] = (KV[d] . relu(q[p])) / (KV[DIM] . relu(q[p]) + eps)
template <int DIM>
__global__ void __launch_bounds__(128) litemla_apply_generic_kernel(const bf16* __restrict__ ms, long long ld,
                                                                    const float* __restrict__ part, int nchunk,
                                                                    bf16* __restrict__ att, long long ldo, int HW, float eps) {
  __shared__ float s_kv[(DIM + 1) * DIM];
  const int h = blockIdx.y, b = blockIdx.z, heads2 = gridDim.y;
  const float* src = part + ((long long)b * heads2 + h) * nchunk * (DIM + 1) * DIM;
  for (int e = threadIdx.x; e < (DIM + 1) * DIM; e += 128) {
    float s = 0.f;
    for (int c = 0; c < nchunk; ++c) s += src[(long long)c * (DIM + 1) * DIM + e];
    s_kv[e] = s;
  }
  __syncthreads();
  const int p = blockIdx.x * 128 + threadIdx.x;
  if (p >= HW) return;
  const bf16* qp = ms + ((long long)b * HW + p) * ld + h * 3 * DIM;
  float q[DIM];
#pragma unroll
  for (int j = 0; j < DIM; ++j) q[j] = fmaxf(__bfloat162float(qp[j]), 0.f);
  float den = 0.f;
#pragma unroll
  for (int j = 0; j < DIM; ++j) den = fmaf(s_kv[DIM * DIM + j], q[j], den);
  const float inv = 1.f / (den + eps);
  bf16* op = att + ((long long)b * HW + p) * ldo + h * DIM;
#pragma unroll 4
  for (int d = 0; d < DIM; ++d) {
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < DIM; ++j) s = fmaf(s_kv[d * DIM + j], q[j], s);
    op[d] = __float2bfloat16(s * inv);
  }
}
}  // namespace es3

using namespace es3;

extern "C" long long es3_litemla_generic_ws_floats(int B, int HW, int heads2, int dim) {
  return (long long)B * heads2 * ceil_div(HW, GA_PX) * (dim + 1) * dim;
}

// ms: [B,HW,ld] bf16 with head h in channels [h*3*dim, (h+1)*3*dim) as q|k|v; att: [B,HW,ldo] bf16, head h in [h*dim, +dim).
extern "C" int es3_litemla_attn_generic(const void* ms, long long ld, float* kv_ws, void* att, long long ldo, int B, int HW,
                                        int heads2, int dim, float eps, void* stream) {
  ES3_REQUIRE(dim == 16 || dim == 32, "es3_litemla_attn_generic: dim=%d not instantiated (16, 32)", dim);
  ES3_REQUIRE(ld >= 3 * dim * heads2 && ldo >= dim * heads2, "es3_litemla_attn_generic: bad ld=%lld ldo=%lld", ld, ldo);
  cudaStream_t st = (cudaStream_t)stream;
  const int nchunk = ceil_div(HW, GA_PX);
  dim3 g1(nchunk, heads2, B), g2(ceil_div(HW, 128), heads2, B);
  if (dim == 16) {
    litemla_kv_generic_kernel<16><<<g1, 256, 0, st>>>((const bf16*)ms, ld, kv_ws, HW);
    litemla_apply_generic_kernel<16><<<g2, 128, 0, st>>>((const bf16*)ms, ld, kv_ws, nchunk, (bf16*)att, ldo, HW, eps);
  } else {
    litemla_kv_generic_kernel<32><<<g1, 256, 0, st>>>((const bf16*)ms, ld, kv_ws, HW);
    litemla_apply_generic_kernel<32><<<g2, 128, 0, st>>>((const bf16*)ms, ld, kv_ws, nchunk, (bf16*)att, ldo, HW, eps);
  }
  ES3_LAUNCH_CHECK("litemla_generic kernels");
  return 0;
}
