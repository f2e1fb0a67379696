// Kernels specific to the RepViT / TinyViT students (sam3/sam3/backbones/repvit.py, tiny_vit.py):
//   * dense 3x3 stride-2 conv with a narrow input (Cin = 32 -> Cout 64..: second patch-embed conv,
//     repvit.py:222-223, tiny_vit.py:75-81) as an implicit GEMM on mma.sync -- 9 taps x (ldmatrix with
//     stride-2 pixel addressing, MMA) per 16 output pixels
//   * SqueezeExcite pieces (timm.layers.SqueezeExcite; repvit.py:136,150): per-image channel means
//     (deterministic two-stage) and the channel-gate multiply.  The two tiny FCs run on es3_gemm_simt.
#include "ptx.cuh"

namespace es3 {
namespace {
__device__ __forceinline__ void cpa16(uint32_t saddr, const void* g, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(saddr), "l"(g), "r"(sz) : "memory");
}
__device__ __forceinline__ void cpa_wait_all() { asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory"); }
}  // namespace

// ---------------------------------------------------------------------------------- conv3x3 s2, Cin = 32 | 48
constexpr int S2_TH = 8, S2_TW = 16, S2_IH = 2 * S2_TH + 1, S2_IW = 2 * S2_TW + 1;

// x [B,H,W,CIN] bf16; w [9][COUT][CIN] bf16 (tap-major, then output channel, K = input channel);
// scale/bias fp32 [COUT] (folded BN); out [B,Ho,Wo,COUT] bf16.  Block 256 = 8 warps, warp = one output row of 16 px.
template <int CIN, int COUT, int ACT>
__global__ void __launch_bounds__(256) conv3x3_s2_c32_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                             const float* __restrict__ scale, const float* __restrict__ bias,
                                                             bf16* __restrict__ out, int H, int W, int Ho, int Wo, int tiles_x) {
  extern __shared__ __align__(16) uint8_t smem[];
  constexpr int S2_CIN = CIN, S2_RS = CIN * 2 + 16, NV = CIN / 8;
  constexpr int TILE_BYTES = S2_IH * S2_IW * S2_RS;
  const uint32_t u_tile = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
  const uint32_t u_w = u_tile + TILE_BYTES;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tile = blockIdx.x, b = blockIdx.y;
  const int oy0 = (tile / tiles_x) * S2_TH, ox0 = (tile % tiles_x) * S2_TW;
  const int iy0 = 2 * oy0 - 1, ix0 = 2 * ox0 - 1;
  const bf16* xb = x + (long long)b * H * W * S2_CIN;
  for (int i = tid; i < S2_IH * S2_IW * NV; i += 256) {
    const int v = i % NV, p = i / NV;
    const int iy = iy0 + p / S2_IW, ix = ix0 + p % S2_IW;
    const bool ok = iy >= 0 && iy < H && ix >= 0 && ix < W;
    cpa16(u_tile + p * S2_RS + v * 16, ok ? xb + ((long long)iy * W + ix) * S2_CIN + v * 8 : xb, ok);
  }
  for (int i = tid; i < 9 * COUT * NV; i += 256) {
    const int v = i % NV, r = i / NV;  // r = tap*COUT + n
    cpa16(u_w + r * S2_RS + v * 16, w + (long long)r * S2_CIN + v * 8, true);
  }
  cpa_wait_all();
  __syncthreads();

  const int a_row = lane & 15, a_kh = lane >> 4;
  const int b_n = (lane & 7) + ((lane >> 4) << 3), b_kh = (lane >> 3) & 1;
  const int g = lane >> 2, t4 = lane & 3;
  float acc[COUT / 8][4];
#pragma unroll
  for (int i = 0; i < COUT / 8; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
#pragma unroll 1
  for (int tap = 0; tap < 9; ++tap) {
    const int ky = tap / 3, kx = tap % 3;
#pragma unroll
    for (int ks = 0; ks < S2_CIN / 16; ++ks) {
      uint32_t af[4];
      ptx::ldsm_x4(u_tile + ((2 * warp + ky) * S2_IW + 2 * a_row + kx) * S2_RS + (ks * 16 + a_kh * 8) * 2, af[0], af[1], af[2], af[3]);
#pragma unroll
      for (int np = 0; np < COUT / 16; ++np) {
        uint32_t b0, b1, b2, b3;
        ptx::ldsm_x4(u_w + (tap * COUT + np * 16 + b_n) * S2_RS + (ks * 16 + b_kh * 8) * 2, b0, b1, b2, b3);
        ptx::mma_16816(acc[2 * np], af, b0, b1);
        ptx::mma_16816(acc[2 * np + 1], af, b2, b3);
      }
    }
  }
  const int oy = oy0 + warp;
  if (oy >= Ho) return;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int ox = ox0 + g + half * 8;
    if (ox >= Wo) continue;
    bf16* dst = out + (((long long)b * Ho + oy) * Wo + ox) * COUT;
#pragma unroll
    for (int nt = 0; nt < COUT / 8; ++nt) {
      const int c = nt * 8 + t4 * 2;
      const float v0 = es3_act_t<ACT>(fmaf(acc[nt][half * 2], scale[c], bias[c]));
      const float v1 = es3_act_t<ACT>(fmaf(acc[nt][half * 2 + 1], scale[c + 1], bias[c + 1]));
      *reinterpret_cast<uint32_t*>(dst + c) = pack_bf16x2(v0, v1);
    }
  }
}

// ---------------------------------------------------------------------------------- SqueezeExcite pieces
// part [B][nchunk][C] partial sums over chunks of 128 pixels; block 256 threads stride the channels.
__global__ void channel_sum_kernel(const bf16* __restrict__ x, float* __restrict__ part, int HW, int C) {
  const int b = blockIdx.y, chunk = blockIdx.x, nchunk = gridDim.x;
  const int p0 = chunk * 128, p1 = min(p0 + 128, HW);
  for (int c = threadIdx.x * 2; c < C; c += blockDim.x * 2) {
    float s0 = 0.f, s1 = 0.f;
    const bf16* xp = x + ((long long)b * HW + p0) * C + c;
    for (int p = p0; p < p1; ++p, xp += C) {
      const float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(xp));
      s0 += f.x; s1 += f.y;
    }
    float* d = part + ((long long)b * nchunk + chunk) * C + c;
    d[0] = s0; d[1] = s1;
  }
}
__global__ void channel_mean_final_kernel(const float* __restrict__ part, float* __restrict__ mean, int nchunk, int C, float inv) {
  const int b = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (int i = 0; i < nchunk; ++i) s += part[((long long)b * nchunk + i) * C + c];
  mean[(long long)b * C + c] = s * inv;
}
// y[b,p,c] = x[b,p,c] * gate[b,c]
__global__ void scale_channels_kernel(const bf16* __restrict__ x, const float* __restrict__ gate, bf16* __restrict__ y, int HW,
                                      int C, long long total8) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total8) return;
  const int cg = C >> 3;
  const int c0 = (int)(i % cg) * 8;
  const long long bp = i / cg;
  const int b = (int)(bp / HW);
  float f[8];
  unpack8(__ldg(reinterpret_cast<const uint4*>(x) + i), f);
  const float4 g0 = __ldg(reinterpret_cast<const float4*>(gate + (long long)b * C + c0));
  const float4 g1 = __ldg(reinterpret_cast<const float4*>(gate + (long long)b * C + c0 + 4));
  f[0] *= g0.x; f[1] *= g0.y; f[2] *= g0.z; f[3] *= g0.w; f[4] *= g1.x; f[5] *= g1.y; f[6] *= g1.z; f[7] *= g1.w;
  reinterpret_cast<uint4*>(y)[i] = pack8(f);
}

}  // namespace es3

using namespace es3;

extern "C" int es3_conv3x3_s2_narrow_bf16(const void* x, const void* w, const float* scale, const float* bias, void* out,
                                          int B, int H, int W, int Cin, int Cout, int act, void* stream) {
  ES3_REQUIRE((Cin == 32 && (Cout == 32 || Cout == 48 || Cout == 64)) || (Cin == 48 && (Cout == 80 || Cout == 96)),
              "es3_conv3x3_s2_narrow_bf16: Cin=%d Cout=%d not instantiated (32: 32/48/64, 48: 80/96)", Cin, Cout);
  ES3_REQUIRE(act == ACT_NONE || act == ACT_GELU, "es3_conv3x3_s2_narrow_bf16: act %d not instantiated", act);
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const int tiles_x = ceil_div(Wo, S2_TW), tiles_y = ceil_div(Ho, S2_TH);
  const size_t rs = (size_t)Cin * 2 + 16;
  const size_t smem = (size_t)S2_IH * S2_IW * rs + (size_t)9 * Cout * rs;
  dim3 grid(tiles_x * tiles_y, B);
  cudaStream_t st = (cudaStream_t)stream;
#define ES3_S2(CI, CO, A)                                                                                                  \
  {                                                                                                                        \
    auto k = conv3x3_s2_c32_kernel<CI, CO, A>;                                                                             \
    ES3_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));                      \
    k<<<grid, 256, smem, st>>>((const bf16*)x, (const bf16*)w, scale, bias, (bf16*)out, H, W, Ho, Wo, tiles_x);           \
  }
#define ES3_S2_ACT(CI, CO)                                                                                                 \
  if (act == ACT_NONE) ES3_S2(CI, CO, ACT_NONE) else ES3_S2(CI, CO, ACT_GELU)
  if (Cin == 32) {
    if (Cout == 64) { ES3_S2_ACT(32, 64) } else if (Cout == 48) { ES3_S2_ACT(32, 48) } else { ES3_S2_ACT(32, 32) }
  } else {
    if (Cout == 80) { ES3_S2_ACT(48, 80) } else { ES3_S2_ACT(48, 96) }
  }
#undef ES3_S2_ACT
#undef ES3_S2
  ES3_LAUNCH_CHECK("conv3x3_s2_c32_kernel");
  return 0;
}

// mean over HW of x [B,HW,C] bf16 -> [B,C] fp32.  ws: B * ceil(HW/128) * C floats.
extern "C" int es3_channel_mean(const void* x, float* ws, float* mean, int B, int HW, int C, void* stream) {
  ES3_REQUIRE(C % 2 == 0, "es3_channel_mean: C must be even");
  const int nchunk = ceil_div(HW, 128);
  cudaStream_t st = (cudaStream_t)stream;
  channel_sum_kernel<<<dim3(nchunk, B), 256, 0, st>>>((const bf16*)x, ws, HW, C);
  ES3_LAUNCH_CHECK("channel_sum_kernel");
  channel_mean_final_kernel<<<dim3(ceil_div(C, 256), B), 256, 0, st>>>(ws, mean, nchunk, C, 1.f / HW);
  ES3_LAUNCH_CHECK("channel_mean_final_kernel");
  return 0;
}

extern "C" int es3_scale_channels(const void* x, const float* gate, void* y, int B, int HW, int C, void* stream) {
  ES3_REQUIRE(C % 8 == 0, "es3_scale_channels: C %% 8 != 0");
  const long long total8 = (long long)B * HW * (C / 8);
  scale_channels_kernel<<<(unsigned)ceil_div(total8, 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)x, gate, (bf16*)y, HW, C, total8);
  ES3_LAUNCH_CHECK("scale_channels_kernel");
  return 0;
}
