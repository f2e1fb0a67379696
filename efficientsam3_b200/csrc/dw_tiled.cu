// Shared-memory tiled depthwise convolution (NHWC bf16, fp32 math) for the stride-2 3x3 convs with C % 32 == 0 (the stride-1
// shapes run on the tensor-core kernel in dw_tc.cu).
//
// Why: the one-thread-per-output kernel in conv.cu re-reads every input pixel KS*KS times through L1/L2.  Here a block stages
// the haloed input tile of CG channels once (cp.async, zero-filled outside the image), every thread produces a strip of 4 output
// pixels x 8 channels from a sliding register window, and weights sit in shared memory.  HBM traffic = input tile (+halo) once +
// output once.
//
// Block: 256 threads.  Tile: TH x TW outputs x CG channels.  smem pixel stride = CG*2 + 16 bytes
// (the pad keeps 16-byte accesses of 8 consecutive pixels on distinct bank groups).
#include "common.cuh"

namespace es3 {

__device__ __forceinline__ void cp_async16_zfill(void* smem, const void* gmem, bool valid) {
  const uint32_t s = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_1() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }

template <int KS, int STRIDE, int CG, int TH, int TW>
struct DwTile {
  static constexpr int IH = (TH - 1) * STRIDE + KS;
  static constexpr int IW = (TW - 1) * STRIDE + KS;
  static constexpr int PIX_BYTES = CG * 2 + 16;
  static constexpr int TILE_BYTES = IH * IW * PIX_BYTES;
  static constexpr int W_FLOATS = KS * KS * CG;
  static constexpr int WB_FLOATS = W_FLOATS + CG;                      // one (tap weights, bias) set
  static constexpr int SMEM = 2 * TILE_BYTES + 2 * WB_FLOATS * 4;   // double-buffered tile + weights (persistent CTAs)
};

// x: [B,H,W,*] bf16 with pixel stride ldx, channel window [c_in0, c_in0 + C) ; out likewise (ldo, c_out0).
// w: [KS*KS][C] fp32 tap-major (scale folded); bias [C] or null.
// Persistent CTAs over work items (tile, channel group, image): while the strips of item i are computed from one shared-memory
// buffer, the haloed tile (cp.async) and the weights of item i + gridDim.x stream into the other -- the one-item-per-CTA version was
// a load -> wait -> compute -> store sequence with nothing overlapped inside a CTA.
template <int KS, int STRIDE, int CG, int TH, int TW, int ACT>
__global__ void __launch_bounds__(256, (2 * (DwTile<KS, STRIDE, CG, TH, TW>::SMEM + 1024) <= 227 * 1024) ? 2 : 1) dw_tiled_kernel(const bf16* x, long long ldx, const float* __restrict__ w,
                                                       const float* __restrict__ bias, bf16* out, long long ldo,
                                                       int H, int W, int C, int Ho, int Wo, int tiles_x, int tiles_per_img,
                                                       int n_cg, int total_items) {
  using T = DwTile<KS, STRIDE, CG, TH, TW>;
  extern __shared__ __align__(16) uint8_t smem[];
  float* s_wb = reinterpret_cast<float*>(smem + 2 * T::TILE_BYTES);     // [2][W_FLOATS + CG]
  constexpr int PAD = KS / 2;
  constexpr int NV = CG / 8;  // 16-byte vectors per pixel

  // item -> (tile, channel group, image); channel group fastest so that neighbouring CTAs share the input tile in L2
  auto decode = [&](int item, int& tile, int& c0, int& b) {
    const int cg = item % n_cg;
    const int r = item / n_cg;
    tile = r % tiles_per_img;
    b = r / tiles_per_img;
    c0 = cg * CG;
  };
  auto stage = [&](int item, int buf) {
    int tile, c0, b;
    decode(item, tile, c0, b);
    const int ty = tile / tiles_x, tx = tile % tiles_x;
    const int iy0 = ty * TH * STRIDE - PAD, ix0 = tx * TW * STRIDE - PAD;
    uint8_t* s_tile = smem + buf * T::TILE_BYTES;
    const bf16* xb = x + (long long)b * H * W * ldx + c0;
    for (int i = threadIdx.x; i < T::IH * T::IW * NV; i += 256) {
      const int v = i % NV, p = i / NV;
      const int py = p / T::IW, px = p % T::IW;
      const int iy = iy0 + py, ix = ix0 + px;
      const bool ok = (iy >= 0 && iy < H && ix >= 0 && ix < W);
      const bf16* src = ok ? xb + ((long long)iy * W + ix) * ldx + v * 8 : xb;
      cp_async16_zfill(s_tile + p * T::PIX_BYTES + v * 16, src, ok);
    }
    float* s_w = s_wb + buf * T::WB_FLOATS;
    for (int i = threadIdx.x; i < T::W_FLOATS; i += 256) {
      const int tap = i / CG, c = i % CG;
      s_w[i] = w[(long long)tap * C + c0 + c];
    }
    for (int i = threadIdx.x; i < CG; i += 256) s_w[T::W_FLOATS + i] = bias ? bias[c0 + i] : 0.f;
    cp_async_commit();
  };

  int item = blockIdx.x;
  if (item >= total_items) return;
  stage(item, 0);
  int buf = 0;
  for (; item < total_items; item += gridDim.x, buf ^= 1) {
    const int next = item + gridDim.x;
    if (next < total_items) {
      stage(next, buf ^ 1);      // the other buffer was released by the __syncthreads that ended the previous iteration
      cp_async_wait_1();         // everything but the group just committed: this item's tile has landed
    } else {
      cp_async_wait_all();
    }
    int tile, c0, b;
    decode(item, tile, c0, b);
    __syncthreads();
    const uint8_t* s_tile = smem + buf * T::TILE_BYTES;
    const float* s_w = s_wb + buf * T::WB_FLOATS;
    const float* s_b = s_w + T::W_FLOATS;
    const int ty = tile / tiles_x, tx = tile % tiles_x;
    const int oy0 = ty * TH, ox0 = tx * TW;

  // ---- compute: item = (strip of 4 outputs along x, 8-channel group)
  constexpr int STRIPS_X = TW / 4;
  constexpr int ITEMS = TH * STRIPS_X * NV;
  constexpr int WIN = 3 * STRIDE + KS;  // input columns covering 4 outputs
  // (unroll 1: with ITEMS = 2 x 256 the compiler fused both iterations into one 150 .. 255-register body -- one resident CTA per SM,
  //  spills in the 5x5 variants)
#pragma unroll 1
  for (int it = threadIdx.x; it < ITEMS; it += 256) {
    const int v = it % NV;
    const int sidx = it / NV;
    const int sy = sidx / STRIPS_X, sx = sidx % STRIPS_X;
    // accumulators, taps and inputs as channel PAIRS: every multiply-add below is one FFMA2 (two fp32 FMAs per issue slot; the
    // scalar version spent 288 of its ~500 instructions per strip on FFMA and sat on the fma pipe)
    float2 acc[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[j][e] = *reinterpret_cast<const float2*>(s_b + v * 8 + 2 * e);
    // (5x5: rows not unrolled -- the unrolled form hoisted all 25 x 8 tap weights into registers: 255 registers and spills)
#pragma unroll(KS == 3 ? 3 : 1)
    for (int ky = 0; ky < KS; ++ky) {
      float2 wk[KS][4];
#pragma unroll
      for (int kx = 0; kx < KS; ++kx) {
        const float4 a = *reinterpret_cast<const float4*>(s_w + (ky * KS + kx) * CG + v * 8);
        const float4 c = *reinterpret_cast<const float4*>(s_w + (ky * KS + kx) * CG + v * 8 + 4);
        wk[kx][0] = make_float2(a.x, a.y); wk[kx][1] = make_float2(a.z, a.w);
        wk[kx][2] = make_float2(c.x, c.y); wk[kx][3] = make_float2(c.z, c.w);
      }
      const uint8_t* rowp = s_tile + ((sy * STRIDE + ky) * T::IW + sx * 4 * STRIDE) * T::PIX_BYTES + v * 16;
#pragma unroll
      for (int col = 0; col < WIN; ++col) {
        float2 f[4];
        unpack8_2(*reinterpret_cast<const uint4*>(rowp + col * T::PIX_BYTES), f);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int kx = col - j * STRIDE;
          if (kx >= 0 && kx < KS) {
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[j][e] = ffma2(f[e], wk[kx][e], acc[j][e]);
          }
        }
      }
    }
    const int oy = oy0 + sy;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float o[8];
#pragma unroll
      for (int e = 0; e < 4; ++e) { o[2 * e] = es3_act_t<ACT>(acc[j][e].x); o[2 * e + 1] = es3_act_t<ACT>(acc[j][e].y); }
      const int ox = ox0 + sx * 4 + j;
      if (oy < Ho && ox < Wo)
        *reinterpret_cast<uint4*>(out + (((long long)b * Ho + oy) * Wo + ox) * ldo + c0 + v * 8) = pack8(o);
    }
  }
    __syncthreads();     // every strip of this item is done with the buffer before the next iteration refills it
  }
}

template <int KS, int STRIDE, int CG, int TH, int TW, int ACT>
static int launch_dw_tiled(const bf16* x, long long ldx, const float* w, const float* bias, bf16* out, long long ldo, int B, int H, int W, int C, int Ho, int Wo, cudaStream_t st) {
  using T = DwTile<KS, STRIDE, CG, TH, TW>;
  auto kern = dw_tiled_kernel<KS, STRIDE, CG, TH, TW, ACT>;
  static bool configured = false;
  if (!configured) {
    ES3_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, T::SMEM));
    configured = true;
  }
  const int tiles_x = ceil_div(Wo, TW), tiles_y = ceil_div(Ho, TH);
  const int n_cg = C / CG;
  const long long total = (long long)tiles_x * tiles_y * n_cg * B;
  ES3_REQUIRE(total < (1LL << 31), "dw_tiled: too many work items");
  static int sm_count = 0;
  if (sm_count == 0) {
    int dev = 0;
    ES3_CHECK_CUDA(cudaGetDevice(&dev));
    ES3_CHECK_CUDA(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));
  }
  const int per_sm = 2 * (T::SMEM + 1024) <= 227 * 1024 ? 2 : 1;       // resident CTAs (shared memory: two buffers each)
  const long long ctas = (long long)sm_count * per_sm;
  kern<<<(unsigned)(total < ctas ? total : ctas), 256, T::SMEM, st>>>(x, ldx, w, bias, out, ldo, H, W, C, Ho, Wo, tiles_x,
                                                                      tiles_x * tiles_y, n_cg, (int)total);
  ES3_LAUNCH_CHECK("dw_tiled_kernel");
  return 0;
}

}  // namespace es3

using namespace es3;

// Depthwise 3x3, stride 2, pad 1, C % 32 == 0.  Same contract as es3_dwconv_bf16.
extern "C" int es3_dwconv_tiled_bf16(const void* x, long long ldx, const float* w, const float* bias, void* out,
                                     long long ldo, int B, int H, int W, int C, int ks, int stride, int act,
                                     void* stream) {
  ES3_REQUIRE(C % 32 == 0 && ldx % 8 == 0 && ldo % 8 == 0, "es3_dwconv_tiled_bf16: C=%d must be a multiple of 32", C);
  ES3_REQUIRE(ks == 3 && stride == 2, "es3_dwconv_tiled_bf16: unsupported ks=%d stride=%d", ks, stride);
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  cudaStream_t st = (cudaStream_t)stream;
  const bf16* xi = (const bf16*)x;
  bf16* o = (bf16*)out;
  switch (act) {
    case ACT_NONE: return launch_dw_tiled<3, 2, 32, 4, 32, ACT_NONE>(xi, ldx, w, bias, o, ldo, B, H, W, C, Ho, Wo, st);
    case ACT_RELU: return launch_dw_tiled<3, 2, 32, 4, 32, ACT_RELU>(xi, ldx, w, bias, o, ldo, B, H, W, C, Ho, Wo, st);
    case ACT_HSWISH: return launch_dw_tiled<3, 2, 32, 4, 32, ACT_HSWISH>(xi, ldx, w, bias, o, ldo, B, H, W, C, Ho, Wo, st);
    case ACT_GELU: return launch_dw_tiled<3, 2, 32, 4, 32, ACT_GELU>(xi, ldx, w, bias, o, ldo, B, H, W, C, Ho, Wo, st);
  }
  ES3_REQUIRE(false, "es3_dwconv_tiled_bf16: activation %d not instantiated", act);
}
