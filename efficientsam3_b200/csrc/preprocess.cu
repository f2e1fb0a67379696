// Stage-1 image preparation on the device, from decoded uint8 (SA1BDataset.__getitem__, stage1/data/sa1b_dataset.py:163-170,
// 216-227): ResizeLongestSide.apply_image_torch (transforms.py:48-54, 79-85) -- F.interpolate(bilinear, align_corners=False,
// antialias=True) on fp32 0..255 values, longest side to S -- then (x - mean) / std and zero padding to S x S.
//
// Ragged batch: uint8 HWC RGB images back to back in one buffer, a host table of (byte offset, h, w) per image.  Two passes
// through an fp32 workspace: horizontal (w -> w', [h][w'][3] per image), then vertical (h -> h') with normalisation, padding
// and the NCHW store.  Thread = output pixel, all three channels; taps and weights are recomputed per thread.
//
// The tap windows and weights are torch's (aten/src/ATen/native/UpSample.h, _compute_indices_min_size_weights_aa), in fp32:
//   scale = in / out, support = scale >= 1 ? scale : 1, invscale = scale >= 1 ? 1 / scale : 1, center = scale (i + 0.5),
//   window [max(int(center - support + 0.5), 0), min(int(center + support + 0.5), in)),
//   w_j = max(0, 1 - |(j - center + 0.5) invscale|), each divided by the window's fp32 sum.
// Every step is an explicitly rounded intrinsic: nvcc would otherwise contract a*b + c into an FMA, which moves `center` by an
// ulp and, at the SA-1B size, shifts whole tap windows.
#include "common.cuh"

namespace es3 {

constexpr int PREP_MAX_IMAGES = 96;   // per launch: the descriptor table travels as a __grid_constant__ kernel parameter (< 4 KB)

struct PrepImage {
  long long src;   // byte offset of the image in the uint8 buffer
  long long ws;    // float offset of its [h][w'][3] rows in the workspace
  int h, w, ho, wo;
};

struct PrepBatch {
  PrepImage img[PREP_MAX_IMAGES];
  float mean[3], std[3];
  int S;
};

// ResizeLongestSide.get_preprocess_shape (transforms.py:79-85), in double as Python evaluates it.
static void preprocess_shape(long long h, long long w, int S, int* ho, int* wo) {
  const double scale = S * 1.0 / (double)(h > w ? h : w);
  const double nh = (double)h * scale, nw = (double)w * scale;
  *ho = (int)(nh + 0.5);
  *wo = (int)(nw + 0.5);
}

// Torch's antialiased bilinear filter for output index i of an in -> out resize.
struct AaTaps {
  float center, invscale;
  int lo, n;
};

__device__ __forceinline__ AaTaps aa_taps(int i, int in, int out) {
  const float scale = __fdiv_rn((float)in, (float)out);
  const float support = scale >= 1.f ? scale : 1.f;
  AaTaps t;
  t.invscale = scale >= 1.f ? __fdiv_rn(1.f, scale) : 1.f;
  t.center = __fmul_rn(scale, __fadd_rn((float)i, 0.5f));
  t.lo = max((int)__fadd_rn(__fsub_rn(t.center, support), 0.5f), 0);
  t.n = min((int)__fadd_rn(__fadd_rn(t.center, support), 0.5f), in) - t.lo;
  return t;
}

__device__ __forceinline__ float aa_weight(const AaTaps& t, int j) {
  const float x = fabsf(__fmul_rn(__fadd_rn(__fsub_rn((float)(t.lo + j), t.center), 0.5f), t.invscale));
  return x < 1.f ? __fsub_rn(1.f, x) : 0.f;
}

__device__ __forceinline__ float aa_total(const AaTaps& t) {
  float s = 0.f;
  for (int j = 0; j < t.n; ++j) s = __fadd_rn(s, aa_weight(t, j));
  return s;
}

__device__ __forceinline__ float aa_normalised(const AaTaps& t, int j, float total) {
  const float w = aa_weight(t, j);
  return total != 0.f ? __fdiv_rn(w, total) : w;
}

// grid (ceil(max w' / 32), ceil(max h / 8), B), block 32 x 8: ws[y][x'][c] = sum_j w_j src[y][lo + j][c]
__global__ void __launch_bounds__(256) prep_horizontal_kernel(const uint8_t* __restrict__ src, float* __restrict__ ws,
                                                              const __grid_constant__ PrepBatch batch) {
  const PrepImage& im = batch.img[blockIdx.z];
  const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y;
  if (x >= im.wo || y >= im.h) return;
  const AaTaps t = aa_taps(x, im.w, im.wo);
  const float total = aa_total(t);
  const uint8_t* p = src + im.src + ((long long)y * im.w + t.lo) * 3;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f;
  for (int j = 0; j < t.n; ++j, p += 3) {
    const float wj = aa_normalised(t, j, total);
    a0 = fmaf(wj, (float)p[0], a0);
    a1 = fmaf(wj, (float)p[1], a1);
    a2 = fmaf(wj, (float)p[2], a2);
  }
  float* o = ws + im.ws + ((long long)y * im.wo + x) * 3;
  o[0] = a0;
  o[1] = a1;
  o[2] = a2;
}

// grid (ceil(S / 32), ceil(S / 8), B), block 32 x 8: out[b][c][y'][x] = (sum_i w_i ws[lo + i][x][c] - mean[c]) / std[c] inside
// (h', w'), +0 outside.
__global__ void __launch_bounds__(256) prep_vertical_kernel(const float* __restrict__ ws, float* __restrict__ out,
                                                            const __grid_constant__ PrepBatch batch) {
  const PrepImage& im = batch.img[blockIdx.z];
  const int S = batch.S;
  const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y;
  if (x >= S || y >= S) return;
  float v0 = 0.f, v1 = 0.f, v2 = 0.f;
  if (y < im.ho && x < im.wo) {
    const AaTaps t = aa_taps(y, im.h, im.ho);
    const float total = aa_total(t);
    const float* p = ws + im.ws + ((long long)t.lo * im.wo + x) * 3;
    const long long step = 3LL * im.wo;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    for (int i = 0; i < t.n; ++i, p += step) {
      const float wi = aa_normalised(t, i, total);
      a0 = fmaf(wi, p[0], a0);
      a1 = fmaf(wi, p[1], a1);
      a2 = fmaf(wi, p[2], a2);
    }
    // SA1BDataset.norm (sa1b_dataset.py:216-219): (x - mean) / std, a subtraction and a true division
    v0 = __fdiv_rn(__fsub_rn(a0, batch.mean[0]), batch.std[0]);
    v1 = __fdiv_rn(__fsub_rn(a1, batch.mean[1]), batch.std[1]);
    v2 = __fdiv_rn(__fsub_rn(a2, batch.mean[2]), batch.std[2]);
  }
  const long long plane = (long long)S * S;
  float* o = out + (long long)blockIdx.z * 3 * plane + (long long)y * S + x;
  o[0] = v0;
  o[plane] = v1;
  o[2 * plane] = v2;
}

}  // namespace es3

using namespace es3;

extern "C" long long es3_prepare_images_ws_floats(const long long* table, int B, int S) {
  if (B < 1 || S < 1) return -1;
  long long n = 0;
  for (int b = 0; b < B; ++b) {
    const long long h = table[3 * b + 1], w = table[3 * b + 2];
    if (h < 1 || w < 1 || h > 65535LL * 8) return -1;
    int ho, wo;
    preprocess_shape(h, w, S, &ho, &wo);
    if (ho < 1 || wo < 1) return -1;
    n += h * wo * 3;
  }
  return n;
}

extern "C" int es3_prepare_images_u8(const unsigned char* src, long long src_bytes, const long long* table, int B, int S,
                                     const float* mean, const float* std, float* ws, float* out, void* stream) {
  ES3_REQUIRE(B >= 1 && B <= PREP_MAX_IMAGES, "es3_prepare_images_u8: %d images (1..%d per call)", B, PREP_MAX_IMAGES);
  ES3_REQUIRE(es3_prepare_images_ws_floats(table, B, S) >= 0,
              "es3_prepare_images_u8: bad size (S = %d, or an image with a side < 1 before or after the resize)", S);
  PrepBatch batch;
  batch.S = S;
  for (int c = 0; c < 3; ++c) {
    batch.mean[c] = mean[c];
    batch.std[c] = std[c];
  }
  long long wsoff = 0;
  int max_h = 0, max_wo = 0;
  for (int b = 0; b < B; ++b) {
    const long long off = table[3 * b], h = table[3 * b + 1], w = table[3 * b + 2];
    ES3_REQUIRE(off >= 0 && off + h * w * 3 <= src_bytes, "es3_prepare_images_u8: image %d ([%lld, +%lld) bytes) outside the %lld-byte buffer",
                b, off, h * w * 3, src_bytes);
    PrepImage& im = batch.img[b];
    im.src = off;
    im.ws = wsoff;
    im.h = (int)h;
    im.w = (int)w;
    preprocess_shape(h, w, S, &im.ho, &im.wo);
    wsoff += h * im.wo * 3;
    max_h = max(max_h, im.h);
    max_wo = max(max_wo, im.wo);
  }
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 block(32, 8);
  prep_horizontal_kernel<<<dim3((max_wo + 31) / 32, (max_h + 7) / 8, B), block, 0, st>>>(src, ws, batch);
  ES3_LAUNCH_CHECK("prep_horizontal_kernel");
  prep_vertical_kernel<<<dim3((S + 31) / 32, (S + 7) / 8, B), block, 0, st>>>(ws, out, batch);
  ES3_LAUNCH_CHECK("prep_vertical_kernel");
  return 0;
}
