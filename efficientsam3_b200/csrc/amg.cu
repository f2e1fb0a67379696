// Post-processing of automatic mask generation ("segment everything", SamAutomaticMaskGenerator in
// efficientsam3_b200/model/automatic_mask_generator.py; the semantics are those of SAM1's segment_anything/utils/amg.py).
//
// The masks are never materialised at crop resolution.  Each pixel of a mask is the bilinear (align_corners=False) sample of
// its low-resolution logits, evaluated by bilinear.cuh exactly as es3_bilinear_nchw_f32 evaluates it, so every statistic here
// is a function of the same fp32 values that kernel would write.
//
//   es3_amg_mask_stats  per batch of decoded masks: the predicted-IoU filter, the stability score (pixel counts above
//                       thr + offset and thr - offset), the box of (v > thr) and the crop-edge test; survivors are appended,
//                       in mask order, to a per-crop arena (low-res logits, box, IoU, stability, point index, device count).
//   es3_box_nms         torchvision.ops.batched_nms with one category, with a defined tie order: a stable descending sort.
//   es3_amg_rle         column-major run-length encoding of the kept masks in the original image frame (and optionally the
//                       uint8 masks), in two passes over the pixels: transitions counted per column, scanned, then written.
//
// All counts are integers reduced with warp reductions and atomics, so every result is exact and independent of the order in
// which CTAs run.
#include "bilinear.cuh"

namespace es3 {

// ------------------------------------------------------------------------------------ mask statistics
constexpr int AMG_THREADS = 256;
constexpr int AMG_STAGE_FLOATS = 12288;   // 48 KB of staged low-res rows per CTA
constexpr int AMG_MAX_BAND = 64;          // output rows per CTA
// per-mask workspace ints: intersections, unions, box of (v > thr) (x min, x max, y min, y max), arena slot or -1
enum { ST_INTER = 0, ST_UNION, ST_XMIN, ST_XMAX, ST_YMIN, ST_YMAX, ST_SLOT, ST_N };

__device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

__global__ void amg_stats_init_kernel(int* __restrict__ ws, int M) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  int* w = ws + (long long)m * ST_N;
  w[ST_INTER] = 0;
  w[ST_UNION] = 0;
  w[ST_XMIN] = INT_MAX;
  w[ST_XMAX] = -1;
  w[ST_YMIN] = INT_MAX;
  w[ST_YMAX] = -1;
  w[ST_SLOT] = -1;
}

// One CTA = a band of output rows of one mask.  The low-res rows the band samples are staged in shared memory (they are read
// ~ (Ho / Hi) x (Wo / Wi) times each); a band whose rows do not fit reads them from global memory instead.
__global__ void __launch_bounds__(AMG_THREADS) amg_stats_kernel(const float* __restrict__ low, const float* __restrict__ iou,
                                                                int Hi, int Wi, int Ho, int Wo, float sy, float sx, int band,
                                                                float thr, float thr_hi, float thr_lo, float iou_thresh,
                                                                int filters, int* __restrict__ ws) {
  __shared__ float s_rows[AMG_STAGE_FLOATS];
  const int m = blockIdx.y;
  if ((filters & 1) && !(__ldg(iou + m) > iou_thresh)) return;   // the IoU filter drops the mask before anything is counted
  const int r0 = blockIdx.x * band, r1 = min(r0 + band, Ho);
  const int ylo = bilinear_tap(r0, sy, Hi).i0, yhi = bilinear_tap(r1 - 1, sy, Hi).i1;   // taps are monotone in the row
  const float* src = low + (long long)m * Hi * Wi + (long long)ylo * Wi;
  const int nst = (yhi - ylo + 1) * Wi;
  const bool staged = nst <= AMG_STAGE_FLOATS;
  if (staged)
    for (int i = threadIdx.x; i < nst; i += AMG_THREADS) s_rows[i] = __ldg(src + i);
  __syncthreads();
  const float* rows = staged ? s_rows : src;
  int inter = 0, uni = 0, xmin = INT_MAX, xmax = -1, ymin = INT_MAX, ymax = -1;
  int oy = r0, ox = threadIdx.x;
  while (ox >= Wo) { ox -= Wo; ++oy; }
  BilinearTap ty = bilinear_tap(oy, sy, Hi);
  for (; oy < r1;) {
    const BilinearTap tx = bilinear_tap(ox, sx, Wi);
    const float* a = rows + (ty.i0 - ylo) * Wi;
    const float* b = rows + (ty.i1 - ylo) * Wi;
    const float v = bilinear_mix(ty, tx, a[tx.i0], a[tx.i1], b[tx.i0], b[tx.i1]);
    inter += v > thr_hi;
    uni += v > thr_lo;
    if (v > thr) {
      xmin = min(xmin, ox); xmax = max(xmax, ox);
      ymin = min(ymin, oy); ymax = max(ymax, oy);
    }
    ox += AMG_THREADS;
    if (ox >= Wo) {
      do { ox -= Wo; ++oy; } while (ox >= Wo);
      if (oy < r1) ty = bilinear_tap(oy, sy, Hi);
    }
  }
  const unsigned full = 0xffffffffu;
  inter = (int)__reduce_add_sync(full, (unsigned)inter);
  uni = (int)__reduce_add_sync(full, (unsigned)uni);
  xmin = __reduce_min_sync(full, xmin); xmax = __reduce_max_sync(full, xmax);
  ymin = __reduce_min_sync(full, ymin); ymax = __reduce_max_sync(full, ymax);
  if ((threadIdx.x & 31) == 0) {
    int* w = ws + (long long)m * ST_N;
    if (inter) atomicAdd(w + ST_INTER, inter);
    if (uni) atomicAdd(w + ST_UNION, uni);
    if (xmax >= 0) {
      atomicMin(w + ST_XMIN, xmin); atomicMax(w + ST_XMAX, xmax);
      atomicMin(w + ST_YMIN, ymin); atomicMax(w + ST_YMAX, ymax);
    }
  }
}

struct AmgFrame {
  int x0, y0, x1, y1;   // crop box, XYXY in the original image
  int W, H;             // original image size
};

// |a - b| <= 20 on integer-valued coordinates: torch.isclose(atol=20, rtol=0) of is_box_near_crop_edge, exactly.
__device__ __forceinline__ bool near20(int a, int b) { return abs(a - b) <= 20; }

// One CTA: filters in mask order, then a block scan places the survivors after the arena's current count.
__global__ void __launch_bounds__(AMG_THREADS) amg_finalize_kernel(const float* __restrict__ iou, int M, int K, float iou_thresh,
                                                                   float stab_thresh, int filters, AmgFrame fr, int point_base,
                                                                   int* __restrict__ ws, int* __restrict__ a_box,
                                                                   float* __restrict__ a_iou, float* __restrict__ a_stab,
                                                                   int* __restrict__ a_point, int* __restrict__ a_count, int cap) {
  __shared__ int s_warp[AMG_THREADS / 32];
  __shared__ int s_base;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_base = *a_count;
  __syncthreads();
  int base = s_base;
  for (int c = 0; c < M; c += AMG_THREADS) {
    const int m = c + threadIdx.x;
    bool keep = false;
    float io = 0.f, st = 0.f;
    int box[4] = {0, 0, 0, 0};
    if (m < M) {
      const int* w = ws + (long long)m * ST_N;
      io = iou[m];
      keep = !(filters & 1) || io > iou_thresh;
      if (keep) {
        st = __fdiv_rn((float)w[ST_INTER], (float)w[ST_UNION]);   // 0 / 0 = NaN, which fails `>=`
        if ((filters & 2) && !(st >= stab_thresh)) keep = false;
      }
      if (keep) {
        if (w[ST_XMAX] >= 0) { box[0] = w[ST_XMIN]; box[1] = w[ST_YMIN]; box[2] = w[ST_XMAX]; box[3] = w[ST_YMAX]; }
        const int ub[4] = {box[0] + fr.x0, box[1] + fr.y0, box[2] + fr.x0, box[3] + fr.y0};
        const int cb[4] = {fr.x0, fr.y0, fr.x1, fr.y1};
        const int ob[4] = {0, 0, fr.W, fr.H};
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (near20(ub[i], cb[i]) && !near20(ub[i], ob[i])) keep = false;
      }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    int off = 0, tot = 0;
#pragma unroll
    for (int i = 0; i < AMG_THREADS / 32; ++i) {
      off += i < warp ? s_warp[i] : 0;
      tot += s_warp[i];
    }
    const int slot = base + off + __popc(bal & lanemask_lt());
    if (m < M) ws[(long long)m * ST_N + ST_SLOT] = keep && slot < cap ? slot : -1;
    if (keep && slot < cap) {
#pragma unroll
      for (int i = 0; i < 4; ++i) a_box[(long long)slot * 4 + i] = box[i];
      a_iou[slot] = io;
      a_stab[slot] = st;
      a_point[slot] = point_base + m / K;
    }
    base += tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) *a_count = base;   // may exceed cap: the caller sized the arena and checks
}

__global__ void amg_compact_kernel(const float* __restrict__ low, long long plane, const int* __restrict__ ws,
                                   float* __restrict__ a_low) {
  const int m = blockIdx.y;
  const int slot = ws[(long long)m * ST_N + ST_SLOT];
  if (slot < 0) return;
  const float* s = low + (long long)m * plane;
  float* d = a_low + (long long)slot * plane;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < plane; i += (long long)gridDim.x * blockDim.x)
    d[i] = __ldg(s + i);
}

// ------------------------------------------------------------------------------------ box NMS
constexpr int NMS_MAX = 65536;
constexpr int NMS_THREADS = 256;

// Total order of the scores, descending: NaN first (as torch.sort), then +inf .. -inf; -0 and +0 are equal.
__device__ __forceinline__ unsigned score_key(float f) {
  if (f != f) return 0xffffffffu;
  if (f == 0.f) return 0x80000000u;
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// rank[i] = #{j : key_j > key_i, or key_j == key_i and j < i}; order[rank[i]] = i.  O(N^2) comparisons, which at the 12288
// candidates of a 64 x 64 grid is a few tens of microseconds across the GPU, and stable by construction.
__global__ void __launch_bounds__(NMS_THREADS) nms_rank_kernel(const float* __restrict__ scores, int N, int* __restrict__ order) {
  __shared__ unsigned s_key[NMS_THREADS];
  const int i = blockIdx.x * NMS_THREADS + threadIdx.x;
  const unsigned ki = i < N ? score_key(scores[i]) : 0u;
  int rank = 0;
  for (int t = 0; t < N; t += NMS_THREADS) {
    __syncthreads();
    if (t + threadIdx.x < N) s_key[threadIdx.x] = score_key(scores[t + threadIdx.x]);
    __syncthreads();
    const int n = min(NMS_THREADS, N - t);
    for (int j = 0; j < n; ++j) {
      const unsigned kj = s_key[j];
      rank += (kj > ki) || (kj == ki && t + j < i);
    }
  }
  if (i < N) order[rank] = i;
}

__device__ __forceinline__ float4 load_box(const int* __restrict__ boxes, int i) {
  const int* b = boxes + (long long)i * 4;
  return make_float4((float)b[0], (float)b[1], (float)b[2], (float)b[3]);
}

// torchvision's nms_kernel_impl (csrc/ops/cpu/nms_kernel.cpp): areas (x2 - x1)(y2 - y1), ovr = inter / (area_i + area_j - inter)
// in fp32, suppression when ovr > the (double) threshold.  Explicit roundings keep the order of the reference's operations.
__device__ __forceinline__ bool iou_above(float4 a, float area_a, float4 b, double thr) {
  const float area_b = __fmul_rn(b.z - b.x, b.w - b.y);
  const float w = fmaxf(0.f, fminf(a.z, b.z) - fmaxf(a.x, b.x));
  const float h = fmaxf(0.f, fminf(a.w, b.w) - fmaxf(a.y, b.y));
  const float inter = __fmul_rn(w, h);
  const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter));
  return (double)ovr > thr;
}

// mask[i][cb] bit k: the box at sorted position i suppresses the one at cb * 64 + k (> i), if i is kept.  Blocks below the
// diagonal are never read and not written.
__global__ void __launch_bounds__(64) nms_mask_kernel(const int* __restrict__ boxes, const int* __restrict__ order, int N, int nb,
                                                      double thr, unsigned long long* __restrict__ mask) {
  const int rb = blockIdx.y, cb = blockIdx.x;
  if (cb < rb) return;
  __shared__ float4 s_box[64];
  const int j0 = cb * 64, nj = min(64, N - j0);
  if ((int)threadIdx.x < nj) s_box[threadIdx.x] = load_box(boxes, order[j0 + threadIdx.x]);
  __syncthreads();
  const int i = rb * 64 + threadIdx.x;
  if (i >= N) return;
  const float4 a = load_box(boxes, order[i]);
  const float area_a = __fmul_rn(a.z - a.x, a.w - a.y);
  unsigned long long bits = 0ull;
  for (int k = (cb == rb ? threadIdx.x + 1 : 0); k < nj; ++k)
    if (iou_above(a, area_a, s_box[k], thr)) bits |= 1ull << k;
  mask[(long long)i * nb + cb] = bits;
}

// One CTA sweeps the sorted boxes: thread 0 resolves a 64-box block against its diagonal word, then every thread folds the
// block's kept rows into the removed words of the later blocks it owns.
__global__ void __launch_bounds__(NMS_THREADS) nms_sweep_kernel(const unsigned long long* __restrict__ mask, const int* __restrict__ order,
                                                                int N, int nb, int* __restrict__ keep, int* __restrict__ count) {
  __shared__ unsigned long long s_removed[NMS_MAX / 64];
  __shared__ int s_kept[64];
  __shared__ int s_nk, s_total;
  for (int i = threadIdx.x; i < nb; i += NMS_THREADS) s_removed[i] = 0ull;
  if (threadIdx.x == 0) s_total = 0;
  __syncthreads();
  for (int b = 0; b < nb; ++b) {
    if (threadIdx.x == 0) {
      unsigned long long w = s_removed[b];
      int nk = 0, total = s_total;
      const int n = min(64, N - b * 64);
      for (int k = 0; k < n; ++k) {
        if ((w >> k) & 1ull) continue;
        const int i = b * 64 + k;
        s_kept[nk++] = i;
        keep[total++] = order[i];
        w |= mask[(long long)i * nb + b];
      }
      s_nk = nk;
      s_total = total;
    }
    __syncthreads();
    const int nk = s_nk;
    for (int cb = b + 1 + threadIdx.x; cb < nb; cb += NMS_THREADS) {
      unsigned long long r = s_removed[cb];
      for (int t = 0; t < nk; ++t) r |= mask[(long long)s_kept[t] * nb + cb];
      s_removed[cb] = r;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *count = s_total;
}

// ------------------------------------------------------------------------------------ RLE
constexpr int RLE_THREADS = 128;

struct AmgRleArgs {
  const float* low;
  int Hi, Wi;
  float sy, sx;
  float thr;
  AmgFrame fr;
};

// Pixel (x, y) of mask k in the original frame: outside the crop 0, inside the bilinear sample at the crop-relative position.
__device__ __forceinline__ bool rle_pixel(const AmgRleArgs& a, const float* __restrict__ p, const BilinearTap& tx, int y) {
  if (y < a.fr.y0 || y >= a.fr.y1) return false;
  const BilinearTap ty = bilinear_tap(y - a.fr.y0, a.sy, a.Hi);
  const float* r0 = p + ty.i0 * a.Wi;
  const float* r1 = p + ty.i1 * a.Wi;
  return bilinear_mix(ty, tx, __ldg(r0 + tx.i0), __ldg(r0 + tx.i1), __ldg(r1 + tx.i0), __ldg(r1 + tx.i1)) > a.thr;
}

__device__ __forceinline__ bool rle_in_cols(const AmgRleArgs& a, int x) { return x >= a.fr.x0 && x < a.fr.x1; }

// The value before column x's first pixel in column-major order: pixel (x - 1, H - 1), or 0 before the first pixel.
__device__ __forceinline__ bool rle_prev(const AmgRleArgs& a, const float* __restrict__ p, int x) {
  if (x == 0 || !rle_in_cols(a, x - 1)) return false;
  return rle_pixel(a, p, bilinear_tap(x - 1 - a.fr.x0, a.sx, a.Wi), a.fr.H - 1);
}

// Pass 1: thread = column of one mask.  Transitions (v[p] != v[p - 1], with v[-1] = 0) and ones per column; the optional uint8
// mask is written row-major, so a warp's stores at one row are contiguous.
__global__ void __launch_bounds__(RLE_THREADS) amg_rle_count_kernel(AmgRleArgs a, int* __restrict__ col_n, int* __restrict__ col_area,
                                                                    uint8_t* __restrict__ bin) {
  const int k = blockIdx.y, x = blockIdx.x * RLE_THREADS + threadIdx.x;
  const int W = a.fr.W, H = a.fr.H;
  if (x >= W) return;
  const float* p = a.low + (long long)k * a.Hi * a.Wi;
  bool prev = rle_prev(a, p, x);
  int n = 0, area = 0;
  uint8_t* bk = bin ? bin + (long long)k * H * W + x : nullptr;
  if (!rle_in_cols(a, x)) {
    n = prev;
    if (bk)
      for (int y = 0; y < H; ++y) bk[(long long)y * W] = 0;
  } else {
    const BilinearTap tx = bilinear_tap(x - a.fr.x0, a.sx, a.Wi);
    for (int y = 0; y < H; ++y) {
      const bool v = rle_pixel(a, p, tx, y);
      n += v != prev;
      area += v;
      prev = v;
      if (bk) bk[(long long)y * W] = v;
    }
  }
  col_n[(long long)k * W + x] = n;
  col_area[(long long)k * W + x] = area;
}

// Per mask: exclusive scan of the column counts in place, the mask's transition total and its area.
__global__ void __launch_bounds__(RLE_THREADS) amg_rle_scan_kernel(int W, int* __restrict__ col_n, const int* __restrict__ col_area,
                                                                   int* __restrict__ n_trans, int* __restrict__ area) {
  __shared__ int s_sum[RLE_THREADS / 32], s_area[RLE_THREADS / 32];
  const int k = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int* cn = col_n + (long long)k * W;
  const int* ca = col_area + (long long)k * W;
  const int per = (W + RLE_THREADS - 1) / RLE_THREADS;
  const int c0 = min(W, threadIdx.x * per), c1 = min(W, c0 + per);
  int s = 0, ar = 0;
  for (int c = c0; c < c1; ++c) { s += cn[c]; ar += ca[c]; }
  int incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  ar = (int)__reduce_add_sync(0xffffffffu, (unsigned)ar);
  if (lane == 31) s_sum[warp] = incl;
  if (lane == 0) s_area[warp] = ar;
  __syncthreads();
  int off = incl - s, tot = 0, atot = 0;
#pragma unroll
  for (int i = 0; i < RLE_THREADS / 32; ++i) {
    off += i < warp ? s_sum[i] : 0;
    tot += s_sum[i];
    atot += s_area[i];
  }
  for (int c = c0; c < c1; ++c) {
    const int n = cn[c];
    cn[c] = off;
    off += n;
  }
  if (threadIdx.x == 0) {
    n_trans[k] = tot;
    area[k] = atot;
  }
}

// Pass 2: the same walk writes each transition's column-major position p at its scanned offset.  A mask with more transitions
// than `cap` writes none (its n_trans tells the caller how large a buffer it needs).
__global__ void __launch_bounds__(RLE_THREADS) amg_rle_write_kernel(AmgRleArgs a, const int* __restrict__ col_off,
                                                                    const int* __restrict__ n_trans, int* __restrict__ pos, int cap) {
  const int k = blockIdx.y, x = blockIdx.x * RLE_THREADS + threadIdx.x;
  const int W = a.fr.W, H = a.fr.H;
  if (x >= W || n_trans[k] > cap) return;
  const float* p = a.low + (long long)k * a.Hi * a.Wi;
  int* out = pos + (long long)k * cap + col_off[(long long)k * W + x];
  bool prev = rle_prev(a, p, x);
  const int colp = x * H;
  if (!rle_in_cols(a, x)) {
    if (prev) *out = colp;
    return;
  }
  const BilinearTap tx = bilinear_tap(x - a.fr.x0, a.sx, a.Wi);
  for (int y = 0; y < H; ++y) {
    const bool v = rle_pixel(a, p, tx, y);
    if (v != prev) *out++ = colp + y;
    prev = v;
  }
}

}  // namespace es3

using namespace es3;

static bool amg_frame_ok(int x0, int y0, int x1, int y1, int W, int H) {
  return W > 0 && H > 0 && (long long)W * H < 2147483647LL && 0 <= x0 && x0 < x1 && x1 <= W && 0 <= y0 && y0 < y1 && y1 <= H;
}

extern "C" long long es3_amg_mask_stats_ws_floats(int M) { return (long long)M * ST_N; }

extern "C" int es3_amg_mask_stats(const float* low, const float* iou, int M, int K, int Hi, int Wi, int crop_x0, int crop_y0,
                                  int crop_x1, int crop_y1, int orig_w, int orig_h, double mask_threshold, double offset,
                                  double pred_iou_thresh, double stability_thresh, int point_base, int* ws, float* arena_low,
                                  int* arena_box, float* arena_iou, float* arena_stab, int* arena_point, int* arena_count,
                                  int arena_cap, void* stream) {
  ES3_REQUIRE(M > 0 && M <= 65535 && K > 0 && M % K == 0 && Hi > 0 && Wi > 0 && (long long)Hi * Wi < 2147483647LL && arena_cap >= 0,
              "es3_amg_mask_stats: bad shape (M=%d K=%d Hi=%d Wi=%d cap=%d)", M, K, Hi, Wi, arena_cap);
  ES3_REQUIRE(amg_frame_ok(crop_x0, crop_y0, crop_x1, crop_y1, orig_w, orig_h),
              "es3_amg_mask_stats: crop box (%d,%d,%d,%d) outside the %dx%d image", crop_x0, crop_y0, crop_x1, crop_y1, orig_w, orig_h);
  ES3_REQUIRE(low && iou && ws && arena_low && arena_box && arena_iou && arena_stab && arena_point && arena_count,
              "es3_amg_mask_stats: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int Ho = crop_y1 - crop_y0, Wo = crop_x1 - crop_x0;
  const float sy = (float)Hi / Ho, sx = (float)Wi / Wo;
  // Rows one band samples: at most (band - 1) sy + 3 (two taps, one rounding of the source coordinate).
  const int cap_rows = AMG_STAGE_FLOATS / Wi;
  int band = (int)((cap_rows - 3) / (double)sy) + 1;
  band = std::max(1, std::min(band, AMG_MAX_BAND));
  // thresholds as the reference forms them: Python floats (thr +- offset in double) compared against fp32 tensors
  const int filters = (pred_iou_thresh > 0.0 ? 1 : 0) | (stability_thresh > 0.0 ? 2 : 0);
  amg_stats_init_kernel<<<(unsigned)ceil_div(M, 256), 256, 0, st>>>(ws, M);
  amg_stats_kernel<<<dim3((unsigned)ceil_div(Ho, band), M), AMG_THREADS, 0, st>>>(
      low, iou, Hi, Wi, Ho, Wo, sy, sx, band, (float)mask_threshold, (float)(mask_threshold + offset),
      (float)(mask_threshold - offset), (float)pred_iou_thresh, filters, ws);
  const AmgFrame fr{crop_x0, crop_y0, crop_x1, crop_y1, orig_w, orig_h};
  amg_finalize_kernel<<<1, AMG_THREADS, 0, st>>>(iou, M, K, (float)pred_iou_thresh, (float)stability_thresh, filters, fr, point_base,
                                                 ws, arena_box, arena_iou, arena_stab, arena_point, arena_count, arena_cap);
  const long long plane = (long long)Hi * Wi;
  amg_compact_kernel<<<dim3((unsigned)std::min<long long>(ceil_div(plane, 256), 64), M), 256, 0, st>>>(low, plane, ws, arena_low);
  ES3_LAUNCH_CHECK("amg_mask_stats kernels");
  return 0;
}

extern "C" long long es3_box_nms_ws_floats(int N) {
  const long long nb = (N + 63) / 64;
  return 2 * (long long)N * nb + N;
}

extern "C" int es3_box_nms(const int* boxes, const float* scores, int N, double iou_threshold, int* keep, int* count, void* ws,
                           void* stream) {
  ES3_REQUIRE(N >= 0 && N <= NMS_MAX, "es3_box_nms: N=%d outside [0, %d]", N, NMS_MAX);
  ES3_REQUIRE(count && ws && (N == 0 || (boxes && scores && keep)), "es3_box_nms: null pointer");
  ES3_REQUIRE(((uintptr_t)ws & 7) == 0, "es3_box_nms: workspace must be 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int nb = (N + 63) / 64;
  unsigned long long* mask = (unsigned long long*)ws;
  int* order = (int*)(mask + (long long)N * nb);
  nms_rank_kernel<<<(unsigned)std::max(1, ceil_div(N, NMS_THREADS)), NMS_THREADS, 0, st>>>(scores, N, order);
  nms_mask_kernel<<<dim3((unsigned)std::max(1, nb), (unsigned)std::max(1, nb)), 64, 0, st>>>(boxes, order, N, nb, iou_threshold, mask);
  nms_sweep_kernel<<<1, NMS_THREADS, 0, st>>>(mask, order, N, nb, keep, count);
  ES3_LAUNCH_CHECK("box_nms kernels");
  return 0;
}

extern "C" long long es3_amg_rle_ws_floats(int K, int W) { return 2 * (long long)K * W; }

extern "C" int es3_amg_rle(const float* low, int K, int Hi, int Wi, int crop_x0, int crop_y0, int crop_x1, int crop_y1, int orig_w,
                           int orig_h, float mask_threshold, int* ws, int* pos, int cap, int* n_trans, int* area, void* bin,
                           void* stream) {
  ES3_REQUIRE(K > 0 && K <= 65535 && Hi > 0 && Wi > 0 && (long long)Hi * Wi < 2147483647LL && cap >= 0,
              "es3_amg_rle: bad shape (K=%d Hi=%d Wi=%d cap=%d)", K, Hi, Wi, cap);
  ES3_REQUIRE(amg_frame_ok(crop_x0, crop_y0, crop_x1, crop_y1, orig_w, orig_h),
              "es3_amg_rle: crop box (%d,%d,%d,%d) outside the %dx%d image", crop_x0, crop_y0, crop_x1, crop_y1, orig_w, orig_h);
  ES3_REQUIRE(low && ws && n_trans && area && (pos || cap == 0), "es3_amg_rle: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  AmgRleArgs a{low, Hi, Wi, (float)Hi / (crop_y1 - crop_y0), (float)Wi / (crop_x1 - crop_x0), mask_threshold,
               AmgFrame{crop_x0, crop_y0, crop_x1, crop_y1, orig_w, orig_h}};
  int* col_n = ws;
  int* col_area = ws + (long long)K * orig_w;
  const dim3 grid((unsigned)ceil_div(orig_w, RLE_THREADS), K);
  amg_rle_count_kernel<<<grid, RLE_THREADS, 0, st>>>(a, col_n, col_area, (uint8_t*)bin);
  amg_rle_scan_kernel<<<K, RLE_THREADS, 0, st>>>(orig_w, col_n, col_area, n_trans, area);
  amg_rle_write_kernel<<<grid, RLE_THREADS, 0, st>>>(a, col_n, n_trans, pos, cap);
  ES3_LAUNCH_CHECK("amg_rle kernels");
  return 0;
}
