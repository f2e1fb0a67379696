// Optimiser half of the stage-1 KD step (SURVEY.md §8 A19/A20), everything that does not depend on the student's backward:
//   * KD-loss backward: d loss / d preds for masked MSE + masked cosine (train_image_encoder_stage1.py:271-307)
//   * loss-scaled global grad norm + non-finite detection over the flat gradient arena
//     (NativeScalerWithGradNormCount: GradScaler.unscale_ + clip_grad_norm_, stage1/utils.py:341-368)
//   * fused AdamW over the flat parameter arena (torch.optim.AdamW semantics, stage1/optimizer.py:6-30: decoupled weight
//     decay on the leading `n_decay` elements only) with the unscale, the clip coefficient and the GradScaler skip-on-inf
//     decision read from device memory: no host synchronisation anywhere in the step, so it can sit in a CUDA graph.
// All three are pure HBM streams: 12 B/elem (loss bwd: read p,t twice from L2, write g), 4 B/elem (norm),
// 28 B/elem (AdamW: read p,g,m,v, write p,m,v).
#include "common.cuh"

namespace es3 {

__device__ __forceinline__ float kd_valid_mask_at(int oy, int ox, int E, int img, int h, int w) {
  // build_valid_mask: bilinear (align_corners=False) resize of the [y < h, x < w] indicator to E x E, > 0.5 (kd_loss.cu)
  const float s = (float)img / (float)E;
  float fy = (oy + 0.5f) * s - 0.5f, fx = (ox + 0.5f) * s - 0.5f;
  if (fy < 0.f) fy = 0.f;
  if (fx < 0.f) fx = 0.f;
  const int y0 = min((int)fy, img - 1), x0 = min((int)fx, img - 1);
  const int y1 = min(y0 + 1, img - 1), x1 = min(x0 + 1, img - 1);
  const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
  const float i00 = (y0 < h && x0 < w) ? 1.f : 0.f, i01 = (y0 < h && x1 < w) ? 1.f : 0.f;
  const float i10 = (y1 < h && x0 < w) ? 1.f : 0.f, i11 = (y1 < h && x1 < w) ? 1.f : 0.f;
  return (hy * (hx * i00 + lx * i01) + ly * (hx * i10 + lx * i11)) > 0.5f ? 1.f : 0.f;
}

// grid (ceil(E*E/256), B); thread = pixel, two passes over the channels (the second one hits L2).
// per_sample [B][3] from es3_kd_loss_fwd: [.., .., mask count].  scale_dev: optional device float (GradScaler loss scale).
__global__ void kd_loss_bwd_kernel(const float* __restrict__ pred, const float* __restrict__ teach, const int* __restrict__ sizes_hw,
                                   const float* __restrict__ per_sample, const float* __restrict__ scale_dev, float gscale,
                                   float cosine_w, int B, int C, int E, int img, float* __restrict__ dpred) {
  const int b = blockIdx.y, HW = E * E;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const float m = kd_valid_mask_at(p / E, p % E, E, img, sizes_hw[b * 2], sizes_hw[b * 2 + 1]);
  const float* pp = pred + (long long)b * C * HW + p;
  const float* tp = teach + (long long)b * C * HW + p;
  float* gp = dpred + (long long)b * C * HW + p;
  if (m == 0.f) {
    for (int c = 0; c < C; ++c) gp[(long long)c * HW] = 0.f;
    return;
  }
  float dot = 0.f, np2 = 0.f, nt2 = 0.f;
#pragma unroll 4
  for (int c = 0; c < C; ++c) {
    const float a = __ldg(pp + (long long)c * HW), t = __ldg(tp + (long long)c * HW);
    dot = fmaf(a, t, dot); np2 = fmaf(a, a, np2); nt2 = fmaf(t, t, nt2);
  }
  const float np = sqrtf(np2), na = fmaxf(np, 1e-8f), nt = fmaxf(sqrtf(nt2), 1e-8f);
  const float up = gscale * (scale_dev ? scale_dev[0] : 1.f) / ((float)B * fmaxf(per_sample[b * 3 + 2], 1.f));
  // d(1 - cos)/da_c = -(t_c / (na nt) - dot a_c / (na^2 nt |a|)), na = max(|a|, eps): the clamp keeps the 1 / na factor of cos
  // constant below eps, but |a|'s own derivative a / |a| is still there (a / |a| := 0 at a = 0, as the norm's backward; text_bwd.cu)
  const float k_t = -cosine_w * up / (na * nt), k_a = np > 0.f ? cosine_w * up * dot / (na * na * np * nt) : 0.f;
  const float k_mse = 2.f * up;
#pragma unroll 4
  for (int c = 0; c < C; ++c) {
    const float a = __ldg(pp + (long long)c * HW), t = __ldg(tp + (long long)c * HW);
    gp[(long long)c * HW] = k_mse * (a - t) + k_t * t + k_a * a;
  }
}

// ---- global grad norm: part[blocks][2] = (sum g^2, non-finite count); norm_ws[0] = sum g^2, norm_ws[1] = non-finite flag
constexpr int GN_THREADS = 256, GN_PER_THREAD = 16;
__global__ void __launch_bounds__(GN_THREADS) grad_sumsq_partial_kernel(const float* __restrict__ g, long long n, float* __restrict__ part) {
  __shared__ float red[2][GN_THREADS / 32];
  const long long base = ((long long)blockIdx.x * GN_THREADS + threadIdx.x) * 4;
  const long long stride = (long long)gridDim.x * GN_THREADS * 4;
  float s = 0.f, bad = 0.f;
  for (long long i = base; i < n; i += stride) {
    if (i + 4 <= n) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(g + i));
      s = fmaf(v.x, v.x, s); s = fmaf(v.y, v.y, s); s = fmaf(v.z, v.z, s); s = fmaf(v.w, v.w, s);
      if (!isfinite(v.x) || !isfinite(v.y) || !isfinite(v.z) || !isfinite(v.w)) bad = 1.f;
    } else {
      for (long long j = i; j < n; ++j) { const float x = g[j]; s = fmaf(x, x, s); if (!isfinite(x)) bad = 1.f; }
    }
  }
  s = warp_sum(s); bad = warp_sum(bad);
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = s; red[1][threadIdx.x >> 5] = bad; }
  __syncthreads();
  if (threadIdx.x < 2) {
    float t = 0.f;
    for (int i = 0; i < GN_THREADS / 32; ++i) t += red[threadIdx.x][i];
    part[blockIdx.x * 2 + threadIdx.x] = t;
  }
}
__global__ void grad_sumsq_final_kernel(const float* __restrict__ part, int nblk, float* __restrict__ norm_ws) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double s = 0.0;
  float bad = 0.f;
  for (int i = 0; i < nblk; ++i) { s += (double)part[i * 2]; bad += part[i * 2 + 1]; }
  norm_ws[0] = (float)s;
  norm_ws[1] = (bad > 0.f || !isfinite((float)s)) ? 1.f : 0.f;
}

// state[0] = loss scale, [1] = growth tracker, [2] = optimiser step count, [3] = last total grad norm (unscaled, pre-clip)
struct AdamWArgs {
  float *p, *m, *v;
  const float* g;
  long long n, n_decay;
  float lr, beta1, beta2, eps, wd, max_norm, inv_world;
  const float* norm_ws;
  const float* state;
};
__global__ void __launch_bounds__(256) adamw_flat_kernel(const AdamWArgs a) {
  if (a.norm_ws[1] != 0.f) return;                       // GradScaler.step: skip the update when infs / nans were found
  const float inv_scale = a.inv_world / a.state[0];
  const float total_norm = sqrtf(a.norm_ws[0]) * inv_scale;
  float coef = 1.f;
  if (a.max_norm > 0.f) coef = fminf(a.max_norm / (total_norm + 1e-6f), 1.f);   // clip_grad_norm_
  const float gmul = inv_scale * coef;
  const float t = a.state[2] + 1.f;
  const float bc1 = 1.f - powf(a.beta1, t), bc2 = 1.f - powf(a.beta2, t);
  const float step_size = a.lr / bc1, inv_sqrt_bc2 = rsqrtf(bc2);
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i >= a.n) return;
  float pv[4], gv[4], mv[4], vv[4];
  const bool full = i + 4 <= a.n;
  if (full) {
    const float4 P = *reinterpret_cast<const float4*>(a.p + i), G = __ldg(reinterpret_cast<const float4*>(a.g + i));
    const float4 M = *reinterpret_cast<const float4*>(a.m + i), V = *reinterpret_cast<const float4*>(a.v + i);
    pv[0] = P.x; pv[1] = P.y; pv[2] = P.z; pv[3] = P.w; gv[0] = G.x; gv[1] = G.y; gv[2] = G.z; gv[3] = G.w;
    mv[0] = M.x; mv[1] = M.y; mv[2] = M.z; mv[3] = M.w; vv[0] = V.x; vv[1] = V.y; vv[2] = V.z; vv[3] = V.w;
  } else {
    for (int j = 0; j < 4; ++j) {
      const bool in = i + j < a.n;
      pv[j] = in ? a.p[i + j] : 0.f; gv[j] = in ? a.g[i + j] : 0.f; mv[j] = in ? a.m[i + j] : 0.f; vv[j] = in ? a.v[i + j] : 0.f;
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float g = gv[j] * gmul;
    float p = pv[j];
    if (i + j < a.n_decay) p *= 1.f - a.lr * a.wd;        // decoupled weight decay, decay group only
    const float m = a.beta1 * mv[j] + (1.f - a.beta1) * g;
    const float v = a.beta2 * vv[j] + (1.f - a.beta2) * g * g;
    const float denom = sqrtf(v) * inv_sqrt_bc2 + a.eps;
    pv[j] = p - step_size * (m / denom);
    mv[j] = m; vv[j] = v;
  }
  if (full) {
    *reinterpret_cast<float4*>(a.p + i) = make_float4(pv[0], pv[1], pv[2], pv[3]);
    *reinterpret_cast<float4*>(a.m + i) = make_float4(mv[0], mv[1], mv[2], mv[3]);
    *reinterpret_cast<float4*>(a.v + i) = make_float4(vv[0], vv[1], vv[2], vv[3]);
  } else {
    for (int j = 0; j < 4 && i + j < a.n; ++j) { a.p[i + j] = pv[j]; a.m[i + j] = mv[j]; a.v[i + j] = vv[j]; }
  }
}
// GradScaler.update (growth 2.0 / backoff 0.5 / interval 2000 by default) + step counter, after the parameter update.
__global__ void scaler_update_kernel(float* __restrict__ state, const float* __restrict__ norm_ws, float inv_world, float growth,
                                     float backoff, int interval, int dynamic) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const bool bad = norm_ws[1] != 0.f;
  state[3] = bad ? INFINITY : sqrtf(norm_ws[0]) * inv_world / state[0];
  if (!bad) state[2] += 1.f;
  if (!dynamic) return;
  if (bad) { state[0] *= backoff; state[1] = 0.f; }
  else {
    state[1] += 1.f;
    if ((int)state[1] >= interval) { state[0] *= growth; state[1] = 0.f; }
  }
}

}  // namespace es3

using namespace es3;

extern "C" int es3_kd_loss_bwd(const float* preds, const float* teacher, const int* sizes_hw, const float* per_sample,
                               const float* scale_dev, float grad_scale, int B, int C, int E, int img_size, float cosine_weight,
                               float* dpreds, void* stream) {
  ES3_REQUIRE(B > 0 && C > 0 && E > 0 && img_size > 0, "es3_kd_loss_bwd: bad shape");
  kd_loss_bwd_kernel<<<dim3(ceil_div(E * E, 256), B), 256, 0, (cudaStream_t)stream>>>(preds, teacher, sizes_hw, per_sample, scale_dev,
                                                                                      grad_scale, cosine_weight, B, C, E, img_size, dpreds);
  ES3_LAUNCH_CHECK("kd_loss_bwd_kernel");
  return 0;
}

extern "C" long long es3_grad_norm_ws_floats(long long n) {
  long long blocks = (n + (long long)GN_THREADS * 4 * GN_PER_THREAD - 1) / ((long long)GN_THREADS * 4 * GN_PER_THREAD);
  if (blocks < 1) blocks = 1;
  if (blocks > 4096) blocks = 4096;
  return blocks * 2;
}

// norm_ws[0] = sum g^2 (raw, still loss-scaled), norm_ws[1] = 1 if any element is inf / nan.  part_ws: es3_grad_norm_ws_floats(n).
extern "C" int es3_grad_norm(const float* g, long long n, float* part_ws, float* norm_ws, void* stream) {
  ES3_REQUIRE(n > 0 && ((uintptr_t)g & 15) == 0, "es3_grad_norm: need n > 0 and a 16-byte aligned arena");
  const int blocks = (int)(es3_grad_norm_ws_floats(n) / 2);
  cudaStream_t st = (cudaStream_t)stream;
  grad_sumsq_partial_kernel<<<blocks, GN_THREADS, 0, st>>>(g, n, part_ws);
  ES3_LAUNCH_CHECK("grad_sumsq_partial_kernel");
  grad_sumsq_final_kernel<<<1, 32, 0, st>>>(part_ws, blocks, norm_ws);
  ES3_LAUNCH_CHECK("grad_sumsq_final_kernel");
  return 0;
}

extern "C" int es3_adamw_flat(float* p, const float* g, float* m, float* v, long long n, long long n_decay, float lr, float beta1,
                              float beta2, float eps, float weight_decay, float max_norm, float inv_world, const float* norm_ws,
                              float* state, int dynamic_scale, float growth, float backoff, int growth_interval, void* stream) {
  ES3_REQUIRE(n > 0 && n_decay >= 0 && n_decay <= n, "es3_adamw_flat: bad sizes n=%lld n_decay=%lld", n, n_decay);
  ES3_REQUIRE((((uintptr_t)p | (uintptr_t)g | (uintptr_t)m | (uintptr_t)v) & 15) == 0, "es3_adamw_flat: arenas must be 16-byte aligned");
  AdamWArgs a{p, m, v, g, n, n_decay, lr, beta1, beta2, eps, weight_decay, max_norm, inv_world, norm_ws, state};
  cudaStream_t st = (cudaStream_t)stream;
  const long long threads = (n + 3) / 4;
  adamw_flat_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(a);
  ES3_LAUNCH_CHECK("adamw_flat_kernel");
  scaler_update_kernel<<<1, 32, 0, st>>>(state, norm_ws, inv_world, growth, backoff, growth_interval, dynamic_scale);
  ES3_LAUNCH_CHECK("scaler_update_kernel");
  return 0;
}
