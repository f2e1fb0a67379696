// Synchronised BatchNorm (nn.SyncBatchNorm in train mode) for the image students: the batch statistics and the BN backward of
// train_bwd.cu, split at the two points where the ranks of a process group exchange data.
//
//   es3_bn_stats_partial     this rank's (count, mean, M2) per channel, fp64 [3][C], from es3_bn_stats' pivot-shifted column
//                            reduction (so |mean| >> std stays accurate)
//   -- all-gather of the [3][C] partials over the group --
//   es3_bn_stats_combine     [W][3][C] combined with Chan's formula in rank order -> mean, invstd, scale, shift (es3_bn_stats'
//                            layout), the running buffers, num_batches_tracked and the total count
//   es3_bn_act_bwd_partial   g = da act'(scale z + shift): this rank's sum g and sum g (z - mean), fp64 [2][C]; adds the rank's own
//                            dgamma / dbeta (as torch's SyncBatchNorm: the gradient exchange averages them)
//   -- all-gather of the [2][C] partials over the group --
//   es3_bn_bwd_coef          [W][2][C] summed in rank order + the total count -> coef [3][C] for the unchanged es3_bn_act_bwd_apply
//
// Every rank combines the same gathered partials in the same order, so the statistics and the running buffers are bit-identical
// across ranks; no float atomics anywhere, so repeats are bit-identical too.
#include "col_reduce.cuh"

namespace es3 {
namespace {

// part [3][C] = (count, mean, M2) of this rank's rows.  grid ceil(C / 8), block 256 (sum_block_partials' map).
__global__ void __launch_bounds__(256) bn_stats_partial_kernel(const bf16* __restrict__ z, const float* __restrict__ ws, int nblk, int C,
                                                               long long M, double* __restrict__ part) {
  double s, q;
  int c;
  if (!sum_block_partials(ws, nblk, C, s, q, c)) return;
  const double n = (double)M;
  const double dm = s / n;                                // mean of (z - pivot)
  part[c] = n;
  part[C + c] = (double)__bfloat162float(z[c]) + dm;
  part[2 * C + c] = fmax(q - s * dm, 0.0);                // sum (z - mean)^2 = sum (z - pivot)^2 - n dm^2
}

// One thread per channel.  Chan's parallel combination over the W ranks in rank order; then es3_bn_stats' finalize.
__global__ void __launch_bounds__(256) bn_stats_combine_kernel(const double* __restrict__ part, int W, int C, float eps, float momentum,
                                                               const float* __restrict__ gamma, const float* __restrict__ beta,
                                                               float* __restrict__ mean, float* __restrict__ invstd,
                                                               float* __restrict__ scale, float* __restrict__ shift,
                                                               float* __restrict__ running_mean, float* __restrict__ running_var,
                                                               long long* __restrict__ num_batches_tracked, double* __restrict__ total) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double n = 0.0, mu = 0.0, m2 = 0.0;
  for (int w = 0; w < W; ++w) {
    const double* p = part + (long long)w * 3 * C;
    const double nb = p[c];
    if (nb <= 0.0) continue;
    const double nn = n + nb, d = p[C + c] - mu;
    mu += d * (nb / nn);
    m2 += p[2 * C + c] + d * d * (n * nb / nn);
    n = nn;
  }
  if (c == 0) {
    if (num_batches_tracked) num_batches_tracked[0] += 1;
    if (total) total[0] = n;
  }
  const double var = n > 0.0 ? m2 / n : 0.0;
  const float is = (float)(1.0 / sqrt(var + (double)eps));
  mean[c] = (float)mu;
  invstd[c] = is;
  const float sc = (gamma ? gamma[c] : 1.f) * is;
  scale[c] = sc;
  shift[c] = (beta ? beta[c] : 0.f) - (float)mu * sc;
  if (running_mean) running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)mu;
  if (running_var) {
    const double unbiased = n > 1.0 ? var * n / (n - 1.0) : var;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unbiased;
  }
}

// part [2][C] = (sum g, sum g (z - mean)) of this rank's rows; dgamma += invstd sum g (z - mean), dbeta += sum g.
// grid ceil(C / 8), block 256.
__global__ void __launch_bounds__(256) bn_bwd_partial_kernel(const float* __restrict__ ws, int nblk, int C, const float* __restrict__ mean,
                                                             const float* __restrict__ invstd, double* __restrict__ part,
                                                             float* __restrict__ dgamma, float* __restrict__ dbeta) {
  double sg, sgz;
  int c;
  if (!sum_block_partials(ws, nblk, C, sg, sgz, c)) return;
  const double sgx = sgz - (double)mean[c] * sg;
  part[c] = sg;
  part[C + c] = sgx;
  if (dgamma) dgamma[c] += (float)((double)invstd[c] * sgx);
  if (dbeta) dbeta[c] += (float)sg;
}

// One thread per channel: the batch-statistics coefficients of bn_bwd_finalize_kernel (mode 2) from the sums over all ranks.
__global__ void __launch_bounds__(256) bn_bwd_coef_kernel(const double* __restrict__ part, int W, int C, const double* __restrict__ total,
                                                          const float* __restrict__ scale, const float* __restrict__ mean,
                                                          const float* __restrict__ invstd, float* __restrict__ coef) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double sg = 0.0, sgx = 0.0;
  for (int w = 0; w < W; ++w) {
    sg += part[(long long)w * 2 * C + c];
    sgx += part[((long long)w * 2 + 1) * C + c];
  }
  const double M = total[0];
  const float sc = scale ? scale[c] : 1.f;
  const double mu = (double)mean[c], is = (double)invstd[c];
  const double mg = sg / M, mgx = is * sgx / M;           // means of g and of g xhat, as bn_bwd_finalize_kernel forms them
  // dz = sc (g - mg - xhat is mgx) = A g + B z + C, xhat = (z - mean) is
  coef[c] = sc;
  coef[C + c] = (float)(-(double)sc * is * mgx);
  coef[2 * C + c] = (float)(-(double)sc * mg + (double)sc * is * mu * mgx);
}

}  // namespace
}  // namespace es3

using namespace es3;

// ------------------------------------------------------------------------------------------ C ABI
extern "C" int es3_bn_stats_partial(const void* z, long long M, int C, float* ws, double* part, void* stream) {
  ES3_REQUIRE(M > 0 && C > 0 && C % 8 == 0, "es3_bn_stats_partial: need M > 0 and C %% 8 == 0 (M=%lld C=%d)", M, C);
  ES3_REQUIRE(((uintptr_t)z & 15) == 0, "es3_bn_stats_partial: z must be 16-byte aligned");
  ES3_REQUIRE(ws && part, "es3_bn_stats_partial: ws / part must not be NULL");
  cudaStream_t st = (cudaStream_t)stream;
  int nblk;
  const int rc = col_reduce_partials(true, ACT_NONE, z, nullptr, nullptr, nullptr, M, C, ws, &nblk, st);
  if (rc) return rc;
  bn_stats_partial_kernel<<<ceil_div(C, 8), 256, 0, st>>>((const bf16*)z, ws, nblk, C, M, part);
  ES3_LAUNCH_CHECK("bn_stats_partial_kernel");
  return 0;
}

extern "C" int es3_bn_stats_combine(const double* part, int W, int C, float eps, float momentum, const float* gamma, const float* beta,
                                    float* mean, float* invstd, float* scale, float* shift, float* running_mean, float* running_var,
                                    long long* num_batches_tracked, double* total, void* stream) {
  ES3_REQUIRE(W > 0 && C > 0 && C % 8 == 0, "es3_bn_stats_combine: need W > 0 and C %% 8 == 0 (W=%d C=%d)", W, C);
  ES3_REQUIRE(part && mean && invstd && scale && shift, "es3_bn_stats_combine: part / mean / invstd / scale / shift must not be NULL");
  bn_stats_combine_kernel<<<ceil_div(C, 256), 256, 0, (cudaStream_t)stream>>>(part, W, C, eps, momentum, gamma, beta, mean, invstd, scale,
                                                                              shift, running_mean, running_var, num_batches_tracked, total);
  ES3_LAUNCH_CHECK("bn_stats_combine_kernel");
  return 0;
}

extern "C" int es3_bn_act_bwd_partial(const void* da, const void* z, const float* scale, const float* shift, int act, const float* mean,
                                      const float* invstd, long long M, int C, float* ws, double* part, float* dgamma, float* dbeta,
                                      void* stream) {
  ES3_REQUIRE(M > 0 && C > 0 && C % 8 == 0, "es3_bn_act_bwd_partial: need M > 0 and C %% 8 == 0 (M=%lld C=%d)", M, C);
  ES3_REQUIRE(mean && invstd && ws && part, "es3_bn_act_bwd_partial: mean / invstd / ws / part must not be NULL");
  cudaStream_t st = (cudaStream_t)stream;
  int nblk;
  const int rc = col_reduce_partials(false, act, z, da, scale, shift, M, C, ws, &nblk, st);
  if (rc) return rc;
  bn_bwd_partial_kernel<<<ceil_div(C, 8), 256, 0, st>>>(ws, nblk, C, mean, invstd, part, dgamma, dbeta);
  ES3_LAUNCH_CHECK("bn_bwd_partial_kernel");
  return 0;
}

extern "C" int es3_bn_bwd_coef(const double* part, int W, int C, const double* total, const float* scale, const float* mean,
                               const float* invstd, float* coef, void* stream) {
  ES3_REQUIRE(W > 0 && C > 0 && C % 8 == 0, "es3_bn_bwd_coef: need W > 0 and C %% 8 == 0 (W=%d C=%d)", W, C);
  ES3_REQUIRE(part && total && mean && invstd && coef, "es3_bn_bwd_coef: part / total / mean / invstd / coef must not be NULL");
  bn_bwd_coef_kernel<<<ceil_div(C, 256), 256, 0, (cudaStream_t)stream>>>(part, W, C, total, scale, mean, invstd, coef);
  ES3_LAUNCH_CHECK("bn_bwd_coef_kernel");
  return 0;
}
