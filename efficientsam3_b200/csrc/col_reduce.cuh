// The two-stage per-channel column reduction of train_bwd.cu, shared with bn_sync.cu (synchronised BatchNorm).
//   stage 1 (col_reduce_partials): per-block fp32 partials part [nblk][2][C] of either the pivot-shifted statistics of z
//            (sum (z - z[0]), sum (z - z[0])^2) or the BN/activation backward sums (sum g, sum g z, g = da act'(scale z + shift));
//   stage 2 (sum_block_partials): the nblk partials of one channel summed in fp64 in a fixed order.
#pragma once
#include "common.cuh"

namespace es3 {

// Launches stage 1 on `st` and returns the number of partial blocks in *nblk.  ws: es3_col_reduce_ws_floats(M, C) floats.
// stats = true: z only (scale / shift / da unused); otherwise act is an Es3Act code for the backward form.
int col_reduce_partials(bool stats, int act, const void* z, const void* da, const float* scale, const float* shift, long long M,
                        int C, float* ws, int* nblk, cudaStream_t st);

// Second stage of the column reductions.  block 256 = 8 channels x 32 lanes: lane l adds partials l, l + 32, ... (double),
// the 32 lanes are then summed in a fixed order.  (One thread per channel walking all <= 1184 partials serially cost
// 35 + 54 launches per step.)
__device__ __forceinline__ bool sum_block_partials(const float* __restrict__ part, int nblk, int C, double& s, double& q, int& c_out) {
  __shared__ double r0[32][9], r1[32][9];
  const int cl = threadIdx.x & 7, lane = threadIdx.x >> 3;
  const int c = blockIdx.x * 8 + cl;
  double a = 0.0, b = 0.0;
  if (c < C) {
    for (int blk = lane; blk < nblk; blk += 32) {
      a += (double)part[((long long)blk * 2) * C + c];
      b += (double)part[((long long)blk * 2 + 1) * C + c];
    }
  }
  r0[lane][cl] = a;
  r1[lane][cl] = b;
  __syncthreads();
  c_out = c;
  if (lane != 0 || c >= C) return false;
  s = 0.0; q = 0.0;
  for (int l = 0; l < 32; ++l) { s += r0[l][cl]; q += r1[l][cl]; }
  return true;
}

}  // namespace es3
