// k5_score.cu -- K5: scoring and test log-likelihood.
//   score : LinearModel.eval / evalInstanceAvro(loglik=false) (models/LinearModel.java:241-257,491-554) and the
//           float cast of RegressionTest (jobs/RegressionTest.java:163).  One warp per record, fp64 accumulate.
//   loglik: RegressionTestLoglik mapper/combiner/reducer (jobs/RegressionTestLoglik.java:124-200) with its float
//           rounding points: per-record float, per-combiner-block float, final float(sum/count).
// HBM-bound streaming kernels (one read of the test matrix).
#include "kernels.cuh"

namespace mlease {

__global__ void __launch_bounds__(256) score_kernel(int Dg, long long nrows, const long long* __restrict__ rowptr,
                                                    const int* __restrict__ colidx, const float* __restrict__ vals, long long ldx,
                                                    const float* __restrict__ offset, const double* __restrict__ model,
                                                    double intercept_term, int binary_feature, float* __restrict__ pred) {
  const int lane = threadIdx.x & 31;
  const long long wg = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long i = wg; i < nrows; i += nw) {
    double a = 0.0;
    if (colidx) {
      for (long long j = rowptr[i] + lane; j < rowptr[i + 1]; j += 32)
        a += model[colidx[j]] * (binary_feature ? 1.0 : (double)vals[j]);
    } else {
      const float* xr = vals + i * ldx;
      for (int k = lane; k < Dg; k += 32) a += model[k] * (binary_feature ? 1.0 : (double)xr[k]);
    }
    a = warp_sum(a);
    if (lane == 0) pred[i] = (float)((offset ? (double)offset[i] : 0.0) + (intercept_term + a));
  }
}

__global__ void loglik_record_kernel(long long nrows, const int* __restrict__ response, const float* __restrict__ pred,
                                     const float* __restrict__ weight, float* __restrict__ ll, int* __restrict__ bad) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nrows) return;
  const int r = response[i];
  if (r != 1 && r != 0 && r != -1) { *bad = 1; ll[i] = 0.f; return; }
  const double w = weight ? (double)weight[i] : 1.0, p = (double)pred[i];
  const double v = (r == 1) ? -log1p(exp(-p)) * w : -log1p(exp(p)) * w;
  ll[i] = (float)v;
}

// one CTA per combiner block: double sum of the block's float logliks and of its weights
__global__ void __launch_bounds__(256) loglik_block_kernel(long long nrows, const float* __restrict__ ll, const float* __restrict__ weight,
                                                           long long block, double* __restrict__ bsum, double* __restrict__ bcnt) {
  __shared__ double s1[8], s2[8];
  const long long b0 = (long long)blockIdx.x * block;
  const long long b1 = min(nrows, b0 + block);
  double a = 0.0, c = 0.0;
  for (long long i = b0 + threadIdx.x; i < b1; i += 256) { a += (double)ll[i]; c += weight ? (double)weight[i] : 1.0; }
  a = warp_sum(a); c = warp_sum(c);
  if ((threadIdx.x & 31) == 0) { s1[threadIdx.x >> 5] = a; s2[threadIdx.x >> 5] = c; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double x = 0.0, y = 0.0;
    for (int w = 0; w < 8; w++) { x += s1[w]; y += s2[w]; }
    bsum[blockIdx.x] = x; bcnt[blockIdx.x] = y;
  }
}

cudaError_t score_launch(int Dg, long long nrows, const long long* rowptr, const int* colidx, const float* vals, long long ldx,
                         const float* offset, const double* d_model, double intercept_term, int binary_feature, float* pred,
                         cudaStream_t st) {
  if (nrows == 0) return cudaSuccess;
  long long blocks = (nrows + 7) / 8;
  if (blocks > 132 * 16) blocks = 132 * 16;
  score_kernel<<<(int)blocks, 256, 0, st>>>(Dg, nrows, rowptr, colidx, vals, ldx, offset, d_model, intercept_term, binary_feature, pred);
  return cudaGetLastError();
}

cudaError_t loglik_launch(long long nrows, const int* response, const float* pred, const float* weight, long long combiner_block,
                          float* d_ll, double* d_block_sum, double* d_block_cnt, int* d_bad, cudaStream_t st) {
  if (nrows == 0) return cudaSuccess;
  loglik_record_kernel<<<(int)((nrows + 255) / 256), 256, 0, st>>>(nrows, response, pred, weight, d_ll, d_bad);
  const long long nb = (nrows + combiner_block - 1) / combiner_block;
  loglik_block_kernel<<<(int)nb, 256, 0, st>>>(nrows, d_ll, weight, combiner_block, d_block_sum, d_block_cnt);
  return cudaGetLastError();
}

}  // namespace mlease
