// k6_postvar.cu -- posterior variance of a fitted model (SURVEY 8f-3):
//   LibLinear.train(..., computePosteriorVar, computeFullPostVar) (llf/LibLinear.java:315-334) as ItemModelTrain calls it
//   (jobs/ItemModelTrain.java:244-276):
//     diagonal : postVar[k] = 1 / H[k],  H[k] = 1/priorVar[k] + sum_i weight_i p_i (1-p_i) x_ik^2
//                (LogisticRegressionL2.hessianDiagonal, llf/LogisticRegressionL2.java:304-327)
//     full     : postVar = diag(H^-1), H = LogisticRegressionL2.hessian (:258-297), inverted by Cholesky
//                (commons-math CholeskyDecomposition in the reference, :321-325; K3's fp64 factorisation + explicit inverse here).
// The tensor-core Gram (bf16 operands) is a preconditioner-grade H; a reported variance needs the Hessian itself, so these
// kernels accumulate it in fp64 from the fp32 data (SIMT; n D'^2 / 2 fp64 FMA for the full matrix).  The diagonal runs over a
// batch of problems (ItemModelTrain's keys, one launch per key chunk and prior) or over a session's one partition.
#include <algorithm>

#include "kernels.cuh"

namespace mlease {

// A batch's rows are numbered across its problems: problem b owns rows [row_start[b], row_start[b+1]) (empty problems allowed).
// One warp per row of the whole batch, so a batch of thousands of keys of a few hundred rows keeps every SM busy; the row's
// problem is the last b with row_start[b] <= r.
__device__ __forceinline__ int postvar_problem_of(const long long* __restrict__ row_start, int nprob, long long r) {
  int lo = 0, hi = nprob - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (row_start[mid] <= r) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// d_r = weight_i p_i (1 - p_i) at the problem's beta (double).  Same score as LogisticRegressionL2.hessian (:261-269).
__global__ void postvar_rowweight_kernel(const Problem* __restrict__ probs, int nprob, const long long* __restrict__ row_start,
                                         int has_bias, double* __restrict__ dvec) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const long long nrows = row_start[nprob];
  for (long long r = warp; r < nrows; r += nwarps) {
    const int b = postvar_problem_of(row_start, nprob, r);
    const Problem& pb = probs[b];
    const long long i = r - row_start[b];
    const double* w = pb.beta;
    double s = 0.0;
    if (pb.X) {
      const float* xr = pb.X + (size_t)i * pb.ldx;
      for (int k = lane; k < pb.Dt; k += 32) s += w[k] * (double)xr[k];          // the bias column is physical (1.0f)
    } else {
      for (long long j = pb.rowptr[i] + lane; j < pb.rowptr[i + 1]; j += 32) s += w[pb.colidx[j]] * (double)pb.vals[j];
    }
    s = warp_sum(s);
    if (lane == 0) {
      if (!pb.X && has_bias) s += w[pb.Dt - 1];
      s += (double)pb.o[i];
      const double p = 1.0 / (1.0 + exp(-(double)pb.y[i] * s));
      dvec[r] = (double)pb.w[i] * p * (1.0 - p);
    }
  }
}

// g_t = q over [0, ldx): the prior precision the diagonal starts from
__global__ void postvar_diag_init_kernel(const Problem* __restrict__ probs) {
  const Problem& pb = probs[blockIdx.x];
  for (int k = threadIdx.x; k < pb.ldx; k += blockDim.x) pb.g_t[k] = pb.q[k];
}

// g_t[k] += d_r x_ik^2 (k < Dt) of each problem, fp64 global atomics.
__global__ void postvar_diag_kernel(const Problem* __restrict__ probs, int nprob, const long long* __restrict__ row_start,
                                    const double* __restrict__ dvec, int has_bias) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const long long nrows = row_start[nprob];
  for (long long r = warp; r < nrows; r += nwarps) {
    const int b = postvar_problem_of(row_start, nprob, r);
    const Problem& pb = probs[b];
    const long long i = r - row_start[b];
    double* H = pb.g_t;
    const double d = dvec[r];
    if (pb.X) {
      const float* xr = pb.X + (size_t)i * pb.ldx;
      for (int k = lane; k < pb.Dt; k += 32) { const double x = (double)xr[k]; atomicAdd(&H[k], d * x * x); }
    } else {
      // duplicates of a column inside a row add BEFORE squaring in the reference's dense x (it requires sorted unique rows, :277);
      // rows with repeated columns are rejected by the caller
      for (long long j = pb.rowptr[i] + lane; j < pb.rowptr[i + 1]; j += 32) { const double x = (double)pb.vals[j]; atomicAdd(&H[pb.colidx[j]], d * x * x); }
      if (has_bias && lane == 0) atomicAdd(&H[pb.Dt - 1], d);
    }
  }
}

// Full Hessian, dense rows: lower 32x32 tiles of  sum_i d_i x_i x_i^T  into Lc (ld = ldh); grid (T, T), blockIdx.y >= blockIdx.x.
__global__ void __launch_bounds__(256) postvar_hess_dense_kernel(const Problem* __restrict__ probs, const double* __restrict__ dvec) {
  const Problem& pb = probs[0];
  const int bi = blockIdx.y, bj = blockIdx.x;
  if (bj > bi) return;
  __shared__ double xa[64][33], xb[64][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // thread owns rows (ty, ty+8, ty+16, ty+24) x column tx of the tile
  double acc[4] = {0, 0, 0, 0};
  for (long long r0 = 0; r0 < pb.n; r0 += 64) {
    for (int e = threadIdx.x; e < 64 * 32; e += 256) {
      const int r = e >> 5, c = e & 31;
      const long long i = r0 + r;
      const int ca = bi * 32 + c, cb = bj * 32 + c;
      const double d = i < pb.n ? dvec[i] : 0.0;
      xa[r][c] = (i < pb.n && ca < pb.Dt) ? d * (double)pb.X[(size_t)i * pb.ldx + ca] : 0.0;
      xb[r][c] = (i < pb.n && cb < pb.Dt) ? (double)pb.X[(size_t)i * pb.ldx + cb] : 0.0;
    }
    __syncthreads();
#pragma unroll 8
    for (int r = 0; r < 64; r++) {
      const double b = xb[r][tx];
#pragma unroll
      for (int q = 0; q < 4; q++) acc[q] += xa[r][ty + 8 * q] * b;
    }
    __syncthreads();
  }
#pragma unroll
  for (int q = 0; q < 4; q++) {
    const int i = bi * 32 + ty + 8 * q, j = bj * 32 + tx;
    if (i < pb.Dt && j <= i) pb.Lc[(size_t)i * pb.ldh + j] += acc[q];
  }
}

// Full Hessian, CSR rows: one warp per row, all ordered entry pairs (the bias is one more entry), lower triangle, fp64 atomics.
__global__ void postvar_hess_csr_kernel(const Problem* __restrict__ probs, const double* __restrict__ dvec, int has_bias) {
  const Problem& pb = probs[0];
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long i = warp; i < pb.n; i += nwarps) {
    const long long j0 = pb.rowptr[i];
    const int len = (int)(pb.rowptr[i + 1] - j0) + (has_bias ? 1 : 0);
    const double d = dvec[i];
    for (long long e = lane; e < (long long)len * len; e += 32) {
      const int a = (int)(e / len), b = (int)(e % len);
      const int ca = a < len - (has_bias ? 1 : 0) ? pb.colidx[j0 + a] : pb.Dt - 1;
      const int cb = b < len - (has_bias ? 1 : 0) ? pb.colidx[j0 + b] : pb.Dt - 1;
      if (ca < cb) continue;
      const double va = a < len - (has_bias ? 1 : 0) ? (double)pb.vals[j0 + a] : 1.0;
      const double vb = b < len - (has_bias ? 1 : 0) ? (double)pb.vals[j0 + b] : 1.0;
      atomicAdd(&pb.Lc[(size_t)ca * pb.ldh + cb], d * va * vb);
    }
  }
}

// Lc = diag(q) on [0, Dt), identity on the padding, zero elsewhere (lower triangle is what the factorisation reads)
__global__ void postvar_init_kernel(const Problem* __restrict__ probs, const double* __restrict__ q) {
  const Problem& pb = probs[0];
  const size_t total = (size_t)pb.ldh * pb.ldh;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int i = (int)(e / pb.ldh), j = (int)(e % pb.ldh);
    pb.Lc[e] = (i == j) ? (i < pb.Dt ? q[i] : 1.0) : 0.0;
  }
}

// Full Hessian of every problem of a batch (CSR rows with strictly increasing column ids): Lc = diag(q) + sum_i d_i x_i x_i^T on
// [0, Dt), the intercept (has_bias) an implicit entry 1 at column Dt - 1, identity on the padding, zero above the diagonal.  CTA =
// (column block bj, row block bi, problem); a lower 32x32 tile densifies 32-row slabs of the problem's rows into shared memory (each
// row's entries in the two column blocks found by a binary search) and every thread sums its 4 cells over the rows in row order:
// no atomics, so each problem's H is a function of its beta and rows alone, whatever else its batch holds.  dvec is numbered
// across the batch's rows (row_start), as postvar_rowweights leaves it.
__global__ void __launch_bounds__(256) postvar_hess_batch_kernel(const Problem* __restrict__ probs, const long long* __restrict__ row_start,
                                                                 const double* __restrict__ dvec, int has_bias) {
  const Problem& pb = probs[blockIdx.z];
  const int bi = blockIdx.y, bj = blockIdx.x;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  double* H = pb.Lc;
  if (bj > bi) {
#pragma unroll
    for (int q = 0; q < 4; q++) H[(size_t)(bi * 32 + ty + 8 * q) * pb.ldh + bj * 32 + tx] = 0.0;
    return;
  }
  __shared__ double xa[32][33], xb[32][33];   // xa = d_i x_i over block bi, xb = x_i over block bj, for 32 rows
  const double* d = dvec + row_start[blockIdx.z];
  const int icol = has_bias ? pb.Dt - 1 : -1;
  double acc[4] = {0, 0, 0, 0};
  for (long long r0 = 0; r0 < pb.n; r0 += 32) {
    for (int e = threadIdx.x; e < 32 * 32; e += 256) { xa[e >> 5][e & 31] = 0.0; xb[e >> 5][e & 31] = 0.0; }
    __syncthreads();
    for (int t = ty; t < 64; t += 8) {   // warp ty: rows ty, ty + 8, .. of the slab, block bi then bj
      const int r = t & 31;
      const long long i = r0 + r;
      if (i >= pb.n) continue;
      const bool A = t < 32;
      const int c0 = (A ? bi : bj) * 32;
      const double s = A ? d[i] : 1.0;
      double* x = A ? xa[r] : xb[r];
      const long long j1 = pb.rowptr[i + 1];
      long long lo = pb.rowptr[i], hi = j1;
      while (lo < hi) { const long long mid = (lo + hi) >> 1; if (pb.colidx[mid] < c0) lo = mid + 1; else hi = mid; }
      const long long j = lo + tx;   // strictly increasing columns: the block's entries are the next 32 at most
      if (j < j1) { const int c = pb.colidx[j]; if (c < c0 + 32) x[c - c0] = s * (double)pb.vals[j]; }
      if (tx == 0 && icol >= c0 && icol < c0 + 32) x[icol - c0] = s;
    }
    __syncthreads();
#pragma unroll 8
    for (int r = 0; r < 32; r++) {
      const double b = xb[r][tx];
#pragma unroll
      for (int q = 0; q < 4; q++) acc[q] += xa[r][ty + 8 * q] * b;
    }
    __syncthreads();
  }
#pragma unroll
  for (int q = 0; q < 4; q++) {
    const int i = bi * 32 + ty + 8 * q, j = bj * 32 + tx;
    double v = j <= i ? acc[q] : 0.0;
    if (i == j) v += i < pb.Dt ? pb.q[i] : 1.0;
    H[(size_t)i * pb.ldh + j] = v;
  }
}

static int postvar_grid(long long nrows) { return (int)std::max(1LL, std::min(1184LL, (nrows + 7) / 8)); }   // 8 warps per CTA
cudaError_t postvar_rowweights(const Problem* d_probs, int nprob, const long long* d_row_start, long long nrows, int has_bias, double* d_dvec,
                               cudaStream_t st, int* launches) {
  postvar_rowweight_kernel<<<postvar_grid(nrows), 256, 0, st>>>(d_probs, nprob, d_row_start, has_bias, d_dvec);
  if (launches) *launches += 1;
  return cudaGetLastError();
}
cudaError_t postvar_diag(const Problem* d_probs, int nprob, const long long* d_row_start, long long nrows, const double* d_dvec, int has_bias,
                         cudaStream_t st, int* launches) {
  postvar_diag_init_kernel<<<nprob, 128, 0, st>>>(d_probs);
  postvar_diag_kernel<<<postvar_grid(nrows), 256, 0, st>>>(d_probs, nprob, d_row_start, d_dvec, has_bias);
  if (launches) *launches += 2;
  return cudaGetLastError();
}
cudaError_t postvar_hessian(const Problem* d_prob, bool csr, int ldh, const double* d_dvec, const double* d_q, int has_bias, cudaStream_t st, int* launches) {
  postvar_init_kernel<<<1184, 256, 0, st>>>(d_prob, d_q);
  if (csr) postvar_hess_csr_kernel<<<1184, 256, 0, st>>>(d_prob, d_dvec, has_bias);
  else { const int T = ldh / 32; postvar_hess_dense_kernel<<<dim3(T, T), 256, 0, st>>>(d_prob, d_dvec); }
  if (launches) *launches += 2;
  return cudaGetLastError();
}
cudaError_t postvar_hessian_batch(const Problem* d_probs, int nprob, int ldh, const long long* d_row_start, const double* d_dvec, int has_bias,
                                  cudaStream_t st, int* launches) {
  const int T = ldh / 32;
  postvar_hess_batch_kernel<<<dim3(T, T, nprob), 256, 0, st>>>(d_probs, d_row_start, d_dvec, has_bias);
  if (launches) *launches += 1;
  return cudaGetLastError();
}

}  // namespace mlease
