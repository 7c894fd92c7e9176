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
#include <cub/device/device_radix_sort.cuh>

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

// ------------------------------------------------------------------------------------------
// The ADMM model's posterior (mlease_admm_posterior): the exact fp64 Hessian sum_i d_i x~_i x~_i^T of a whole resident partition,
// added into a sum over partitions.  CSR rows (strictly increasing columns) are walked column by column as the sparse Gram walks
// them (gram_csr_column_kernel): with the intercept an implicit last entry of every row, the lower triangle's column c1 is
//     H[c2][c1] = sum over the rows r listing c1 of d_r x_{r,c1} x_{r,c2},   c2 >= c1 in the row's suffix from c1 to its intercept,
// so every entry read is a product and the column needs only the positions of its entries.  Positions are those of the row-order
// operand of the sparse Gram's column index (row r at [rowptr[r] + r, rowptr[r + 1] + r], its intercept last): the session's own
// index where it built one, else one built for the call; rowof[] maps a position back to its row.
// Determinism: a column belongs to one CTA, which walks its rows in row order (staged HC_STAGE at a time).  Its cells are dealt to
// the CTA's warps by 32-column groups ((c2 >> 5) & 7), and a warp adds a row's products to its own cells only -- one lane per cell
// (a row lists a column once) -- with a __syncwarp between rows: every cell is a plain fp64 sum over its rows in row order, no
// atomics, whatever CTA runs the column or when.  The CTAs take columns from a counter in descending order of their work (the summed
// suffix lengths of their rows) so that the costly columns of a skewed dictionary start first.  The intercept's own cell, sum_i d_i,
// is a fixed-order block reduction.  The work is sum_i n_i (n_i + 1) / 2 fp64 FMAs with n_i the row's entries plus its intercept:
// ~5e9 at 1M x 10k x 1 %; every warp reads every suffix of its column (from L1 after the first), each adds only its cells' products.
// ------------------------------------------------------------------------------------------
constexpr int HC_THREADS = 256;
constexpr int HC_WARPS = HC_THREADS / 32;
constexpr int HC_STAGE = 256;        // column positions staged per step
constexpr int HC_CELLS = 12288;      // fp64 cells of a column window: 96 KB, two CTAs an SM

// rowof[q] = r for every position q of row r (its entries and its intercept)
__global__ void __launch_bounds__(256) postvar_rowof_kernel(long long n, const long long* __restrict__ rowptr, uint32_t* __restrict__ rowof) {
  const int lane = threadIdx.x & 31;
  const long long nw = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += nw)
    for (long long j = rowptr[r] + lane; j <= rowptr[r + 1]; j += 32) rowof[j + r] = (uint32_t)r;
}

// cost[c] = the products column c's walk forms (the suffix lengths of its positions, intercept included), cols[c] = c
__global__ void __launch_bounds__(256) postvar_colcost_kernel(int Dt, const long long* __restrict__ rowptr, const uint32_t* __restrict__ offs,
                                                              const uint32_t* __restrict__ pos, const uint32_t* __restrict__ rowof,
                                                              unsigned long long* __restrict__ cost, int* __restrict__ cols) {
  const int lane = threadIdx.x & 31;
  const int nw = (gridDim.x * blockDim.x) >> 5;
  for (int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < Dt; c += nw) {
    unsigned long long s = 0;
    for (uint32_t i = offs[c] + lane; i < offs[c + 1]; i += 32) {
      const uint32_t q = pos[i], r = rowof[q];
      s += (unsigned long long)(rowptr[r + 1] + r + 1 - q);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) s += __shfl_down_sync(0xffffffffu, s, d);
    if (lane == 0) { cost[c] = s; cols[c] = c; }
  }
}

struct HessCsr {
  long long n;
  const long long* rowptr;
  const int* colidx;
  const float* vals;
  const double* d;
  const uint32_t *offs, *pos, *rowof;
  const int* order;   // columns, costliest first
  int* next;          // column counter (0 before the launch)
  int Dt, ldh;
  double* H;          // += into the lower triangle, ld = ldh
};

__global__ void __launch_bounds__(HC_THREADS, 2) postvar_hess_col_kernel(HessCsr a) {
  extern __shared__ __align__(16) unsigned char hc_smem_raw[];
  double* acc = reinterpret_cast<double*>(hc_smem_raw);
  __shared__ long long sj[HC_STAGE];
  __shared__ int slen[HC_STAGE];
  __shared__ double sx[HC_STAGE];
  __shared__ double red[HC_WARPS];
  __shared__ int s_k;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int hot = a.Dt - 1, W = min(a.Dt, HC_CELLS);
  while (true) {
    if (threadIdx.x == 0) s_k = atomicAdd(a.next, 1);
    __syncthreads();
    const int k = s_k;
    __syncthreads();
    if (k >= a.Dt) return;
    const int c1 = a.order[k];
    if (c1 == hot) {   // every row's intercept squared: sum_i d_i
      double s = 0.0;
      for (long long r = threadIdx.x; r < a.n; r += HC_THREADS) s += a.d[r];
      s = warp_sum(s);
      if (lane == 0) red[warp] = s;
      __syncthreads();
      if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < HC_WARPS; w++) t += red[w];
        a.H[(size_t)hot * a.ldh + hot] += t;
      }
      continue;
    }
    const uint32_t p0 = a.offs[c1], p1 = a.offs[c1 + 1];
    for (int w0 = c1; w0 < a.Dt; w0 += W) {
      const int w1 = min(a.Dt, w0 + W);
      for (int e = threadIdx.x; e < w1 - w0; e += HC_THREADS) acc[e] = 0.0;
      __syncthreads();
      for (uint32_t b0 = p0; b0 < p1; b0 += HC_STAGE) {
        const int cnt = (int)min((uint32_t)HC_STAGE, p1 - b0);
        if (threadIdx.x < cnt) {
          const uint32_t q = a.pos[b0 + threadIdx.x], r = a.rowof[q];
          const long long j = (long long)q - r;
          sj[threadIdx.x] = j;
          slen[threadIdx.x] = (int)(a.rowptr[r + 1] - j);   // stored entries from c1 on; the intercept follows
          sx[threadIdx.x] = a.d[r] * (double)a.vals[j];
        }
        __syncthreads();
        for (int t = 0; t < cnt; t++) {
          const long long j = sj[t];
          const int len = slen[t];
          const double x = sx[t];
          for (int e = lane; e <= len; e += 32) {
            const int c2 = e < len ? a.colidx[j + e] : hot;
            if (c2 >= w0 && c2 < w1 && ((c2 >> 5) & (HC_WARPS - 1)) == warp) acc[c2 - w0] += x * (e < len ? (double)a.vals[j + e] : 1.0);
          }
          __syncwarp();
        }
        __syncthreads();
      }
      for (int e = threadIdx.x; e < w1 - w0; e += HC_THREADS) a.H[(size_t)(w0 + e) * a.ldh + c1] += acc[e];
      __syncthreads();
    }
  }
}

// Diagonal mode, CSR: diag[c] += sum over the positions of column c of d_r x_rc^2 (x = 1 at the intercept), in row order per lane
// then warp_sum
__global__ void __launch_bounds__(256) postvar_diag_col_kernel(int Dt, const long long* __restrict__ rowptr, const float* __restrict__ vals,
                                                               const double* __restrict__ d, const uint32_t* __restrict__ offs,
                                                               const uint32_t* __restrict__ pos, const uint32_t* __restrict__ rowof,
                                                               double* __restrict__ diag) {
  const int lane = threadIdx.x & 31;
  const int nw = (gridDim.x * blockDim.x) >> 5;
  for (int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < Dt; c += nw) {
    double s = 0.0;
    for (uint32_t i = offs[c] + lane; i < offs[c + 1]; i += 32) {
      const uint32_t q = pos[i], r = rowof[q];
      const long long j = (long long)q - r;
      const double x = j < rowptr[r + 1] ? (double)vals[j] : 1.0;
      s += d[r] * x * x;
    }
    s = warp_sum(s);
    if (lane == 0) diag[c] += s;
  }
}

// Diagonal mode, dense rows (the intercept is the physical column Dt - 1 of 1.0f): diag[k] += sum_i d_i x_ik^2 in row order
__global__ void __launch_bounds__(256) postvar_diag_dense_kernel(long long n, int Dt, const float* __restrict__ X, int ldx, const double* __restrict__ d,
                                                                 double* __restrict__ diag) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= Dt) return;
  double s = 0.0;
  for (long long i = 0; i < n; i++) { const double x = (double)X[(size_t)i * ldx + k]; s += d[i] * x * x; }
  diag[k] += s;
}

// Lc = Hs + diag(q) on the lower triangle of [0, Dt), identity on the padding, zero above the diagonal (as chol_prep leaves it)
__global__ void postvar_lc_kernel(const double* __restrict__ Hs, const double* __restrict__ q, int Dt, int ldh, double* __restrict__ Lc) {
  const size_t total = (size_t)ldh * ldh;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int i = (int)(e / ldh), j = (int)(e % ldh);
    Lc[e] = (i < Dt && j <= i) ? Hs[e] + (i == j ? q[i] : 0.0) : (i == j ? 1.0 : 0.0);
  }
}

// the lower triangle of [0, Dt) (ld ldh) to / from packed rows (i (i + 1) / 2 + j): the all-reduce sends Dt (Dt + 1) / 2 doubles
__global__ void postvar_pack_kernel(double* __restrict__ H, int Dt, int ldh, double* __restrict__ packed, int unpack) {
  const size_t total = (size_t)Dt * (Dt + 1) / 2;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    int i = (int)((sqrt(8.0 * (double)e + 1.0) - 1.0) * 0.5);
    while ((size_t)i * (i + 1) / 2 > e) i--;
    while ((size_t)(i + 1) * (i + 2) / 2 <= e) i++;
    const int j = (int)(e - (size_t)i * (i + 1) / 2);
    if (unpack) H[(size_t)i * ldh + j] = packed[e];
    else packed[e] = H[(size_t)i * ldh + j];
  }
}

cudaError_t postvar_rowof(long long n, const long long* rowptr, uint32_t* rowof, cudaStream_t st) {
  postvar_rowof_kernel<<<(int)std::max(1LL, std::min((n + 7) / 8, 132LL * 32)), 256, 0, st>>>(n, rowptr, rowof);
  return cudaGetLastError();
}

cudaError_t postvar_hessian_csr_cols(long long n, const long long* rowptr, const int* colidx, const float* vals, const double* d_dvec,
                                     const uint32_t* offs, const uint32_t* pos, const uint32_t* rowof, int Dt, int ldh, double* H, cudaStream_t st) {
  static bool configured[64] = {};
  static int sms[64] = {};
  cudaError_t e = set_smem_once(postvar_hess_col_kernel, HC_CELLS * sizeof(double), configured);
  if (e != cudaSuccess) return e;
  int dev = 0, nsm = 0;
  if ((e = cudaGetDevice(&dev)) != cudaSuccess) return e;
  if (dev >= 0 && dev < 64 && sms[dev]) nsm = sms[dev];
  else {
    if ((e = cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) sms[dev] = nsm;
  }
  const size_t smem = (size_t)std::min(Dt, HC_CELLS) * sizeof(double);
  // the column order: descending cost, ties in column order (stable sort)
  unsigned long long *cost = nullptr, *cost_s = nullptr;
  int *cols = nullptr, *order = nullptr, *next = nullptr;
  void* tmp = nullptr;
  size_t tmp_bytes = 0;
  auto run = [&]() -> cudaError_t {
    cudaError_t r;
    if ((r = cudaMallocAsync(&cost, (size_t)Dt * 8, st)) != cudaSuccess) return r;
    if ((r = cudaMallocAsync(&cost_s, (size_t)Dt * 8, st)) != cudaSuccess) return r;
    if ((r = cudaMallocAsync(&cols, (size_t)Dt * 4, st)) != cudaSuccess) return r;
    if ((r = cudaMallocAsync(&order, (size_t)Dt * 4, st)) != cudaSuccess) return r;
    if ((r = cudaMallocAsync(&next, 4, st)) != cudaSuccess) return r;
    if ((r = cudaMemsetAsync(next, 0, 4, st)) != cudaSuccess) return r;
    postvar_colcost_kernel<<<std::max(1, std::min((Dt + 7) / 8, 132 * 32)), 256, 0, st>>>(Dt, rowptr, offs, pos, rowof, cost, cols);
    if ((r = cudaGetLastError()) != cudaSuccess) return r;
    if ((r = cub::DeviceRadixSort::SortPairsDescending(nullptr, tmp_bytes, cost, cost_s, cols, order, Dt, 0, 64, st)) != cudaSuccess) return r;
    if ((r = cudaMallocAsync(&tmp, tmp_bytes ? tmp_bytes : 16, st)) != cudaSuccess) return r;
    if ((r = cub::DeviceRadixSort::SortPairsDescending(tmp, tmp_bytes, cost, cost_s, cols, order, Dt, 0, 64, st)) != cudaSuccess) return r;
    HessCsr a{n, rowptr, colidx, vals, d_dvec, offs, pos, rowof, order, next, Dt, ldh, H};
    postvar_hess_col_kernel<<<std::max(1, std::min(Dt, 2 * nsm)), HC_THREADS, smem, st>>>(a);
    return cudaGetLastError();
  };
  e = run();
  for (void* p : {(void*)cost, (void*)cost_s, (void*)cols, (void*)order, (void*)next, tmp})
    if (p) { cudaError_t e2 = cudaFreeAsync(p, st); if (e == cudaSuccess) e = e2; }
  return e;
}

cudaError_t postvar_hessian_dense_add(const Problem* d_prob, int ldh, const double* d_dvec, cudaStream_t st) {
  const int T = ldh / 32;
  postvar_hess_dense_kernel<<<dim3(T, T), 256, 0, st>>>(d_prob, d_dvec);
  return cudaGetLastError();
}

cudaError_t postvar_diag_csr_cols(const long long* rowptr, const float* vals, const double* d_dvec, const uint32_t* offs, const uint32_t* pos,
                                  const uint32_t* rowof, int Dt, double* diag, cudaStream_t st) {
  postvar_diag_col_kernel<<<std::max(1, std::min((Dt + 7) / 8, 132 * 32)), 256, 0, st>>>(Dt, rowptr, vals, d_dvec, offs, pos, rowof, diag);
  return cudaGetLastError();
}

cudaError_t postvar_diag_dense(long long n, int Dt, const float* X, int ldx, const double* d_dvec, double* diag, cudaStream_t st) {
  postvar_diag_dense_kernel<<<(Dt + 127) / 128, 128, 0, st>>>(n, Dt, X, ldx, d_dvec, diag);
  return cudaGetLastError();
}

cudaError_t postvar_lc(const double* Hs, const double* d_q, int Dt, int ldh, double* Lc, cudaStream_t st) {
  postvar_lc_kernel<<<1184, 256, 0, st>>>(Hs, d_q, Dt, ldh, Lc);
  return cudaGetLastError();
}

cudaError_t postvar_pack(double* H, int Dt, int ldh, double* packed, int unpack, cudaStream_t st) {
  postvar_pack_kernel<<<1184, 256, 0, st>>>(H, Dt, ldh, packed, unpack);
  return cudaGetLastError();
}

}  // namespace mlease
