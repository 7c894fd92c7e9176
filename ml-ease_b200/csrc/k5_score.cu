// k5_score.cu -- K5: scoring and test log-likelihood.
//   score : LinearModel.eval / evalInstanceAvro(loglik=false) (models/LinearModel.java:241-257,491-554) and the
//           float cast of RegressionTest (jobs/RegressionTest.java:163).  One warp per record, fp64 accumulate.
//   loglik: RegressionTestLoglik mapper/combiner/reducer (jobs/RegressionTestLoglik.java:124-200) with its float
//           rounding points: per-record float, per-combiner-block float, final float(sum/count).
//   keyed : ItemModelTest / ItemModelTestLoglik, the same two computations with one model (and one reducer) per key.
// HBM-bound streaming kernels (one read of the test matrix).
#include <cub/device/device_radix_sort.cuh>

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

// ---- ItemModelTest (jobs/ItemModelTest.java:181-211): every record scored with its key's model, for LP lambdas at once ----
// table [key - k0][Dg][LP] fp32: the chunk's models scattered dense, so one LP-wide load per stored value serves every lambda
// of the group.  The arithmetic of each lambda is score_kernel's (same lane stride, fp64 products and sums, warp_sum, final
// float cast), which makes a pred bitwise equal to mlease_score on that key's rows with that key's model.
template <int LP>
__device__ __forceinline__ void load_lp(const float* p, float (&t)[LP]) {
  if constexpr (LP == 4) { const float4 v = *reinterpret_cast<const float4*>(p); t[0] = v.x; t[1] = v.y; t[2] = v.z; t[3] = v.w; }
  else if constexpr (LP == 2) { const float2 v = *reinterpret_cast<const float2*>(p); t[0] = v.x; t[1] = v.y; }
  else t[0] = *p;
}

template <int LP>
__global__ void __launch_bounds__(256) score_keyed_kernel(int Dg, int k0, int k1, long long r0, long long r1, const long long* __restrict__ krs,
                                                          const long long* __restrict__ rowptr, const int* __restrict__ colidx,
                                                          const float* __restrict__ vals, const float* __restrict__ offset,
                                                          const float* __restrict__ table, const double* __restrict__ term, int K, int G,
                                                          int binary_feature, long long nrows, float* __restrict__ pred, int* __restrict__ bad) {
  const int lane = threadIdx.x & 31;
  const long long wg = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long i = r0 + wg; i < r1; i += nw) {
    int lo = k0, hi = k1;   // krs[lo] <= i < krs[hi]: row i belongs to key lo once hi = lo + 1
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (krs[mid] <= i) lo = mid; else hi = mid; }
    const float* tk = table + (size_t)(lo - k0) * Dg * LP;
    double a[LP];
#pragma unroll
    for (int q = 0; q < LP; q++) a[q] = 0.0;
    for (long long j = rowptr[i] + lane; j < rowptr[i + 1]; j += 32) {
      const int c = colidx[j];
      if ((unsigned)c >= (unsigned)Dg) { *bad = 1; continue; }
      float t[LP];
      load_lp<LP>(tk + (size_t)c * LP, t);
      const double v = binary_feature ? 1.0 : (double)vals[j];
#pragma unroll
      for (int q = 0; q < LP; q++) a[q] += (double)t[q] * v;
    }
#pragma unroll
    for (int q = 0; q < LP; q++) a[q] = warp_sum(a[q]);
    if (lane == 0) {
      const double o = offset ? (double)offset[i] : 0.0;
#pragma unroll
      for (int q = 0; q < LP; q++)
        if (q < G) pred[(size_t)q * nrows + i] = (float)(o + (term[(size_t)q * K + lo] + a[q]));
    }
  }
}

// one warp per (lambda of the group, key of the chunk): its model's coefficients into the table; the intercept (column Dg)
// is not a table column, it enters through term
__global__ void __launch_bounds__(256) keyed_table_scatter_kernel(int Dg, int K, int k0, int nk, int G, int LP, const long long* __restrict__ mp,
                                                                  const int* __restrict__ mc, const float* __restrict__ mv, float* __restrict__ table) {
  const int lane = threadIdx.x & 31;
  const long long w = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= (long long)nk * G) return;
  const int q = (int)(w / nk), kk = (int)(w % nk);
  const long long m = (long long)q * K + k0 + kk;
  for (long long e = mp[m] + lane; e < mp[m + 1]; e += 32) {
    const int c = mc[e];
    if (c < Dg) table[((size_t)kk * Dg + c) * LP + q] = mv[e];
  }
}

cudaError_t score_keyed_chunk(int Dg, int K, int k0, int k1, long long r0, long long r1, const long long* krs, const long long* rowptr,
                              const int* colidx, const float* vals, const float* offset, int G, const long long* mp, const int* mc,
                              const float* mv, const double* term, int binary_feature, long long nrows, float* table, float* pred,
                              int* d_bad, cudaStream_t st) {
  const int LP = G == 1 ? 1 : G == 2 ? 2 : 4;
  const int nk = k1 - k0;
  cudaError_t e = cudaMemsetAsync(table, 0, (size_t)nk * Dg * LP * sizeof(float), st);
  if (e != cudaSuccess) return e;
  const long long warps = (long long)nk * G;
  keyed_table_scatter_kernel<<<(int)((warps + 7) / 8), 256, 0, st>>>(Dg, K, k0, nk, G, LP, mp, mc, mv, table);
  if (r1 > r0) {
    long long blocks = (r1 - r0 + 7) / 8;
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (LP == 1) score_keyed_kernel<1><<<(int)blocks, 256, 0, st>>>(Dg, k0, k1, r0, r1, krs, rowptr, colidx, vals, offset, table, term, K, G, binary_feature, nrows, pred, d_bad);
    else if (LP == 2) score_keyed_kernel<2><<<(int)blocks, 256, 0, st>>>(Dg, k0, k1, r0, r1, krs, rowptr, colidx, vals, offset, table, term, K, G, binary_feature, nrows, pred, d_bad);
    else score_keyed_kernel<4><<<(int)blocks, 256, 0, st>>>(Dg, k0, k1, r0, r1, krs, rowptr, colidx, vals, offset, table, term, K, G, binary_feature, nrows, pred, d_bad);
  }
  return cudaGetLastError();
}

// ---- ItemModelTestLoglik (jobs/ItemModelTestLoglik.java:60-142) ----
// mapper: float loglik per (record, pred-map key) entry; the entries are then sorted stably by (key, combiner group), so each
// (key, group) run is one combiner call and a key's runs follow each other in group order
__global__ void keyed_loglik_entry_kernel(long long n, int nkeys, long long ngroups, const int* __restrict__ key, const int* __restrict__ group,
                                          const int* __restrict__ response, const float* __restrict__ weight, const float* __restrict__ pred,
                                          float* __restrict__ ll, long long* __restrict__ skey, int* __restrict__ idx, int* __restrict__ bad) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = response[i], k = key[i], g = group[i];
  int b = 0;
  if (r != 1 && r != 0 && r != -1) b |= 1;
  if (k < 0 || k >= nkeys) b |= 2;
  if (g < 0 || g >= ngroups || (i > 0 && group[i - 1] > g)) b |= 4;
  if (b) atomicOr(bad, b);
  const double w = weight ? (double)weight[i] : 1.0, p = (double)pred[i];
  ll[i] = (float)((r == 1) ? -log1p(exp(-p)) * w : -log1p(exp(p)) * w);
  skey[i] = b ? 0 : (long long)k * ngroups + g;
  idx[i] = (int)i;
}

__device__ __forceinline__ long long lower_bound_ll(const long long* a, long long lo, long long hi, long long v) {
  while (lo < hi) { const long long mid = (lo + hi) >> 1; if (a[mid] < v) lo = mid + 1; else hi = mid; }
  return lo;
}

// one warp per key: each (key, group) run is a combiner call, float(double sum of the float logliks) and the double sum of the
// weights; the reducer adds the runs in group order in double and divides
__global__ void __launch_bounds__(256) keyed_loglik_reduce_kernel(long long n, int nkeys, long long ngroups, const long long* __restrict__ skey,
                                                                  const int* __restrict__ idx, const float* __restrict__ ll,
                                                                  const float* __restrict__ weight, float* __restrict__ out_ll,
                                                                  double* __restrict__ out_cnt) {
  const int lane = threadIdx.x & 31;
  const long long k = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (k >= nkeys) return;
  const long long lo = lower_bound_ll(skey, 0, n, k * ngroups), hi = lower_bound_ll(skey, lo, n, (k + 1) * ngroups);
  double sum = 0.0, cnt = 0.0;
  for (long long s = lo; s < hi;) {
    const long long e = lower_bound_ll(skey, s, hi, skey[s] + 1);
    double a = 0.0, c = 0.0;
    for (long long j = s + lane; j < e; j += 32) { const int t = idx[j]; a += (double)ll[t]; c += weight ? (double)weight[t] : 1.0; }
    a = warp_sum(a); c = warp_sum(c);
    sum += (double)(float)a;
    cnt += c;
    s = e;
  }
  if (lane == 0) { out_ll[k] = (float)(sum / cnt); out_cnt[k] = cnt; }
}

cudaError_t loglik_keyed_launch(long long n, int nkeys, long long ngroups, const int* key, const int* group, const int* response,
                                const float* weight, const float* pred, float* d_ll, long long* d_skey, long long* d_skey_sorted,
                                int* d_idx, int* d_idx_sorted, void* d_tmp, size_t* tmp_bytes, int* d_bad, float* d_out_ll,
                                double* d_out_cnt, cudaStream_t st) {
  int end_bit = 1;
  while (end_bit < 63 && ((long long)nkeys * ngroups - 1) >> end_bit) end_bit++;
  if (!d_tmp)   // size query
    return cub::DeviceRadixSort::SortPairs(nullptr, *tmp_bytes, d_skey, d_skey_sorted, d_idx, d_idx_sorted, (int)n, 0, end_bit, st);
  keyed_loglik_entry_kernel<<<(int)((n + 255) / 256), 256, 0, st>>>(n, nkeys, ngroups, key, group, response, weight, pred, d_ll, d_skey, d_idx, d_bad);
  cudaError_t e = cub::DeviceRadixSort::SortPairs(d_tmp, *tmp_bytes, d_skey, d_skey_sorted, d_idx, d_idx_sorted, (int)n, 0, end_bit, st);
  if (e != cudaSuccess) return e;
  keyed_loglik_reduce_kernel<<<(int)((nkeys + 7) / 8), 256, 0, st>>>(n, nkeys, ngroups, d_skey_sorted, d_idx_sorted, d_ll, weight, d_out_ll, d_out_cnt);
  return cudaGetLastError();
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
