// k5_score.cu -- K5: scoring and test log-likelihood.
//   score : LinearModel.eval / evalInstanceAvro(loglik=false) (models/LinearModel.java:241-257,491-554) and the
//           float cast of RegressionTest (jobs/RegressionTest.java:163).  One warp per record, fp64 accumulate.
//   loglik: RegressionTestLoglik mapper/combiner/reducer (jobs/RegressionTestLoglik.java:124-200) with its float
//           rounding points: per-record float, per-combiner-block float, final float(sum/count).
//   keyed : ItemModelTest / ItemModelTestLoglik, the same two computations with one model (and one reducer) per key; with a
//           variance list per model (ItemModelTrain's posteriorVar), also each record's predictive variance.
// HBM-bound streaming kernels (one read of the test matrix).
#include <cub/device/device_radix_sort.cuh>

#include <cmath>
#include <string>
#include <vector>

#include "host.cuh"

namespace mlease {

__global__ void __launch_bounds__(256) score_kernel(int Dg, long long nrows, const long long* __restrict__ rowptr,
                                                    const int* __restrict__ colidx, const float* __restrict__ vals, long long ldx,
                                                    const float* __restrict__ offset, const double* __restrict__ model,
                                                    double intercept_term, int binary_feature, float* __restrict__ pred,
                                                    int* __restrict__ bad) {
  const int lane = threadIdx.x & 31;
  const long long wg = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long i = wg; i < nrows; i += nw) {
    double a = 0.0;
    if (colidx) {
      for (long long j = rowptr[i] + lane; j < rowptr[i + 1]; j += 32) {
        const int c = colidx[j];
        if ((unsigned)c >= (unsigned)Dg) { atomicOr(bad, 1); continue; }   // never read outside the model, nor the intercept
        a += model[c] * (binary_feature ? 1.0 : (double)vals[j]);
      }
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

// WITH_VAR (mlease_score_keyed_var): a second [key - k0][Dg][LP] table holds each model's diagonal posterior variance (var_default
// where its list names no column), and pred_var = float(sum v x^2 + vterm) beside pred, in fp64 with the same lane stride.  Rows
// must then list strictly ascending columns (bad |= 2): a repeated column would count as two independent terms of the variance.
template <int LP, bool WITH_VAR>
__global__ void __launch_bounds__(256) score_keyed_kernel(int Dg, int k0, int k1, long long r0, long long r1, const long long* __restrict__ krs,
                                                          const long long* __restrict__ rowptr, const int* __restrict__ colidx,
                                                          const float* __restrict__ vals, const float* __restrict__ offset,
                                                          const float* __restrict__ table, const double* __restrict__ term, int K, int G,
                                                          int binary_feature, long long nrows, long long row_base, float* __restrict__ pred,
                                                          int* __restrict__ bad, const float* __restrict__ vtable,
                                                          const double* __restrict__ vterm, float* __restrict__ pred_var) {
  // rowptr, offset and pred hold rows [row_base, ...): a streamed key range indexes its own copy of them
  rowptr -= row_base;
  if (offset) offset -= row_base;
  pred -= row_base;
  if constexpr (WITH_VAR) pred_var -= row_base;
  const int lane = threadIdx.x & 31;
  const long long wg = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long i = r0 + wg; i < r1; i += nw) {
    int lo = k0, hi = k1;   // krs[lo] <= i < krs[hi]: row i belongs to key lo once hi = lo + 1
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (krs[mid] <= i) lo = mid; else hi = mid; }
    const float* tk = table + (size_t)(lo - k0) * Dg * LP;
    double a[LP], va[LP];
#pragma unroll
    for (int q = 0; q < LP; q++) { a[q] = 0.0; if constexpr (WITH_VAR) va[q] = 0.0; }
    const long long j0 = rowptr[i];
    for (long long j = j0 + lane; j < rowptr[i + 1]; j += 32) {
      const int c = colidx[j];
      if ((unsigned)c >= (unsigned)Dg) { *bad = 1; continue; }
      if constexpr (WITH_VAR) { if (j > j0 && colidx[j - 1] >= c) { atomicOr(bad, 2); continue; } }
      float t[LP];
      load_lp<LP>(tk + (size_t)c * LP, t);
      const double v = binary_feature ? 1.0 : (double)vals[j];
#pragma unroll
      for (int q = 0; q < LP; q++) a[q] += (double)t[q] * v;
      if constexpr (WITH_VAR) {
        float s[LP];
        load_lp<LP>(vtable + ((size_t)(lo - k0) * Dg + c) * LP, s);
        const double v2 = v * v;
#pragma unroll
        for (int q = 0; q < LP; q++) va[q] += (double)s[q] * v2;
      }
    }
#pragma unroll
    for (int q = 0; q < LP; q++) { a[q] = warp_sum(a[q]); if constexpr (WITH_VAR) va[q] = warp_sum(va[q]); }
    if (lane == 0) {
      const double o = offset ? (double)offset[i] : 0.0;
#pragma unroll
      for (int q = 0; q < LP; q++)
        if (q < G) {
          pred[(size_t)q * nrows + i] = (float)(o + (term[(size_t)q * K + lo] + a[q]));
          if constexpr (WITH_VAR) pred_var[(size_t)q * nrows + i] = (float)(va[q] + vterm[(size_t)q * K + lo]);
        }
    }
  }
}

// one warp per (lambda of the group, key of the chunk): its model's coefficients into the table; the intercept (column Dg)
// is not a table column, it enters through term.  fill (variance lists): every column of the model's slice starts at fill[m].
__global__ void __launch_bounds__(256) keyed_table_scatter_kernel(int Dg, int K, int k0, int nk, int G, int LP, const long long* __restrict__ mp,
                                                                  const int* __restrict__ mc, const float* __restrict__ mv, float* __restrict__ table,
                                                                  const float* __restrict__ fill) {
  const int lane = threadIdx.x & 31;
  const long long w = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= (long long)nk * G) return;
  const int q = (int)(w / nk), kk = (int)(w % nk);
  const long long m = (long long)q * K + k0 + kk;
  if (fill) {
    for (int c = lane; c < Dg; c += 32) table[((size_t)kk * Dg + c) * LP + q] = fill[m];
    __syncwarp();
  }
  for (long long e = mp[m] + lane; e < mp[m + 1]; e += 32) {
    const int c = mc[e];
    if (c < Dg) table[((size_t)kk * Dg + c) * LP + q] = mv[e];
  }
}

// The variance lists of mlease_score_keyed_var on the device, for one group of up to four lambdas (at()); all null for
// mlease_score_keyed.  vterm[m]: the listed intercept variance, 0 without one, NaN for an empty list.
struct KeyedVar {
  const long long* vp = nullptr;
  const int* vc = nullptr;
  const float* vv = nullptr;
  const float* vdef = nullptr;
  const double* vterm = nullptr;
  float* vtable = nullptr;
  float* pred_var = nullptr;
  explicit operator bool() const { return vp != nullptr; }
  KeyedVar at(int l0, int K, long long nrows) const {
    if (!vp) return *this;
    KeyedVar r = *this;
    r.vp += (size_t)l0 * K; r.vdef += (size_t)l0 * K; r.vterm += (size_t)l0 * K; r.pred_var += (size_t)l0 * nrows;
    return r;
  }
};

// mlease_score_keyed_cov: each record's predictive variance under the full posterior of its key's model, pred_var = float(x_L^T Sigma
// x_L + sum over unlisted columns of v_c x_c^2), x_L the record's entries the model lists plus the intercept at 1 when the list ends
// with it.  Sigma is the model's packed lower triangle over its list (entry (a, b), a >= b, at cov_ptr[m] + a(a+1)/2 + b); an empty
// block gives NaN.  v_c = 1 / lambda_map[c] where that is > 0, else var_default[m].  One warp per record and model: each entry's
// position in the list comes from a binary search, then the lanes walk the flat pair space of 256-entry tiles of the row (a tile
// with itself, then with each earlier tile), fp64, each lane over a fixed set of pairs in a fixed order, then warp_sum: bitwise
// repeatable, and the same for a record whichever range or chunk scores it.
constexpr int COV_TILE = 256;
struct KeyedCov {
  const long long* cp = nullptr;
  const double* cv = nullptr;
  const float* lm = nullptr;
  const float* vdef = nullptr;
  float* pred_var = nullptr;
  explicit operator bool() const { return cp != nullptr; }
};
__device__ __forceinline__ int cov_row_of(long long e) {   // the row a of flat lower-triangle entry e
  int a = (int)((sqrt(8.0 * (double)e + 1.0) - 1.0) * 0.5);
  while ((long long)a * (a + 1) / 2 > e) a--;
  while ((long long)(a + 1) * (a + 2) / 2 <= e) a++;
  return a;
}
__global__ void __launch_bounds__(256) score_keyed_cov_kernel(int Dg, int k0, int k1, long long r0, long long r1, const long long* __restrict__ krs,
                                                              const long long* __restrict__ rowptr, const int* __restrict__ colidx,
                                                              const float* __restrict__ vals, const long long* __restrict__ mp,
                                                              const int* __restrict__ mc, const long long* __restrict__ cp,
                                                              const double* __restrict__ cv, const float* __restrict__ lm,
                                                              const float* __restrict__ vdef, int K, int G, int binary_feature, long long nrows,
                                                              long long row_base, float* __restrict__ pred_var, int* __restrict__ bad) {
  __shared__ int spos[8][2][COV_TILE];
  __shared__ double sx[8][2][COV_TILE];
  rowptr -= row_base;
  pred_var -= row_base;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const long long wg = (long long)blockIdx.x * (blockDim.x >> 5) + w;
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long i = r0 + wg; i < r1; i += nw) {
    int lo = k0, hi = k1;
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (krs[mid] <= i) lo = mid; else hi = mid; }
    const long long j0 = rowptr[i], j1 = rowptr[i + 1];
    for (int q = 0; q < G; q++) {
      const long long m = (long long)q * K + lo;
      const long long e0 = mp[m];
      const int n = (int)(mp[m + 1] - e0);
      const double* S = cv + cp[m];
      if (cp[m + 1] == cp[m]) { if (lane == 0) pred_var[(size_t)q * nrows + i] = __int_as_float(0x7fc00000); continue; }
      const int* L = mc + e0;
      const int pI = (n > 0 && L[n - 1] == Dg) ? n - 1 : -1;
      const double vd = (double)vdef[m];
      auto sig = [&](int a, int b) { return a >= b ? S[(long long)a * (a + 1) / 2 + b] : S[(long long)b * (b + 1) / 2 + a]; };
      // tile t of the row's entries into buffer slot: list positions (-1: unlisted or out of range) and values; first: the diagonal
      // pass also adds the unlisted terms and the entries' pairs with the intercept
      auto load = [&](long long t0, int slot, bool first, double& acc) {
        for (int t = lane; t < COV_TILE; t += 32) {
          const long long j = t0 + t;
          int p = -1; double x = 0.0;
          if (j < j1) {
            const int c = colidx[j];
            x = binary_feature ? 1.0 : (double)vals[j];
            if ((unsigned)c >= (unsigned)Dg) { if (first) atomicOr(bad, 1); x = 0.0; }
            else {
              if (first && j > j0 && colidx[j - 1] >= c) atomicOr(bad, 2);
              int a = 0, b = n;
              while (a < b) { const int mid = (a + b) >> 1; if (L[mid] < c) a = mid + 1; else b = mid; }
              if (a < n && L[a] == c) {
                p = a;
                if (first && pI >= 0) acc += 2.0 * x * sig(pI, p);
              } else if (first) {
                acc += (lm && lm[c] > 0.f ? 1.0 / (double)lm[c] : vd) * x * x;
              }
            }
          }
          spos[w][slot][t] = p; sx[w][slot][t] = x;
        }
        __syncwarp();
      };
      double acc = 0.0;
      for (long long ta = j0; ta < j1; ta += COV_TILE) {
        const int Ta = (int)min((long long)COV_TILE, j1 - ta);
        load(ta, 0, true, acc);
        const long long tri = (long long)Ta * (Ta + 1) / 2;
        for (long long e = lane; e < tri; e += 32) {
          const int a = cov_row_of(e), b = (int)(e - (long long)a * (a + 1) / 2);
          const int pa = spos[w][0][a], pb = spos[w][0][b];
          if (pa >= 0 && pb >= 0) acc += (a == b ? 1.0 : 2.0) * sx[w][0][a] * sx[w][0][b] * sig(pa, pb);
        }
        for (long long tb = j0; tb < ta; tb += COV_TILE) {
          double unused = 0.0;
          load(tb, 1, false, unused);
          for (int e = lane; e < Ta * COV_TILE; e += 32) {
            const int a = e / COV_TILE, b = e % COV_TILE;
            const int pa = spos[w][0][a], pb = spos[w][1][b];
            if (pa >= 0 && pb >= 0) acc += 2.0 * sx[w][0][a] * sx[w][1][b] * sig(pa, pb);
          }
          __syncwarp();
        }
        __syncwarp();
      }
      if (lane == 0 && pI >= 0) acc += sig(pI, pI);
      acc = warp_sum(acc);
      if (lane == 0) pred_var[(size_t)q * nrows + i] = (float)acc;
    }
  }
}

// mlease_score_var: score_kernel's pred (the same sum, the same rounding) and pred_var = float(g^T Sigma g), g = the record's entries
// and gI at the intercept (column Dg, after every stored column).  Diagonal Sigma (var): each lane its entries, lane 0 the intercept,
// then warp_sum.  Dense Sigma (cov, ld Dg + 1, lower triangle read): the pair space of the row's 256-entry tiles as
// score_keyed_cov_kernel walks it (a tile with itself, then with each earlier tile), the intercept's pairs added in the diagonal
// tile's pass: each lane a fixed set of pairs in a fixed order, then warp_sum.  bad: 1 column out of range, 2 not ascending.
__global__ void __launch_bounds__(256) score_var_kernel(int Dg, long long nrows, const long long* __restrict__ rowptr, const int* __restrict__ colidx,
                                                        const float* __restrict__ vals, const float* __restrict__ offset,
                                                        const double* __restrict__ model, double intercept_term, double gI, int binary_feature,
                                                        const double* __restrict__ var, const double* __restrict__ cov, float* __restrict__ pred,
                                                        float* __restrict__ pred_var, int* __restrict__ bad) {
  __shared__ int scol[8][2][COV_TILE];
  __shared__ double sx[8][2][COV_TILE];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const long long wg = (long long)blockIdx.x * (blockDim.x >> 5) + w;
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  const size_t ld = (size_t)Dg + 1;
  for (long long i = wg; i < nrows; i += nw) {
    const long long j0 = rowptr[i], j1 = rowptr[i + 1];
    double a = 0.0;
    for (long long j = j0 + lane; j < j1; j += 32) {
      const int c = colidx[j];
      if ((unsigned)c >= (unsigned)Dg) { atomicOr(bad, 1); continue; }   // never read outside the model
      a += model[c] * (binary_feature ? 1.0 : (double)vals[j]);
    }
    a = warp_sum(a);
    if (lane == 0) pred[i] = (float)((offset ? (double)offset[i] : 0.0) + (intercept_term + a));
    double acc = 0.0;
    if (var) {
      for (long long j = j0 + lane; j < j1; j += 32) {
        const int c = colidx[j];
        if ((unsigned)c >= (unsigned)Dg) { atomicOr(bad, 1); continue; }
        if (j > j0 && colidx[j - 1] >= c) atomicOr(bad, 2);
        const double x = binary_feature ? 1.0 : (double)vals[j];
        acc += var[c] * x * x;
      }
      if (lane == 0) acc += var[Dg] * gI * gI;
    } else {
      auto load = [&](long long t0, int slot, bool first) {
        for (int t = lane; t < COV_TILE; t += 32) {
          const long long j = t0 + t;
          int c = -1; double x = 0.0;
          if (j < j1) {
            c = colidx[j];
            x = binary_feature ? 1.0 : (double)vals[j];
            if ((unsigned)c >= (unsigned)Dg) { if (first) atomicOr(bad, 1); c = -1; x = 0.0; }
            else {
              if (first && j > j0 && colidx[j - 1] >= c) atomicOr(bad, 2);
              if (first) acc += 2.0 * gI * x * cov[(size_t)Dg * ld + c];
            }
          }
          scol[w][slot][t] = c; sx[w][slot][t] = x;
        }
        __syncwarp();
      };
      for (long long ta = j0; ta < j1; ta += COV_TILE) {
        const int Ta = (int)min((long long)COV_TILE, j1 - ta);
        load(ta, 0, true);
        const long long tri = (long long)Ta * (Ta + 1) / 2;
        for (long long e = lane; e < tri; e += 32) {
          const int p = cov_row_of(e), q = (int)(e - (long long)p * (p + 1) / 2);
          const int ca = scol[w][0][p], cb = scol[w][0][q];
          if (ca >= 0 && cb >= 0) acc += (p == q ? 1.0 : 2.0) * sx[w][0][p] * sx[w][0][q] * cov[(size_t)max(ca, cb) * ld + min(ca, cb)];
        }
        for (long long tb = j0; tb < ta; tb += COV_TILE) {
          load(tb, 1, false);
          for (int e = lane; e < Ta * COV_TILE; e += 32) {
            const int p = e / COV_TILE, q = e % COV_TILE;
            const int ca = scol[w][0][p], cb = scol[w][1][q];
            if (ca >= 0 && cb >= 0) acc += 2.0 * sx[w][0][p] * sx[w][1][q] * cov[(size_t)max(ca, cb) * ld + min(ca, cb)];
          }
          __syncwarp();
        }
        __syncwarp();
      }
      if (lane == 0) acc += gI * gI * cov[(size_t)Dg * ld + Dg];
    }
    acc = warp_sum(acc);
    if (lane == 0) pred_var[i] = (float)acc;
  }
}

static cudaError_t score_keyed_chunk(int Dg, int K, int k0, int k1, long long r0, long long r1, const long long* krs, const long long* rowptr,
                                     const int* colidx, const float* vals, const float* offset, int G, const long long* mp, const int* mc,
                                     const float* mv, const double* term, int binary_feature, long long nrows, long long row_base, float* table,
                                     float* pred, int* d_bad, const KeyedVar& var, const KeyedCov& cov, cudaStream_t st) {
  const int LP = G == 1 ? 1 : G == 2 ? 2 : 4;
  const int nk = k1 - k0;
  const size_t tbytes = (size_t)nk * Dg * LP * sizeof(float);
  cudaError_t e = cudaMemsetAsync(table, 0, tbytes, st);
  if (e == cudaSuccess && var) e = cudaMemsetAsync(var.vtable, 0, tbytes, st);   // the unused lanes of a group of three
  if (e != cudaSuccess) return e;
  const long long warps = (long long)nk * G;
  keyed_table_scatter_kernel<<<(int)((warps + 7) / 8), 256, 0, st>>>(Dg, K, k0, nk, G, LP, mp, mc, mv, table, nullptr);
  if (var) keyed_table_scatter_kernel<<<(int)((warps + 7) / 8), 256, 0, st>>>(Dg, K, k0, nk, G, LP, var.vp, var.vc, var.vv, var.vtable, var.vdef);
  if (r1 > r0) {
    long long blocks = (r1 - r0 + 7) / 8;
    if (blocks > 132 * 16) blocks = 132 * 16;
#define MLEASE_SCORE_KEYED(LP_, V_)                                                                                                     \
  score_keyed_kernel<LP_, V_><<<(int)blocks, 256, 0, st>>>(Dg, k0, k1, r0, r1, krs, rowptr, colidx, vals, offset, table, term, K, G,   \
                                                           binary_feature, nrows, row_base, pred, d_bad, var.vtable, var.vterm, var.pred_var)
    if (var) {
      if (LP == 1) MLEASE_SCORE_KEYED(1, true); else if (LP == 2) MLEASE_SCORE_KEYED(2, true); else MLEASE_SCORE_KEYED(4, true);
    } else {
      if (LP == 1) MLEASE_SCORE_KEYED(1, false); else if (LP == 2) MLEASE_SCORE_KEYED(2, false); else MLEASE_SCORE_KEYED(4, false);
    }
#undef MLEASE_SCORE_KEYED
    if (cov)
      score_keyed_cov_kernel<<<(int)blocks, 256, 0, st>>>(Dg, k0, k1, r0, r1, krs, rowptr, colidx, vals, mp, mc, cov.cp, cov.cv, cov.lm,
                                                          cov.vdef, K, G, binary_feature, nrows, row_base, cov.pred_var, d_bad);
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

static cudaError_t loglik_keyed_launch(long long n, int nkeys, long long ngroups, const int* key, const int* group, const int* response,
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

static cudaError_t score_launch(int Dg, long long nrows, const long long* rowptr, const int* colidx, const float* vals, long long ldx,
                                const float* offset, const double* d_model, double intercept_term, int binary_feature, float* pred,
                                int* d_bad, cudaStream_t st) {
  if (nrows == 0) return cudaSuccess;
  long long blocks = (nrows + 7) / 8;
  if (blocks > 132 * 16) blocks = 132 * 16;
  score_kernel<<<(int)blocks, 256, 0, st>>>(Dg, nrows, rowptr, colidx, vals, ldx, offset, d_model, intercept_term, binary_feature, pred,
                                            d_bad);
  return cudaGetLastError();
}

static cudaError_t loglik_launch(long long nrows, const int* response, const float* pred, const float* weight, long long combiner_block,
                                 float* d_ll, double* d_block_sum, double* d_block_cnt, int* d_bad, cudaStream_t st) {
  if (nrows == 0) return cudaSuccess;
  loglik_record_kernel<<<(int)((nrows + 255) / 256), 256, 0, st>>>(nrows, response, pred, weight, d_ll, d_bad);
  const long long nb = (nrows + combiner_block - 1) / combiner_block;
  loglik_block_kernel<<<(int)nb, 256, 0, st>>>(nrows, d_ll, weight, combiner_block, d_block_sum, d_block_cnt);
  return cudaGetLastError();
}

// ItemModelTest.  The rows are uploaded once for every lambda.  Keys are taken in chunks whose dense coefficient table fits
// SCORE_KEYED_TABLE_CAP and a quarter of the free device memory; a chunk's rows are one contiguous range because rows come grouped
// by key.  A key's table slice (Dg * 16 B) is reused by all its rows from L2 while the rows stream from HBM once per group of
// four lambdas.
static constexpr size_t SCORE_KEYED_TABLE_CAP = size_t(1) << 30;

// the row checks of score_keyed_kernel, read back
static int keyed_bad(int bad) {
  if (bad & 1) return fail(MLEASE_ERR_INVALID, "colidx out of range [0, num_features)");
  if (bad & 2) return fail(MLEASE_ERR_INVALID, "colidx must be strictly ascending within a row");
  return 0;
}

// Host copies of mlease_score_keyed_var's variance lists, checked; absent for mlease_score_keyed.
struct KeyedVarHost {
  std::vector<long long> vp;
  std::vector<int> vc;
  std::vector<float> vv, vdef;
  std::vector<double> vterm;
  size_t bytes() const { return vp.size() * 8 + vc.size() * 4 + vv.size() * 4 + vdef.size() * 4 + vterm.size() * 8; }
  int upload(DevMem& t, KeyedVar& d, cudaStream_t st) const {
    if (int rc = to_device(t, (const long long*)vp.data(), vp.size(), &d.vp, st)) return rc;
    if (int rc = to_device(t, (const int*)vc.data(), vc.size(), &d.vc, st)) return rc;
    if (int rc = to_device(t, (const float*)vv.data(), vv.size(), &d.vv, st)) return rc;
    if (int rc = to_device(t, (const float*)vdef.data(), vdef.size(), &d.vdef, st)) return rc;
    return to_device(t, (const double*)vterm.data(), vterm.size(), &d.vterm, st);
  }
};

}  // namespace mlease

using namespace mlease;

extern "C" {

int mlease_score(int32_t device, void* stream, int32_t Dg, int64_t nrows, const int64_t* rowptr, const int32_t* colidx, const float* vals,
                 int64_t ldx, const float* offset, const double* model, int32_t num_click_replicates, int32_t binary_feature, float* pred) {
  if (!vals || !model || !pred || nrows < 0) return fail(MLEASE_ERR_INVALID, "bad argument");
  if (int rc = open_device(device, nullptr)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  DevMem t;
  const long long* d_rp = nullptr; const int* d_ci = nullptr; const float* d_v = nullptr; const float* d_o = nullptr; const double* d_m = nullptr;
  long long nnz = nrows * ldx;
  int* d_bad;
  if (int rc = t.get(&d_bad, 1, true)) return rc;
  if (colidx) {
    if (!rowptr) return fail(MLEASE_ERR_INVALID, "null rowptr");
    long long last;
    CK(cudaMemcpy(&last, rowptr + nrows, 8, cudaMemcpyDefault));
    if (last < 0) return fail(MLEASE_ERR_INVALID, "rowptr[nrows] < 0");
    nnz = last;
    if (int rc = to_device(t, (const long long*)rowptr, (size_t)nrows + 1, &d_rp, st)) return rc;
    if (int rc = check_rowptr(st, nrows, d_rp, d_bad, "")) return rc;
    if (int rc = to_device(t, colidx, (size_t)nnz, &d_ci, st)) return rc;
  }
  if (int rc = to_device(t, vals, (size_t)nnz, &d_v, st)) return rc;
  if (int rc = to_device(t, offset, (size_t)nrows, &d_o, st)) return rc;
  if (int rc = to_device(t, model, (size_t)Dg + 1, &d_m, st)) return rc;
  double b;
  CK(cudaMemcpy(&b, model + Dg, 8, cudaMemcpyDefault));
  // intercept term  -log(n - 1 + n exp(-b))  (models/LinearModel.java:243-244)
  const double ic = -std::log((double)num_click_replicates - 1 + (double)num_click_replicates * std::exp(-b));
  const bool pred_dev = is_device_ptr(pred);
  float* d_pred = pred;
  if (!pred_dev) { if (int rc = t.get(&d_pred, (size_t)nrows, false)) return rc; }
  CK(cudaMemsetAsync(d_bad, 0, 4, st));
  CK(score_launch(Dg, nrows, d_rp, d_ci, d_v, ldx, d_o, d_m, ic, binary_feature, d_pred, d_bad, st));
  int bad = 0;
  CK(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, st));
  if (!pred_dev) CK(cudaMemcpyAsync(pred, d_pred, (size_t)nrows * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return keyed_bad(bad);
}

int mlease_score_var(int32_t device, void* stream, int32_t Dg, int64_t nrows, const int64_t* rowptr, const int32_t* colidx, const float* vals,
                     const float* offset, const double* model, int32_t num_click_replicates, int32_t binary_feature, const double* var,
                     const double* cov, float* pred, float* pred_var) {
  if (!vals || !model || !pred || !pred_var || nrows < 0 || Dg <= 0) return fail(MLEASE_ERR_INVALID, "bad argument");
  if (!colidx || !rowptr) return fail(MLEASE_ERR_INVALID, "score_var takes CSR rows only (rowptr and colidx), not dense input");
  if ((var != nullptr) == (cov != nullptr)) return fail(MLEASE_ERR_INVALID, "exactly one of var and cov must be given");
  if (int rc = open_device(device, nullptr)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  DevMem t;
  long long nnz;
  CK(cudaMemcpy(&nnz, rowptr + nrows, 8, cudaMemcpyDefault));
  if (nnz < 0) return fail(MLEASE_ERR_INVALID, "rowptr[nrows] < 0");
  int* d_bad;
  if (int rc = t.get(&d_bad, 1, true)) return rc;
  const long long* d_rp; const int* d_ci; const float *d_v, *d_o; const double *d_m, *d_var, *d_cov;
  if (int rc = to_device(t, (const long long*)rowptr, (size_t)nrows + 1, &d_rp, st)) return rc;
  if (int rc = check_rowptr(st, nrows, d_rp, d_bad, "")) return rc;
  CK(cudaMemsetAsync(d_bad, 0, 4, st));
  if (int rc = to_device(t, colidx, (size_t)nnz, &d_ci, st)) return rc;
  if (int rc = to_device(t, vals, (size_t)nnz, &d_v, st)) return rc;
  if (int rc = to_device(t, offset, (size_t)nrows, &d_o, st)) return rc;
  if (int rc = to_device(t, model, (size_t)Dg + 1, &d_m, st)) return rc;
  if (int rc = to_device(t, var, (size_t)Dg + 1, &d_var, st)) return rc;
  if (int rc = to_device(t, cov, (size_t)(Dg + 1) * (Dg + 1), &d_cov, st)) return rc;
  double b;
  CK(cudaMemcpy(&b, model + Dg, 8, cudaMemcpyDefault));
  const double n = (double)num_click_replicates;
  const double ic = -std::log(n - 1 + n * std::exp(-b));   // as mlease_score
  const double gI = n * std::exp(-b) / (n - 1 + n * std::exp(-b));
  float* d_pred = pred;
  float* d_pv = pred_var;
  if (!is_device_ptr(pred)) { if (int rc = t.get(&d_pred, (size_t)nrows, false)) return rc; }
  if (!is_device_ptr(pred_var)) { if (int rc = t.get(&d_pv, (size_t)nrows, false)) return rc; }
  if (nrows > 0) {
    const long long blocks = std::min<long long>((nrows + 7) / 8, 132LL * 16);
    score_var_kernel<<<(int)blocks, 256, 0, st>>>(Dg, nrows, d_rp, d_ci, d_v, d_o, d_m, ic, gI, binary_feature, d_var, d_cov, d_pred, d_pv, d_bad);
    CK(cudaGetLastError());
  }
  int bad = 0;
  CK(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, st));
  if (d_pred != pred) CK(cudaMemcpyAsync(pred, d_pred, (size_t)nrows * 4, cudaMemcpyDeviceToHost, st));
  if (d_pv != pred_var) CK(cudaMemcpyAsync(pred_var, d_pv, (size_t)nrows * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return keyed_bad(bad);
}

int mlease_test_loglik(int32_t device, void* stream, int64_t nrows, const int32_t* response, const float* pred, const float* weight,
                       int64_t combiner_block, float* out_loglik, double* out_count) {
  if (!response || !pred || !out_loglik || !out_count || nrows <= 0) return fail(MLEASE_ERR_INVALID, "bad argument");
  if (int rc = open_device(device, nullptr)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  DevMem t;
  const int* d_r; const float* d_p; const float* d_w;
  if (int rc = to_device(t, (const int*)response, (size_t)nrows, &d_r, st)) return rc;
  if (int rc = to_device(t, pred, (size_t)nrows, &d_p, st)) return rc;
  if (int rc = to_device(t, weight, (size_t)nrows, &d_w, st)) return rc;
  const bool combine = combiner_block > 0;
  const long long blk = combine ? combiner_block : 4096;
  const long long nb = (nrows + blk - 1) / blk;
  float* d_ll; double *d_bs, *d_bc; int* d_bad;
  if (int rc = t.get(&d_ll, (size_t)nrows, false)) return rc;
  if (int rc = t.get(&d_bs, (size_t)nb, false)) return rc;
  if (int rc = t.get(&d_bc, (size_t)nb, false)) return rc;
  if (int rc = t.get(&d_bad, 1, false)) return rc;
  CK(cudaMemsetAsync(d_bad, 0, 4, st));
  CK(loglik_launch(nrows, d_r, d_p, d_w, blk, d_ll, d_bs, d_bc, d_bad, st));
  std::vector<double> bs(nb), bc(nb);
  int bad = 0;
  CK(cudaMemcpyAsync(bs.data(), d_bs, nb * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(bc.data(), d_bc, nb * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (bad) return fail(MLEASE_ERR_INVALID, "response should be 1,0 or -1!");
  double sum = 0, n = 0;
  for (long long b = 0; b < nb; b++) {
    sum += combine ? (double)(float)bs[b] : bs[b];   // combiner casts its partial sum to float (jobs/RegressionTestLoglik.java:197)
    n += bc[b];
  }
  *out_loglik = (float)(sum / n);                    // reducer (:173)
  *out_count = n;
  return 0;
}

}  // extern "C"

namespace mlease {

// mlease_score_keyed, and mlease_score_keyed_var when var_ptr is given: the variance lists are copied to the host and checked
// like the models, and every table, slice and copy of pred gets its variance twin.
static int score_keyed(int32_t device, void* stream, int32_t Dg, int32_t K, const int64_t* key_rowstart, const int64_t* rowptr,
                       const int32_t* colidx, const float* vals, const float* offset, int32_t L, const int64_t* model_ptr,
                       const int32_t* model_col, const float* model_val, const int64_t* var_ptr, const int32_t* var_col,
                       const float* var_val, const float* var_default, int32_t binary_feature, float* pred, float* pred_var,
                       const int64_t* cov_ptr = nullptr, const double* cov_val = nullptr, const float* lambda_map = nullptr) {
  if (Dg <= 0 || K < 0 || L <= 0 || !key_rowstart || !rowptr || !colidx || !vals || !model_ptr || !pred) return fail(MLEASE_ERR_INVALID, "bad argument");
  if ((var_ptr || cov_ptr) && (!var_default || !pred_var)) return fail(MLEASE_ERR_INVALID, "bad argument");
  if (int rc = open_device(device, nullptr)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  // host copies of the index arrays that decide the chunks and of the models, which are checked and give the intercept terms
  std::vector<long long> krs((size_t)K + 1);
  CK(cudaMemcpy(krs.data(), key_rowstart, krs.size() * 8, cudaMemcpyDefault));
  if (krs[0] != 0) return fail(MLEASE_ERR_INVALID, "key_rowstart[0] must be 0");
  for (int k = 0; k < K; k++) if (krs[k + 1] < krs[k]) return fail(MLEASE_ERR_INVALID, "key_rowstart must be non-decreasing");
  const long long nrows = krs[K], M = (long long)L * K;
  std::vector<long long> mp((size_t)M + 1);
  CK(cudaMemcpy(mp.data(), model_ptr, mp.size() * 8, cudaMemcpyDefault));
  if (mp[0] != 0) return fail(MLEASE_ERR_INVALID, "model_ptr[0] must be 0");
  for (long long m = 0; m < M; m++) if (mp[m + 1] < mp[m]) return fail(MLEASE_ERR_INVALID, "model_ptr must be non-decreasing");
  const long long nme = mp[M];
  if (nme > 0 && (!model_col || !model_val)) return fail(MLEASE_ERR_INVALID, "null model_col / model_val");
  std::vector<int> mc((size_t)nme);
  std::vector<float> mv((size_t)nme);
  if (nme > 0) {
    CK(cudaMemcpy(mc.data(), model_col, (size_t)nme * 4, cudaMemcpyDefault));
    CK(cudaMemcpy(mv.data(), model_val, (size_t)nme * 4, cudaMemcpyDefault));
  }
  // intercept term -log(0 + 1 exp(-b)) of LinearModel.eval with num_click_replicates = 1 (models/LinearModel.java:243-244), b = 0 for
  // a model without an intercept entry, the empty model included (jobs/ItemModelTest.java:189-197)
  std::vector<double> term((size_t)M);
  for (long long m = 0; m < M; m++) {
    for (long long e = mp[m]; e < mp[m + 1]; e++) {
      if (mc[e] < 0 || mc[e] > Dg) return fail(MLEASE_ERR_INVALID, "model_col out of range (model " + std::to_string(m) + ")");
      if (e > mp[m] && mc[e] <= mc[e - 1]) return fail(MLEASE_ERR_INVALID, "model_col must be strictly ascending within a model (model " + std::to_string(m) + ")");
    }
    const double b = (mp[m + 1] > mp[m] && mc[mp[m + 1] - 1] == Dg) ? (double)mv[mp[m + 1] - 1] : 0.0;
    term[m] = -std::log(1.0 - 1 + 1.0 * std::exp(-b));
  }
  KeyedVarHost vh;
  const KeyedVarHost* var = var_ptr ? &vh : nullptr;
  if (var) {
    // the same checks for the variance lists, and every variance finite and >= 0; vterm = the listed intercept variance, 0 when the
    // list does not name the intercept (as term), NaN for an empty list (no posterior for this model)
    vh.vp.resize((size_t)M + 1);
    vh.vdef.resize((size_t)M);
    CK(cudaMemcpy(vh.vp.data(), var_ptr, vh.vp.size() * 8, cudaMemcpyDefault));
    if (M > 0) CK(cudaMemcpy(vh.vdef.data(), var_default, (size_t)M * 4, cudaMemcpyDefault));
    if (vh.vp[0] != 0) return fail(MLEASE_ERR_INVALID, "var_ptr[0] must be 0");
    for (long long m = 0; m < M; m++) if (vh.vp[m + 1] < vh.vp[m]) return fail(MLEASE_ERR_INVALID, "var_ptr must be non-decreasing");
    const long long nve = vh.vp[M];
    if (nve > 0 && (!var_col || !var_val)) return fail(MLEASE_ERR_INVALID, "null var_col / var_val");
    vh.vc.resize((size_t)nve);
    vh.vv.resize((size_t)nve);
    if (nve > 0) {
      CK(cudaMemcpy(vh.vc.data(), var_col, (size_t)nve * 4, cudaMemcpyDefault));
      CK(cudaMemcpy(vh.vv.data(), var_val, (size_t)nve * 4, cudaMemcpyDefault));
    }
    vh.vterm.resize((size_t)M);
    for (long long m = 0; m < M; m++) {
      auto bad = [m](const char* what) { return fail(MLEASE_ERR_INVALID, std::string(what) + " (model " + std::to_string(m) + ")"); };
      if (!(std::isfinite(vh.vdef[m]) && vh.vdef[m] >= 0.f)) return bad("var_default must be finite and >= 0");
      for (long long e = vh.vp[m]; e < vh.vp[m + 1]; e++) {
        if (vh.vc[e] < 0 || vh.vc[e] > Dg) return bad("var_col out of range");
        if (e > vh.vp[m] && vh.vc[e] <= vh.vc[e - 1]) return bad("var_col must be strictly ascending within a model");
        if (!(std::isfinite(vh.vv[e]) && vh.vv[e] >= 0.f)) return bad("var_val must be finite and >= 0");
      }
      const long long e1 = vh.vp[m + 1];
      vh.vterm[m] = e1 == vh.vp[m] ? std::nan("") : vh.vc[e1 - 1] == Dg ? (double)vh.vv[e1 - 1] : 0.0;
    }
  }
  // mlease_score_keyed_cov: every block the packed lower triangle over its model's list, or empty; finite values; lambda_map >= 0
  std::vector<long long> cph;
  std::vector<double> cvh;
  std::vector<float> lmh, cdef;
  if (cov_ptr) {
    cph.resize((size_t)M + 1);
    cdef.resize((size_t)M);
    CK(cudaMemcpy(cph.data(), cov_ptr, cph.size() * 8, cudaMemcpyDefault));
    if (M > 0) CK(cudaMemcpy(cdef.data(), var_default, (size_t)M * 4, cudaMemcpyDefault));
    if (cph[0] != 0) return fail(MLEASE_ERR_INVALID, "cov_ptr[0] must be 0");
    for (long long m = 0; m < M; m++) {
      auto bad = [m](const std::string& what) { return fail(MLEASE_ERR_INVALID, what + " (model " + std::to_string(m) + ")"); };
      const long long n = mp[m + 1] - mp[m], sz = cph[m + 1] - cph[m];
      if (sz != 0 && sz != n * (n + 1) / 2)
        return bad("covariance block of " + std::to_string(sz) + " entries: a model listing " + std::to_string(n) + " columns needs " +
                   std::to_string(n * (n + 1) / 2) + ", or 0 for no posterior");
      if (!(std::isfinite(cdef[m]) && cdef[m] >= 0.f)) return bad("var_default must be finite and >= 0");
    }
    const long long nce = cph[M];
    if (nce > 0 && !cov_val) return fail(MLEASE_ERR_INVALID, "null cov_val");
    cvh.resize((size_t)nce);
    if (nce > 0) CK(cudaMemcpy(cvh.data(), cov_val, (size_t)nce * 8, cudaMemcpyDefault));
    for (long long e = 0; e < nce; e++)
      if (!std::isfinite(cvh[e])) return fail(MLEASE_ERR_INVALID, "cov_val must be finite (entry " + std::to_string(e) + ")");
    if (lambda_map) {
      lmh.resize((size_t)Dg);
      CK(cudaMemcpy(lmh.data(), lambda_map, (size_t)Dg * 4, cudaMemcpyDefault));
      for (float x : lmh) if (!(x >= 0.f) || !std::isfinite(x)) return fail(MLEASE_ERR_INVALID, "lambda_map: entries must be > 0, or 0 for a feature without one");
    }
  }
  if (nrows == 0) return 0;
  long long nnz;
  CK(cudaMemcpy(&nnz, rowptr + nrows, 8, cudaMemcpyDefault));
  if (nnz < 0) return fail(MLEASE_ERR_INVALID, "rowptr[nrows] < 0");
  const bool with_pv = var || cov_ptr;   // a pred_var output
  const bool pred_dev = is_device_ptr(pred), pred_var_dev = with_pv && is_device_ptr(pred_var);
  const size_t key_bytes = (size_t)Dg * (L >= 3 ? 4 : L) * sizeof(float) * (var ? 2 : 1);   // var: the variance table too
  // keys per table chunk within a budget
  auto chunk_keys = [&](size_t b) {
    return std::max<long long>(1, std::min<long long>(K, (long long)(std::min(SCORE_KEYED_TABLE_CAP, b / 4) / key_bytes)));
  };
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  const size_t budget = keyed_budget(free_b);
  // resident (one range) when the rows, the pred array and the model table fit the budget next to the models; else key ranges whose
  // rows, offsets and pred slice fit a quarter of the budget stream, each one table chunk
  const size_t models = ((size_t)M + 1) * 8 + (size_t)nme * 8 + (size_t)M * 8 + ((size_t)K + 1) * 8 + (var ? var->bytes() : 0) +
                        cph.size() * 8 + cvh.size() * 8 + lmh.size() * 4 + cdef.size() * 4;
  size_t rows = 0;
  if (!is_device_ptr(rowptr)) rows += ((size_t)nrows + 1) * 8;
  if (!is_device_ptr(colidx)) rows += (size_t)nnz * 4;
  if (!is_device_ptr(vals)) rows += (size_t)nnz * 4;
  if (offset && !is_device_ptr(offset)) rows += (size_t)nrows * 4;
  if (!pred_dev) rows += (size_t)L * nrows * 4;
  if (with_pv && !pred_var_dev) rows += (size_t)L * nrows * 4;
  std::vector<long long> ranges{0, K}, nnz_at{0, nnz}, row_at;   // nnz_at / row_at: rowptr / the row at the range bounds
  long long kpc = 0;
  const bool streamed = models + rows + std::min(SCORE_KEYED_TABLE_CAP, budget / 4) > budget;
  if (streamed) {
    std::vector<long long> off;   // rowptr at the key boundaries
    if (int rc = gather_rowptr(rowptr, krs, off)) return rc;
    // the ranges' entry counts come from these; every range's own rows are checked on the device before a kernel indexes by them
    if (off[0] < 0) return fail(MLEASE_ERR_INVALID, "rowptr[0] < 0");
    for (int k = 0; k < K; k++)
      if (off[k + 1] < off[k]) return fail(MLEASE_ERR_INVALID, "rowptr must never decrease (key " + std::to_string(k) + ")");
    const size_t pred_bytes = 4 * (size_t)L * (with_pv ? 2 : 1);   // a row's pred (and pred_var) slice
    kpc = chunk_keys(budget);
    ranges = plan_ranges(K, budget / 4, kpc, [&](long long k) {
      return (size_t)(krs[k + 1] - krs[k]) * (16 + 4 + pred_bytes) + (size_t)(off[k + 1] - off[k]) * 8;
    }, nullptr);
    nnz_at.clear();
    for (long long k : ranges) nnz_at.push_back(off[k]);
  }
  const int nr = (int)ranges.size() - 1;
  for (long long k : ranges) row_at.push_back(krs[k]);
  // the rows are copied straight from the caller's arrays: through the fit's pinned bounce buffers, streamed scoring of 4096 keys x
  // 1000 rows x 256 features took 2.3 s instead of 1.35 s (H100 80GB HBM3, 700 W)
  enum { RP, CI, V, O };
  RangeRing ring(st, {{rowptr, 8, RangeSrc::ROWPTR}, {colidx, 4, RangeSrc::ENTRY}, {vals, 4, RangeSrc::ENTRY}, {offset, 4, RangeSrc::ROW}},
                 row_at, nnz_at, 0, Dg, streamed, false);
  long long max_rows = 0;
  for (int c = 0; c < nr; c++) max_rows = std::max(max_rows, row_at[c + 1] - row_at[c]);
  DevMem t;
  const long long *d_krs, *d_mp; const int* d_mc; const float* d_mv; const double* d_term;
  if (int rc = to_device(t, (const long long*)krs.data(), krs.size(), &d_krs, st)) return rc;
  if (int rc = to_device(t, (const long long*)mp.data(), mp.size(), &d_mp, st)) return rc;
  if (int rc = to_device(t, (const int*)mc.data(), mc.size(), &d_mc, st)) return rc;
  if (int rc = to_device(t, (const float*)mv.data(), mv.size(), &d_mv, st)) return rc;
  if (int rc = to_device(t, (const double*)term.data(), term.size(), &d_term, st)) return rc;
  KeyedVar dvar;
  if (var) { if (int rc = var->upload(t, dvar, st)) return rc; }
  // a resident call writes straight into device pred / pred_var; otherwise each range's slice is copied back
  float* d_pred = pred;
  if (streamed || !pred_dev) { if (int rc = t.get(&d_pred, (size_t)L * max_rows, false)) return rc; }
  if (var) {
    dvar.pred_var = pred_var;
    if (streamed || !pred_var_dev) { if (int rc = t.get(&dvar.pred_var, (size_t)L * max_rows, false)) return rc; }
  }
  KeyedCov dcov;
  if (cov_ptr) {
    if (int rc = to_device(t, (const long long*)cph.data(), cph.size(), &dcov.cp, st)) return rc;
    if (int rc = to_device(t, (const double*)cvh.data(), cvh.size(), &dcov.cv, st)) return rc;
    if (int rc = to_device(t, (const float*)cdef.data(), cdef.size(), &dcov.vdef, st)) return rc;
    if (lambda_map) { if (int rc = to_device(t, (const float*)lmh.data(), lmh.size(), &dcov.lm, st)) return rc; }
    dcov.pred_var = pred_var;
    if (streamed || !pred_var_dev) { if (int rc = t.get(&dcov.pred_var, (size_t)L * max_rows, false)) return rc; }
  }
  float* const d_pred_var = var ? dvar.pred_var : dcov.pred_var;
  int* d_bad;   // [0] the row checks of the kernels, [1] check_rowptr's flag
  if (int rc = t.get(&d_bad, 2, false)) return rc;
  CK(cudaMemsetAsync(d_bad, 0, 4, st));
  if (int rc = ring.open()) return rc;
  float* d_table = nullptr;
  std::vector<long long> bounds{0};
  for (int c = 0; c < nr; c++) {
    const void* v[4];
    if (int rc = ring.view(c, v)) return rc;
    const long long r0 = row_at[c], n = row_at[c + 1] - r0, z0 = nnz_at[c], nz = nnz_at[c + 1] - z0;
    DevMem rt;   // the range's device copies of host input
    const long long* rp; const int* ci; const float *vv, *o;
    if (int rc = to_device(rt, (const long long*)v[RP], (size_t)n + 1, &rp, st)) return rc;
    if (int rc = to_device(rt, (const int*)v[CI], (size_t)nz, &ci, st)) return rc;
    if (int rc = to_device(rt, (const float*)v[V], (size_t)nz, &vv, st)) return rc;
    if (int rc = to_device(rt, (const float*)v[O], (size_t)n, &o, st)) return rc;
    if (z0) rebase_rowptr(st, n, rp, z0, (long long*)rp);   // in place: a range after the first is in a ring slot
    if (int rc = check_rowptr(st, n, rp, d_bad + 1, "keys " + std::to_string(ranges[c]) + ".." + std::to_string(ranges[c + 1] - 1) + ": "))
      return rc;
    if (!d_table) {   // a resident call's table chunks fit the memory left after its upload
      if (!ring.staged()) { CK(cudaMemGetInfo(&free_b, &total_b)); kpc = chunk_keys(keyed_budget(free_b)); }
      if (int rc = t.get(&d_table, (size_t)kpc * key_bytes / sizeof(float), false)) return rc;
      if (var) dvar.vtable = d_table + (size_t)kpc * key_bytes / 2 / sizeof(float);
    }
    const std::vector<long long> chunks = plan_ranges(ranges[c + 1] - ranges[c], SIZE_MAX, kpc, nullptr, nullptr);
    for (size_t j = 1; j < chunks.size(); j++) {
      const int k0 = (int)(ranges[c] + chunks[j - 1]), k1 = (int)(ranges[c] + chunks[j]);
      bounds.push_back(k1);
      if (krs[k1] == krs[k0]) continue;
      for (int l0 = 0; l0 < L; l0 += 4) {
        KeyedCov cg = dcov;   // the group's models: blocks, defaults and pred_var rows from l0 on
        if (cg) { cg.cp += (size_t)l0 * K; cg.vdef += (size_t)l0 * K; cg.pred_var += (size_t)l0 * n; }
        CK(score_keyed_chunk(Dg, K, k0, k1, krs[k0], krs[k1], d_krs, rp, ci, vv, o, std::min(4, L - l0), d_mp + (size_t)l0 * K, d_mc, d_mv,
                             d_term + (size_t)l0 * K, binary_feature, n, r0, d_table, d_pred + (size_t)l0 * n, d_bad, dvar.at(l0, K, n), cg, st));
      }
    }
    if (int rc = ring.done(c)) return rc;
    if (int rc = ring.start(c + 1)) return rc;
    if (n > 0 && d_pred != pred) CK(cudaMemcpy2DAsync(pred + r0, (size_t)nrows * 4, d_pred, (size_t)n * 4, (size_t)n * 4, L, cudaMemcpyDefault, st));
    if (n > 0 && with_pv && d_pred_var != pred_var)
      CK(cudaMemcpy2DAsync(pred_var + r0, (size_t)nrows * 4, d_pred_var, (size_t)n * 4, (size_t)n * 4, L, cudaMemcpyDefault, st));
  }
  int bad = 0;
  CK(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  keyed_record(bounds, ring.staged(), ring.stage_ms, ring.wait_ms);
  return keyed_bad(bad);
}

}  // namespace mlease

extern "C" {

int mlease_score_keyed(int32_t device, void* stream, int32_t Dg, int32_t K, const int64_t* key_rowstart, const int64_t* rowptr,
                       const int32_t* colidx, const float* vals, const float* offset, int32_t L, const int64_t* model_ptr,
                       const int32_t* model_col, const float* model_val, int32_t binary_feature, float* pred) {
  return score_keyed(device, stream, Dg, K, key_rowstart, rowptr, colidx, vals, offset, L, model_ptr, model_col, model_val, nullptr, nullptr,
                     nullptr, nullptr, binary_feature, pred, nullptr);
}

int mlease_score_keyed_var(int32_t device, void* stream, int32_t Dg, int32_t K, const int64_t* key_rowstart, const int64_t* rowptr,
                           const int32_t* colidx, const float* vals, const float* offset, int32_t G, const int64_t* model_ptr,
                           const int32_t* model_col, const float* model_val, const int64_t* var_ptr, const int32_t* var_col,
                           const float* var_val, const float* var_default, int32_t binary_feature, float* pred, float* pred_var) {
  if (!var_ptr) return fail(MLEASE_ERR_INVALID, "bad argument");
  return score_keyed(device, stream, Dg, K, key_rowstart, rowptr, colidx, vals, offset, G, model_ptr, model_col, model_val, var_ptr, var_col,
                     var_val, var_default, binary_feature, pred, pred_var);
}

int mlease_score_keyed_cov(int32_t device, void* stream, int32_t Dg, int32_t K, const int64_t* key_rowstart, const int64_t* rowptr,
                           const int32_t* colidx, const float* vals, const float* offset, int32_t G, const int64_t* model_ptr,
                           const int32_t* model_col, const float* model_val, const int64_t* cov_ptr, const double* cov_val,
                           const float* lambda_map, const float* var_default, int32_t binary_feature, float* pred, float* pred_var) {
  if (!cov_ptr) return fail(MLEASE_ERR_INVALID, "bad argument");
  return score_keyed(device, stream, Dg, K, key_rowstart, rowptr, colidx, vals, offset, G, model_ptr, model_col, model_val, nullptr, nullptr,
                     nullptr, var_default, binary_feature, pred, pred_var, cov_ptr, cov_val, lambda_map);
}

int mlease_test_loglik_keyed(int32_t device, void* stream, int64_t n, const int32_t* entry_key, const int32_t* entry_group,
                             const int32_t* response, const float* weight, const float* pred, int32_t num_keys, float* out_loglik,
                             double* out_count) {
  if (n <= 0 || n > INT32_MAX || num_keys <= 0 || !entry_key || !entry_group || !response || !pred || !out_loglik || !out_count)
    return fail(MLEASE_ERR_INVALID, "bad argument");
  if (int rc = open_device(device, nullptr)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  DevMem t;
  const int *d_k, *d_g, *d_r; const float *d_p, *d_w;
  if (int rc = to_device(t, (const int*)entry_key, (size_t)n, &d_k, st)) return rc;
  if (int rc = to_device(t, (const int*)entry_group, (size_t)n, &d_g, st)) return rc;
  if (int rc = to_device(t, (const int*)response, (size_t)n, &d_r, st)) return rc;
  if (int rc = to_device(t, pred, (size_t)n, &d_p, st)) return rc;
  if (int rc = to_device(t, weight, (size_t)n, &d_w, st)) return rc;
  int last_group = 0;
  CK(cudaMemcpy(&last_group, entry_group + n - 1, 4, cudaMemcpyDefault));
  if (last_group < 0) return fail(MLEASE_ERR_INVALID, "entry_group must be non-decreasing and >= 0");
  const long long ngroups = (long long)last_group + 1;
  float* d_ll; long long *d_skey, *d_skey_s; int *d_idx, *d_idx_s, *d_bad; float* d_oll; double* d_ocnt; char* d_tmp;
  size_t tmp_bytes = 0;
  CK(loglik_keyed_launch(n, num_keys, ngroups, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                         nullptr, &tmp_bytes, nullptr, nullptr, nullptr, st));
  if (int rc = t.get(&d_ll, (size_t)n, false)) return rc;
  if (int rc = t.get(&d_skey, (size_t)n, false)) return rc;
  if (int rc = t.get(&d_skey_s, (size_t)n, false)) return rc;
  if (int rc = t.get(&d_idx, (size_t)n, false)) return rc;
  if (int rc = t.get(&d_idx_s, (size_t)n, false)) return rc;
  if (int rc = t.get(&d_bad, 1, false)) return rc;
  if (int rc = t.get(&d_oll, (size_t)num_keys, false)) return rc;
  if (int rc = t.get(&d_ocnt, (size_t)num_keys, false)) return rc;
  if (int rc = t.get(&d_tmp, tmp_bytes, false)) return rc;
  CK(cudaMemsetAsync(d_bad, 0, 4, st));
  CK(loglik_keyed_launch(n, num_keys, ngroups, d_k, d_g, d_r, d_w, d_p, d_ll, d_skey, d_skey_s, d_idx, d_idx_s, d_tmp, &tmp_bytes, d_bad,
                         d_oll, d_ocnt, st));
  int bad = 0;
  CK(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(out_loglik, d_oll, (size_t)num_keys * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(out_count, d_ocnt, (size_t)num_keys * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (bad & 1) return fail(MLEASE_ERR_INVALID, "response should be 1,0 or -1!");   // jobs/ItemModelTestLoglik.java:74-77
  if (bad & 2) return fail(MLEASE_ERR_INVALID, "entry_key out of range [0, num_keys)");
  if (bad & 4) return fail(MLEASE_ERR_INVALID, "entry_group must be non-decreasing and >= 0");
  return 0;
}

}  // extern "C"
