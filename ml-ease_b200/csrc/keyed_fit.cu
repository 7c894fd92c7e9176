// keyed_fit.cu -- K independent fits per prior over one upload of the rows: RegressionNaiveTrain (mlease_naive_train,
// mlease_naive_train_dense) and ItemModelTrain (mlease_item_model_train), both with sparse outputs (mlease_*_train_sparse), and
// ItemModelTrain with each key's full posterior covariance (mlease_item_model_train_cov) or under per-key prior lists
// (mlease_item_model_train_prior).
#include <cub/block/block_scan.cuh>

#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "host.cuh"

using namespace mlease;

namespace {
// beta = 0, prior mean m and precision q of every problem; intercept_mean (NULL or [nprob]): problem b's prior mean at the
// intercept (column Dt - 1) instead of m's
__global__ void naive_init_kernel(const Problem* probs, const double* m, const double* q, const double* intercept_mean) {
  const Problem& pb = probs[blockIdx.x];
  for (int k = threadIdx.x; k < pb.ldx; k += blockDim.x) {
    pb.beta[k] = 0.0; pb.q[k] = q[k];
    pb.m[k] = (intercept_mean && k == pb.Dt - 1) ? intercept_mean[blockIdx.x] : m[k];
  }
}
// out[b][k] = beta (hdiag: the Hessian diagonal g_t that postvar_diag left) of problem b, 0 where mask[b][k] == 0
__global__ void gather_beta_kernel(const Problem* probs, int Dt, double* out, const unsigned char* mask, int hdiag) {
  const Problem& pb = probs[blockIdx.x];
  const double* v = hdiag ? pb.g_t : pb.beta;
  for (int k = threadIdx.x; k < Dt; k += blockDim.x)
    out[(size_t)blockIdx.x * Dt + k] = (!mask || mask[(size_t)blockIdx.x * Dt + k]) ? v[k] : 0.0;
}
// mask[b][c] = 1 for every feature listed in some row of problem b (+ the intercept)
__global__ void naive_present_kernel(const Problem* probs, int Dt, int has_bias, unsigned char* mask) {
  const Problem& pb = probs[blockIdx.x];
  unsigned char* mk = mask + (size_t)blockIdx.x * Dt;
  const long long j0 = pb.rowptr[0], j1 = pb.rowptr[pb.n];
  for (long long j = j0 + threadIdx.x; j < j1; j += blockDim.x) mk[pb.colidx[j]] = 1;
  if (threadIdx.x == 0 && has_bias) mk[Dt - 1] = 1;
}
// naive_init_kernel for problems in their keys' own column spaces: column c < Dk of problem b is global column cols[span[2b] + c]
// (Dk = span[2b + 1] - span[2b]) and takes its q and m from the global [ldx] vectors; the intercept (column Dt - 1) takes the global
// column Dg's (or intercept_mean[b]); the padding between them and beyond Dt gets q = 1, m = 0, which no row touches
__global__ void local_init_kernel(const Problem* probs, const double* m, const double* q, const double* intercept_mean, const int* cols,
                                  const long long* span, int Dg) {
  const Problem& pb = probs[blockIdx.x];
  const int* c = cols + span[2 * blockIdx.x];
  const int dk = (int)(span[2 * blockIdx.x + 1] - span[2 * blockIdx.x]);
  for (int k = threadIdx.x; k < pb.ldx; k += blockDim.x) {
    pb.beta[k] = 0.0;
    if (k < dk) { pb.q[k] = q[c[k]]; pb.m[k] = m[c[k]]; }
    else if (k == pb.Dt - 1) { pb.q[k] = q[Dg]; pb.m[k] = intercept_mean ? intercept_mean[blockIdx.x] : m[Dg]; }
    else { pb.q[k] = 1.0; pb.m[k] = 0.0; }
  }
}
// mask[b][c] = 1 for every column the rows rows[2b] .. rows[2b + 1] of rp / ci list (+ the intercept, column Dt - 1); count[b] = the
// mask's ones.  The keys of a sparse chunk that have no column list (sparse_gather_kernel compacts the same mask rows).
__global__ void span_present_kernel(const long long* rp, const int* ci, const long long* rows, int Dt, int has_bias, unsigned char* mask,
                                    int* count) {
  unsigned char* mk = mask + (size_t)blockIdx.x * Dt;
  const long long j0 = rp[rows[2 * blockIdx.x]], j1 = rp[rows[2 * blockIdx.x + 1]];
  for (long long j = j0 + threadIdx.x; j < j1; j += blockDim.x) mk[ci[j]] = 1;
  if (threadIdx.x == 0 && has_bias) mk[Dt - 1] = 1;
  __syncthreads();
  __shared__ int total;
  if (threadIdx.x == 0) total = 0;
  __syncthreads();
  int c = 0;
  for (int k = threadIdx.x; k < Dt; k += blockDim.x) c += mk[k];
  atomicAdd(&total, c);
  __syncthreads();
  if (threadIdx.x == 0) count[blockIdx.x] = total;
}
// Where problem b of a batch writes its list in a chunk's slab: entries dst .. of out.  dk >= 0: the list is cols[s0 .. s0 + dk)
// (then the intercept); dk < 0: no list, the ones of mask row mrow in column order (the intercept's included).  Per-key priors: the
// key's prior list is entries p0 .. p0 + pn of its range's PriorDev (pn = 0 without one)
struct GatherJob { long long dst, s0; int dk, mrow; long long p0; int pn; };
// A key range's per-key prior lists on the device (mlease_item_model_train_prior), entries numbered from the range's first key's;
// col NULL: the call has none
struct PriorDev { const int* col; const double* mean; const double* var; };
constexpr int GATHER_THREADS = 256;
// the first index i of the ascending a[0 .. n) with a[i] >= x
__device__ __forceinline__ int lower_index(const int* a, int n, int x) {
  int lo = 0, hi = n;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[mid] < x) lo = mid + 1; else hi = mid; }
  return lo;
}
// the index of x in the ascending a[0 .. n), or -1
__device__ __forceinline__ int find_index(const int* a, int n, int x) {
  const int i = lower_index(a, n, x);
  return i < n && a[i] == x ? i : -1;
}
// One problem per block: beta (hdiag: 1 / g_t, IEEE fp64 like the host's 1.0 / x) at the problem's listed columns into out, and the
// global column ids into out_col (NULL: already written).  A local problem (local = 1) holds its list's columns at 0 .. dk - 1 and
// the intercept at Dt - 1; a global-width one holds global column c at c.  Per-key priors (pr.col): the list is the union of the
// listed columns and the key's prior-only columns (prior entries its rows do not list), ascending, then the intercept; a prior-only
// column takes its entry's mean (hdiag: its variance, or 1 / q[c] where that is 0), never a value of the fit.
__global__ void sparse_gather_kernel(const Problem* probs, const GatherJob* jobs, const int* cols, const unsigned char* mask, int local,
                                     int Dg, int has_bias, int hdiag, double* out, int* out_col, PriorDev pr, const double* q) {
  using Scan = cub::BlockScan<int, GATHER_THREADS>;
  __shared__ typename Scan::TempStorage scan;
  __shared__ int carry;
  const Problem& pb = probs[blockIdx.x];
  const GatherJob jb = jobs[blockIdx.x];
  const double* v = hdiag ? pb.g_t : pb.beta;
  auto put = [&](long long e, int src, int col) {
    out[jb.dst + e] = hdiag ? __ddiv_rn(1.0, v[src]) : v[src];
    if (out_col) out_col[jb.dst + e] = col;
  };
  const int pn = pr.col ? jb.pn : 0;
  const int* pc = pn ? pr.col + jb.p0 : nullptr;
  auto put_prior = [&](long long e, int i, int col) {   // prior entry i of the key, a prior-only column
    const double pv = pr.var[jb.p0 + i];
    out[jb.dst + e] = hdiag ? (pv > 0.0 ? pv : __ddiv_rn(1.0, q[col])) : pr.mean[jb.p0 + i];
    if (out_col) out_col[jb.dst + e] = col;
  };
  if (jb.dk >= 0) {
    const int* c = cols + jb.s0;
    if (!pn) {
      for (int i = threadIdx.x; i < jb.dk; i += blockDim.x) put(i, local ? i : c[i], c[i]);
      if (threadIdx.x == 0 && has_bias) put(jb.dk, pb.Dt - 1, Dg);
      return;
    }
    // listed column i: after i listed columns and the prior-only entries below c[i] -- the prior entries below it (lb) less those
    // that are listed (a scan over the listed columns that have an entry)
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int t0 = 0; t0 < jb.dk; t0 += GATHER_THREADS) {
      const int i = t0 + threadIdx.x;
      int lb = 0, h = 0;
      if (i < jb.dk) { lb = lower_index(pc, pn, c[i]); h = lb < pn && pc[lb] == c[i]; }
      int pos, tile;
      Scan(scan).ExclusiveSum(h, pos, tile);
      if (i < jb.dk) put(i + lb - (carry + pos), local ? i : c[i], c[i]);
      __syncthreads();
      if (threadIdx.x == 0) carry += tile;
      __syncthreads();
    }
    // prior-only entry: after the prior-only entries before it and the listed columns below it
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int t0 = 0; t0 < pn; t0 += GATHER_THREADS) {
      const int i = t0 + threadIdx.x;
      int lb = 0, f = 0;
      if (i < pn && pc[i] != Dg) { lb = lower_index(c, jb.dk, pc[i]); f = !(lb < jb.dk && c[lb] == pc[i]); }
      int pos, tile;
      Scan(scan).ExclusiveSum(f, pos, tile);
      if (f) put_prior(carry + pos + lb, i, pc[i]);
      __syncthreads();
      if (threadIdx.x == 0) carry += tile;
      __syncthreads();
    }
    if (threadIdx.x == 0 && has_bias) put(jb.dk + carry, pb.Dt - 1, Dg);
    return;
  }
  const unsigned char* mk = mask + (size_t)jb.mrow * pb.Dt;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int t0 = 0; t0 < pb.Dt; t0 += GATHER_THREADS) {
    const int k = t0 + threadIdx.x;
    int f = k < pb.Dt ? mk[k] : 0, e = -1;
    if (!f && pn && k < Dg) { e = find_index(pc, pn, k); f = e >= 0; }
    int pos, tile;
    Scan(scan).ExclusiveSum(f, pos, tile);
    if (f) { if (e < 0) put(carry + pos, k, k); else put_prior(carry + pos, e, k); }
    __syncthreads();
    if (threadIdx.x == 0) carry += tile;
    __syncthreads();
  }
}
// naive_init_kernel (span NULL: global width, mask[b] the columns the rows list) and local_init_kernel (cols / span) under per-key
// priors: each column as they set it, then a column the rows list (local: the list's columns and the intercept) that has an entry
// in its key's prior list (a binary search of jobs[b]'s) takes the entry's mean, and the precision 1 / var when var > 0.  Prior-only
// columns, unlisted columns and the padding keep their q and m.
__global__ void prior_init_kernel(const Problem* probs, const double* m, const double* q, const double* intercept_mean, const int* cols,
                                  const long long* span, const unsigned char* mask, int Dg, const GatherJob* jobs, PriorDev pr) {
  const Problem& pb = probs[blockIdx.x];
  const GatherJob jb = jobs[blockIdx.x];
  const int* pc = pr.col + jb.p0;
  const int* c = span ? cols + span[2 * blockIdx.x] : nullptr;
  const int dk = span ? (int)(span[2 * blockIdx.x + 1] - span[2 * blockIdx.x]) : 0;
  for (int k = threadIdx.x; k < pb.ldx; k += blockDim.x) {
    pb.beta[k] = 0.0;
    int g = -1;   // the global column of k where the rows list it
    double qk, mk;
    if (span) {
      if (k < dk) { g = c[k]; qk = q[g]; mk = m[g]; }
      else if (k == pb.Dt - 1) { g = Dg; qk = q[Dg]; mk = intercept_mean ? intercept_mean[blockIdx.x] : m[Dg]; }
      else { qk = 1.0; mk = 0.0; }
    } else {
      qk = q[k]; mk = (intercept_mean && k == pb.Dt - 1) ? intercept_mean[blockIdx.x] : m[k];
      if (k < pb.Dt && mask[(size_t)blockIdx.x * pb.Dt + k]) g = k;
    }
    if (g >= 0 && jb.pn) {
      const int e = find_index(pc, jb.pn, g);
      if (e >= 0) {
        mk = pr.mean[jb.p0 + e];
        const double v = pr.var[jb.p0 + e];
        if (v > 0.0) qk = 1.0 / v;
      }
    }
    pb.q[k] = qk; pb.m[k] = mk;
  }
}
// count[b] = the prior-only columns of key b (jobs[b]): the entries of its prior list that its rows do not list -- not in its column
// list (dk >= 0) or 0 in its row of mask; the intercept is always listed
__global__ void prior_only_count_kernel(const GatherJob* jobs, const int* cols, const unsigned char* mask, int Dt, int Dg, PriorDev pr,
                                        int* count) {
  const GatherJob jb = jobs[blockIdx.x];
  __shared__ int total;
  if (threadIdx.x == 0) total = 0;
  __syncthreads();
  int n = 0;
  for (int i = threadIdx.x; i < jb.pn; i += blockDim.x) {
    const int g = pr.col[jb.p0 + i];
    if (g == Dg) continue;
    n += (jb.dk >= 0 ? find_index(cols + jb.s0, jb.dk, g) >= 0 : mask[(size_t)jb.mrow * Dt + g] != 0) ? 0 : 1;
  }
  atomicAdd(&total, n);
  __syncthreads();
  if (threadIdx.x == 0) count[blockIdx.x] = total;
}
// The checks of the prior lists of nk keys (offs[i] .. offs[i + 1] of col / mean / var: key kbase + i): a column outside [0, Dg],
// columns not strictly ascending, a mean that is not finite, a variance that is negative or not finite.  bad = the smallest
// (key << 3 | reason) found (reasons 1 .. 4 in that order), left as is when all pass; nonint[i] = key i's entries less its intercept's.
__global__ void prior_check_kernel(const long long* offs, int kbase, const int* col, const double* mean, const double* var, int Dg,
                                   unsigned long long* bad, int* nonint) {
  const long long e0 = offs[blockIdx.x], e1 = offs[blockIdx.x + 1];
  for (long long e = e0 + threadIdx.x; e < e1; e += blockDim.x) {
    const int c = col[e];
    int why = 0;
    if (c < 0 || c > Dg) why = 1;
    else if (e > e0 && col[e - 1] >= c) why = 2;
    else if (!isfinite(mean[e])) why = 3;
    else if (!(var[e] >= 0.0) || isinf(var[e])) why = 4;
    if (why) atomicMin(bad, ((unsigned long long)(kbase + blockIdx.x) << 3) | (unsigned long long)why);
  }
  if (threadIdx.x == 0) nonint[blockIdx.x] = (int)(e1 - e0) - (e1 > e0 && col[e1 - 1] == Dg ? 1 : 0);
}
// Where problem b of a batch writes its posterior in a chunk's slab: its list of n entries starts at entry dst of the variances (and
// of the column ids the model gather wrote), the packed lower triangle of its covariance at entry cdst of the covariance slab (cdst
// < 0: variances only)
struct CovJob { long long dst, cdst; int n; };
// One problem per block, from the explicit inverse Hinv = Sigma of its Hessian: the variances diag(Sigma) over its list and (cdst >= 0)
// the lower triangle of Sigma over it, row-major: entry (a, b), a >= b, at cdst + a(a+1)/2 + b.  A local problem's entry a is its
// column a, the last entry (the intercept) its column Dt - 1; a global-width problem's entry a is the global column col names.
__global__ void cov_gather_kernel(const Problem* probs, const CovJob* jobs, int local, const int* col, double* var, double* cov) {
  const Problem& pb = probs[blockIdx.x];
  const CovJob jb = jobs[blockIdx.x];
  auto hcol = [&](int a) -> size_t { return local ? (a < jb.n - 1 ? a : pb.Dt - 1) : col[jb.dst + a]; };
  for (int a = threadIdx.x; a < jb.n; a += blockDim.x) { const size_t c = hcol(a); var[jb.dst + a] = pb.Hinv[c * pb.ldh + c]; }
  if (jb.cdst < 0) return;
  const long long tot = (long long)jb.n * (jb.n + 1) / 2;
  for (long long e = threadIdx.x; e < tot; e += blockDim.x) {
    int a = (int)((sqrt(8.0 * (double)e + 1.0) - 1.0) * 0.5);   // the row of entry e, corrected for rounding
    while ((long long)a * (a + 1) / 2 > e) a--;
    while ((long long)(a + 1) * (a + 2) / 2 <= e) a++;
    const int b = (int)(e - (long long)a * (a + 1) / 2);
    cov[jb.cdst + e] = pb.Hinv[hcol(a) * pb.ldh + hcol(b)];
  }
}

// count[0] += the problems whose factorisation found a non-positive pivot (K3 leaves Ctrl::fail = 1)
__global__ void cov_fail_kernel(const Problem* probs, int nprob, int* count) {
  int c = 0;
  for (int b = threadIdx.x; b < nprob; b += blockDim.x) c += probs[b].ctrl->fail == 1 ? 1 : 0;
  if (c) atomicAdd(count, c);
}

// One prior of a keyed fit: precision q and mean m of every coefficient ([ldx], the intercept at Dg, 1 / 0 on the padding)
struct KeyedPrior { std::vector<double> q, m; };

// The sparse output of mlease_*_train_sparse: key k's list is entries key_ptr[k] .. key_ptr[k + 1] of col, prior p's values at
// model[p * cap + e] (and var).  NULL in KeyedFit: the dense [prior][K][Dt] arrays.
struct SparseOut { int64_t cap; int64_t* key_ptr; int32_t* col; };
// The covariance output of mlease_item_model_train_cov: key k's block is entries ptr[k] .. ptr[k + 1] of val, prior p's at
// val[p * cap + e]; val NULL: variances only (ptr unused)
struct CovOut { int64_t cap; int64_t* ptr; double* val; };
// The per-key priors of mlease_item_model_train_prior, host-or-device as the caller passed them: key k's entries are ptr[k] ..
// ptr[k + 1] of col (ascending, Dg = the intercept), mean and var (0: the column's usual variance)
struct KeyPriorIn { const int64_t* ptr; const int32_t* col; const double* mean; const double* var; };
// prior entries checked per pass of prior_check_kernel (a larger key is checked on its own), 20 B each on the device
constexpr size_t PRIOR_CHECK_BYTES = size_t(20) << 24;
// the widest system whose explicit inverse K3 forms (wider ones keep it factored, cholesky_factored_direction)
constexpr int COV_MAX_WIDTH = 2048;
// solve_batch of a covariance call whose batch would be matrix-free: solve_group splits it
constexpr int SPLIT_BATCH = -1;
// A chunk's sparse results on the device: the lists of its fitted keys, contiguous in key order, [prior][n] values and n column ids.
// off / len (by key - k0): a key's entries in the slab; mrow: its row of mask (-1: it has a column list).  Covariance calls: [prior]
// [ncov] packed blocks, coff a key's block
struct Slab {
  int k0 = 0;
  long long n = 0, ncov = 0;
  double* model = nullptr; double* var = nullptr; int* col = nullptr; double* cov = nullptr;
  unsigned char* mask = nullptr;
  std::vector<long long> off, len, coff;
  std::vector<int> mrow;
};

// K independent fits per prior, processed in lockstep chunks of keys: the rows are uploaded ONCE and serve every prior (the reference
// fans each record out once per reducer through the shuffle, jobs/RegressionNaiveTrain.java:228-241, jobs/ItemModelTrain.java:256-258).
// Key k owns rows [key_rowstart[k], key_rowstart[k+1]); keys with fewer than data_size_threshold rows, or none, are skipped (model 0).
// intercept_mean (host, [K] or NULL): key k's prior mean of the intercept, replacing the priors' m[Dg].  out_model / out_var (NULL = no
// variance) are [prior][K][Dt]; var = 1 / (q + sum_i w_i p_i (1-p_i) x_ik^2) at the fit, hence 1/q for a feature the key's rows do not list.
// the input checks of keyed_fit, then the device (the callers read their prior arrays between the two)
int keyed_fit_check(int32_t device, int32_t Dg, const int64_t* rowptr, const int32_t* colidx, int64_t ldx_in, int32_t binary_feature, int* num_sms) {
  const bool csr = rowptr != nullptr;
  if (csr && !colidx) return fail(MLEASE_ERR_INVALID, "null colidx");
  if (!csr && binary_feature) return fail(MLEASE_ERR_INVALID, "binary.feature needs CSR input (every listed feature counts as 1)");
  if (!csr && ldx_in < Dg) return fail(MLEASE_ERR_INVALID, "ldx < num_features");
  return open_device(device, num_sms);
}

// The device arrays the problems of a chunk point into; element 0 of the row arrays is row row0 of the call (its range's first)
struct ChunkRows {
  long long row0 = 0;
  signed char* y = nullptr; float* w = nullptr; float* o = nullptr;
  float* X = nullptr;
  const long long* rp = nullptr; const int* ci = nullptr; float* v = nullptr;   // rp: offsets into ci / v
  int csr_unique = 0;
  const KeyCols* kc = nullptr;   // the column spaces of keys kbase.. (CSR calls wider than 32 columns), else NULL
  int kbase = 0;
  PriorDev pd{nullptr, nullptr, nullptr};   // the range's per-key prior lists, entries from prior_ptr[pbase_key] on
  long long pbase = 0;                      // prior_ptr at the range's first key
};

// One keyed fit call, over the key ranges of the keyed pipeline (key_ranges.cu).  Resident (the whole upload and the first chunk's
// state fit the budget): one range, every row uploaded once, then solved in chunks of keys.  Streamed: contiguous key ranges, each
// holding its own rows next to its solver state within a quarter of the budget and solved as one chunk, the rows of range c+1
// staged through the ring while range c is solved.  Each range passes the row checks before any of its rows is read, so rows
// sorted and unique (csr_unique) is a property of the range.  Neither mode changes what a key's fit computes: a streamed range
// solves exactly as a resident call on that range's keys alone.  The mode and the plan are host arithmetic on the shapes, the CSR
// offsets at the key boundaries and the free memory, never on the values.
// Column spaces (CSR): a key whose Dk distinct listed columns give round_up(Dk + 1, 32) < round_up(Dg + 1, 32) is solved in its own
// space of Dt_k = round_up(Dk + 1, 32) columns: its Dk listed features in ascending order, padding (q = 1, m = 0, no row touches it,
// so beta stays 0 there) and the intercept at Dt_k - 1.  Every other key runs at the global width Dt = Dg + 1.  The choice and the
// shape depend on the key's own rows alone, never on which keys share its call, chunk or streamed range; each chunk runs one batch
// per width.  Dense sink: outputs are scattered back to the global columns, a feature the key does not list keeping 0 in the model
// and 1/q in the variance.  Sparse sink (sp): each chunk's lists are gathered on the device into a slab and copied out once per prior.
// Covariance (cv, with sp and out_var): after each prior's fit, every batch assembles its problems' exact fp64 Hessians into Lc, K3
// factorises and inverts them, and the variances (and packed covariance blocks) over each key's list are gathered from Hinv.
struct KeyedFit {
  int num_sms; cudaStream_t st; int32_t K, Dg; const int64_t* key_rowstart; const int64_t* rowptr; const int32_t* colidx; const float* vals;
  int64_t ldx_in; const int32_t* response; const float* weight; const float* offset; bool has_intercept; int32_t data_size_threshold;
  int32_t binary_feature; const std::vector<KeyedPrior>& priors; const double* intercept_mean; double* out_model; double* out_var;
  int32_t* skipped;
  const SparseOut* sp;                    // the output sink: NULL = dense out_model / out_var; else the lists (out_model / out_var their values)
  const CovOut* cv;                       // NULL, or the full posterior (out_var = diag(Sigma)) and its blocks
  const KeyPriorIn* kp;                   // NULL, or per-key priors (sparse sink only): each range uploads its keys' lists
  bool csr = false;
  std::vector<long long> pptr;            // per-key priors: host copy of prior_ptr
  std::vector<int> pnon;                  // per-key priors: each key's entries other than the intercept's
  int L = 0, Dt = 0, ldx = 0, Dp = 0, ldh = 0;
  std::vector<long long> krs, key_nnz0;   // key_nnz0: CSR rowptr at the key boundaries
  std::vector<int> todo;                  // the keys that are fitted
  bool lists = false;                     // CSR with Dt > 32: a key may be narrower than Dt, so every range builds its column lists
  std::vector<int> kdt;                   // the width (Dt or Dt_k) of each key's problems, known once its range's lists exist
  int sp_key = 0;                         // sparse: key_ptr[0 .. sp_key] are written
  Counters cnt;

  bool solves(int k) const { const long long nk = krs[k + 1] - krs[k]; return !(nk < data_size_threshold || nk <= 0); }   // (:379-382)
  // the width of a key of dk distinct columns; with dk = its stored entries, a bound on it before the lists exist
  int local_dt(long long dk) const { const int w = round_up((int)std::min<long long>(dk, Dg) + 1, 32); return w < ldh ? w : Dt; }
  int bound_dt(int k) const { return lists ? local_dt(key_nnz0[k + 1] - key_nnz0[k]) : Dt; }
  // device bytes of a fitted key of n rows at width w: Xt (n*Dp*2) + Hpart + Lc per problem (+ the row weights of the variance)
  size_t state_bytes(long long n, int w) const {
    const size_t x = (size_t)round_up(w, 4), p = (size_t)round_up((int)x, 128), h = (size_t)round_up(w, 32);
    return (size_t)n * p * 2 + p * p * 4 + 3 * h * h * 8 + 2 * h * 32 * 8 + 64 * x + (out_var ? (size_t)n * 8 : 0);
  }
  // entries of a fitted CSR key's list at most: its stored entries (and prior entries other than the intercept's) or the dictionary,
  // whichever is smaller, and the intercept
  long long list_bound(int k) const {
    return std::min<long long>(key_nnz0[k + 1] - key_nnz0[k] + (kp ? pnon[k] : 0), Dg) + (has_intercept ? 1 : 0);
  }
  // device bytes of the prior lists of keys [k0, k1)
  size_t prior_bytes(long long k0, long long k1) const { return kp ? (size_t)(pptr[k1] - pptr[k0]) * 20 : 0; }
  int check_priors();
  // device bytes of a fitted key's entries in its chunk's slab (values of every prior, variances, column ids, covariance blocks); 0 for
  // the dense sink.  len: the key's list length when known, else (< 0) its bound
  size_t slab_bytes(int k, long long len = -1) const {
    if (!sp) return 0;
    const size_t n = (size_t)(len < 0 ? list_bound(k) : len);
    return n * ((size_t)L * 8 * (out_var ? 2 : 1) + 4) + (cv && cv->val ? n * (n + 1) / 2 * 8 * (size_t)L : 0);
  }
  // the lists of keys [k0, k1) over the range's colidx ci (entries from key_nnz0[k0] on), and the widths they give
  int build_lists(int k0, int k1, const int* ci, cudaStream_t s, DevMem& mem, KeyCols* kc) {
    std::vector<long long> koff(key_nnz0.begin() + k0, key_nnz0.begin() + k1 + 1);
    for (auto& o : koff) o -= key_nnz0[k0];
    if (int rc = key_columns(s, mem, koff, ci, kc)) return rc;
    for (int k = k0; k < k1; k++)
      kdt[k] = kc->listed[k - k0] ? local_dt(kc->start[k - k0 + 1] - kc->start[k - k0]) : Dt;
    return 0;
  }
  // device bytes of the lists of keys [k0, k1)
  size_t list_bytes(int k0, int k1) const {
    if (!lists) return 0;
    long long mx = 0;
    for (int k = k0; k < k1; k++) mx = std::max(mx, key_nnz0[k + 1] - key_nnz0[k]);
    return key_columns_bytes(key_nnz0[k1] - key_nnz0[k0], mx, k1 - k0);
  }
  void init_outputs() {
    if (skipped) for (int k = 0; k < K; k++) skipped[k] = solves(k) ? 0 : 1;   // "data size < threshold": no model
    if (cv && cv->val) cv->ptr[0] = 0;
    if (sp) { sp->key_ptr[0] = 0; return; }   // a list is written with its chunk
    for (size_t e = 0; e < (size_t)L * K * Dt; e++) out_model[e] = 0.0;
    if (out_var)   // a key without rows has no fit: every variance is the prior's
      for (int l = 0; l < L; l++)
        for (int k = 0; k < K; k++)
          for (int j = 0; j < Dt; j++) out_var[((size_t)l * K + k) * Dt + j] = 1.0 / priors[l].q[j];
  }
  // sparse: empty lists for keys sp_key .. k1 - 1 (the keys before k1 that no chunk fitted)
  void close_lists(int k1) {
    for (; sp_key < k1; sp_key++) {
      sp->key_ptr[sp_key + 1] = sp->key_ptr[sp_key];
      if (cv && cv->val) cv->ptr[sp_key + 1] = cv->ptr[sp_key];
    }
  }
  int run();
  int solve_chunk(const int* keys, int nprob, const ChunkRows& cr, int* dflag, int* hflag);
  int solve_batch(const int* keys, int nprob, int width, const ChunkRows& cr, int* dflag, int* hflag, Slab* sl);
  int solve_group(const int* keys, int nprob, int width, const ChunkRows& cr, int* dflag, int* hflag, Slab* sl);
  int open_slab(const int* keys, int nprob, const ChunkRows& cr, DevMem& mem, Slab* sl);
  int posterior_cov(Batch& B, bool local, const long long* drs, long long nrows, double* dvec, const CovJob* dcjobs, Slab* sl, int l,
                    int* dfail, const Ctrl* factor, const Ctrl* reset);
  int write_slab(const int* keys, int nprob, const Slab& sl);
};

int KeyedFit::run() {
  csr = rowptr != nullptr;
  L = (int)priors.size();
  Dt = Dg + 1; ldx = round_up(Dt, 4); Dp = round_up(ldx, 128); ldh = round_up(Dt, 32);
  krs.resize(K + 1);
  CK(cudaMemcpy(krs.data(), key_rowstart, (size_t)(K + 1) * 8, cudaMemcpyDefault));
  const long long ntot = krs[K];
  for (int k = 0; k < K; k++) if (krs[k + 1] < krs[k]) return fail(MLEASE_ERR_INVALID, "key_rowstart must be non-decreasing");
  for (int k = 0; k < K; k++) if (solves(k)) todo.push_back(k);
  kdt.assign(K, Dt);
  if (csr) {
    // rowptr at the key boundaries and at row 0, read without uploading the rows: each key's stored entries bound its width
    std::vector<long long> idx(krs);
    idx.push_back(0);
    if (int rc = gather_rowptr(rowptr, idx, key_nnz0)) return rc;
    if (key_nnz0.back() != 0) return fail(MLEASE_ERR_INVALID, "rowptr[0] must be 0");
    key_nnz0.pop_back();
    // the ranges' entry counts come from these; every range's own rows are checked on the device before a kernel indexes by them
    for (int k = 0; k < K; k++)
      if (key_nnz0[k + 1] < key_nnz0[k]) return fail(MLEASE_ERR_INVALID, "rowptr must never decrease (key " + std::to_string(k) + ")");
    // any key may list fewer columns than the dictionary holds (the bound above only caps its width): every range builds its lists
    lists = ldh > 32 && !todo.empty();
  }
  if (kp) { if (int rc = check_priors()) return rc; }   // before anything is written or indexed by the lists
  if (sp) {   // the lists' room, checked before any row is read
    long long need = 0;
    for (int k : todo) need += list_bound(k);
    if (sp->cap < need)
      return fail(MLEASE_ERR_INVALID, "capacity " + std::to_string(sp->cap) + " is too small: the keys' lists need up to " +
                                          std::to_string(need) + " entries (the sum over fitted keys of min(stored entries" +
                                          (kp ? " + non-intercept prior entries" : "") + ", num_features)" + (has_intercept ? " + 1)" : ")"));
  }
  // resident (one range) when the whole upload (rows, labels, key boundaries, the temporaries of host input, the column lists) and
  // the first chunk's state fit the budget
  size_t free_b, total_b;
  CK(cudaMemGetInfo(&free_b, &total_b));
  const size_t budget = keyed_budget(free_b);
  const long long nnz = csr ? key_nnz0[K] : 0;
  const bool host_rows = !is_device_ptr(csr ? (const void*)colidx : (const void*)vals);
  size_t up = (size_t)ntot * 9 + (is_device_ptr(response) ? 0 : (size_t)ntot * 12);
  if (csr) up += (size_t)nnz * 4 + (host_rows ? (size_t)nnz * 4 + (size_t)(ntot + 1) * 8 : 0) + (size_t)(K + 1) * 16 + list_bytes(0, K) + prior_bytes(0, K);
  else up += (size_t)ntot * ldx * 4 + (host_rows ? (size_t)256 << 20 : 0);
  const size_t first = todo.empty() ? 0 : state_bytes(krs[todo[0] + 1] - krs[todo[0]], bound_dt(todo[0])) + slab_bytes(todo[0]);
  const bool streamed = up + first > budget;
  std::vector<long long> ranges{0, K};
  if (streamed) {
    // streamed: ranges whose rows (staged copy + the solver's layout, the column lists) and fitted keys' state (at the bound of
    // their widths) fit a quarter of the budget
    ranges = plan_ranges(K, budget / 4, 16384, [&](long long k) -> size_t {
      const size_t n = (size_t)(krs[k + 1] - krs[k]);
      size_t b = n * (12 + 9);
      b += csr ? n * 16 + (size_t)(key_nnz0[k + 1] - key_nnz0[k]) * 8 + list_bytes(k, k + 1) + prior_bytes(k, k + 1) : n * ((size_t)ldx_in + ldx) * 4;
      return b + (solves(k) ? state_bytes(n, bound_dt(k)) + slab_bytes((int)k) : 0);
    }, [&](long long k) { return solves(k); });
  }
  const int nr = (int)ranges.size() - 1;
  std::vector<long long> row_at, nnz_at;
  for (long long k : ranges) { row_at.push_back(krs[k]); if (csr) nnz_at.push_back(key_nnz0[k]); }
  enum { RP, CI, V, Y, W, O };   // the sources; the dense rows are V
  RangeRing ring(st, {{rowptr, 8, RangeSrc::ROWPTR}, {colidx, 4, RangeSrc::ENTRY}, {vals, 4, csr ? RangeSrc::ENTRY : RangeSrc::DENSE},
                      {response, 4, RangeSrc::ROW}, {weight, 4, RangeSrc::ROW}, {offset, 4, RangeSrc::ROW}}, row_at, nnz_at, ldx_in, Dg,
                      streamed, true);
  long long max_rows = 0;
  for (int c = 0; c < nr; c++) max_rows = std::max(max_rows, row_at[c + 1] - row_at[c]);
  DevMem t;
  PinnedMem pinned;
  signed char* dy; float *dw, *dofs, *dX = nullptr; int* dflag; int* hflag;
  if (int rc = t.get(&dy, (size_t)max_rows, false)) return rc;
  if (int rc = t.get(&dw, (size_t)max_rows, false)) return rc;
  if (int rc = t.get(&dofs, (size_t)max_rows, false)) return rc;
  if (int rc = t.get(&dflag, 16, false)) return rc;
  if (int rc = pinned.get(&hflag, 16, false)) return rc;
  if (!csr) { if (int rc = t.get(&dX, (size_t)max_rows * ldx, false)) return rc; }
  if (int rc = ring.open()) return rc;
  std::vector<long long> bounds{0};
  for (int c = 0; c < nr; c++) {
    const void* v[6];
    if (int rc = ring.view(c, v)) return rc;
    const int k0 = (int)ranges[c], k1 = (int)ranges[c + 1];
    const long long n = row_at[c + 1] - row_at[c];
    DevMem rt;   // the range's device copies of host input and its column lists
    KeyCols kc;
    ChunkRows cr;
    cr.row0 = row_at[c]; cr.y = dy; cr.w = dw; cr.o = dofs; cr.X = dX;
    // the range's checks, before any kernel reads its rows
    if (csr) {
      const long long z0 = nnz_at[c], nz = nnz_at[c + 1] - z0;
      if (int rc = to_device(rt, (const long long*)v[RP], (size_t)n + 1, &cr.rp, st)) return rc;
      if (int rc = to_device(rt, (const int*)v[CI], (size_t)nz, &cr.ci, st)) return rc;
      cr.v = (float*)v[V];   // a ring slot: the range's own copy
      if (!ring.staged()) {  // the caller's values are copied even when they live on the device: binary.feature rewrites them
        if (int rc = rt.get(&cr.v, (size_t)nz, false)) return rc;
        CK(cudaMemcpyAsync(cr.v, vals, (size_t)nz * 4, cudaMemcpyDefault, st));
      }
      if (z0) rebase_rowptr(st, n, cr.rp, z0, (long long*)cr.rp);   // in place: a range after the first is in a ring slot
      if (int rc = check_rowptr(st, n, cr.rp, dflag, "keys " + std::to_string(k0) + ".." + std::to_string(k1 - 1) + ": ")) return rc;
      CK(cudaMemsetAsync(dflag, 0, 8, st));
      check_csr(st, n, nz, cr.rp, cr.ci, cr.v, Dg, binary_feature, dflag);
      CK(cudaMemcpyAsync(hflag, dflag, 8, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      if (hflag[0]) return fail(MLEASE_ERR_INVALID, "feature index out of range");
      cr.csr_unique = hflag[1] ? 0 : 1;
      if (cv && !cr.csr_unique)
        return fail(MLEASE_ERR_INVALID, "the full Hessian needs rows with strictly increasing column ids (llf/LogisticRegressionL2.java:277)");
      if (lists) {
        if (int rc = build_lists(k0, k1, cr.ci, st, rt, &kc)) return rc;
        cr.kc = &kc; cr.kbase = k0;
      }
      if (kp) {   // the range's slice of the prior lists (check_priors passed them all)
        const long long p0 = pptr[k0], pn = pptr[k1] - p0;
        int* pc; double *pm, *pv;
        if (int rc = rt.get(&pc, (size_t)pn, false)) return rc;
        if (int rc = rt.get(&pm, (size_t)pn, false)) return rc;
        if (int rc = rt.get(&pv, (size_t)pn, false)) return rc;
        CK(cudaMemcpyAsync(pc, kp->col + p0, (size_t)pn * 4, cudaMemcpyDefault, st));
        CK(cudaMemcpyAsync(pm, kp->mean + p0, (size_t)pn * 8, cudaMemcpyDefault, st));
        CK(cudaMemcpyAsync(pv, kp->var + p0, (size_t)pn * 8, cudaMemcpyDefault, st));
        cr.pd = PriorDev{pc, pm, pv}; cr.pbase = p0;
      }
    } else {
      if (int rc = upload_dense_rows(dX, ldx, (const float*)v[V], ldx_in, n, Dg, has_intercept ? 1 : 0, st)) return rc;
    }
    if (int rc = ingest_labels(st, n, (const int32_t*)v[Y], (const float*)v[W], (const float*)v[O], dy, dw, dofs, dflag, hflag, nullptr))
      return rc;
    if (c == 0) init_outputs();   // the first range's rows passed their checks
    if (int rc = ring.start(c + 1)) return rc;
    // the range's fitted keys in chunks: a streamed range is one chunk, a resident call's chunks fit the memory left after its upload
    std::vector<int> keys;
    for (int k = k0; k < k1; k++) if (solves(k)) keys.push_back(k);
    size_t cap = SIZE_MAX;
    if (!ring.staged()) { CK(cudaMemGetInfo(&free_b, &total_b)); cap = keyed_budget(free_b) / 2; }
    const std::vector<long long> chunks = plan_ranges((long long)keys.size(), cap, 16384, [&](long long i) {
      const int k = keys[i];
      // a covariance call counts a listed key's blocks at their exact size: the bound squared overshoots wide keys many times
      const long long len = cv && cr.kc && cr.kc->listed[k - cr.kbase] ? cr.kc->start[k - cr.kbase + 1] - cr.kc->start[k - cr.kbase] + 1 : -1;
      return state_bytes(krs[k + 1] - krs[k], kdt[k]) + slab_bytes(k, len);
    }, nullptr);
    for (size_t j = 1; j < chunks.size(); j++) {
      if (int rc = solve_chunk(keys.data() + chunks[j - 1], (int)(chunks[j] - chunks[j - 1]), cr, dflag, hflag)) return rc;
      bounds.push_back(chunks[j] < (long long)keys.size() ? keys[chunks[j]] : k1);
    }
    if (bounds.back() != k1) bounds.push_back(k1);
    if (int rc = ring.done(c)) return rc;
  }
  if (sp) close_lists(K);
  keyed_record(bounds, ring.staged(), ring.stage_ms, ring.wait_ms);
  if (cnt.not_converged) return fail(MLEASE_ERR_NUMERIC, "Model fitting error! (" + std::to_string(cnt.not_converged) + " fits did not converge)");
  return 0;
}

// The per-key priors' checks, before the call writes anything: prior_ptr on the host (one value per key), every entry on the device
// in passes over contiguous key slices of at most PRIOR_CHECK_BYTES; each key's non-intercept entries into pnon for the list bound
int KeyedFit::check_priors() {
  pptr.resize((size_t)K + 1);
  CK(cudaMemcpy(pptr.data(), kp->ptr, (size_t)(K + 1) * 8, cudaMemcpyDefault));
  if (pptr[0] != 0) return fail(MLEASE_ERR_INVALID, "prior_ptr[0] must be 0 (key 0)");
  for (int k = 0; k < K; k++)
    if (pptr[k + 1] < pptr[k]) return fail(MLEASE_ERR_INVALID, "prior_ptr must never decrease (key " + std::to_string(k) + ")");
  pnon.assign(K, 0);
  if (pptr[K] == 0) return 0;
  const std::vector<long long> sl = plan_ranges(K, PRIOR_CHECK_BYTES, 1 << 20, [&](long long k) { return (size_t)(pptr[k + 1] - pptr[k]) * 20; },
                                                nullptr);
  long long mx = 0, mk = 0;
  for (size_t s = 1; s < sl.size(); s++) { mx = std::max(mx, pptr[sl[s]] - pptr[sl[s - 1]]); mk = std::max(mk, sl[s] - sl[s - 1]); }
  DevMem t;
  int *pc, *nonint; double *pm, *pv; long long* offs; unsigned long long* bad;
  if (int rc = t.get(&pc, (size_t)mx, false)) return rc;
  if (int rc = t.get(&pm, (size_t)mx, false)) return rc;
  if (int rc = t.get(&pv, (size_t)mx, false)) return rc;
  if (int rc = t.get(&offs, (size_t)mk + 1, false)) return rc;
  if (int rc = t.get(&nonint, (size_t)mk, false)) return rc;
  if (int rc = t.get(&bad, 1, false)) return rc;
  std::vector<long long> o;
  for (size_t s = 1; s < sl.size(); s++) {
    const long long k0 = sl[s - 1], k1 = sl[s], p0 = pptr[k0], pn = pptr[k1] - p0;
    o.resize((size_t)(k1 - k0 + 1));
    for (long long k = k0; k <= k1; k++) o[k - k0] = pptr[k] - p0;
    CK(cudaMemcpyAsync(offs, o.data(), o.size() * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(pc, kp->col + p0, (size_t)pn * 4, cudaMemcpyDefault, st));
    CK(cudaMemcpyAsync(pm, kp->mean + p0, (size_t)pn * 8, cudaMemcpyDefault, st));
    CK(cudaMemcpyAsync(pv, kp->var + p0, (size_t)pn * 8, cudaMemcpyDefault, st));
    CK(cudaMemsetAsync(bad, 0xff, 8, st));
    prior_check_kernel<<<(unsigned)(k1 - k0), 128, 0, st>>>(offs, (int)k0, pc, pm, pv, Dg, bad, nonint);
    CK(cudaGetLastError());
    unsigned long long hbad = 0;
    CK(cudaMemcpyAsync(&hbad, bad, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(pnon.data() + k0, nonint, (size_t)(k1 - k0) * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (hbad != ~0ull) {
      static const char* why[] = {"", "a prior column outside [0, num_features]", "prior columns that are not strictly ascending",
                                  "a prior mean that is not finite", "a prior variance that is negative or not finite"};
      return fail(MLEASE_ERR_INVALID, "key " + std::to_string(hbad >> 3) + ": " + why[hbad & 7]);
    }
  }
  return 0;
}

// the problems keys[0, nprob) over the rows of cr, every prior, into out_model / out_var: one batch per width, narrowest first
int KeyedFit::solve_chunk(const int* keys, int nprob, const ChunkRows& cr, int* dflag, int* hflag) {
  std::vector<int> widths;
  for (int b = 0; b < nprob; b++) widths.push_back(kdt[keys[b]]);
  std::sort(widths.begin(), widths.end());
  widths.erase(std::unique(widths.begin(), widths.end()), widths.end());
  if (cv)   // before any of the chunk's keys is solved
    for (int b = 0; b < nprob; b++)
      if (round_up(kdt[keys[b]], 32) > COV_MAX_WIDTH)
        return fail(MLEASE_ERR_INVALID, "key " + std::to_string(keys[b]) + ": its posterior covariance needs the explicit inverse of a " +
                                            std::to_string(kdt[keys[b]]) + "-column system (" + (kdt[keys[b]] == Dt ? "the global width" : "its own column space") +
                                            "), which exists for at most " + std::to_string(COV_MAX_WIDTH) + " columns");
  DevMem sm;   // the sparse sink's slab
  Slab slab;
  if (sp) { if (int rc = open_slab(keys, nprob, cr, sm, &slab)) return rc; }
  std::vector<int> group;
  for (int w : widths) {
    group.clear();
    for (int b = 0; b < nprob; b++) if (kdt[keys[b]] == w) group.push_back(keys[b]);
    if (int rc = solve_group(group.data(), (int)group.size(), w, cr, dflag, hflag, sp ? &slab : nullptr)) return rc;
  }
  return sp ? write_slab(keys, nprob, slab) : 0;
}

// solve_batch; a covariance call's batch that would be matrix-free (its Hessians, factors and inverses do not fit the device) is
// solved in halves instead
int KeyedFit::solve_group(const int* keys, int nprob, int w, const ChunkRows& cr, int* dflag, int* hflag, Slab* sl) {
  const int rc = solve_batch(keys, nprob, w, cr, dflag, hflag, sl);
  if (rc != SPLIT_BATCH) return rc;
  if (nprob == 1)
    return fail(MLEASE_ERR_CUDA, "key " + std::to_string(keys[0]) + ": its Hessian, factor and inverse (" + std::to_string(w) +
                                     " columns) do not fit the free device memory");
  const int h = nprob / 2;
  if (int r = solve_group(keys, h, w, cr, dflag, hflag, sl)) return r;
  return solve_group(keys + h, nprob - h, w, cr, dflag, hflag, sl);
}

// The slab of the chunk keys[0, nprob) (ascending, fitted): each key's list length (from its column list, or for a key without one
// from the presence mask of its rows, read back here), its offset, and the device arrays
int KeyedFit::open_slab(const int* keys, int nprob, const ChunkRows& cr, DevMem& mem, Slab* sl) {
  const int k0 = keys[0], nk = keys[nprob - 1] - k0 + 1;
  sl->k0 = k0;
  sl->off.assign(nk, 0); sl->len.assign(nk, 0); sl->mrow.assign(nk, -1);
  std::vector<long long> rows;   // range-local row bounds of the keys without a list
  for (int b = 0; b < nprob; b++) {
    const int k = keys[b];
    if (cr.kc && cr.kc->listed[k - cr.kbase])
      sl->len[k - k0] = cr.kc->start[k - cr.kbase + 1] - cr.kc->start[k - cr.kbase] + (has_intercept ? 1 : 0);
    else {
      sl->mrow[k - k0] = (int)(rows.size() / 2);
      rows.push_back(krs[k] - cr.row0); rows.push_back(krs[k + 1] - cr.row0);
    }
  }
  const int nu = (int)rows.size() / 2;
  std::vector<int> count(nu), pcount(kp ? nprob : 0);
  if (nu) {
    long long* drows; int* dcount;
    if (int rc = mem.get(&sl->mask, (size_t)nu * Dt, false)) return rc;
    if (int rc = mem.get(&drows, rows.size(), false)) return rc;
    if (int rc = mem.get(&dcount, (size_t)nu, false)) return rc;
    CK(cudaMemsetAsync(sl->mask, 0, (size_t)nu * Dt, st));
    CK(cudaMemcpyAsync(drows, rows.data(), rows.size() * 8, cudaMemcpyHostToDevice, st));
    span_present_kernel<<<nu, 256, 0, st>>>(cr.rp, cr.ci, drows, Dt, has_intercept ? 1 : 0, sl->mask, dcount);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(count.data(), dcount, (size_t)nu * 4, cudaMemcpyDeviceToHost, st));
  }
  std::vector<GatherJob> pj(pcount.size());   // per-key priors: each key's list, or mask row, and its prior entries
  if (kp) {
    for (int b = 0; b < nprob; b++) {
      const int k = keys[b];
      GatherJob& j = pj[b];
      j.mrow = sl->mrow[k - k0]; j.dk = -1;
      if (j.mrow < 0) { j.s0 = cr.kc->start[k - cr.kbase]; j.dk = (int)(cr.kc->start[k - cr.kbase + 1] - j.s0); }
      j.p0 = pptr[k] - cr.pbase; j.pn = (int)(pptr[k + 1] - pptr[k]);
    }
    GatherJob* dpj; int* dpcount;
    if (int rc = mem.get(&dpj, pj.size(), false)) return rc;
    if (int rc = mem.get(&dpcount, pj.size(), false)) return rc;
    CK(cudaMemcpyAsync(dpj, pj.data(), pj.size() * sizeof(GatherJob), cudaMemcpyHostToDevice, st));
    prior_only_count_kernel<<<nprob, 128, 0, st>>>(dpj, cr.kc ? cr.kc->d_cols : nullptr, sl->mask, Dt, Dg, cr.pd, dpcount);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(pcount.data(), dpcount, pj.size() * 4, cudaMemcpyDeviceToHost, st));
  }
  if (nu || kp) CK(cudaStreamSynchronize(st));
  for (int i = 0; i < nk; i++) if (sl->mrow[i] >= 0) sl->len[i] = count[sl->mrow[i]];
  for (size_t b = 0; b < pcount.size(); b++) sl->len[keys[b] - k0] += pcount[b];   // the union with the prior-only columns
  for (int i = 0; i < nk; i++) { sl->off[i] = sl->n; sl->n += sl->len[i]; }
  if (cv && cv->val) {
    // the lengths are fixed: the chunk's blocks must fit the room left, checked before the chunk writes anything
    sl->coff.assign(nk, 0);
    for (int i = 0; i < nk; i++) { sl->coff[i] = sl->ncov; sl->ncov += sl->len[i] * (sl->len[i] + 1) / 2; }
    const long long need = cv->ptr[sp_key] + sl->ncov;
    if (need > cv->cap)
      return fail(MLEASE_ERR_INVALID, "cov_capacity " + std::to_string(cv->cap) + " is too small: the covariance blocks of keys 0 .. " +
                                          std::to_string(keys[nprob - 1]) + " need " + std::to_string(need) + " entries");
    if (int rc = mem.get(&sl->cov, (size_t)L * sl->ncov, false)) return rc;
  }
  if (int rc = mem.get(&sl->model, (size_t)L * sl->n, false)) return rc;
  if (out_var) { if (int rc = mem.get(&sl->var, (size_t)L * sl->n, false)) return rc; }
  return mem.get(&sl->col, (size_t)sl->n, false);
}

// the chunk's slab into the caller's lists: entries key_ptr[keys[0]] .. of every prior, and key_ptr up to the chunk's last key
int KeyedFit::write_slab(const int* keys, int nprob, const Slab& sl) {
  close_lists(keys[0]);
  const long long e0 = sp->key_ptr[keys[0]];
  for (int l = 0; l < L; l++) {
    CK(cudaMemcpyAsync(out_model + l * sp->cap + e0, sl.model + l * sl.n, (size_t)sl.n * 8, cudaMemcpyDeviceToHost, st));
    if (out_var) CK(cudaMemcpyAsync(out_var + l * sp->cap + e0, sl.var + l * sl.n, (size_t)sl.n * 8, cudaMemcpyDeviceToHost, st));
  }
  if (cv && cv->val)
    for (int l = 0; l < L; l++)
      CK(cudaMemcpyAsync(cv->val + l * cv->cap + cv->ptr[keys[0]], sl.cov + l * sl.ncov, (size_t)sl.ncov * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(sp->col + e0, sl.col, (size_t)sl.n * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  for (int k = keys[0]; k <= keys[nprob - 1]; k++) {
    sp->key_ptr[k + 1] = sp->key_ptr[k] + sl.len[k - sl.k0];
    if (cv && cv->val) cv->ptr[k + 1] = cv->ptr[k] + sl.len[k - sl.k0] * (sl.len[k - sl.k0] + 1) / 2;
  }
  sp_key = keys[nprob - 1] + 1;
  return 0;
}

// the problems keys[0, nprob) of width w: Dt (today's global-width problems), or the keys' own column spaces (w < Dt); results into
// the dense outputs, or with sl into the chunk's slab
int KeyedFit::solve_batch(const int* keys, int nprob, int w, const ChunkRows& cr, int* dflag, int* hflag, Slab* sl) {
  const bool local = w != Dt;
  Batch B;
  B.nprob = nprob; B.Dt = w; B.ldx = round_up(w, 4); B.csr = csr; B.has_bias = has_intercept ? 1 : 0;
  // a local batch's members depend on the call (its chunk, its width group): without the slot pipeline a key's path, hence a one-row
  // key's bits, do not depend on them
  B.lockstep = local;
  B.h.resize(B.nprob);
  std::vector<long long> span(local ? 2 * (size_t)nprob : 0);   // each problem's list in cr.kc's columns
  std::vector<long long> row_start(B.nprob + 1, 0);   // the chunk's rows numbered across its problems (batched variance)
  for (int b = 0; b < B.nprob; b++) {
    const int k = keys[b];
    const long long r = krs[k] - cr.row0;
    Problem& p = B.h[b];
    std::memset(&p, 0, sizeof(Problem));
    p.n = krs[k + 1] - krs[k];
    p.y = cr.y + r; p.w = cr.w + r; p.o = cr.o + r;
    if (csr) {
      // a key = a row range of the CSR: the row pointers keep their offsets into colidx / vals
      p.rowptr = cr.rp + r; p.colidx = cr.ci; p.vals = cr.v; p.nnz_hint = key_nnz0[k + 1] - key_nnz0[k]; p.csr_unique = cr.csr_unique;
      if (local) {   // the same entries, each naming its index in the key's list
        p.colidx = cr.kc->d_lci;
        span[2 * b] = cr.kc->start[k - cr.kbase]; span[2 * b + 1] = cr.kc->start[k - cr.kbase + 1];
      }
    } else {
      p.X = cr.X + (size_t)r * ldx;
    }
    row_start[b + 1] = row_start[b] + p.n;
  }
  if (int rc = batch_alloc(B, num_sms, 0)) return rc;
  if (cv && B.matfree) return SPLIT_BATCH;   // the Hessians need the Gram path's Lc and Hinv
  DevMem ct;   // the batch's temporaries: freed with it, before the next batch_alloc
  double *dm, *dq, *dout = nullptr, *dim = nullptr, *dvec = nullptr; long long *drs = nullptr, *dspan = nullptr; unsigned char* dmask = nullptr;
  GatherJob* djobs = nullptr;
  CovJob* dcjobs = nullptr;
  int* dfail = nullptr;              // covariance: pivot failures of the batch's factorisations, all priors
  PinnedMem cp;
  Ctrl *factor_ctl = nullptr, *reset_ctl = nullptr;
  if (int rc = ct.get(&dm, (size_t)ldx, false)) return rc;
  if (int rc = ct.get(&dq, (size_t)ldx, false)) return rc;
  if (sl) {
    // each problem's list: its column list (local, or a global-width key that has one), else its row of the slab's mask
    std::vector<GatherJob> jobs(B.nprob);
    for (int b = 0; b < B.nprob; b++) {
      const int k = keys[b];
      GatherJob& j = jobs[b];
      j.dst = sl->off[k - sl->k0]; j.mrow = sl->mrow[k - sl->k0]; j.s0 = 0; j.dk = -1;
      if (j.mrow < 0) { j.s0 = cr.kc->start[k - cr.kbase]; j.dk = (int)(cr.kc->start[k - cr.kbase + 1] - j.s0); }
      if (kp) { j.p0 = pptr[k] - cr.pbase; j.pn = (int)(pptr[k + 1] - pptr[k]); }
    }
    if (int rc = ct.get(&djobs, jobs.size(), false)) return rc;
    CK(cudaMemcpyAsync(djobs, jobs.data(), jobs.size() * sizeof(GatherJob), cudaMemcpyHostToDevice, st));
    std::vector<CovJob> cjobs(cv ? B.nprob : 0);
    for (size_t b = 0; b < cjobs.size(); b++) {
      const int i = keys[b] - sl->k0;
      cjobs[b] = CovJob{sl->off[i], cv->val ? sl->coff[i] : -1, (int)sl->len[i]};
    }
    if (cv) {
      if (int rc = ct.get(&dfail, 1, true)) return rc;
      if (int rc = cp.get(&factor_ctl, (size_t)B.nprob, true)) return rc;
      if (int rc = cp.get(&reset_ctl, (size_t)B.nprob, true)) return rc;
      for (int b = 0; b < B.nprob; b++) factor_ctl[b].need_hess = 1;
      if (int rc = ct.get(&dcjobs, cjobs.size(), false)) return rc;
      CK(cudaMemcpyAsync(dcjobs, cjobs.data(), cjobs.size() * sizeof(CovJob), cudaMemcpyHostToDevice, st));
    }
    CK(cudaStreamSynchronize(st));   // jobs and cjobs are released here
  } else {
    if (int rc = ct.get(&dout, (size_t)B.nprob * w, false)) return rc;
  }
  if (intercept_mean) {
    std::vector<double> im(B.nprob);
    for (int b = 0; b < B.nprob; b++) im[b] = intercept_mean[keys[b]];
    if (int rc = ct.get(&dim, (size_t)B.nprob, false)) return rc;
    CK(cudaMemcpyAsync(dim, im.data(), im.size() * 8, cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));   // im is released here
  }
  if (out_var) {
    if (int rc = ct.get(&dvec, (size_t)row_start[B.nprob], false)) return rc;
    if (int rc = ct.get(&drs, row_start.size(), false)) return rc;
    CK(cudaMemcpyAsync(drs, row_start.data(), row_start.size() * 8, cudaMemcpyHostToDevice, st));
  }
  if (local) {
    if (int rc = ct.get(&dspan, span.size(), false)) return rc;
    CK(cudaMemcpyAsync(dspan, span.data(), span.size() * 8, cudaMemcpyHostToDevice, st));
  } else if (csr && (!sl || kp)) {
    // features absent from a key's rows are not part of its dataset, hence not of its model (llf/LibLinear.java:343-350; the only
    // prior mean a caller may set per key is the intercept's, which every dataset holds, so :374-383 adds nothing): mask them out
    // (the sparse sink reports only the listed columns).  Per-key priors: the mask says which columns take a prior entry in the fit
    if (int rc = ct.get(&dmask, (size_t)B.nprob * Dt, false)) return rc;
    CK(cudaMemsetAsync(dmask, 0, (size_t)B.nprob * Dt, st));
    naive_present_kernel<<<B.nprob, 256, 0, st>>>(B.d, Dt, has_intercept ? 1 : 0, dmask);
  }
  // a local problem's column c < Dk is global column cols[c]; its intercept (column w - 1) is global column Dg
  auto scatter = [&](double* dst, const double* x, int b, bool inv) {
    const long long s0 = span[2 * b], dk = span[2 * b + 1] - s0;
    const int* cols = cr.kc->cols.data() + s0;
    for (long long c = 0; c < dk; c++) dst[cols[c]] = inv ? 1.0 / x[c] : x[c];
    dst[Dg] = inv ? 1.0 / x[w - 1] : x[w - 1];
  };
  std::vector<double> xs(sl ? 0 : (size_t)B.nprob * w);
  for (int l = 0; l < L; l++) {
    CK(cudaMemcpyAsync(dm, priors[l].m.data(), ldx * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(dq, priors[l].q.data(), ldx * 8, cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));   // dq / dm are reused by the next prior
    if (kp) prior_init_kernel<<<B.nprob, 128, 0, st>>>(B.d, dm, dq, dim, local ? cr.kc->d_cols : nullptr, local ? dspan : nullptr, dmask, Dg,
                                                        djobs, cr.pd);
    else if (local) local_init_kernel<<<B.nprob, 128, 0, st>>>(B.d, dm, dq, dim, cr.kc->d_cols, dspan, Dg);
    else naive_init_kernel<<<B.nprob, 128, 0, st>>>(B.d, dm, dq, dim);
    B.mirror.clear();                // the factors of the previous prior belong to another prior
    if (int rc = batch_xupdate(B, st, 2e-7, 100, 0, 1, hflag, dflag, cnt)) return rc;
    if (sl) {   // the listed values straight into the slab (column ids with the first prior); no read-back until the chunk is done
      const int* kcols = cr.kc ? cr.kc->d_cols : nullptr;
      sparse_gather_kernel<<<B.nprob, GATHER_THREADS, 0, st>>>(B.d, djobs, kcols, sl->mask, local ? 1 : 0, Dg, B.has_bias, 0,
                                                               sl->model + l * sl->n, l == 0 ? sl->col : nullptr, cr.pd, dq);
      CK(cudaGetLastError());
      if (cv) {
        if (int rc = posterior_cov(B, local, drs, row_start[B.nprob], dvec, dcjobs, sl, l, dfail, factor_ctl, reset_ctl)) return rc;
      } else if (out_var) {
        CK(postvar_rowweights(B.d, B.nprob, drs, row_start[B.nprob], B.has_bias, dvec, st, nullptr));
        CK(postvar_diag(B.d, B.nprob, drs, row_start[B.nprob], dvec, B.has_bias, st, nullptr));
        sparse_gather_kernel<<<B.nprob, GATHER_THREADS, 0, st>>>(B.d, djobs, kcols, sl->mask, local ? 1 : 0, Dg, B.has_bias, 1,
                                                                 sl->var + l * sl->n, nullptr, cr.pd, dq);
        CK(cudaGetLastError());
      }
      continue;
    }
    gather_beta_kernel<<<B.nprob, 128, 0, st>>>(B.d, w, dout, dmask, 0);
    CK(cudaMemcpyAsync(xs.data(), dout, xs.size() * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (int b = 0; b < B.nprob; b++) {
      double* dst = out_model + ((size_t)l * K + keys[b]) * Dt;
      if (local) scatter(dst, xs.data() + (size_t)b * w, b, false);
      else std::memcpy(dst, xs.data() + (size_t)b * Dt, Dt * 8);
      if (!has_intercept) dst[Dg] = 0.0;
    }
    if (out_var) {
      // posteriorVar, diagonal (llf/LibLinear.java:328-333): one pass over the batch's rows for all of its keys
      CK(postvar_rowweights(B.d, B.nprob, drs, row_start[B.nprob], B.has_bias, dvec, st, nullptr));
      CK(postvar_diag(B.d, B.nprob, drs, row_start[B.nprob], dvec, B.has_bias, st, nullptr));
      gather_beta_kernel<<<B.nprob, 128, 0, st>>>(B.d, w, dout, nullptr, 1);
      CK(cudaMemcpyAsync(xs.data(), dout, xs.size() * 8, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      for (int b = 0; b < B.nprob; b++) {
        double* dst = out_var + ((size_t)l * K + keys[b]) * Dt;
        if (local) scatter(dst, xs.data() + (size_t)b * w, b, true);   // unlisted features keep init_outputs' 1/q
        else for (int j = 0; j < Dt; j++) dst[j] = 1.0 / xs[(size_t)b * Dt + j];
      }
    }
  }
  if (dfail) {
    int bad = 0;
    CK(cudaMemcpyAsync(&bad, dfail, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (bad) return fail(MLEASE_ERR_NUMERIC, "Model fitting error! (Hessian not positive definite in " + std::to_string(bad) + " fit(s))");
  }
  return 0;
}

// The full posterior of prior l's fits, the batch's x-update just done (llf/LibLinear.java:315-326): row weights at each fit, the
// exact Hessians into Lc, K3's factorisation without prep and its explicit inverse, then the variances and covariance blocks over
// each key's list into the slab.  The control blocks are left as reset_ctrl leaves them: no factor, so the next prior's x-update
// rebuilds from its start point exactly as after the sparse call's diagonal variance (the fits do not change).
// The pivot failures are counted on the device into dfail, which the batch reads once after its last prior; factor / reset: the
// control blocks before the factorisation (need_hess = 1) and after it (zero), pinned so that the copies stay asynchronous.
int KeyedFit::posterior_cov(Batch& B, bool local, const long long* drs, long long nrows, double* dvec, const CovJob* dcjobs, Slab* sl, int l,
                            int* dfail, const Ctrl* factor, const Ctrl* reset) {
  CK(postvar_rowweights(B.d, B.nprob, drs, nrows, B.has_bias, dvec, st, nullptr));
  CK(postvar_hessian_batch(B.d, B.nprob, B.ldh, drs, dvec, B.has_bias, st, nullptr));
  CK(cudaMemcpyAsync(B.d_ctrl, factor, (size_t)B.nprob * sizeof(Ctrl), cudaMemcpyHostToDevice, st));
  CK(cholesky_launch(B.d, B.nprob, B.ldh, st, nullptr, 0, 1, 1));
  cov_gather_kernel<<<B.nprob, 256, 0, st>>>(B.d, dcjobs, local ? 1 : 0, sl->col, sl->var + l * sl->n, cv->val ? sl->cov + l * sl->ncov : nullptr);
  cov_fail_kernel<<<1, 256, 0, st>>>(B.d, B.nprob, dfail);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(B.d_ctrl, reset, (size_t)B.nprob * sizeof(Ctrl), cudaMemcpyHostToDevice, st));
  B.mirror.clear();
  return 0;
}

// callers run keyed_fit_check first
int keyed_fit(int num_sms, cudaStream_t st, int32_t K, int32_t Dg, const int64_t* key_rowstart, const int64_t* rowptr, const int32_t* colidx,
              const float* vals, int64_t ldx_in, const int32_t* response, const float* weight, const float* offset, bool has_intercept,
              int32_t data_size_threshold, int32_t binary_feature, const std::vector<KeyedPrior>& priors, const double* intercept_mean,
              double* out_model, double* out_var, int32_t* skipped, const SparseOut* sp, const CovOut* cv = nullptr,
              const KeyPriorIn* kp = nullptr) {
  KeyedFit f{num_sms, st, K, Dg, key_rowstart, rowptr, colidx, vals, ldx_in, response, weight, offset, has_intercept, data_size_threshold,
             binary_feature, priors, intercept_mean, out_model, out_var, skipped, sp, cv, kp};
  return f.run();
}
// host copy of a host-or-device array (NULL -> empty)
template <class T> int host_copy(const T* in, size_t count, std::vector<T>& out) {
  out.clear();
  if (!in) return 0;
  out.resize(count);
  CK(cudaMemcpy(out.data(), in, count * sizeof(T), cudaMemcpyDefault));
  return 0;
}

// ------------------------------------------------------------------------------------------
// RegressionNaiveTrain: K independent fits per lambda (keyed_fit), into the dense outputs or (sp) the sparse lists
// ------------------------------------------------------------------------------------------
int naive_train(int32_t device, void* stream, int32_t K, int32_t Dg, const int64_t* key_rowstart, const int64_t* rowptr,
                const int32_t* colidx, const float* vals, int64_t ldx_in, const int32_t* response, const float* weight,
                const float* offset, int32_t L, const float* lambdas, const float* lambda_map, float prior_mean,
                int32_t penalize_intercept, int32_t has_intercept, int32_t data_size_threshold, int32_t binary_feature,
                double* out_model, int32_t* skipped, const SparseOut* sp) {
  int num_sms = 0;
  if (int rc = keyed_fit_check(device, Dg, rowptr, colidx, ldx_in, binary_feature, &num_sms)) return rc;
  std::vector<float> lm, lams;
  if (int rc = host_copy(lambda_map, (size_t)Dg, lm)) return rc;
  if (int rc = host_copy(lambdas, (size_t)L, lams)) return rc;
  const int ldx = round_up(Dg + 1, 4);
  std::vector<KeyedPrior> priors(L);
  for (int l = 0; l < L; l++) {
    // prior (jobs/RegressionNaiveTrain.java:333-343,395): variance 1/lambdaMap[k] for listed features, 1/lambda otherwise,
    // 100000 for the intercept unless penalised; mean prior.mean; the fit starts at 0 (null initParam)
    const float lambda = lams[l];
    std::vector<double>& q = priors[l].q; std::vector<double>& m = priors[l].m;
    q.assign(ldx, 1.0); m.assign(ldx, 0.0);
    for (int k = 0; k < Dg; k++) {
      q[k] = (!lm.empty() && lm[k] > 0.f) ? 1.0 / (1.0 / (double)lm[k]) : 1.0 / (1.0 / (double)lambda);
      m[k] = (double)prior_mean;
    }
    // without an intercept the bias column is 0 and its coefficient stays at 0
    q[Dg] = has_intercept ? (penalize_intercept ? 1.0 / (1.0 / (double)lambda) : 1.0 / 100000.0) : 1.0;
    m[Dg] = has_intercept ? (double)prior_mean : 0.0;
  }
  return keyed_fit(num_sms, (cudaStream_t)stream, K, Dg, key_rowstart, rowptr, colidx, vals, ldx_in, response, weight, offset, has_intercept != 0,
                   data_size_threshold, binary_feature, priors, nullptr, out_model, nullptr, skipped, sp);
}

// ------------------------------------------------------------------------------------------
// ItemModelTrain (jobs/ItemModelTrain.java:226-276): per key, one fit per (intercept lambda, default lambda) in config order, the
// intercept's prior mean the key's own; diagonal posterior variance on request.  Dense outputs, or (sp) the sparse lists, with (cv)
// the full posterior or (kp) per-key prior lists
// ------------------------------------------------------------------------------------------
int item_model_train(int32_t device, void* stream, int32_t K, int32_t Dg, const int64_t* key_rowstart, const int64_t* rowptr,
                     const int32_t* colidx, const float* vals, const int32_t* response, const float* weight, const float* offset,
                     const double* intercept_prior_mean, int32_t IL, const float* intercept_lambdas, int32_t DL,
                     const float* default_lambdas, const float* lambda_map, int32_t binary_feature, int32_t compute_var,
                     double* out_model, double* out_var, const SparseOut* sp, const CovOut* cv = nullptr,
                     const KeyPriorIn* kp = nullptr) {
  int num_sms = 0;
  if (int rc = keyed_fit_check(device, Dg, rowptr, colidx, 0, binary_feature, &num_sms)) return rc;
  std::vector<float> lm, il, dl;
  std::vector<double> im;
  if (int rc = host_copy(lambda_map, (size_t)Dg, lm)) return rc;
  if (int rc = host_copy(intercept_lambdas, (size_t)IL, il)) return rc;
  if (int rc = host_copy(default_lambdas, (size_t)DL, dl)) return rc;
  if (int rc = host_copy(intercept_prior_mean, (size_t)K, im)) return rc;
  // the reference divides by every lambda (:262) and turns lambda.map entries into variances 1/lambda (:205-206)
  for (float x : il) if (!(x > 0.f)) return fail(MLEASE_ERR_INVALID, "intercept.lambdas: every lambda must be > 0 (got " + std::to_string(x) + ")");
  for (float x : dl) if (!(x > 0.f)) return fail(MLEASE_ERR_INVALID, "default.lambdas: every lambda must be > 0 (got " + std::to_string(x) + ")");
  for (float x : lm) if (x < 0.f || x != x) return fail(MLEASE_ERR_INVALID, "lambda_map: entries must be > 0, or 0 for a feature without one");
  const int ldx = round_up(Dg + 1, 4);
  std::vector<KeyedPrior> priors((size_t)IL * DL);
  for (int a = 0; a < IL; a++)
    for (int b = 0; b < DL; b++) {
      // priorVar (:194-216, :262): 1/lambdaMap[k] for a listed feature, 1/interceptLambda for the intercept, 1/defaultLambda otherwise;
      // mean 0 except the intercept's (per key, intercept_prior_mean)
      std::vector<double>& q = priors[(size_t)a * DL + b].q; std::vector<double>& m = priors[(size_t)a * DL + b].m;
      q.assign(ldx, 1.0); m.assign(ldx, 0.0);
      for (int k = 0; k < Dg; k++) q[k] = (!lm.empty() && lm[k] > 0.f) ? 1.0 / (1.0 / (double)lm[k]) : 1.0 / (1.0 / (double)dl[b]);
      q[Dg] = 1.0 / (1.0 / (double)il[a]);
    }
  return keyed_fit(num_sms, (cudaStream_t)stream, K, Dg, key_rowstart, rowptr, colidx, vals, 0, response, weight, offset, true, 0, binary_feature,
                   priors, im.data(), out_model, compute_var ? out_var : nullptr, nullptr, sp, cv, kp);
}
}  // namespace

extern "C" {

int mlease_naive_train(int32_t device, void* stream, int32_t K, int32_t Dg, const int64_t* key_rowstart, const int64_t* rowptr,
                       const int32_t* colidx, const float* vals, int64_t ldx_in, const int32_t* response, const float* weight,
                       const float* offset, int32_t L, const float* lambdas, const float* lambda_map, float prior_mean,
                       int32_t penalize_intercept, int32_t has_intercept, int32_t data_size_threshold, int32_t binary_feature,
                       double* out_model, int32_t* skipped) {
  if (K <= 0 || Dg <= 0 || L <= 0 || !lambdas || !key_rowstart || !vals || !response || !out_model) return fail(MLEASE_ERR_INVALID, "bad argument");
  return naive_train(device, stream, K, Dg, key_rowstart, rowptr, colidx, vals, ldx_in, response, weight, offset, L, lambdas, lambda_map,
                     prior_mean, penalize_intercept, has_intercept, data_size_threshold, binary_feature, out_model, skipped, nullptr);
}

int mlease_naive_train_sparse(int32_t device, void* stream, int32_t K, int32_t Dg, const int64_t* key_rowstart, const int64_t* rowptr,
                              const int32_t* colidx, const float* vals, const int32_t* response, const float* weight, const float* offset,
                              int32_t L, const float* lambdas, const float* lambda_map, float prior_mean, int32_t penalize_intercept,
                              int32_t has_intercept, int32_t data_size_threshold, int32_t binary_feature, int64_t capacity,
                              int64_t* out_key_ptr, int32_t* out_col, double* out_model, int32_t* skipped) {
  if (K <= 0 || Dg <= 0 || L <= 0 || !lambdas || !key_rowstart || !rowptr || !colidx || !vals || !response || capacity < 0 || !out_key_ptr ||
      !out_col || !out_model)
    return fail(MLEASE_ERR_INVALID, "bad argument");
  const SparseOut sp{capacity, out_key_ptr, out_col};
  return naive_train(device, stream, K, Dg, key_rowstart, rowptr, colidx, vals, 0, response, weight, offset, L, lambdas, lambda_map,
                     prior_mean, penalize_intercept, has_intercept, data_size_threshold, binary_feature, out_model, skipped, &sp);
}

int mlease_item_model_train(int32_t device, void* stream, int32_t K, int32_t Dg, const int64_t* key_rowstart, const int64_t* rowptr,
                            const int32_t* colidx, const float* vals, const int32_t* response, const float* weight, const float* offset,
                            const double* intercept_prior_mean, int32_t IL, const float* intercept_lambdas, int32_t DL,
                            const float* default_lambdas, const float* lambda_map, int32_t binary_feature, int32_t compute_var,
                            double* out_model, double* out_var) {
  if (K <= 0 || Dg <= 0 || IL <= 0 || DL <= 0 || !intercept_lambdas || !default_lambdas || !key_rowstart || !rowptr || !vals || !response ||
      !intercept_prior_mean || !out_model || (compute_var && !out_var))
    return fail(MLEASE_ERR_INVALID, "bad argument");
  return item_model_train(device, stream, K, Dg, key_rowstart, rowptr, colidx, vals, response, weight, offset, intercept_prior_mean, IL,
                          intercept_lambdas, DL, default_lambdas, lambda_map, binary_feature, compute_var, out_model, out_var, nullptr);
}

int mlease_item_model_train_sparse(int32_t device, void* stream, int32_t K, int32_t Dg, const int64_t* key_rowstart, const int64_t* rowptr,
                                   const int32_t* colidx, const float* vals, const int32_t* response, const float* weight, const float* offset,
                                   const double* intercept_prior_mean, int32_t IL, const float* intercept_lambdas, int32_t DL,
                                   const float* default_lambdas, const float* lambda_map, int32_t binary_feature, int32_t compute_var,
                                   int64_t capacity, int64_t* out_key_ptr, int32_t* out_col, double* out_model, double* out_var) {
  if (K <= 0 || Dg <= 0 || IL <= 0 || DL <= 0 || !intercept_lambdas || !default_lambdas || !key_rowstart || !rowptr || !colidx || !vals ||
      !response || !intercept_prior_mean || capacity < 0 || !out_key_ptr || !out_col || !out_model || (compute_var && !out_var))
    return fail(MLEASE_ERR_INVALID, "bad argument");
  const SparseOut sp{capacity, out_key_ptr, out_col};
  return item_model_train(device, stream, K, Dg, key_rowstart, rowptr, colidx, vals, response, weight, offset, intercept_prior_mean, IL,
                          intercept_lambdas, DL, default_lambdas, lambda_map, binary_feature, compute_var, out_model, out_var, &sp);
}

int mlease_item_model_train_cov(int32_t device, void* stream, int32_t K, int32_t Dg, const int64_t* key_rowstart, const int64_t* rowptr,
                                const int32_t* colidx, const float* vals, const int32_t* response, const float* weight, const float* offset,
                                const double* intercept_prior_mean, int32_t IL, const float* intercept_lambdas, int32_t DL,
                                const float* default_lambdas, const float* lambda_map, int32_t binary_feature, int64_t capacity,
                                int64_t* out_key_ptr, int32_t* out_col, double* out_model, double* out_var, int64_t cov_capacity,
                                int64_t* out_cov_ptr, double* out_cov) {
  if (K <= 0 || Dg <= 0 || IL <= 0 || DL <= 0 || !intercept_lambdas || !default_lambdas || !key_rowstart || !rowptr || !colidx || !vals ||
      !response || !intercept_prior_mean || capacity < 0 || !out_key_ptr || !out_col || !out_model || !out_var ||
      (out_cov && (cov_capacity < 0 || !out_cov_ptr)))
    return fail(MLEASE_ERR_INVALID, "bad argument");
  const SparseOut sp{capacity, out_key_ptr, out_col};
  const CovOut cv{cov_capacity, out_cov ? out_cov_ptr : nullptr, out_cov};
  return item_model_train(device, stream, K, Dg, key_rowstart, rowptr, colidx, vals, response, weight, offset, intercept_prior_mean, IL,
                          intercept_lambdas, DL, default_lambdas, lambda_map, binary_feature, 1, out_model, out_var, &sp, &cv);
}

int mlease_item_model_train_prior(int32_t device, void* stream, int32_t K, int32_t Dg, const int64_t* key_rowstart, const int64_t* rowptr,
                                  const int32_t* colidx, const float* vals, const int32_t* response, const float* weight, const float* offset,
                                  const double* intercept_prior_mean, int32_t IL, const float* intercept_lambdas, int32_t DL,
                                  const float* default_lambdas, const float* lambda_map, int32_t binary_feature, int32_t compute_var,
                                  int64_t capacity, int64_t* out_key_ptr, int32_t* out_col, double* out_model, double* out_var,
                                  const int64_t* prior_ptr, const int32_t* prior_col, const double* prior_mean, const double* prior_var) {
  if (K <= 0 || Dg <= 0 || IL <= 0 || DL <= 0 || !intercept_lambdas || !default_lambdas || !key_rowstart || !rowptr || !colidx || !vals ||
      !response || !intercept_prior_mean || capacity < 0 || !out_key_ptr || !out_col || !out_model || (compute_var && !out_var) ||
      !prior_ptr || !prior_col || !prior_mean || !prior_var)
    return fail(MLEASE_ERR_INVALID, "bad argument");
  const SparseOut sp{capacity, out_key_ptr, out_col};
  const KeyPriorIn kp{prior_ptr, prior_col, prior_mean, prior_var};
  return item_model_train(device, stream, K, Dg, key_rowstart, rowptr, colidx, vals, response, weight, offset, intercept_prior_mean, IL,
                          intercept_lambdas, DL, default_lambdas, lambda_map, binary_feature, compute_var, out_model, out_var, &sp, nullptr, &kp);
}

int mlease_naive_train_dense(int32_t device, void* stream, int32_t K, int32_t Dg, const int64_t* key_rowstart, const float* X, int64_t ldx_in,
                             const int32_t* response, const float* weight, const float* offset, float lambda, const float* lambda_map,
                             float prior_mean, int32_t penalize_intercept, int32_t has_intercept, int32_t data_size_threshold,
                             double* out_model, int32_t* skipped) {
  return mlease_naive_train(device, stream, K, Dg, key_rowstart, nullptr, nullptr, X, ldx_in, response, weight, offset, 1, &lambda, lambda_map,
                            prior_mean, penalize_intercept, has_intercept, data_size_threshold, 0, out_model, skipped);
}

}  // extern "C"
