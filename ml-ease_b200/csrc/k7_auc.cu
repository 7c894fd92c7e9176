// k7_auc.cu -- mlease_test_auc: the weighted ROC AUC (Mann-Whitney U, tied pairs count 1/2) of every set of predictions, and of
// every (set, key) pair, on the GPU.
//
// Per set: the rows' predictions become 32-bit orderable keys (-0.0 folded onto +0.0) and one device-wide stable radix sort
// (4 passes) puts the set's rows in (pred, row) order.  For per-key results a second stable radix sort of the rows' key ids
// (ceil(log2 K) bits) carries the (pred key, row) pairs of that order, which leaves them in (key, pred, row) order: a key's rows
// come out where they went in, at [krs[k], krs[k+1]), so segment boundaries are known without a search.
//
// U, P and N of a segment are a fold of the segment's records in sorted order under the associative summary of auc_sum(): tiles of
// AUC_TILE records start at the segment's start, one warp folds a tile (each lane a contiguous run of records, then a fixed shuffle
// tree), and one warp per segment folds its tiles the same way.  Every association depends only on the segment's length, so an
// AUC is bitwise the same whatever other keys or sets share the call, and from run to run.  No atomics and no decoupled look-back
// touch a floating-point value.
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "host.cuh"

namespace mlease {
namespace {

constexpr int AUC_LANE = 32;                    // records a lane folds in a tile
constexpr int AUC_TILE = 32 * AUC_LANE;         // records of one tile (one warp)

// The summary of a run of records in ascending prediction order: positive / negative weight P, N, the U of the pairs inside it,
// the weights of its first and last tie group (Pf, Nf, Pl, Nl) with their keys vf, vl, whether it is one tie group, and empty.
struct AucSum {
  double P, N, U, Pf, Nf, Pl, Nl;
  unsigned vf, vl;
  int single, empty;
};

__device__ __forceinline__ AucSum auc_empty() { AucSum s{}; s.empty = 1; return s; }

// A followed by B (every key of A <= every key of B): B's positives beat A's negatives, except the pairs of a tie group that spans
// the boundary, which count 1/2 either way.
__device__ __forceinline__ AucSum auc_sum(const AucSum& a, const AucSum& b) {
  if (a.empty) return b;
  if (b.empty) return a;
  const bool eq = a.vl == b.vf;
  AucSum r;
  r.U = a.U + b.U + (eq ? (b.P * a.N - 0.5 * b.Pf * a.Nl) + 0.5 * a.Pl * b.Nf : b.P * a.N);
  r.P = a.P + b.P;
  r.N = a.N + b.N;
  if (a.single && eq) { r.Pf = a.Pf + b.Pf; r.Nf = a.Nf + b.Nf; } else { r.Pf = a.Pf; r.Nf = a.Nf; }
  if (b.single && eq) { r.Pl = a.Pl + b.Pl; r.Nl = a.Nl + b.Nl; } else { r.Pl = b.Pl; r.Nl = b.Nl; }
  r.vf = a.vf; r.vl = b.vl;
  r.single = a.single && b.single && eq;
  r.empty = 0;
  return r;
}

__device__ __forceinline__ AucSum auc_leaf(unsigned v, float lw) {
  const double w = fabs((double)lw);
  AucSum s;
  s.P = signbit(lw) ? 0.0 : w; s.N = signbit(lw) ? w : 0.0; s.U = 0.0;
  s.Pf = s.Pl = s.P; s.Nf = s.Nl = s.N;
  s.vf = s.vl = v; s.single = 1; s.empty = 0;
  return s;
}

__device__ __forceinline__ AucSum auc_shfl_down(const AucSum& s, int o) {
  AucSum r;
  r.P = __shfl_down_sync(0xffffffffu, s.P, o); r.N = __shfl_down_sync(0xffffffffu, s.N, o);
  r.U = __shfl_down_sync(0xffffffffu, s.U, o);
  r.Pf = __shfl_down_sync(0xffffffffu, s.Pf, o); r.Nf = __shfl_down_sync(0xffffffffu, s.Nf, o);
  r.Pl = __shfl_down_sync(0xffffffffu, s.Pl, o); r.Nl = __shfl_down_sync(0xffffffffu, s.Nl, o);
  r.vf = __shfl_down_sync(0xffffffffu, s.vf, o); r.vl = __shfl_down_sync(0xffffffffu, s.vl, o);
  r.single = __shfl_down_sync(0xffffffffu, s.single, o); r.empty = __shfl_down_sync(0xffffffffu, s.empty, o);
  return r;
}

// lane 0 gets lane 0's run, then lane 1's, ... in order: at each step lane l (a multiple of 2o) adds the contiguous run of lane l + o
__device__ __forceinline__ AucSum auc_warp_fold(AucSum s) {
  const int lane = threadIdx.x & 31;
  for (int o = 1; o < 32; o <<= 1) {
    const AucSum t = auc_shfl_down(s, o);
    if ((lane & (2 * o - 1)) == 0 && lane + o < 32) s = auc_sum(s, t);
  }
  return s;
}

// Where the records of a pass come from: ROWS the rows in row order with one tie group (weights only), SORTED the set sort's keys
// and rows, PACKED the key sort's (key << 32 | row) pairs.
enum { SRC_ROWS = 0, SRC_SORTED = 1, SRC_PACKED = 2 };

template <int SRC>
__device__ __forceinline__ AucSum auc_record(long long q, const unsigned* skey, const int* srow, const unsigned long long* spk,
                                             const float* lw) {
  if (SRC == SRC_ROWS) return auc_leaf(0u, lw[q]);
  if (SRC == SRC_SORTED) return auc_leaf(skey[q], lw[srow[q]]);
  const unsigned long long p = spk[q];
  return auc_leaf((unsigned)(p >> 32), lw[(int)(unsigned)p]);
}

// one warp per tile: tile t covers [tile_start[t], min(tile_start[t] + AUC_TILE, seg_end[tile_seg[t]])) of the pass's records
template <int SRC>
__global__ void __launch_bounds__(256) auc_tile_kernel(long long ntiles, const long long* __restrict__ tile_start,
                                                       const int* __restrict__ tile_seg, const long long* __restrict__ seg_end,
                                                       const unsigned* __restrict__ skey, const int* __restrict__ srow,
                                                       const unsigned long long* __restrict__ spk, const float* __restrict__ lw,
                                                       AucSum* __restrict__ out) {
  const long long t = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (t >= ntiles) return;
  const int lane = threadIdx.x & 31;
  const long long end = min(tile_start[t] + AUC_TILE, seg_end[tile_seg[t]]);
  const long long lo = tile_start[t] + (long long)lane * AUC_LANE, hi = min(lo + AUC_LANE, end);
  AucSum s = auc_empty();
  for (long long q = lo; q < hi; q++) s = auc_sum(s, auc_record<SRC>(q, skey, srow, spk, lw));
  s = auc_warp_fold(s);
  if (lane == 0) out[t] = s;
}

// one warp per segment over its tiles [seg_t0[g], seg_t0[g + 1]): auc[g] = U / (P N) (NaN when P or N is 0); pn[2g], pn[2g + 1] =
// P, N when pn is not NULL
__global__ void __launch_bounds__(256) auc_segment_kernel(int nseg, const long long* __restrict__ seg_t0, const AucSum* __restrict__ tiles,
                                                          double* __restrict__ auc, double* __restrict__ pn) {
  const long long g = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (g >= nseg) return;
  const int lane = threadIdx.x & 31;
  const long long t0 = seg_t0[g], nt = seg_t0[g + 1] - t0, per = (nt + 31) / 32;
  const long long lo = t0 + min(nt, lane * per), hi = t0 + min(nt, (lane + 1) * per);
  AucSum s = auc_empty();
  for (long long t = lo; t < hi; t++) s = auc_sum(s, tiles[t]);
  s = auc_warp_fold(s);
  if (lane == 0) {
    const bool def = !s.empty && s.P > 0.0 && s.N > 0.0;
    if (auc) auc[g] = def ? s.U / (s.P * s.N) : __longlong_as_double(0x7ff8000000000000LL);
    if (pn) { pn[2 * g] = s.empty ? 0.0 : s.P; pn[2 * g + 1] = s.empty ? 0.0 : s.N; }
  }
}

// the checks of the shared row inputs: bad bit 1 = a response other than 1, 0, -1; bit 2 = a negative or NaN weight.  lw[i] = the
// row's weight, negated for a negative (the sign bit is the label, so a zero weight of either label adds nothing); kid[i] = the
// row's key (upper bound in krs - 1), if kid is not NULL
__global__ void auc_rows_kernel(long long n, const int* __restrict__ response, const float* __restrict__ weight, int nkeys,
                                const long long* __restrict__ krs, float* __restrict__ lw, int* __restrict__ kid, int* __restrict__ bad) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = response[i];
  const float w = weight ? weight[i] : 1.f;
  int b = 0;
  if (r != 1 && r != 0 && r != -1) b |= 1;
  if (!(w >= 0.f)) b |= 2;
  if (b) atomicOr(bad, b);
  lw[i] = r == 1 ? fabsf(w) : -fabsf(w);
  if (kid) {
    int lo = 0, hi = nkeys - 1;   // the last k with krs[k] <= i: krs[k + 1] > i, so row i is key k's
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (krs[mid] <= i) lo = mid; else hi = mid - 1; }
    kid[i] = lo;
  }
}

// one set: key[i] = the orderable bits of pred[i] (+0.0 for -0.0; a NaN sets bad bit 4), row[i] = i
__global__ void auc_keys_kernel(long long n, const float* __restrict__ pred, unsigned* __restrict__ key, int* __restrict__ row,
                                int* __restrict__ bad) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float p = pred[i];
  if (p != p) atomicOr(bad, 4);
  const unsigned u = p == 0.f ? 0u : __float_as_uint(p);
  key[i] = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  row[i] = (int)i;
}

// the key sort's input, in the set's sorted order: kq[q] = kid[row], pk[q] = key << 32 | row
__global__ void auc_pack_kernel(long long n, const unsigned* __restrict__ skey, const int* __restrict__ srow, const int* __restrict__ kid,
                                int* __restrict__ kq, unsigned long long* __restrict__ pk) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  const int r = srow[q];
  kq[q] = kid[r];
  pk[q] = ((unsigned long long)skey[q] << 32) | (unsigned)r;
}

// The tiles of a list of segments [start[g], end[g]) of one pass, host side: seg_t0 (nseg + 1), tile_start, tile_seg.
struct SegPlan {
  std::vector<long long> end, tile_start;
  std::vector<long long> t0{0};
  std::vector<int> tile_seg;
  void add(long long a, long long b) {
    for (long long q = a; q < b; q += AUC_TILE) { tile_start.push_back(q); tile_seg.push_back((int)end.size()); }
    end.push_back(b);
    t0.push_back((long long)tile_start.size());
  }
  int nseg() const { return (int)end.size(); }
  long long ntiles() const { return (long long)tile_start.size(); }
};

// the plan on the device
struct DevPlan {
  long long ntiles = 0;
  int nseg = 0;
  const long long *tile_start = nullptr, *end = nullptr, *t0 = nullptr;
  const int* tile_seg = nullptr;
};

int upload_plan(DevMem& mem, const SegPlan& p, DevPlan* d, cudaStream_t st) {
  d->ntiles = p.ntiles(); d->nseg = p.nseg();
  if (int rc = to_device(mem, p.tile_start.data(), p.tile_start.size(), &d->tile_start, st)) return rc;
  if (int rc = to_device(mem, p.end.data(), p.end.size(), &d->end, st)) return rc;
  if (int rc = to_device(mem, p.tile_seg.data(), p.tile_seg.size(), &d->tile_seg, st)) return rc;
  if (int rc = to_device(mem, p.t0.data(), p.t0.size(), &d->t0, st)) return rc;
  return 0;
}

// one pass: every segment of the plan folded from src; results as auc_segment_kernel writes them
template <int SRC>
cudaError_t auc_pass(const DevPlan& p, const unsigned* skey, const int* srow, const unsigned long long* spk, const float* lw,
                     AucSum* d_tiles, double* auc, double* pn, cudaStream_t st) {
  if (p.ntiles > 0)
    auc_tile_kernel<SRC><<<(unsigned)((p.ntiles + 7) / 8), 256, 0, st>>>(p.ntiles, p.tile_start, p.tile_seg, p.end, skey, srow, spk,
                                                                          lw, d_tiles);
  if (p.nseg > 0) auc_segment_kernel<<<(unsigned)((p.nseg + 7) / 8), 256, 0, st>>>(p.nseg, p.t0, d_tiles, auc, pn);
  return cudaGetLastError();
}

}  // namespace
}  // namespace mlease

using namespace mlease;

extern "C" {

int mlease_test_auc(int32_t device, void* stream, int64_t n, int32_t num_sets, const float* pred, const int32_t* response,
                    const float* weight, int32_t num_keys, const int64_t* key_rowstart, double* out_auc, double* out_weight,
                    double* out_key_auc, double* out_key_weight) {
  if (n < 1 || n > INT32_MAX) return fail(MLEASE_ERR_INVALID, "nrows must be in [1, 2^31 - 1]");
  if (num_sets < 1) return fail(MLEASE_ERR_INVALID, "num_sets must be >= 1");
  if (!pred || !response) return fail(MLEASE_ERR_INVALID, "pred and response are required");
  if (num_keys < 0 || (num_keys > 0 && !key_rowstart)) return fail(MLEASE_ERR_INVALID, "key_rowstart must have num_keys + 1 entries");
  if (!out_auc && !out_key_auc) return fail(MLEASE_ERR_INVALID, "out_auc and out_key_auc are both NULL: nothing to compute");
  if (int rc = open_device(device, nullptr)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int K = num_keys, S = num_sets;
  std::vector<long long> krs(K + 1, 0);
  krs[K] = n;
  if (K > 0) {
    CK(cudaMemcpy(krs.data(), key_rowstart, (size_t)(K + 1) * 8, cudaMemcpyDefault));
    if (krs[0] != 0) return fail(MLEASE_ERR_INVALID, "key_rowstart must start at 0");
    for (int k = 0; k < K; k++)
      if (krs[k + 1] < krs[k]) return fail(MLEASE_ERR_INVALID, "key_rowstart decreases at key " + std::to_string(k));
    if (krs[K] != n) return fail(MLEASE_ERR_INVALID, "key_rowstart must end at nrows");
  }
  const bool want_set = out_auc != nullptr, want_key = out_key_auc != nullptr && K > 0;
  SegPlan all, keys;
  all.add(0, n);
  for (int k = 0; k < K; k++) keys.add(krs[k], krs[k + 1]);
  int key_bits = 1;
  while (key_bits < 31 && ((long long)K - 1) >> key_bits) key_bits++;

  // device bytes: what every set shares, then what each set of a chunk adds (its predictions, when they come from the host)
  const size_t un = (size_t)n;
  size_t tmp_set = 0, tmp_key = 0;
  CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_set, (unsigned*)nullptr, (unsigned*)nullptr, (int*)nullptr, (int*)nullptr, (int)n, 0, 32, st));
  if (want_key)
    CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_key, (int*)nullptr, (int*)nullptr, (unsigned long long*)nullptr,
                                       (unsigned long long*)nullptr, (int)n, 0, key_bits, st));
  const long long max_tiles = std::max(all.ntiles(), keys.ntiles());
  const size_t fixed = (is_device_ptr(response) ? 0 : 4 * un) + (weight && !is_device_ptr(weight) ? 4 * un : 0) + 4 * un /* lw */ +
                       16 * un /* set sort keys and rows, in and out */ + (want_key ? 4 * un /* kid */ + 16 * un /* pk in, out */ : 0) +
                       std::max(tmp_set, tmp_key) + (size_t)max_tiles * sizeof(AucSum) +
                       (size_t)(all.ntiles() + keys.ntiles()) * 12 + (size_t)(2 * K + 4) * 16 + (size_t)(K + 1) * 24 + 4096;
  const size_t per_set = (is_device_ptr(pred) ? 0 : 4 * un) + (size_t)(K + 1) * 8;
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  const size_t budget = keyed_budget(free_b);
  if (fixed + per_set > budget)
    return fail(MLEASE_ERR_INVALID, "mlease_test_auc: one set needs " + std::to_string(fixed + per_set) + " device bytes, " +
                                        std::to_string(budget) + " are available");
  const int chunk = (int)std::min<size_t>((size_t)S, (budget - fixed) / per_set);

  DevMem t;
  const int *d_resp; const float* d_w;
  if (int rc = to_device(t, (const int*)response, un, &d_resp, st)) return rc;
  if (int rc = to_device(t, weight, un, &d_w, st)) return rc;
  const long long* d_krs = nullptr;
  if (int rc = to_device(t, krs.data(), krs.size(), &d_krs, st)) return rc;
  DevPlan p_all, p_keys;
  if (int rc = upload_plan(t, all, &p_all, st)) return rc;
  if (int rc = upload_plan(t, keys, &p_keys, st)) return rc;
  float* d_lw; int *d_kid = nullptr, *d_bad; unsigned *d_key, *d_skey; int *d_row, *d_srow; unsigned long long *d_pk = nullptr, *d_spk = nullptr;
  AucSum* d_tiles; char* d_tmp; double *d_out, *d_pn;
  if (int rc = t.get(&d_lw, un, false)) return rc;
  if (int rc = t.get(&d_bad, 1, true)) return rc;
  if (int rc = t.get(&d_key, un, false)) return rc;
  if (int rc = t.get(&d_skey, un, false)) return rc;
  if (int rc = t.get(&d_row, un, false)) return rc;
  if (int rc = t.get(&d_srow, un, false)) return rc;
  if (want_key) {
    if (int rc = t.get(&d_kid, un, false)) return rc;
    if (int rc = t.get(&d_pk, un, false)) return rc;
    if (int rc = t.get(&d_spk, un, false)) return rc;
  }
  if (int rc = t.get(&d_tiles, (size_t)std::max<long long>(max_tiles, 1), false)) return rc;
  if (int rc = t.get(&d_tmp, std::max(tmp_set, tmp_key), false)) return rc;
  if (int rc = t.get(&d_out, (size_t)chunk * (K + 1), false)) return rc;
  if (int rc = t.get(&d_pn, (size_t)2 * (K + 1), false)) return rc;
  float* d_chunk = nullptr;
  if (!is_device_ptr(pred))
    if (int rc = t.get(&d_chunk, (size_t)chunk * un, false)) return rc;

  // the rows' checks come back before any set is touched
  const unsigned rblocks = (unsigned)((n + 255) / 256);
  auc_rows_kernel<<<rblocks, 256, 0, st>>>(n, d_resp, d_w, K, d_krs, d_lw, d_kid, d_bad);
  CK(cudaGetLastError());
  int bad = 0;
  CK(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (bad & 1) return fail(MLEASE_ERR_INVALID, "response should be 1,0 or -1!");
  if (bad & 2) return fail(MLEASE_ERR_INVALID, "weight must be >= 0 and not NaN");

  // the weights, in row order (one tie group): over all rows, and per key
  std::vector<double> w_all(2, 0.0), w_key((size_t)2 * K, 0.0);
  CK(auc_pass<SRC_ROWS>(p_all, nullptr, nullptr, nullptr, d_lw, d_tiles, nullptr, d_pn, st));
  CK(cudaMemcpyAsync(w_all.data(), d_pn, 16, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (K > 0) {
    CK(auc_pass<SRC_ROWS>(p_keys, nullptr, nullptr, nullptr, d_lw, d_tiles, nullptr, d_pn, st));
    CK(cudaMemcpyAsync(w_key.data(), d_pn, (size_t)16 * K, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }

  std::vector<double> auc_h(want_set ? (size_t)S : 0), kauc_h(want_key ? (size_t)S * K : 0);
  std::vector<long long> bounds{0};
  for (int s0 = 0; s0 < S; s0 += chunk) {
    const int s1 = std::min(S, s0 + chunk);
    const float* d_pred = pred + (size_t)s0 * un;
    if (d_chunk) {
      CK(cudaMemcpyAsync(d_chunk, d_pred, (size_t)(s1 - s0) * un * 4, cudaMemcpyHostToDevice, st));
      d_pred = d_chunk;
    }
    for (int s = s0; s < s1; s++) {
      double* o = d_out + (size_t)(s - s0) * (K + 1);
      auc_keys_kernel<<<rblocks, 256, 0, st>>>(n, d_pred + (size_t)(s - s0) * un, d_key, d_row, d_bad);
      CK(cudaGetLastError());
      size_t tb = tmp_set;
      CK(cub::DeviceRadixSort::SortPairs(d_tmp, tb, d_key, d_skey, d_row, d_srow, (int)n, 0, 32, st));
      if (want_set) CK(auc_pass<SRC_SORTED>(p_all, d_skey, d_srow, nullptr, d_lw, d_tiles, o, nullptr, st));
      if (want_key) {
        int* d_kq = (int*)d_key;   // the set sort's inputs are free again
        int* d_skq = d_row;
        auc_pack_kernel<<<rblocks, 256, 0, st>>>(n, d_skey, d_srow, d_kid, d_kq, d_pk);
        CK(cudaGetLastError());
        tb = tmp_key;
        CK(cub::DeviceRadixSort::SortPairs(d_tmp, tb, d_kq, d_skq, d_pk, d_spk, (int)n, 0, key_bits, st));
        CK(auc_pass<SRC_PACKED>(p_keys, nullptr, nullptr, d_spk, d_lw, d_tiles, o + 1, nullptr, st));
      }
    }
    CK(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, st));
    std::vector<double> h((size_t)(s1 - s0) * (K + 1));
    CK(cudaMemcpyAsync(h.data(), d_out, h.size() * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (bad & 4) return fail(MLEASE_ERR_INVALID, "pred holds NaN");
    for (int s = s0; s < s1; s++) {
      const double* hs = h.data() + (size_t)(s - s0) * (K + 1);
      if (want_set) auc_h[s] = hs[0];
      if (want_key) std::copy(hs + 1, hs + 1 + K, kauc_h.begin() + (size_t)s * K);
    }
    bounds.push_back(s1);
  }
  keyed_record(bounds, bounds.size() > 2, 0.0, 0.0);
  if (out_auc) std::copy(auc_h.begin(), auc_h.end(), out_auc);
  if (out_weight) std::copy(w_all.begin(), w_all.end(), out_weight);
  if (out_key_auc && K > 0) std::copy(kauc_h.begin(), kauc_h.end(), out_key_auc);
  if (out_key_weight && K > 0) std::copy(w_key.begin(), w_key.end(), out_key_weight);
  return 0;
}

}  // extern "C"
