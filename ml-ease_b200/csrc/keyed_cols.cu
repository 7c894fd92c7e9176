// keyed_cols.cu -- the column space of each key of a keyed CSR fit: its sorted distinct column list (a segmented sort over the key
// boundaries, then a run-length pass) and the key-local column index of every stored entry.
#include <climits>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>

#include <algorithm>
#include <vector>

#include "host.cuh"

namespace mlease {

namespace {

// entries sorted per pass: bounds the pass's temporaries (key_columns_bytes); a larger key is sorted on its own
constexpr long long KC_SLAB = 1LL << 28;

int kc_grid(long long n) { return (int)std::max<long long>(1, std::min<long long>((n + 255) / 256, 4096)); }

// head[j] = 1 where a run of equal columns starts in the sorted slab, head[s] = 0 (the scan's total)
__global__ void kc_run_heads_kernel(long long s, const int* __restrict__ sorted, long long* __restrict__ head) {
  for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j <= s; j += (long long)gridDim.x * blockDim.x)
    head[j] = j == s ? 0 : ((j == 0 || sorted[j] != sorted[j - 1]) ? 1 : 0);
}
// every key with entries starts a run, even when its first column equals the previous key's last
__global__ void kc_key_heads_kernel(int nk, const int* __restrict__ offs, long long* __restrict__ head) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nk && offs[i] < offs[i + 1]) head[offs[i]] = 1;
}
// pos: exclusive scan of the heads, so pos[j] is the run of entry j and the runs of key i are [pos[offs[i]], pos[offs[i + 1]])
__global__ void kc_compact_kernel(long long s, const int* __restrict__ sorted, const long long* __restrict__ pos, int* __restrict__ cols) {
  for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j < s; j += (long long)gridDim.x * blockDim.x)
    if (pos[j + 1] != pos[j]) cols[pos[j]] = sorted[j];
}
__global__ void kc_key_start_kernel(int nk, const int* __restrict__ offs, const long long* __restrict__ pos, long long* __restrict__ start) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= nk) start[i] = pos[offs[i]];
}
// one CTA per key: lci[j] = the index of ci[j] in its key's ascending list (a lower bound; the column is always there)
__global__ void kc_local_index_kernel(const int* __restrict__ offs, const long long* __restrict__ start, const int* __restrict__ cols,
                                      const int* __restrict__ ci, int* __restrict__ lci) {
  const int k = blockIdx.x;
  const int* c = cols + start[k];
  const int dk = (int)(start[k + 1] - start[k]);
  for (long long j = offs[k] + (long long)threadIdx.x; j < offs[k + 1]; j += blockDim.x) {   // 64-bit: offs may reach INT_MAX
    const int x = ci[j];
    int lo = 0, hi = dk;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (c[mid] < x) lo = mid + 1; else hi = mid; }
    lci[j] = lo;
  }
}

}  // namespace

size_t key_columns_bytes(long long nnz, long long max_key_nnz, int nkeys) {
  const long long slab = std::min(nnz, std::max(KC_SLAB, max_key_nnz));
  // the lists and lci (8 B an entry), the sorted slab, its run offsets and CUB's copy of the keys (~16 B an entry), per-key offsets
  return (size_t)nnz * 8 + (size_t)slab * 24 + (size_t)nkeys * 32;
}

int key_columns(cudaStream_t st, DevMem& mem, const std::vector<long long>& koff, const int* ci, KeyCols* kc) {
  const int nk = (int)koff.size() - 1;
  const long long nnz = koff[nk];
  kc->start.assign((size_t)nk + 1, 0);
  kc->listed.assign((size_t)nk, 1);
  if (int rc = mem.get(&kc->d_cols, (size_t)nnz, false)) return rc;
  if (int rc = mem.get(&kc->d_lci, (size_t)nnz, false)) return rc;
  long long ubase = 0;
  std::vector<long long> ks;
  for (int k0 = 0; k0 < nk;) {
    int k1 = k0 + 1;
    while (k1 < nk && koff[k1 + 1] - koff[k0] <= KC_SLAB) k1++;
    const long long e0 = koff[k0], s = koff[k1] - e0;
    const int ns = k1 - k0;
    if (s > INT_MAX) {   // one key of more entries than one sort takes: no list, it keeps the global width
      kc->listed[k0] = 0;
      kc->start[k0 + 1] = ubase;
      k0 = k1;
      continue;
    }
    if (s == 0) {
      for (int i = 1; i <= ns; i++) kc->start[k0 + i] = ubase;
      k0 = k1;
      continue;
    }
    DevMem t;   // the slab's temporaries
    std::vector<int> offs((size_t)ns + 1);
    for (int i = 0; i <= ns; i++) offs[i] = (int)(koff[k0 + i] - e0);
    int *d_offs, *sorted; long long *pos, *d_ks;
    if (int rc = t.get(&d_offs, offs.size(), false)) return rc;
    if (int rc = t.get(&sorted, (size_t)s, false)) return rc;
    if (int rc = t.get(&pos, (size_t)s + 1, false)) return rc;
    if (int rc = t.get(&d_ks, (size_t)ns + 1, false)) return rc;
    CK(cudaMemcpyAsync(d_offs, offs.data(), offs.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    size_t sort_b = 0, scan_b = 0;
    CK(cub::DeviceSegmentedSort::SortKeys(nullptr, sort_b, ci + e0, sorted, (int)s, ns, d_offs, d_offs + 1, st));
    CK(cub::DeviceScan::ExclusiveSum(nullptr, scan_b, pos, pos, s + 1, st));
    char* tmp;
    if (int rc = t.get(&tmp, std::max(sort_b, scan_b), false)) return rc;
    CK(cub::DeviceSegmentedSort::SortKeys(tmp, sort_b, ci + e0, sorted, (int)s, ns, d_offs, d_offs + 1, st));
    kc_run_heads_kernel<<<kc_grid(s + 1), 256, 0, st>>>(s, sorted, pos);
    kc_key_heads_kernel<<<(ns + 255) / 256, 256, 0, st>>>(ns, d_offs, pos);
    CK(cub::DeviceScan::ExclusiveSum(tmp, scan_b, pos, pos, s + 1, st));
    kc_compact_kernel<<<kc_grid(s), 256, 0, st>>>(s, sorted, pos, kc->d_cols + ubase);
    kc_key_start_kernel<<<(ns + 256) / 256, 256, 0, st>>>(ns, d_offs, pos, d_ks);
    kc_local_index_kernel<<<ns, 256, 0, st>>>(d_offs, d_ks, kc->d_cols + ubase, ci + e0, kc->d_lci + e0);
    CK(cudaGetLastError());
    ks.resize((size_t)ns + 1);
    CK(cudaMemcpyAsync(ks.data(), d_ks, ks.size() * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (int i = 1; i <= ns; i++) kc->start[k0 + i] = ubase + ks[i];
    ubase += ks[ns];
    k0 = k1;
  }
  kc->cols.resize((size_t)ubase);
  CK(cudaMemcpyAsync(kc->cols.data(), kc->d_cols, (size_t)ubase * sizeof(int), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return 0;
}

}  // namespace mlease
