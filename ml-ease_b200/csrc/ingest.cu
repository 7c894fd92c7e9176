// ingest.cu -- data into device memory: labels, CSR checks, dense rows into the padded layout, and the derived lists of an
// uploaded CSR partition.  Shared by the session upload and the keyed fits.
#include <algorithm>
#include <cstring>
#include <string>

#include "host.cuh"

namespace mlease {

namespace {

__global__ void fill_bias_pad_kernel(float* X, long long n, int ldx, int Dg, int has_bias) {
  const int npad = ldx - Dg;
  const long long total = n * npad;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long i = e / npad;
    const int c = Dg + (int)(e % npad);
    X[i * ldx + c] = (c == Dg && has_bias) ? 1.0f : 0.0f;
  }
}
// response {1,0,-1} -> int8 {+1,-1,-1} (llf/LibLinearDataset.java:419-422); weight >= 0 (:428-429)
__global__ void convert_labels_kernel(long long n, const int* resp, const float* w_in, const float* o_in, signed char* y, float* w,
                                      float* o, int* bad) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int r = resp[i];
    if (r != 1 && r != 0 && r != -1) atomicOr(bad, 1);
    y[i] = (r == 1) ? 1 : -1;
    const float ww = w_in ? w_in[i] : 1.0f;
    if (!(ww >= 0.f)) atomicOr(bad, 2);
    w[i] = ww;
    o[i] = o_in ? o_in[i] : 0.0f;
  }
}
// rowptr[0] >= 0 and rowptr[i] <= rowptr[i + 1]: reads the n + 1 row pointers only, so it is safe on any rowptr
__global__ void check_rowptr_kernel(long long n, const long long* rowptr, int* bad) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t == 0 && rowptr[0] < 0) atomicOr(bad, 1);
  for (long long i = t; i < n; i += (long long)gridDim.x * blockDim.x)
    if (rowptr[i + 1] < rowptr[i]) { atomicOr(bad, 1); break; }
}
__global__ void check_rows_sorted_kernel(long long n, const long long* rowptr, const int* colidx, int* bad) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    for (long long j = rowptr[i] + 1; j < rowptr[i + 1]; j++)
      if (colidx[j] <= colidx[j - 1]) { atomicOr(bad, 8); break; }
}
// max |a[i]| as the bit pattern of a non-negative float (order preserving), NaN ignored
__global__ void absmax_kernel(long long n, const float* __restrict__ a, unsigned* __restrict__ out) {
  float m = 0.f;
  for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (long long)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(a[j]));
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));
}
// sum over rows of (k_i + 1)(k_i + 2) / 2 (k_i stored values plus the intercept): the products, lower triangle, of one sparse
// CSR Gram build
__global__ void csr_gram_pairs_kernel(long long n, const long long* __restrict__ rowptr, unsigned long long* __restrict__ out) {
  unsigned long long s = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = (unsigned long long)(rowptr[i + 1] - rowptr[i]);
    s += (k + 1) * (k + 2) / 2;
  }
  for (int d = 16; d > 0; d >>= 1) s += __shfl_down_sync(0xffffffffu, s, d);
  if ((threadIdx.x & 31) == 0) atomicAdd(out, s);
}
__global__ void check_csr_kernel(long long nnz, const int* colidx, float* vals, int Dg, int binary, int* bad) {
  for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < nnz; j += (long long)gridDim.x * blockDim.x) {
    const int c = colidx[j];
    if (c < 0 || c >= Dg) atomicOr(bad, 4);
    if (binary) vals[j] = 1.0f;
  }
}
__global__ void gather_i64_kernel(const long long* src, const long long* idx, int n, long long* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = src[idx[i]];
}
__global__ void rebase_rowptr_kernel(long long n, const long long* src, long long base, long long* dst) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (long long)gridDim.x * blockDim.x) dst[i] = src[i] - base;
}
__global__ void repack_rows_kernel(float* dst, int ldx, const float* src, long long ld_in, long long rows, int Dg) {
  const long long total = rows * Dg;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long i = e / Dg;
    const int c = (int)(e - i * Dg);
    dst[i * ldx + c] = src[i * ld_in + c];
  }
}

}  // namespace

bool is_device_ptr(const void* p) {
  cudaPointerAttributes a;
  const bool dev = cudaPointerGetAttributes(&a, p) == cudaSuccess && (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged);
  cudaGetLastError();
  return dev;
}

bool is_dma_ptr(const void* p) {
  cudaPointerAttributes a;
  const bool dma = cudaPointerGetAttributes(&a, p) == cudaSuccess &&
                   (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged || a.type == cudaMemoryTypeHost);
  cudaGetLastError();
  return dma;
}

int gather_rowptr(const int64_t* rowptr, const std::vector<long long>& idx, std::vector<long long>& out) {
  out.resize(idx.size());
  if (!is_device_ptr(rowptr)) {
    for (size_t i = 0; i < idx.size(); i++) out[i] = rowptr[idx[i]];
    return 0;
  }
  DevMem t;
  long long *d_idx, *d_out;
  if (int rc = t.get(&d_idx, idx.size(), false)) return rc;
  if (int rc = t.get(&d_out, idx.size(), false)) return rc;
  CK(cudaMemcpy(d_idx, idx.data(), idx.size() * 8, cudaMemcpyHostToDevice));
  gather_i64_kernel<<<(int)((idx.size() + 255) / 256), 256>>>((const long long*)rowptr, d_idx, (int)idx.size(), d_out);
  CK(cudaMemcpy(out.data(), d_out, idx.size() * 8, cudaMemcpyDeviceToHost));
  return 0;
}

int ingest_labels(cudaStream_t st, long long n, const int32_t* response, const float* weight, const float* offset, signed char* y, float* w,
                  float* o, int* d_flag, int* h_flag, float* wmax) {
  DevMem t;   // device copies of host input: freed on every return path
  const int* d_r; const float *d_w, *d_o;
  if (int rc = to_device(t, (const int*)response, (size_t)n, &d_r, st)) return rc;
  if (int rc = to_device(t, weight, (size_t)n, &d_w, st)) return rc;
  if (int rc = to_device(t, offset, (size_t)n, &d_o, st)) return rc;
  CK(cudaMemsetAsync(d_flag, 0, 8, st));
  if (n > 0) {
    convert_labels_kernel<<<(int)std::min<long long>((n + 255) / 256, 4096), 256, 0, st>>>(n, d_r, d_w, d_o, y, w, o, d_flag);
    if (wmax) absmax_kernel<<<(int)std::min<long long>((n + 255) / 256, 2048), 256, 0, st>>>(n, w, (unsigned*)(d_flag + 1));
  }
  CK(cudaMemcpyAsync(h_flag, d_flag, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (h_flag[0] & 1) return fail(MLEASE_ERR_INVALID, "response (only 1, 0, -1 are allowed)");
  if (h_flag[0] & 2) return fail(MLEASE_ERR_INVALID, "weight cannot < 0");
  if (wmax && n > 0) std::memcpy(wmax, h_flag + 1, 4);
  return 0;
}

int check_rowptr(cudaStream_t st, long long n, const long long* rowptr, int* d_flag, const std::string& who) {
  int bad = 0;
  CK(cudaMemsetAsync(d_flag, 0, 4, st));
  check_rowptr_kernel<<<(int)std::max<long long>(1, std::min<long long>((n + 255) / 256, 4096)), 256, 0, st>>>(n, rowptr, d_flag);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(&bad, d_flag, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (bad) return fail(MLEASE_ERR_INVALID, who + "rowptr must start at >= 0 and never decrease");
  return 0;
}

void check_csr(cudaStream_t st, long long n, long long nnz, const long long* rowptr, const int* colidx, float* vals, int Dg, int binary,
               int* d_flag) {
  if (nnz <= 0) return;
  check_csr_kernel<<<(int)std::min<long long>((nnz + 255) / 256, 4096), 256, 0, st>>>(nnz, colidx, vals, Dg, binary, d_flag);
  check_rows_sorted_kernel<<<(int)std::min<long long>((n + 255) / 256, 4096), 256, 0, st>>>(n, rowptr, colidx, d_flag + 1);
}

void rebase_rowptr(cudaStream_t st, long long n, const long long* src, long long base, long long* dst) {
  rebase_rowptr_kernel<<<(int)std::min<long long>((n + 256) / 256, 4096), 256, 0, st>>>(n, src, base, dst);
}

int upload_dense_rows(float* dst, int ldx, const float* src, long long ld_in, long long n, int Dg, int has_bias, cudaStream_t st) {
  // The rows are re-pitched by a kernel: the copy engine moves short pitched rows far below its bandwidth, over PCIe as well as
  // on the device.  A host source streams in contiguous chunks through two staging buffers on a copy stream, each chunk
  // repacked into the padded layout on `st`.
  if (is_device_ptr(src)) {
    repack_rows_kernel<<<4096, 256, 0, st>>>(dst, ldx, src, ld_in, n, Dg);
  } else {
    const long long chunk_rows = std::max<long long>(1, (128LL << 20) / (ld_in * 4));
    struct Staging {   // the events + the copy stream, released on every return path
      cudaEvent_t h2d_done[2] = {nullptr, nullptr}, repack_done[2] = {nullptr, nullptr};
      cudaStream_t cs = nullptr;
      ~Staging() {
        for (int b = 0; b < 2; b++) { if (h2d_done[b]) cudaEventDestroy(h2d_done[b]); if (repack_done[b]) cudaEventDestroy(repack_done[b]); }
        if (cs) cudaStreamDestroy(cs);
      }
    } sg;
    DevMem bufs;
    float* buf[2];
    CK(cudaStreamCreateWithFlags(&sg.cs, cudaStreamNonBlocking));
    for (int b = 0; b < 2; b++) {
      if (int rc = bufs.get(&buf[b], (size_t)chunk_rows * ld_in, false)) return rc;
      CK(cudaEventCreateWithFlags(&sg.h2d_done[b], cudaEventDisableTiming));
      CK(cudaEventCreateWithFlags(&sg.repack_done[b], cudaEventDisableTiming));
    }
    int ci = 0;
    for (long long r0 = 0; r0 < n; r0 += chunk_rows, ci++) {
      const int b = ci & 1;
      const long long rows = std::min(chunk_rows, n - r0);
      if (ci >= 2) CK(cudaStreamWaitEvent(sg.cs, sg.repack_done[b], 0));
      const size_t bytes = ((size_t)(rows - 1) * ld_in + Dg) * 4;
      CK(cudaMemcpyAsync(buf[b], src + r0 * ld_in, bytes, cudaMemcpyHostToDevice, sg.cs));
      CK(cudaEventRecord(sg.h2d_done[b], sg.cs));
      CK(cudaStreamWaitEvent(st, sg.h2d_done[b], 0));
      repack_rows_kernel<<<2048, 256, 0, st>>>(dst + r0 * ldx, ldx, buf[b], ld_in, rows, Dg);
      CK(cudaEventRecord(sg.repack_done[b], st));
    }
    CK(cudaStreamSynchronize(sg.cs));
    CK(cudaStreamSynchronize(st));
  }
  fill_bias_pad_kernel<<<1024, 256, 0, st>>>(dst, n, ldx, Dg, has_bias);
  return 0;
}

// Checks and derived lists of one uploaded CSR partition (feature range, |value| max, block-major Gram list, K1 segment
// lists). Runs on s->stream; mlease_add_partition_csr defers it by one call so that it overlaps the next partition's H2D copy.
int csr_build_layout(mlease_session* s, PartData& pd) {
  Problem& d = pd.data;
  if (d.nnz_hint <= 0) return 0;
  const long long nrows = d.n, nnz = d.nnz_hint;
  const std::string who = "partition " + std::to_string(pd.pid) + ": ";
  // every kernel below indexes by rowptr: its rows must lie inside [0, nnz], which a rowptr that starts at 0 and never decreases
  // guarantees (a decreasing one makes rows overlap, and the block-major list would get more than nnz + nrows entries)
  if (int rc = check_rowptr(s->stream, nrows, d.rowptr, s->d_flag, who)) return rc;
  // one read-back of the checks and the scalars: d_flag[0] range, [1] sorted, [2] |value| max, [3] row L1 max, [4, 6) Gram products.
  // A range error is reported before the lists below index by colidx; the reductions read column ids as values only.
  int* f = s->d_flag;
  CK(cudaMemsetAsync(f, 0, 24, s->stream));
  check_csr(s->stream, nrows, nnz, d.rowptr, d.colidx, const_cast<float*>(d.vals), s->Dg, s->cfg.binary_feature, f);   // the session's copy
  absmax_kernel<<<(int)std::min<long long>((nnz + 255) / 256, 2048), 256, 0, s->stream>>>(nnz, d.vals, (unsigned*)(f + 2));
  CK(csr_row_l1_max(nrows, d.rowptr, d.vals, (unsigned*)(f + 3), s->stream));
  csr_gram_pairs_kernel<<<(int)std::min<long long>((nrows + 255) / 256, 2048), 256, 0, s->stream>>>(nrows, d.rowptr, (unsigned long long*)(f + 4));
  CK(cudaMemcpyAsync(s->h_flag, f, 24, cudaMemcpyDeviceToHost, s->stream));
  CK(cudaStreamSynchronize(s->stream));
  if (s->h_flag[0]) return fail(MLEASE_ERR_INVALID, who + "feature index out of range");
  d.csr_unique = s->h_flag[1] ? 0 : 1;
  std::memcpy(&d.vmax, s->h_flag + 2, 4);
  std::memcpy(&d.rowl1, s->h_flag + 3, 4);
  unsigned long long pairs = 0;
  std::memcpy(&pairs, s->h_flag + 4, 8);
  // the Gram producers index the entry list with 32 bits; the list holds one bias entry per row (session batches always have the
  // intercept, column Dg)
  // A matrix-free session (hessian_policy 2) builds no Gram, so it skips the block-major list (n D'/512 offsets + 6 B per entry)
  // and the column index of the sparse Gram (4 B per entry)
  if (d.csr_unique && nnz + nrows < (1LL << 32) - 64 && s->cfg.hessian_policy != 2) {
    d.nblk128 = round_up(s->ldx, 128) / 128;
    d.bm_groups = (nrows + 31) / 32;
    d.bm_entries = nnz + nrows;
    long long* bo; unsigned short* bk; float* bv;
    if (int rc = s->mem.get(&bo, (size_t)d.nblk128 * d.bm_groups + 1, true)) return rc;
    if (int rc = s->mem.get(&bk, (size_t)d.bm_entries, true)) return rc;
    if (int rc = s->mem.get(&bv, (size_t)d.bm_entries, true)) return rc;
    CK(csr_bm_offsets(nrows, d.rowptr, d.colidx, s->Dg, d.nblk128, d.bm_groups, bo, s->stream));
    CK(csr_bm_fill(nrows, d.rowptr, d.colidx, d.vals, s->Dg, d.nblk128, d.bm_groups, bo, bk, bv, s->stream));
    d.bm_offs = bo; d.bm_keys = bk; d.bm_vals = bv;
    d.gram_pairs = (double)pairs;   // products of one sparse Gram build (the kernel choice of batch_alloc)
    // the sparse Gram's column index (4 B per entry), only where that kernel can run
    if (nrows <= gram_sparse_max_rows() && s->Dt <= gram_sparse_max_cols()) {
      uint32_t *co, *cp;
      if (int rc = s->mem.get(&co, (size_t)s->Dt + 1, true)) return rc;
      if (int rc = s->mem.get(&cp, (size_t)d.bm_entries, true)) return rc;
      CK(csr_col_index(nrows, d.rowptr, d.colidx, s->Dg, d.bm_entries, co, cp, s->stream));
      d.gc_offs = co; d.gc_pos = cp;
    }
  }
  if (d.csr_unique && nnz + nrows < (1LL << 32) - 64) {
    // segment lists of the fused multi-lambda K1
    int S = 0, rows = 0, LP = 0; size_t smem = 0;
    if (k1f_plan(nrows, s->ldx, s->L, s->num_sms, &S, &rows, &LP, &smem)) {
      int *perm, *depth; long long* goff; unsigned short *row16, *col16; float* val; long long total;
      CK(k1f_build(nrows, s->Dg, nnz, d.rowptr, d.colidx, d.vals, S, rows, &d.sg_ngrp, &perm, &depth, &goff, &row16, &val, &total, &col16,
                   s->stream));
      d.sg_S = S; d.sg_rows = rows;
      d.sg_perm = perm; d.sg_depth = depth; d.sg_goff = goff; d.sg_row16 = row16; d.sg_val = val; d.sg_col16 = col16;
      for (void* p : {(void*)perm, (void*)depth, (void*)goff, (void*)row16, (void*)val, (void*)col16}) s->mem.adopt(p);
    }
  }
  return 0;
}

}  // namespace mlease
