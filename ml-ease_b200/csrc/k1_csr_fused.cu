// k1_csr_fused.cu -- K1 for CSR partitions, all lambda-problems of a partition in ONE pass, no atomics.
//
// Replaces LogisticRegressionL2.fun + grad (llf/LogisticRegressionL2.java:156-225: the sparse passes Xv :115-129 and XTv :131-150)
// for the L reducers that share a partition (reducers = nblocks x #lambda, jobs/RegressionAdmmTrain.java:355): they read the
// same rows, so one load of (column, value) feeds L margins and L gradient sums.
//
// A CTA owns one SEGMENT of a partition's rows (sg_rows consecutive rows, a few thousand):
//   phase A (row-major, the CSR arrays): half-warp per row, s_il = sum_j v_ij beta_l[c_ij] (+ bias) with the L betas
//            interleaved in shared memory (one LDS.128 serves all lambdas), sigmoid / loss / IRLS weight per lambda,
//            residuals r_il = -w_i y_i (1 - p_il) into shared memory r_s[row][l]; sqrt(d_il) to sdvec when a Gram follows.
//   phase B (column-major, the segment list built at upload): the segment's entries regrouped by COLUMN: lane = column,
//            32 columns of similar length per group (columns sorted by their count inside the segment, so the padding of a
//            group to its longest column is a few per cent), entries stored [k][lane] = (row16, value).  A warp walks a
//            group: coalesced loads, r gathered from shared memory, g_c += v r in registers -- a segmented sum with no
//            atomics and a fixed order (row order): deterministic like the dense kernel.
// Per-segment partial gradients go to gpart_f[segment][column] (fp32, one writer per element); k1_partial_reduce_kernel adds
// the segments in fp64 in segment order.  HBM traffic per partition pass: 6 B (the CSR values + a 16-bit copy of the column ids,
// sg_col16) + ~6.2 B (segment list) per stored value + 9 B per row, for ALL lambdas together.
// MODE K1_HV / K1_DIAG (matrix-free solver, common.cuh): phase A computes t_il = d_il (x_i . v_l) (v_l = hv_vf, interleaved like
// beta) or t_il = d_il, with d_il = sqrt(d_il)^2 from sdvec of the last gradient pass; phase B is the same column sum of
// x_ic t_il (x_ic^2 t_il for the diagonal).  The problems taking part are those with Ctrl::cg_active.
#include <cub/cub.cuh>

#include <algorithm>

#include "kernels.cuh"

namespace mlease {

constexpr int K1F_THREADS = 768;   // 24 warps, <= 85 registers per thread
constexpr int K1F_HW = 16;         // lanes per row in phase A
constexpr int K1F_NCH = 7;         // register-resident 16-entry chunks per row (112 entries)

template <int LP> struct VecOf;
template <> struct VecOf<1> { using T = float; };
template <> struct VecOf<2> { using T = float2; };
template <> struct VecOf<4> { using T = float4; };
__device__ __forceinline__ float vget(const float& v, int) { return v; }
__device__ __forceinline__ float vget(const float2& v, int i) { return i == 0 ? v.x : v.y; }
__device__ __forceinline__ float vget(const float4& v, int i) { return i == 0 ? v.x : i == 1 ? v.y : i == 2 ? v.z : v.w; }

template <int LP, int MODE>
__global__ void __launch_bounds__(K1F_THREADS, 1) k1_csr_fused_kernel(const Problem* __restrict__ probs, int L, int has_bias, int force_emit) {
  using V = typename VecOf<LP>::T;
  const int b0 = blockIdx.y * L;
  const Problem& p0 = probs[b0];
  const int seg = blockIdx.x;
  __shared__ int s_act, s_emit;
  if (threadIdx.x == 0) {
    int a = 0, e = 0;
    for (int l = 0; l < L; l++) {
      Ctrl* c = probs[b0 + l].ctrl;
      if (MODE != K1_GRAD ? (c->cg_active != 0) : (!c->done && !c->skip_eval)) {   // skip_eval: the start-point gradient of this x-update is known without a pass (k4_consensus.cu)
        a |= 1 << l;
        if (force_emit >= 0 ? (force_emit != 0) : (c->emit != 0)) e |= 1 << l;
        if (seg == 0) c->k1_chunks = p0.sg_S;
      }
    }
    s_act = a; s_emit = e;
  }
  __syncthreads();
  const int act = s_act, emit = s_emit;
  if (!act) return;
  extern __shared__ __align__(16) float k1f_sm[];
  const int ldx = p0.ldx, Dt = p0.Dt;
  V* beta_s = reinterpret_cast<V*>(k1f_sm);              // [ldx] interleaved betas
  V* r_s = beta_s + ldx;                                  // [sg_rows] interleaved residuals
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = K1F_THREADS >> 5;
  {
    // 4 columns per thread: one 16-byte load per lambda, written as the LP-wide interleaved vectors of the 4 columns
    const float* src[LP];
#pragma unroll
    for (int l = 0; l < LP; l++)
      src[l] = (MODE != K1_DIAG && l < L && ((act >> l) & 1)) ? (MODE == K1_GRAD ? probs[b0 + l].beta_tf : probs[b0 + l].hv_vf) : nullptr;
    float4* bs4 = reinterpret_cast<float4*>(k1f_sm);
    for (int k4 = tid; k4 < (ldx >> 2); k4 += K1F_THREADS) {
      float q[LP][4];
#pragma unroll
      for (int l = 0; l < LP; l++) {
        const float4 t = src[l] ? __ldg(reinterpret_cast<const float4*>(src[l]) + k4) : make_float4(0.f, 0.f, 0.f, 0.f);
        q[l][0] = t.x; q[l][1] = t.y; q[l][2] = t.z; q[l][3] = t.w;
      }
#pragma unroll
      for (int m = 0; m < LP; m++) {   // float e = 4m..4m+3 of the 4 LP values: column e / LP, lambda e % LP
        float o[4];
#pragma unroll
        for (int u = 0; u < 4; u++) o[u] = q[(4 * m + u) % LP][(4 * m + u) / LP];
        bs4[(size_t)k4 * LP + m] = make_float4(o[0], o[1], o[2], o[3]);
      }
    }
  }
  __syncthreads();
  const long long n = p0.n;
  const long long rb = (long long)seg * p0.sg_rows, re = min(n, rb + p0.sg_rows);
  // ------------------------------------------------------------------ phase A: margins, weights, residuals
  const long long* __restrict__ rp = p0.rowptr;
  const signed char* __restrict__ yv = p0.y;
  const float* __restrict__ wv = p0.w;
  const float* __restrict__ ov = p0.o;
  const int sub = lane >> 4, sl = lane & 15;
  // After the half-warp reduction below, the 16 lanes of a row hold the LP margins distributed: lane sl owns lambda
  // lam_of = bits (3,2) of sl for LP = 4 (bit 3 for LP = 2), and the lanes with (sl & 3) == 0 do that lambda's sigmoid / loss /
  // residual -- the L sigmoids of a row run in parallel lanes instead of one lane doing them one after the other.
  const int lam_of = LP == 4 ? (sl >> 2) : (LP == 2 ? (sl >> 3) : 0);
  const bool lam_lane = (LP == 4 ? (sl & 3) == 0 : (LP == 2 ? (sl & 7) == 0 : sl == 0));
  const bool lam_on = lam_lane && lam_of < L && ((act >> lam_of) & 1);
  const bool lam_emit = lam_on && ((emit >> lam_of) & 1);
  const float bias_l = has_bias ? reinterpret_cast<const float*>(beta_s)[(size_t)(Dt - 1) * LP + lam_of] : 0.f;
  float* __restrict__ sd_l = (MODE != K1_GRAD ? lam_on : lam_emit) ? probs[b0 + lam_of].sdvec : nullptr;
  float* r_sf = reinterpret_cast<float*>(r_s);
  float loss = 0.f, rsum = 0.f;
  const long long rstep = 2LL * nw;
  long long i = rb + 2 * warp + sub;
  long long j0 = 0;
  int len = 0;
  if (i < re) { j0 = __ldg(rp + i); len = (int)(__ldg(rp + i + 1) - j0); }
  for (long long ib = rb + 2 * warp; ib < re; ib += rstep) {
    const bool has_row = i < re;
    const float* __restrict__ vr = p0.vals + j0;
    const unsigned short* __restrict__ cr = p0.sg_col16 + j0;
    float v[K1F_NCH];
    int c[K1F_NCH];
#pragma unroll
    for (int q = 0; q < K1F_NCH; q++) {
      const bool ok = sl + K1F_HW * q < len;
      v[q] = ok ? __ldg(vr + sl + K1F_HW * q) : 0.f;
      c[q] = ok ? (int)__ldg(cr + sl + K1F_HW * q) : 0;   // unsigned: ids >= 32768 stay positive
    }
    float yy = 0.f, ww = 0.f, oo = 0.f;
    if (has_row) { yy = (float)__ldg(yv + i); ww = __ldg(wv + i); oo = __ldg(ov + i); }
    const long long in = i + rstep;
    long long j0n = 0;
    int lenn = 0;
    if (in < re) { j0n = __ldg(rp + in); lenn = (int)(__ldg(rp + in + 1) - j0n); }
    float a[LP];
#pragma unroll
    for (int l = 0; l < LP; l++) a[l] = 0.f;
#pragma unroll
    for (int q = 0; q < K1F_NCH; q++) {
      const V bb = beta_s[c[q]];
#pragma unroll
      for (int l = 0; l < LP; l++) a[l] = fmaf(v[q], vget(bb, l), a[l]);
    }
    for (int j = K1F_NCH * K1F_HW + sl; j < len; j += K1F_HW) {
      const float vj = __ldg(vr + j);
      const V bb = beta_s[(int)__ldg(cr + j)];
#pragma unroll
      for (int l = 0; l < LP; l++) a[l] = fmaf(vj, vget(bb, l), a[l]);
    }
    // transposed half-warp reduction: LP values x 16 lanes -> one value per lane (5 shuffles for LP = 4 instead of 16)
    float av;
    if constexpr (LP == 4) {
      const bool up = (sl & 8) != 0;
      const float k0 = (up ? a[2] : a[0]) + __shfl_xor_sync(0xffffffffu, up ? a[0] : a[2], 8);
      const float k1 = (up ? a[3] : a[1]) + __shfl_xor_sync(0xffffffffu, up ? a[1] : a[3], 8);
      const bool up2 = (sl & 4) != 0;
      av = (up2 ? k1 : k0) + __shfl_xor_sync(0xffffffffu, up2 ? k0 : k1, 4);
      av += __shfl_xor_sync(0xffffffffu, av, 2);
      av += __shfl_xor_sync(0xffffffffu, av, 1);
    } else if constexpr (LP == 2) {
      const bool up = (sl & 8) != 0;
      av = (up ? a[LP - 1] : a[0]) + __shfl_xor_sync(0xffffffffu, up ? a[0] : a[LP - 1], 8);
      av += __shfl_xor_sync(0xffffffffu, av, 4);
      av += __shfl_xor_sync(0xffffffffu, av, 2);
      av += __shfl_xor_sync(0xffffffffu, av, 1);
    } else {
      av = a[0];
#pragma unroll
      for (int m = K1F_HW / 2; m >= 1; m >>= 1) av += __shfl_xor_sync(0xffffffffu, av, m);
    }
    if constexpr (MODE != K1_GRAD) {
      if (lam_lane && has_row) {
        float tv = 0.f;
        if (lam_on) {
          const float sd = sd_l[i];
          tv = sd * sd;
          if constexpr (MODE == K1_HV) tv *= av + bias_l;
          rsum += tv;
        }
        r_sf[(size_t)(i - rb) * LP + lam_of] = tv;
      }
    } else if (lam_lane && has_row) {
      const float t = yy * (av + bias_l + oo);
      const float e = __expf(-fabsf(t));
      const float inv = __frcp_rn(1.f + e);
      const float p = t >= 0.f ? inv : e * inv;
      const float qq = t >= 0.f ? e * inv : inv;
      const float r = lam_on ? -ww * yy * qq : 0.f;
      r_sf[(size_t)(i - rb) * LP + lam_of] = r;
      if (lam_on) {
        loss += ww * ((t >= 0.f ? 0.f : -t) - __logf(inv));
        rsum += r;
        if (lam_emit) sd_l[i] = sqrtf(ww * p * qq);   // the Gram kernel assembles the scaled rows itself
      }
    }
    i = in; j0 = j0n; len = lenn;
  }
  // loss / bias-gradient partials of this segment: the two rows of a warp, then one fp64 sum per lambda in warp order
  __shared__ float red[2][LP][K1F_THREADS / 32];
  {
    const float la = loss + __shfl_down_sync(0xffffffffu, loss, 16);
    const float lb = rsum + __shfl_down_sync(0xffffffffu, rsum, 16);
    if (lam_lane && sub == 0) { red[0][lam_of][warp] = la; red[1][lam_of][warp] = lb; }
  }
  __syncthreads();   // r_s complete, red complete
  if (tid < LP && tid < L && ((act >> tid) & 1)) {
    double sa = 0.0, sb = 0.0;
    for (int wq = 0; wq < nw; wq++) { sa += (double)red[0][tid][wq]; sb += (double)red[1][tid][wq]; }
    const Problem& pl = probs[b0 + tid];
    if (MODE == K1_GRAD) pl.fpart[seg] = sa;
    if (has_bias) pl.gpart_f[(size_t)seg * ldx + Dt - 1] = (float)sb;
  }
  // ------------------------------------------------------------------ phase B: column sums from the segment list
  const int ngrp = p0.sg_ngrp;
  const int* __restrict__ perm = p0.sg_perm + (size_t)seg * ngrp * 32;
  const int* __restrict__ depth = p0.sg_depth + (size_t)seg * ngrp;
  const long long* __restrict__ goff = p0.sg_goff + (size_t)seg * ngrp;
  const unsigned short* __restrict__ r16 = p0.sg_row16;
  const float* __restrict__ sv = p0.sg_val;
  for (int g = warp; g < ngrp; g += nw) {
    const int col = __ldg(perm + g * 32 + lane);
    const int dep = __ldg(depth + g);
    const unsigned short* __restrict__ pr = r16 + (size_t)__ldg(goff + g) * 32 + lane;
    const float* __restrict__ pv = sv + (size_t)__ldg(goff + g) * 32 + lane;
    float acc[LP];
#pragma unroll
    for (int l = 0; l < LP; l++) acc[l] = 0.f;
    int k = 0;
    constexpr int UB = 8;   // 16 independent loads in flight per lane: phase B is pure latency otherwise
    for (; k + UB <= dep; k += UB) {
      unsigned short rw[UB];
      float vv[UB];
#pragma unroll
      for (int u = 0; u < UB; u++) { rw[u] = __ldg(pr + (k + u) * 32); vv[u] = __ldg(pv + (k + u) * 32); }
#pragma unroll
      for (int u = 0; u < UB; u++) {
        const V rr = r_s[rw[u]];
        const float xv = MODE == K1_DIAG ? vv[u] * vv[u] : vv[u];
#pragma unroll
        for (int l = 0; l < LP; l++) acc[l] = fmaf(xv, vget(rr, l), acc[l]);
      }
    }
    if (k < dep) {   // tail: predicated loads (padding value 0 * r_s[0])
      unsigned short rw[UB];
      float vv[UB];
#pragma unroll
      for (int u = 0; u < UB; u++) {
        const bool ok = k + u < dep;
        rw[u] = ok ? __ldg(pr + (k + u) * 32) : (unsigned short)0;
        vv[u] = ok ? __ldg(pv + (k + u) * 32) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < UB; u++) {
        const V rr = r_s[rw[u]];
        const float xv = MODE == K1_DIAG ? vv[u] * vv[u] : vv[u];
#pragma unroll
        for (int l = 0; l < LP; l++) acc[l] = fmaf(xv, vget(rr, l), acc[l]);
      }
    }
    if (col >= 0) {
#pragma unroll
      for (int l = 0; l < LP; l++)
        if (l < L && ((act >> l) & 1)) probs[b0 + l].gpart_f[(size_t)seg * ldx + col] = acc[l];
    }
  }
}

// ------------------------------------------------------------------------------------------
// segment-list builder (once per partition upload)
// ------------------------------------------------------------------------------------------
// cnt[seg][c] = stored values of column c in the rows of segment seg (shared-memory counters, one CTA per segment)
__global__ void __launch_bounds__(1024) k1f_count_kernel(long long n, int sg_rows, int Dg, const long long* __restrict__ rowptr, const int* __restrict__ colidx,
                                                        int* __restrict__ cnt) {
  extern __shared__ int k1f_cnt_sm[];
  const int seg = blockIdx.x;
  for (int c = threadIdx.x; c < Dg; c += blockDim.x) k1f_cnt_sm[c] = 0;
  __syncthreads();
  const long long rb = (long long)seg * sg_rows, re = min(n, rb + sg_rows);
  if (rb < re) {
    const long long j0 = rowptr[rb], j1 = rowptr[re];
    for (long long j = j0 + threadIdx.x; j < j1; j += blockDim.x) atomicAdd(&k1f_cnt_sm[colidx[j]], 1);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < Dg; c += blockDim.x) cnt[(size_t)seg * Dg + c] = k1f_cnt_sm[c];
}
__global__ void k1f_iota_kernel(int S, int Dg, int* __restrict__ ids, int* __restrict__ seg_offs) {
  const size_t tot = (size_t)S * Dg;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < tot; e += (size_t)gridDim.x * blockDim.x) ids[e] = (int)(e % Dg);
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s <= S; s += gridDim.x * blockDim.x) seg_offs[s] = s * Dg;
}
// from the per-segment descending (count, column) lists: lane slots, group depths, column -> slot
__global__ void k1f_groups_kernel(int S, int Dg, int ngrp, const int* __restrict__ cnt_sorted, const int* __restrict__ col_sorted, int* __restrict__ perm,
                                  int* __restrict__ depth, long long* __restrict__ depth64, int* __restrict__ inv) {
  const size_t tot = (size_t)S * ngrp * 32;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < tot; e += (size_t)gridDim.x * blockDim.x) {
    const int seg = (int)(e / ((size_t)ngrp * 32)), slot = (int)(e % ((size_t)ngrp * 32));
    int col = -1;
    if (slot < Dg) {
      col = col_sorted[(size_t)seg * Dg + slot];
      inv[(size_t)seg * Dg + col] = slot;
    }
    perm[e] = col;
    if ((slot & 31) == 0) {
      const int d = slot < Dg ? cnt_sorted[(size_t)seg * Dg + slot] : 0;   // descending order: the group's first column is its longest
      depth[(size_t)seg * ngrp + (slot >> 5)] = d;
      depth64[(size_t)seg * ngrp + (slot >> 5)] = d;
    }
  }
}
// pass 1 (parallel): per stored value, the row id inside its segment and the position of its column's lane slot:
// (first 32-lane row of the column's group) * 32 + lane.  The value's final place is that + 32 * (its rank in the column).
__global__ void k1f_rowid_kernel(long long n, int sg_rows, int Dg, int ngrp, const long long* __restrict__ rowptr, const int* __restrict__ colidx,
                                 const int* __restrict__ inv, const long long* __restrict__ goff, unsigned short* __restrict__ ent_row,
                                 unsigned* __restrict__ ent_base) {
  const int lane = threadIdx.x & 31;
  const long long nw = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += nw) {
    const int seg = (int)(i / sg_rows);
    const unsigned short r = (unsigned short)(i - (long long)seg * sg_rows);
    const int* __restrict__ iv = inv + (size_t)seg * Dg;
    const long long* __restrict__ go = goff + (size_t)seg * ngrp;
    for (long long j = rowptr[i] + lane; j < rowptr[i + 1]; j += 32) {
      const int slot = iv[colidx[j]];
      ent_row[j] = r;
      ent_base[j] = (unsigned)(go[slot >> 5] * 32 + (slot & 31));
    }
  }
}
// 16-bit copy of the column ids for phase A (k1f_plan admits no partition wider than 55 296 columns)
__global__ void k1f_col16_kernel(long long nnz, const int* __restrict__ colidx, unsigned short* __restrict__ col16) {
  for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < nnz; j += (long long)gridDim.x * blockDim.x)
    col16[j] = (unsigned short)colidx[j];
}
// pass 2a: column histogram of every chunk of a segment's stored values (K1F_CHUNKS chunks per segment, consecutive in the CSR)
constexpr int K1F_CHUNKS = 8;
__device__ __forceinline__ void k1f_chunk_range(long long j0, long long j1, int chunk, long long* a, long long* b) {
  const long long per = (((j1 - j0) + K1F_CHUNKS - 1) / K1F_CHUNKS + 31) / 32 * 32;
  *a = min(j1, j0 + (long long)chunk * per);
  *b = min(j1, *a + per);
}
__global__ void __launch_bounds__(256) k1f_hist_kernel(long long n, int sg_rows, int Dg, const long long* __restrict__ rowptr, const int* __restrict__ colidx,
                                                      unsigned short* __restrict__ hist) {
  extern __shared__ int k1f_hist_sm[];
  const int seg = blockIdx.x, chunk = blockIdx.y;
  for (int c = threadIdx.x; c < Dg; c += blockDim.x) k1f_hist_sm[c] = 0;
  __syncthreads();
  const long long rb = (long long)seg * sg_rows, re = min(n, rb + sg_rows);
  if (rb < re) {
    long long a, b;
    k1f_chunk_range(rowptr[rb], rowptr[re], chunk, &a, &b);
    for (long long j = a + threadIdx.x; j < b; j += blockDim.x) atomicAdd(&k1f_hist_sm[colidx[j]], 1);
  }
  __syncthreads();
  unsigned short* out = hist + ((size_t)seg * K1F_CHUNKS + chunk) * Dg;
  for (int c = threadIdx.x; c < Dg; c += blockDim.x) out[c] = (unsigned short)k1f_hist_sm[c];
}
// pass 2b: one warp per (segment, chunk) walks the chunk's stored values IN ORDER (they are contiguous in the CSR arrays, row
// after row), 32 at a time; its per-column counters start at the number of entries the earlier chunks hold, so every column's
// entries end up in row order: a fixed summation order for phase B.  Lanes of one step that hit the same column (possible when
// a step spans two short rows) are ranked by lane = by row.
__global__ void __launch_bounds__(32) k1f_fill_kernel(long long n, int sg_rows, int Dg, const long long* __restrict__ rowptr,
                                                     const int* __restrict__ colidx, const float* __restrict__ vals,
                                                     const unsigned short* __restrict__ ent_row, const unsigned* __restrict__ ent_base,
                                                     const unsigned short* __restrict__ hist, unsigned short* __restrict__ row16,
                                                     float* __restrict__ sval) {
  extern __shared__ unsigned short k1f_fill_sm[];
  const int seg = blockIdx.x, chunk = blockIdx.y, lane = threadIdx.x;
  for (int c = lane; c < Dg; c += 32) {
    int s0 = 0;
    for (int q = 0; q < chunk; q++) s0 += hist[((size_t)seg * K1F_CHUNKS + q) * Dg + c];
    k1f_fill_sm[c] = (unsigned short)s0;
  }
  __syncwarp();
  const long long rb = (long long)seg * sg_rows, re = min(n, rb + sg_rows);
  if (rb >= re) return;
  long long j0, j1;
  k1f_chunk_range(rowptr[rb], rowptr[re], chunk, &j0, &j1);
  // the loads of a step do not depend on the counters: keep the next step's in flight while this one is ranked and stored
  auto ld = [&](long long jb, int& c, float& v, unsigned short& r, unsigned& b) {
    const long long j = jb + lane;
    const bool ok = j < j1;
    c = ok ? __ldg(colidx + j) : -1 - lane;          // inactive lanes: distinct negative keys
    v = ok ? __ldg(vals + j) : 0.f;
    r = ok ? __ldg(ent_row + j) : (unsigned short)0;
    b = ok ? __ldg(ent_base + j) : 0u;
  };
  int cn; float vn; unsigned short rn; unsigned bn;
  ld(j0, cn, vn, rn, bn);
  for (long long jb = j0; jb < j1; jb += 32) {
    const int c = cn; const float v = vn; const unsigned short r = rn; const unsigned b = bn;
    ld(jb + 32, cn, vn, rn, bn);
    const bool ok = c >= 0;
    const unsigned m = __match_any_sync(0xffffffffu, c);
    const int rank = __popc(m & ((1u << lane) - 1u));
    int k = 0;
    if (ok) k = k1f_fill_sm[c] + rank;
    __syncwarp();
    if (ok && (m >> (lane + 1)) == 0) k1f_fill_sm[c] = (unsigned short)(k + 1);   // highest lane of the group: count + group size
    __syncwarp();
    if (ok) {
      const size_t pos = (size_t)b + (size_t)k * 32;
      row16[pos] = r;
      sval[pos] = v;
    }
  }
}

// Segment size for a partition: sg_rows * 4 * LP bytes of residuals next to ldx * 4 * LP bytes of betas in one CTA's shared memory,
// at most 65535 rows (16-bit row ids), and a multiple-of-SM-count number of segments when the partition is large enough.
bool k1f_plan(long long n, int ldx, int L, int num_sms, int* S_out, int* rows_out, int* LP_out, size_t* smem_out) {
  if (L > 4 || n <= 0) return false;
  const int LP = L <= 1 ? 1 : (L == 2 ? 2 : 4);
  const size_t cap = 220 * 1024;
  const size_t beta_b = (size_t)ldx * 4 * LP;
  if ((size_t)ldx * 4 > 200 * 1024) return false;                     // the builder counts columns in shared memory
  if (beta_b + (size_t)1024 * 4 * LP > cap) return false;
  const long long max_rows = std::min<long long>((long long)((cap - beta_b) / (4 * LP)), 65535);
  long long S = (n + max_rows - 1) / max_rows;
  if (n >= (long long)num_sms * 512) S = (S + num_sms - 1) / num_sms * num_sms;        // whole waves of one CTA per SM
  else S = std::max<long long>(S, std::min<long long>(num_sms, (n + 511) / 512));       // small partitions: a few CTAs
  const long long rows = (n + S - 1) / S;
  *S_out = (int)S; *rows_out = (int)rows; *LP_out = LP;
  *smem_out = beta_b + (size_t)rows * 4 * LP;
  return true;
}

template <typename T>
static cudaError_t k1f_tmp_alloc(T** p, cudaStream_t st, size_t bytes) { return cudaMallocAsync((void**)p, bytes, st); }

// Builds the segment list of one partition.  All outputs are cudaMalloc'ed here and owned by the caller.
cudaError_t k1f_build(long long n, int Dg, long long nnz, const long long* rowptr, const int* colidx, const float* vals, int S, int sg_rows, int* ngrp_out,
                      int** perm_out, int** depth_out, long long** goff_out, unsigned short** row16_out, float** val_out, long long* total_out,
                      unsigned short** col16_out, cudaStream_t st) {
  const int ngrp = (Dg + 31) / 32;
  cudaError_t e;
  int *cnt = nullptr, *cnt_s = nullptr, *ids = nullptr, *ids_s = nullptr, *offs = nullptr, *inv = nullptr, *perm = nullptr, *depth = nullptr;
  long long *goff = nullptr, *d64 = nullptr;
  unsigned short* row16 = nullptr;
  unsigned short* col16 = nullptr;
  unsigned short* ent_row = nullptr;
  unsigned* ent_base = nullptr;
  unsigned short* hist = nullptr;
  float* sval = nullptr;
  void* tmp = nullptr;
  const size_t sd = (size_t)S * Dg;
  auto cleanup = [&](bool all) {
    // temporaries come from the stream-ordered allocator: cudaFree would wait for the whole device, including the next partition's H2D copy
    void* tmps[] = {cnt, cnt_s, ids, ids_s, offs, inv, d64, tmp, ent_row, ent_base, hist};
    for (void* t : tmps) if (t) cudaFreeAsync(t, st);
    if (all) { cudaFree(perm); cudaFree(depth); cudaFree(goff); cudaFree(row16); cudaFree(sval); cudaFree(col16); }
  };
#define K1F_CK(x) do { e = (x); if (e != cudaSuccess) { cleanup(true); return e; } } while (0)
  K1F_CK(k1f_tmp_alloc(&cnt, st, sd * 4)); K1F_CK(k1f_tmp_alloc(&cnt_s, st, sd * 4)); K1F_CK(k1f_tmp_alloc(&ids, st, sd * 4)); K1F_CK(k1f_tmp_alloc(&ids_s, st, sd * 4));
  K1F_CK(k1f_tmp_alloc(&offs, st, (size_t)(S + 1) * 4)); K1F_CK(k1f_tmp_alloc(&inv, st, sd * 4));
  K1F_CK(cudaMalloc(&perm, (size_t)S * ngrp * 32 * 4)); K1F_CK(cudaMalloc(&depth, (size_t)S * ngrp * 4));
  K1F_CK(cudaMalloc(&goff, ((size_t)S * ngrp + 1) * 8)); K1F_CK(k1f_tmp_alloc(&d64, st, ((size_t)S * ngrp + 1) * 8));
  K1F_CK(cudaFuncSetAttribute(k1f_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Dg * 4));
  k1f_count_kernel<<<S, 1024, (size_t)Dg * 4, st>>>(n, sg_rows, Dg, rowptr, colidx, cnt);
  k1f_iota_kernel<<<1024, 256, 0, st>>>(S, Dg, ids, offs);
  K1F_CK(cudaGetLastError());
  size_t tb = 0;
  K1F_CK(cub::DeviceSegmentedRadixSort::SortPairsDescending(nullptr, tb, cnt, cnt_s, ids, ids_s, (int)sd, S, offs, offs + 1, 0, 17, st));
  size_t tb2 = 0;
  K1F_CK(cub::DeviceScan::ExclusiveSum(nullptr, tb2, d64, goff, (int)((size_t)S * ngrp + 1), st));
  K1F_CK(k1f_tmp_alloc(&tmp, st, std::max(std::max(tb, tb2), (size_t)16)));
  K1F_CK(cub::DeviceSegmentedRadixSort::SortPairsDescending(tmp, tb, cnt, cnt_s, ids, ids_s, (int)sd, S, offs, offs + 1, 0, 17, st));
  K1F_CK(cudaMemsetAsync(d64, 0, ((size_t)S * ngrp + 1) * 8, st));
  k1f_groups_kernel<<<2048, 256, 0, st>>>(S, Dg, ngrp, cnt_s, ids_s, perm, depth, d64, inv);
  K1F_CK(cudaGetLastError());
  K1F_CK(cub::DeviceScan::ExclusiveSum(tmp, tb2, d64, goff, (int)((size_t)S * ngrp + 1), st));
  long long total = 0;
  K1F_CK(cudaMemcpyAsync(&total, goff + (size_t)S * ngrp, 8, cudaMemcpyDeviceToHost, st));
  K1F_CK(cudaStreamSynchronize(st));
  K1F_CK(cudaMalloc(&row16, std::max<size_t>((size_t)total * 32 * 2, 16)));
  K1F_CK(cudaMalloc(&sval, std::max<size_t>((size_t)total * 32 * 4, 16)));
  K1F_CK(cudaMemsetAsync(row16, 0, (size_t)total * 32 * 2, st));
  K1F_CK(cudaMemsetAsync(sval, 0, (size_t)total * 32 * 4, st));
  if ((size_t)total * 32 >= ((size_t)1 << 32)) { cleanup(true); return cudaErrorInvalidValue; }   // 32-bit slot positions
  K1F_CK(k1f_tmp_alloc(&ent_row, st, std::max<size_t>((size_t)nnz * 2, 16)));
  K1F_CK(k1f_tmp_alloc(&ent_base, st, std::max<size_t>((size_t)nnz * 4, 16)));
  k1f_rowid_kernel<<<2368, 256, 0, st>>>(n, sg_rows, Dg, ngrp, rowptr, colidx, inv, goff, ent_row, ent_base);
  K1F_CK(k1f_tmp_alloc(&hist, st, sd * K1F_CHUNKS * 2));
  K1F_CK(cudaFuncSetAttribute(k1f_hist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Dg * 4));
  k1f_hist_kernel<<<dim3(S, K1F_CHUNKS), 256, (size_t)Dg * 4, st>>>(n, sg_rows, Dg, rowptr, colidx, hist);
  K1F_CK(cudaFuncSetAttribute(k1f_fill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Dg * 2));
  k1f_fill_kernel<<<dim3(S, K1F_CHUNKS), 32, (size_t)Dg * 2, st>>>(n, sg_rows, Dg, rowptr, colidx, vals, ent_row, ent_base, hist, row16, sval);
  K1F_CK(cudaMalloc(&col16, std::max<size_t>((size_t)nnz * 2, 16)));
  k1f_col16_kernel<<<2048, 256, 0, st>>>(nnz, colidx, col16);
  K1F_CK(cudaGetLastError());
  K1F_CK(cudaStreamSynchronize(st));
#undef K1F_CK
  cleanup(false);
  *ngrp_out = ngrp; *perm_out = perm; *depth_out = depth; *goff_out = goff; *row16_out = row16; *val_out = sval; *total_out = total; *col16_out = col16;
  return cudaSuccess;
}

cudaError_t k1f_launch(const Problem* d_probs, int ngroups, int L, int S, int LP, size_t smem, int has_bias, int force_emit, cudaStream_t st, int* launches,
                       int mode) {
  cudaError_t e;
  const dim3 grid(S, ngroups);
#define K1F_GO(LPV, M)                                                                                                     \
  e = cudaFuncSetAttribute(k1_csr_fused_kernel<LPV, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);             \
  if (e != cudaSuccess) return e;                                                                                            \
  k1_csr_fused_kernel<LPV, M><<<grid, K1F_THREADS, smem, st>>>(d_probs, L, has_bias, force_emit);
#define K1F_GO_LP(M) if (LP == 1) { K1F_GO(1, M) } else if (LP == 2) { K1F_GO(2, M) } else { K1F_GO(4, M) }
  if (mode == K1_HV) { K1F_GO_LP(K1_HV) } else if (mode == K1_DIAG) { K1F_GO_LP(K1_DIAG) } else { K1F_GO_LP(K1_GRAD) }
#undef K1F_GO_LP
#undef K1F_GO
  if (launches) *launches += 1;
  return cudaGetLastError();
}

}  // namespace mlease
