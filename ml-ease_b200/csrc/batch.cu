// batch.cu -- a batch of equally shaped problems: allocation and the choice of its solver paths (K1 grid, CSR Gram kernel, matrix-free
// or Gram path, split-K), its Gram and K1 launches, and the Newton slot pipeline of one x-update.
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "host.cuh"

namespace mlease {

namespace {

// End-of-slot poll for large batches (one CTA): flag_out[0] = running | emit << 1; and, for the Gram / Cholesky launches of
// the NEXT slot, the problems that may rebuild there (running and emit set) are copied, as Problem structs, into `compact`
// and counted in flag_out[1]: a rebuild slot then launches grids over those only instead of over thousands of finished fits.
__global__ void poll2_kernel(const Problem* probs, int nprob, int* flag_out, Problem* compact) {
  __shared__ int s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  int running = 0, emit = 0;
  for (int b = threadIdx.x; b < nprob; b += blockDim.x) {
    const Ctrl* c = probs[b].ctrl;
    if (!c->done) {
      running = 1;
      if (c->emit) { emit = 1; compact[atomicAdd(&s_cnt, 1)] = probs[b]; }   // order is irrelevant: the problems are independent
    }
  }
  running = __syncthreads_or(running);
  emit = __syncthreads_or(emit);
  if (threadIdx.x == 0) { flag_out[0] = running | (emit << 1); flag_out[1] = s_cnt; }
}

}  // namespace

// Bytes the Gram path allocates for a batch beyond the O(D') solver state: split-K Gram partials (one slice at least), the fp64
// factor, L^-1 and H^-1, the diagonal-block side buffers, the bf16 Y of wide systems (~26 D'^2 per problem) and the CSR operands
// (B.csr_gram must be set: one byte an entry for the wgmma kernel, one 32-bit word for the sparse kernel).
static int csr_operand_bytes(int csr_gram) { return csr_gram == CSR_GRAM_SPARSE ? 4 : 1; }
static double gram_path_bytes(const Batch& B) {
  const double Dp = round_up(B.ldx, 128), ldh = round_up(B.Dt, 32);
  double per = Dp * Dp * 4.0 + 3.0 * ldh * ldh * 8.0 + 2.0 * ldh * 32 * 8.0 + (cholesky_factored_direction((int)ldh) ? ldh * ldh * 2.0 : 0.0);
  double bytes = per * B.nprob;
  for (auto& p : B.h) bytes += (double)csr_operand_bytes(B.csr_gram) * (double)p.bm_entries;
  return bytes;
}

// Cost of one CSR Gram build of a partition (seconds; only the comparison matters).  wgmma: every 128 x 128 lower tile times every
// 32-row group on the tensor pipe, plus the producers' run loads (each 128-column block's run of every 32-row group is read once per
// tile it belongs to: nblk + 1 tiles, `reads` entries in all), which is what makes its rate fall at small n and high density.
// Sparse (column kernel): per product (a suffix word loaded and multiplied, one native shared atomic add), per entry (one position
// of the column index, the first run of its suffix loaded) and per cell of the lower triangle (each column's clear and epilogue:
// one rounding and one strided store a cell), with the whole device busy; a grid of fewer CTAs than two an SM is that much slower.
// Relative least-squares fits of tools/time_gram.py (REPS=3) over 0.3 - 20 % density at 10k features (DESIGN.md section 4): the
// wgmma constants on an H100 80GB HBM3 at a 400 W power limit, the sparse ones on an H100 80GB HBM3 at a 700 W power limit (the
// wgmma times there are within 3.5 % of the 400 W ones).  The sparse model is within 10.2 % and the wgmma model within 9.5 % of every
// measured shape, so near the crossover (~3 % at 10k features) the rule may pick a kernel up to ~10 % slower than the other.
constexpr double GRAM_WGMMA_S_PER_MAC = 1.317e-15, GRAM_WGMMA_S_PER_READ = 4.315e-12;
constexpr double GRAM_SPARSE_S_PER_PAIR = 3.084e-12, GRAM_SPARSE_S_PER_ENTRY = 1.174e-10, GRAM_SPARSE_S_PER_CELL = 5.048e-13;
static double gram_cost(const Problem& p, int Dp, int kind, int num_sms) {
  const double nblk = Dp / 128, tiles = nblk * (nblk + 1) / 2, groups = (double)((p.n + 31) / 32);
  if (kind == CSR_GRAM_WGMMA)
    return tiles * 128.0 * 128.0 * 32.0 * groups * GRAM_WGMMA_S_PER_MAC + (nblk + 1) * (double)p.bm_entries * GRAM_WGMMA_S_PER_READ;
  const double ctas = std::min(Dp, 2 * num_sms);   // gram_launch_csr_sparse's grid per problem
  return (p.gram_pairs * GRAM_SPARSE_S_PER_PAIR + (double)p.bm_entries * GRAM_SPARSE_S_PER_ENTRY +
          0.5 * Dp * (Dp + 1.0) * GRAM_SPARSE_S_PER_CELL) * std::max(1.0, 2.0 * num_sms / ctas);
}

// Allocate the per-problem solver state.  Data pointers (X, y, ...) and n must be filled in h[] first.
// hessian_policy 2 builds the batch matrix-free (Newton-CG on Hv passes, O(D') state per problem); with any other policy the batch
// is built matrix-free when what the Gram path would allocate exceeds the free device memory (it could not run at all).
// CSR Gram batches pick their kernel from the data: the sparse kernel when its cost model is lower and every partition is within
// its row and column limits (gram_sparse_max_rows, gram_sparse_max_cols), else the wgmma kernel.  csr_gram_force (a test hook's setting) overrides the choice.
int batch_alloc(Batch& B, int num_sms, int hessian_policy, int csr_gram_force) {
  const int nprob = B.nprob, ldx = B.ldx;
  B.Dp = round_up(B.ldx, 128);
  B.ldh = round_up(B.Dt, 32);
  long long maxn = 1;
  for (auto& p : B.h) maxn = std::max(maxn, p.n);
  // K1 grid: rows per tile and CTAs per SM of the kernel (CSR: 64-row tiles, 1024-thread CTAs at 64 registers, one per SM)
  int R = 64, cps = 1;
  if (!B.csr) {
    int S, G;
    size_t smem;
    if (!k1_dense_plan(ldx, &R, &S, &G, &smem, &cps))
      return fail(MLEASE_ERR_INVALID, "dense partitions support at most 4095 features (+intercept); use CSR input beyond that");
  }
  const long long row_tiles = (maxn + R - 1) / R;
  B.k1_dyn = (nprob > 1 && nprob <= 32) ? nprob : 0;
  if (B.k1_dyn) B.k1_grid = (int)std::max(1LL, std::min((long long)num_sms * cps, (long long)nprob * row_tiles));
  else B.k1_grid = (int)std::max(1LL, std::min(row_tiles, (long long)std::max(1, (num_sms * cps) / std::max(1, nprob))));
  B.gram_from_csr = B.csr ? 1 : 0;
  for (auto& p : B.h) if (!p.bm_offs) B.gram_from_csr = 0;
  B.csr_fx = B.gram_from_csr;
  if (hessian_policy == 2 && B.csr) {
    B.csr_fx = 1;
    for (auto& p : B.h) if (!p.csr_unique) B.csr_fx = 0;
  }
  // fused multi-lambda CSR K1: every problem has segment lists, the groups are whole, and the shared-memory vectors fit
  B.k1_fused = 0;
  if (B.csr && B.csr_fx && B.group_L >= 1 && B.group_L <= 4 && nprob % B.group_L == 0) {
    bool ok = true;
    for (auto& p : B.h) if (!p.sg_perm || p.sg_S != B.h[0].sg_S || p.sg_rows != B.h[0].sg_rows) ok = false;
    if (ok) {
      B.k1f_LP = B.group_L <= 1 ? 1 : (B.group_L == 2 ? 2 : 4);
      B.k1f_smem = (size_t)ldx * 4 * B.k1f_LP + (size_t)B.h[0].sg_rows * 4 * B.k1f_LP;
      if (B.k1f_smem <= 224 * 1024) { B.k1_fused = 1; B.k1_dyn = 0; B.k1_grid = B.h[0].sg_S; }
    }
  }
  const int gpart_rows = B.k1_fused ? 1 : B.k1_grid;   // the fused kernel keeps its partials in gpart_f (fp32)
  // Hv passes are modes of the deterministic CSR K1 kernels (sorted unique rows, fixed-point or segment-list accumulation)
  if (hessian_policy == 2 && !B.csr)
    return fail(MLEASE_ERR_INVALID, "hessian_policy 2 (matrix-free Newton-CG) needs CSR partitions; dense partitions (at most 4095 features) use the Gram path");
  if (hessian_policy == 2 && !B.csr_fx)
    return fail(MLEASE_ERR_INVALID, "hessian_policy 2 (matrix-free Newton-CG) needs CSR rows with strictly increasing column ids");
  B.matfree = hessian_policy == 2 ? 1 : 0;
  // the CSR Gram kernel first: its operand's size enters the memory check below
  B.csr_gram = 0;
  if (B.gram_from_csr && !B.matfree) {
    double t_sparse = 0, t_wgmma = 0;
    // the upload builds the sparse kernel's column index wherever both of its limits hold
    bool rows_fit = true, indexed = true;
    for (auto& p : B.h) {
      t_sparse += gram_cost(p, B.Dp, CSR_GRAM_SPARSE, num_sms);
      t_wgmma += gram_cost(p, B.Dp, CSR_GRAM_WGMMA, num_sms);
      if (p.n > gram_sparse_max_rows()) rows_fit = false;
      if (!p.gc_pos) indexed = false;
    }
    const bool fits = rows_fit && indexed && B.Dt <= gram_sparse_max_cols();
    B.csr_gram = (fits && t_sparse < t_wgmma) ? CSR_GRAM_SPARSE : CSR_GRAM_WGMMA;
    if (csr_gram_force == CSR_GRAM_SPARSE && !rows_fit)
      return fail(MLEASE_ERR_INVALID, "the sparse CSR Gram's int64 sums hold at most 2^27 rows per partition");
    if (csr_gram_force == CSR_GRAM_SPARSE && !fits)
      return fail(MLEASE_ERR_INVALID, "the sparse CSR Gram's operand word holds column ids below 2^20 (features + intercept)");
    if (csr_gram_force) B.csr_gram = csr_gram_force;
  }
  if (!B.matfree && B.csr && B.gram_from_csr) {
    // the Gram path's bytes plus the O(D') state allocated with it (vectors, L-BFGS pairs, per-CTA partials, sqrt(d) per row) and
    // a margin for the session's own vectors: a Gram path that would only just fit is not taken
    double state = 0;
    for (auto& p : B.h) state += 8.0 * (double)p.n;
    state += (double)nprob * (8.0 * ((9 + 2 * BFGS_M + gpart_rows) * (double)ldx + B.k1_grid + 8) + 16.0 * ldx +
                              (B.k1_fused ? 4.0 * B.k1_grid * ldx : 0.0));
    size_t free_b = 0, total_b = 0;
    CK(cudaMemGetInfo(&free_b, &total_b));
    if (gram_path_bytes(B) + state + (256.0 * 1024 * 1024) > (double)free_b) { B.matfree = 1; B.csr_gram = 0; }
  }
  // Cost model for the rebuild policy (seconds, order of magnitude only: the policy compares the two with a factor of 8): one K1
  // pass streams the partition at ~5 TB/s; a rebuild is n*Dt^2 flop at ~1 PFLOP/s (tensor-core Gram, lower triangle) plus
  // ~Dt^3 fp64 flop at ~5 TFLOP/s (Cholesky + inverse).
  {
    double bytes = 0;
    for (auto& p : B.h) bytes = std::max(bytes, B.csr ? 8.0 * (double)p.nnz_hint + 17.0 * (double)p.n : (double)p.n * 4.0 * ldx);
    const double t_pass = bytes / 5e12 + 20e-6;
    const double t_rebuild = (double)maxn * B.Dt * B.Dt / 1e15 + (double)B.Dt * B.Dt * B.Dt / 5e12 + 300e-6;
    // only wide systems qualify: small ones (NaiveTrain's per-key fits, cold-started every time) are launch-bound, not
    // flop-bound, and a mid-update rebuild saves them many lock-step slots
    B.rebuild_is_expensive = (t_rebuild > 8.0 * t_pass && B.Dt > 2048 && !B.matfree) ? 1 : 0;
  }
  // Gram decomposition (the sparse kernel walks columns: no tiles)
  constexpr int MAX_TILES = 1 << 18;   // lower 128x128 tiles of Dp up to ~90k
  const bool tiled = !B.matfree && B.csr_gram != CSR_GRAM_SPARSE;
  std::vector<short> tiles(tiled ? 2 * (size_t)MAX_TILES : 2);
  B.ntiles = tiled ? gram_tile_list(B.Dp, tiles.data(), MAX_TILES, B.gram_from_csr) : 0;
  if (B.ntiles <= 0 && tiled) return fail(MLEASE_ERR_INVALID, "Gram tile list overflow");
  if (tiled) {   // the sparse kernel has no split-K: one slice
    const long long ksteps = (maxn + 63) / 64;
    const long long base = (long long)B.ntiles * nprob;   // CTAs
    const long long cap = std::max(1, num_sms);
    int best = 1;
    double best_eff = 0;
    for (int s = 1; s <= 16; s++) {
      if (s > ksteps) break;
      const long long ctas = base * s;
      const double eff = (double)ctas / (double)(((ctas + cap - 1) / cap) * cap);
      if (eff > best_eff + 1e-9) { best_eff = eff; best = s; }
      if (eff >= 0.93 && ctas >= 2LL * cap) { best = s; break; }
    }
    // bound the split-K scratch to 1 GiB per batch
    while (best > 1 && (double)best * B.Dp * B.Dp * 4.0 * nprob > 1024.0 * 1024 * 1024) best--;
    B.gram_slices = best;
  }
  // matrix-free: the CG vectors r, p, z, Hp and diag(H) per problem instead of the L-BFGS pairs (no secant pairs are kept there)
  // doubles per problem, rounded up to a multiple of 4: every problem's vectors start 32-byte aligned (the triangular GEMVs and the
  // Hv passes read qf / tf / hv_vf as float4); the K1 partial count k1_grid (fused: its segment count) may be odd
  const size_t nd_prob = ((9 + (B.matfree ? 5 : 2 * BFGS_M)) * (size_t)ldx + 2 * BFGS_M + (size_t)gpart_rows * ldx + (size_t)B.k1_grid + 8 + 3) & ~(size_t)3;
  const size_t nd = (size_t)nprob * nd_prob;
  const size_t nf = (size_t)nprob * 4 * ldx;
  double* dd; float* ff; float* hp = nullptr; double* lc = nullptr; double* ld = nullptr; double* ldi = nullptr; double* yi = nullptr; double* hi = nullptr;
  if (int rc = B.mem.get(&dd, nd, true)) return rc;
  if (int rc = B.mem.get(&ff, nf, true)) return rc;
  float* gpf = nullptr;
  if (B.k1_fused)
    if (int rc = B.mem.get(&gpf, (size_t)nprob * B.k1_grid * ldx, true)) return rc;
  __nv_bfloat16* hif = nullptr;
  if (!B.matfree) {
    if (int rc = B.mem.get(&hp, (size_t)nprob * B.gram_slices * B.Dp * B.Dp, true)) return rc;
    if (int rc = B.mem.get(&lc, (size_t)nprob * B.ldh * B.ldh, true)) return rc;
    if (int rc = B.mem.get(&ld, (size_t)nprob * B.ldh * 32, true)) return rc;
    if (int rc = B.mem.get(&ldi, (size_t)nprob * B.ldh * 32, true)) return rc;
    if (int rc = B.mem.get(&yi, (size_t)nprob * B.ldh * B.ldh, true)) return rc;
    if (int rc = B.mem.get(&hi, (size_t)nprob * B.ldh * B.ldh, true)) return rc;
    if (cholesky_factored_direction(B.ldh))
      if (int rc = B.mem.get(&hif, (size_t)nprob * B.ldh * B.ldh, true)) return rc;
  }
  if (int rc = B.mem.get(&B.d_ctrl, (size_t)nprob, true)) return rc;
  if (int rc = B.mem.get(&B.d, (size_t)nprob, true)) return rc;
  if (nprob > 64 || B.lockstep)
    if (int rc = B.mem.get(&B.d_compact, (size_t)nprob, true)) return rc;
  if (int rc = B.mem.get(&B.d_tmaps, nprob, true)) return rc;
  if (int rc = B.mem.get(&B.d_tiles, (size_t)B.ntiles * 2, true)) return rc;
  CK(cudaMemcpy(B.d_tiles, tiles.data(), (size_t)B.ntiles * 2 * sizeof(short), cudaMemcpyHostToDevice));
  std::vector<CUtensorMap> maps(nprob);
  std::vector<size_t> pool_off(nprob);
  size_t pool_bytes = 0;
  for (int b = 0; b < nprob; b++) {
    pool_off[b] = pool_bytes;
    const bool windows = B.csr_fx && k1_csr_window(ldx) > 0;   // then a second [n] vector (row residuals) follows sdvec
    // CSR: sdvec (+ rvec), then the operand of the entry list (e4m3 bytes or sparse-kernel words; none in a matrix-free batch);
    // else the bf16 operand Xt
    const size_t need = B.csr_fx ? (((size_t)B.h[b].n * sizeof(float) * (windows ? 2 : 1) + 255) & ~(size_t)255) +
                                       (B.matfree ? 0 : (size_t)csr_operand_bytes(B.csr_gram) * (size_t)B.h[b].bm_entries)
                                        : (size_t)B.h[b].n * B.Dp * sizeof(__nv_bfloat16);
    pool_bytes += (need + 255) & ~(size_t)255;
  }
  unsigned char* pool = nullptr;
  if (int rc = B.mem.get(&pool, pool_bytes, true)) return rc;
  for (int b = 0; b < nprob; b++) {
    Problem& p = B.h[b];
    p.ldx = ldx; p.Dt = B.Dt; p.Dp = B.Dp; p.ldh = B.ldh; p.self_idx = b;
    p.k1_ctas = B.k1_grid;
    p.gram_slices = B.gram_slices;
    double* const q0 = dd;
    double* q = dd;
    p.beta = q; q += ldx; p.beta_t = q; q += ldx; p.m = q; q += ldx; p.q = q; q += ldx;
    p.g_t = q; q += ldx; p.g_acc = q; q += ldx; p.dir = q; q += ldx; p.x_d = q; q += ldx;
    p.qf = reinterpret_cast<float*>(q); p.tf = p.qf + ldx; q += ldx;   // one double-vector slot holds the two fp32 vectors of the triangular GEMVs
    if (!B.matfree) { p.bfgs_S = q; q += (size_t)BFGS_M * ldx; p.bfgs_Y = q; q += (size_t)BFGS_M * ldx; }
    p.bfgs_rho = q; q += BFGS_M; p.bfgs_alpha = q; q += BFGS_M;
    p.gpart = q; q += (size_t)gpart_rows * ldx;
    p.hv_vf = p.qf;
    if (B.matfree) { p.cg_r = q; q += ldx; p.cg_p = q; q += ldx; p.cg_z = q; q += ldx; p.cg_Hp = q; q += ldx; p.cg_diag = q; q += ldx; }
    p.gpart_f = gpf ? gpf + (size_t)b * B.k1_grid * ldx : nullptr;
    p.fpart = q; q += B.k1_grid + 8;
    dd = q0 + nd_prob;
    float* f = ff;
    p.beta_tf = f; f += ldx; p.u_f = f; f += ldx; p.uplusx_f = f; f += ldx; p.x_f = f; f += ldx;
    ff = f;
    p.Hpart = hp ? hp + (size_t)b * B.gram_slices * B.Dp * B.Dp : nullptr;
    p.Lc = lc ? lc + (size_t)b * B.ldh * B.ldh : nullptr;
    p.Ldiag = ld ? ld + (size_t)b * B.ldh * 32 : nullptr;
    p.Ldinv = ldi ? ldi + (size_t)b * B.ldh * 32 : nullptr;
    p.Yinv = yi ? yi + (size_t)b * B.ldh * B.ldh : nullptr;
    p.Hinv = hi ? hi + (size_t)b * B.ldh * B.ldh : nullptr;
    p.Ysym = hif ? hif + (size_t)b * B.ldh * B.ldh : nullptr;
    p.ctrl = B.d_ctrl + b;
    // Gram operand state, carved out of ONE allocation for the whole batch (NaiveTrain batches hold thousands of problems:
    // one cudaMalloc / cudaFree each would cost more than the fits)
    if (B.csr_fx) {
      p.sdvec = reinterpret_cast<float*>(pool + pool_off[b]);
      p.rvec = k1_csr_window(ldx) > 0 ? p.sdvec + p.n : nullptr;
      unsigned char* op = B.matfree ? nullptr : pool + pool_off[b] + (((size_t)p.n * sizeof(float) * (p.rvec ? 2 : 1) + 255) & ~(size_t)255);
      p.bm_e4m3 = B.csr_gram == CSR_GRAM_SPARSE ? nullptr : op;
      p.bm_word = B.csr_gram == CSR_GRAM_SPARSE ? reinterpret_cast<uint32_t*>(op) : nullptr;
      p.gram_from_csr = B.gram_from_csr;
      p.csr_gram = B.csr_gram;
      std::memset(&maps[b], 0, sizeof(CUtensorMap));
    } else {
      p.gram_from_csr = 0;
      p.csr_gram = 0;
      p.gram_scale = 1.f; p.gram_unscale = 1.f;   // bf16 dense-operand Gram: no operand scale
      p.Xt = reinterpret_cast<__nv_bfloat16*>(pool + pool_off[b]);
      if (gram_make_tensor_map(&maps[b], p.Xt, p.n, B.Dp) != 0) return fail(MLEASE_ERR_CUDA, "cuTensorMapEncodeTiled failed");
    }
  }
  CK(cudaMemcpy(B.d_tmaps, maps.data(), (size_t)nprob * sizeof(CUtensorMap), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(B.d, B.h.data(), (size_t)nprob * sizeof(Problem), cudaMemcpyHostToDevice));
  return 0;
}

// One Gram build of the problems d_probs[0 .. n) with the batch's kernel (force / share: see gram_wgmma_kernel)
cudaError_t batch_gram(const Batch& B, const Problem* d_probs, int n, int force, cudaStream_t st, int* launches, int share) {
  if (B.csr_gram == CSR_GRAM_SPARSE) return gram_launch_csr_sparse(d_probs, n, B.Dp, force, st, launches, share);
  if (B.gram_from_csr) return gram_launch_csr_wgmma(d_probs, n, B.d_tiles, B.ntiles, B.gram_slices, force, st, launches, share);
  return gram_launch_wgmma(d_probs, n, B.d_tmaps, B.d_tiles, B.ntiles, B.gram_slices, force, st, launches, share);
}

// flops one Gram build of problem p runs: 2 per product the sparse kernel forms, n Dt (Dt + 1) (lower triangle) for the wgmma kernels
static double gram_build_flops(const Batch& B, const Problem& p) {
  return B.csr_gram == CSR_GRAM_SPARSE ? 2.0 * p.gram_pairs : (double)p.n * (double)B.Dt * (double)(B.Dt + 1);
}

// K1 of a slot: the fused multi-lambda CSR kernel when the batch has segment lists, the per-problem kernels otherwise.
// mode K1_HV / K1_DIAG: the Hessian-vector / Hessian-diagonal pass of the problems with Ctrl::cg_active (CSR batches whose rows
// are sorted and unique only).
cudaError_t batch_k1(Batch& B, int force_emit, cudaStream_t st, int* launches, int mode) {
  if (mode != K1_GRAD && !(B.csr && B.csr_fx)) return cudaErrorInvalidValue;
  if (B.k1_fused)
    return k1f_launch(B.d, B.nprob / B.group_L, B.group_L, B.h[0].sg_S, B.k1f_LP, B.k1f_smem, B.has_bias, force_emit, st, launches, mode);
  return k1_launch(B.d, B.nprob, B.csr, B.ldx, B.has_bias, B.k1_grid, force_emit, st, launches, B.csr_fx, B.k1_dyn, mode);
}

// The factorisation of a rebuild slot over d_hess[0 .. n_hess) (the whole batch, or poll2_kernel's compacted copies).  share =
// group_L > 1 (cold start, d_hess = B.d): every problem's H is its group leader's Gram + its own diag(q); share_fact (equal rho
// too): only the leaders factorise, the followers take the leader's outcome and a copy of its H^-1.  skip_prep: Lc already holds H.
int batch_factor(Batch& B, const Problem* d_hess, int n_hess, int share, bool share_fact, int skip_prep, cudaStream_t st, int* launches) {
  // a follower still on a shared factor whose owner refactorises here takes a copy of the owner's bytes first
  if (B.ysym_shared) CK(cholesky_detach_followers(B.d, B.nprob, B.ldh, st, launches));
  if (share_fact) CK(cholesky_share_begin(B.d, B.nprob, share, st, launches));
  CK(cholesky_launch(d_hess, n_hess, B.ldh, st, launches, share, skip_prep));
  if (share_fact) {
    CK(cholesky_share_end(B.d, B.nprob, share, st, launches));
    if (cholesky_factored_direction(B.ldh)) B.ysym_shared = true;
    const size_t hh = (size_t)B.ldh * B.ldh;
    for (int b = 0; b < B.nprob; b++) {
      if (b % share == 0) continue;
      const Problem& lead = B.h[b - b % share];
      // wide systems work on the factored form Y = L^-1 (bf16, Ysym): that is all a follower needs
      if (!cholesky_factored_direction(B.ldh)) CK(cudaMemcpyAsync(B.h[b].Hinv, lead.Hinv, hh * sizeof(double), cudaMemcpyDeviceToDevice, st));
      // (Ysym is not copied: chol_share_end_kernel points the follower's Ctrl::ysym_use at the leader's)
    }
  }
  B.has_factor = true;
  return 0;
}

// Matrix-free direction of the problems that accepted a point this slot: diagonal pass, then CG steps in chunks of CG_CHUNK
// (Hv pass -> fixed-order reduction -> CG update each), one pinned read-back of the "any CG running" flag per chunk.
// Problems whose CG has finished return at once from every kernel of a chunk.
static int mf_direction(Batch& B, const SlotCtx& x) {
  constexpr int CG_CHUNK = 4;
  Profiler& pf = *x.pf;
  cudaStream_t st = x.st;
  int& launches = *x.launches;
  pf.begin(2, st);
  CK(cg_begin(B.d, B.nprob, st, &launches));
  CK(batch_k1(B, 0, st, &launches, K1_DIAG));
  CK(hv_reduce(B.d, B.nprob, B.Dt, 2, st, &launches));
  CK(cg_init(B.d, B.nprob, B.Dt, st, &launches));
  pf.end(st);
  for (int steps = 0; steps < CG_MAX_STEPS; steps += CG_CHUNK) {
    for (int j = 0; j < CG_CHUNK; j++) {
      pf.begin(2, st);
      CK(batch_k1(B, 0, st, &launches, K1_HV));
      CK(hv_reduce(B.d, B.nprob, B.Dt, 1, st, &launches));
      CK(cg_step(B.d, B.nprob, B.Dt, st, &launches));
      pf.end(st);
    }
    CK(cg_poll(B.d, B.nprob, x.d_flag + 2, st, &launches));
    CK(cudaMemcpyAsync(x.h_flag + 2, x.d_flag + 2, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (!x.h_flag[2]) break;
  }
  return 0;
}

// One slot's launches of an x-update: K1, the decide kernel, the Gram / Cholesky launches of a rebuild (with_hess), the
// matrix-free direction, newton_solve / newton_finish and, for large batches (x.poll), the end-of-slot poll.  spec: see
// k1_reduce_decide_kernel.  batch_xupdate and the slot-trace test hook both run their slots through this function.
int batch_slot(Batch& B, const SlotCtx& x, int slot_idx, bool with_hess, bool spec) {
  Profiler& pf = *x.pf;
  cudaStream_t st = x.st;
  int& launches = *x.launches;
  pf.begin(0, st);
  CK(batch_k1(B, B.matfree ? 1 : -1, st, &launches));   // matrix-free: every pass leaves sqrt(d) of its point for the Hv passes
  pf.end(st);
  pf.begin(1, st);
  CK(k1_reduce_decide(B.d, B.nprob, B.Dt, st, &launches, spec ? 1 : 0));
  pf.end(st);
  if (with_hess && x.n_hess > 0) {
    pf.begin(2, st);
    // cold start of a multi-lambda run: the L problems of a partition all sit at beta = 0, their Grams are the same
    const int share = (slot_idx == 0) ? x.share_first_gram : 0;
    if (share > 1)
      for (int b = 0; b < B.nprob; b++) if (b % share != 0) *x.shared_flops += gram_build_flops(B, B.h[b]);
    CK(batch_gram(B, x.d_hess, x.n_hess, 0, st, &launches, share));
    pf.end(st);
    pf.begin(3, st);
    const bool share_fact = share > 1 && x.share_first_factor;   // same rho too: same H, one factorisation per group
    if (int rc = batch_factor(B, x.d_hess, x.n_hess, share, share_fact, 0, st, &launches)) return rc;
    pf.end(st);
  }
  if (B.matfree)
    if (int rc = mf_direction(B, x)) return rc;
  pf.begin(1, st);
  if (B.matfree) CK(newton_finish(B.d, B.nprob, B.Dt, st, &launches));
  else CK(newton_solve(B.d, B.nprob, B.ldh, st, &launches, B.group_L));
  if (x.poll) { poll2_kernel<<<1, 256, 0, st>>>(B.d, B.nprob, x.d_flag, B.d_compact); launches++; }
  pf.end(st);
  return 0;
}

// One x-update for every problem of the batch: beta (init), m, q must already be on the device.
int batch_xupdate(Batch& B, cudaStream_t st, double xtol, int max_newton, int policy, int invalidate, int* h_flag, int* d_flag,
                  Counters& cnt, Profiler* prof, int share_first_gram, int share_first_factor) {
  Profiler nop;
  Profiler& pf = prof ? *prof : nop;
  int launches = 0;
  if (B.matfree) policy = 2;   // also when the batch was made matrix-free by the memory rule
  CK(newton_begin(B.d, B.nprob, xtol, max_newton, policy, invalidate, B.rebuild_is_expensive, st, &launches));
  // The first slot's flags are known on the host: every problem is running, and a rebuild is due iff the policy says
  // always, the factors were invalidated, or the mirrored control blocks say so (no factor yet / refresh requested).
  // small batches read the whole control array back each slot (one sync, no poll kernel) and pipeline their slots
  const bool small = B.nprob <= 64 && !B.lockstep;
  int flag = 1;
  {
    bool emit0 = policy == 1 || invalidate || B.mirror.empty();
    for (auto& c : B.mirror) if (!c.hess_valid || c.refresh_next) emit0 = true;
    if (emit0 && !B.matfree) flag |= 2;
  }
  B.mirror.resize(B.nprob);
  std::vector<Ctrl>& hc = B.mirror;
  int slots = 0;
  const Problem* d_hess = B.d;   // problems the Gram / Cholesky grids run over (large batches: compacted by poll2_kernel)
  int n_hess = B.nprob;
  double shared_flops = 0;   // Gram builds that were not run because the group's first problem stood in for them
  // One slot's launches (batch_slot).  with_hess: the Gram / Cholesky launches of a rebuild are included; spec: see k1_reduce_decide_kernel.
  auto enqueue_slot = [&](int slot_idx, bool with_hess, bool spec) -> int {
    const SlotCtx x{st, &pf, &launches, d_hess, n_hess, share_first_gram, share_first_factor, &shared_flops, h_flag, d_flag, !small};
    return batch_slot(B, x, slot_idx, with_hess, spec);
  };
  if (small) {
    // Slot pipeline: the host runs ONE slot ahead of what it knows.  While slot s executes, slot s+1 is already enqueued in
    // speculative form (no rebuild launches; a rebuild that turns out to be due is deferred by the decide kernel and shows
    // up as `emit` in the flags, after which a regular rebuild slot follows).  The read-back of the control blocks goes to
    // pinned double buffers and is awaited per slot (event), so the GPU never idles on the host between slots; a finished
    // x-update leaves at most one slot of early-exit kernels behind.
    for (int i = 0; i < 2; i++) {
      if (!B.h_ctrl[i]) if (int rc = B.pinned.get(&B.h_ctrl[i], B.nprob, false)) return rc;
      if (!B.slot_ev[i]) CK(cudaEventCreateWithFlags(&B.slot_ev[i], cudaEventDisableTiming));
    }
    const bool may_spec = policy == 0;
    auto flags_of = [&](const Ctrl* c, bool* all_valid) {
      int f = 0; bool v = true;
      for (int b = 0; b < B.nprob; b++) if (!c[b].done) { f |= 1; if (c[b].emit) f |= 2; if (!c[b].hess_valid) v = false; }
      *all_valid = v;
      return f;
    };
    auto finish_slot = [&](int idx) -> int {
      CK(cudaMemcpyAsync(B.h_ctrl[idx & 1], B.d_ctrl, (size_t)B.nprob * sizeof(Ctrl), cudaMemcpyDeviceToHost, st));
      CK(cudaEventRecord(B.slot_ev[idx & 1], st));
      return 0;
    };
    // what is known before slot 0: every problem runs; a rebuild is due iff emit0; factors are valid iff the mirror says so
    bool known_valid = !(flag & 2);
    if (int rc = enqueue_slot(0, (flag & 2) != 0, false)) return rc;
    if (int rc = finish_slot(0)) return rc;
    int s_cur = 0;          // newest slot in flight whose outcome is not known yet
    bool next_in_flight = false;
    int known_flag = flag;  // flags as of the newest COMPLETED slot (before slot 0: the host-side prediction)
    while (true) {
      // speculate slot s_cur + 1 on what is known (the state BEFORE slot s_cur): no rebuild pending, every factor valid
      const bool spec_next = may_spec && known_valid && !(known_flag & 2) && s_cur + 1 < 400;
      if (spec_next) {
        if (int rc = enqueue_slot(s_cur + 1, false, true)) return rc;
        if (int rc = finish_slot(s_cur + 1)) return rc;
        next_in_flight = true;
      }
      CK(cudaEventSynchronize(B.slot_ev[s_cur & 1]));
      std::memcpy(hc.data(), B.h_ctrl[s_cur & 1], (size_t)B.nprob * sizeof(Ctrl));
      slots = s_cur + 1;
      known_flag = flags_of(hc.data(), &known_valid);
      if (!(known_flag & 1) || slots >= 400) break;          // finished (a speculative slot in flight is a no-op)
      if (next_in_flight) { s_cur++; next_in_flight = false; continue; }
      if (int rc = enqueue_slot(s_cur + 1, (known_flag & 2) != 0, false)) return rc;
      if (int rc = finish_slot(s_cur + 1)) return rc;
      s_cur++;
    }
    flag = known_flag;
  }
  while (!small && (flag & 1) && slots < 400) {
    if (int rc = enqueue_slot(slots, (flag & 2) != 0, false)) return rc;
    CK(cudaMemcpyAsync(h_flag, d_flag, 2 * sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    flag = h_flag[0];
    n_hess = h_flag[1];
    d_hess = B.d_compact;
    slots++;
  }
  if (!small) {
    CK(cudaMemcpyAsync(hc.data(), B.d_ctrl, (size_t)B.nprob * sizeof(Ctrl), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  cnt.launches += launches;
  cnt.last_slots = slots;
  int bad_spd = 0, bad_ls = 0;
  if (pf.on) CK(cudaStreamSynchronize(st));   // a trailing speculative slot may still be running: its events must have completed
  pf.resolve();
  for (int b = 0; b < B.nprob; b++) {
    const Ctrl& c = hc[b];
    const Problem& p = B.h[b];
    const double rowbytes = B.csr ? 17.0 : (4.0 * B.ldx + 9.0);
    cnt.k1_bytes += (double)c.evals * ((double)p.n * rowbytes + (B.csr ? 8.0 * (double)p.nnz_hint : 0.0));
    cnt.gram_flops += (double)c.hess_builds * gram_build_flops(B, p);
    cnt.k1_emit_bytes += (double)c.hess_builds * (double)p.n * (double)B.Dp * 2.0;
  }
  cnt.gram_flops -= shared_flops;
  if (B.csr) {
    // the problems of a group advance in lock step from the first slot and drop out as they converge: slot t serves the
    // problems with evals > t, so a group's passes = max evals, and the lambdas served in total = sum of evals
    const int gl = std::max(1, B.group_L);
    for (int g0 = 0; g0 + gl <= B.nprob; g0 += gl) {
      int mx = 0; long long sum = 0;
      for (int l = 0; l < gl; l++) { mx = std::max(mx, hc[g0 + l].evals); sum += hc[g0 + l].evals; }
      const Problem& p = B.h[g0];
      cnt.k1_shared_bytes += (double)mx * (8.0 * (double)p.nnz_hint + 9.0 * (double)p.n) + (double)sum * 8.0 * (double)p.n;
    }
  }
  for (auto& c : hc) {
    cnt.k1_passes += c.evals; cnt.newton_steps += c.newton_steps; cnt.rejected += c.rejects; cnt.gram_builds += c.hess_builds;
    if (c.fail == 3 || !c.done) cnt.not_converged++;
    if (c.fail == 1) bad_spd++;
    if (c.fail == 2) bad_ls++;
  }
  if (bad_spd) return fail(MLEASE_ERR_NUMERIC, "Model fitting error! (Hessian not positive definite in " + std::to_string(bad_spd) + " problem(s))");
  if (bad_ls) return fail(MLEASE_ERR_NUMERIC, "Model fitting error! (line search failed in " + std::to_string(bad_ls) + " problem(s))");
  return 0;
}

}  // namespace mlease
