// kernels.cuh -- launcher declarations shared by the translation units of libmlease_b200.so
#pragma once
#include "common.cuh"

namespace mlease {

// the dynamic shared-memory attribute is per device: set it once for every device this process launches on
template <typename K>
inline cudaError_t set_smem_once(K kernel, size_t bytes, bool (&configured)[64]) {
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) configured[dev] = true;
  }
  return cudaSuccess;
}

// K1 (k1_score_grad.cu)
bool k1_dense_plan(int ldx, int* R_out, int* S_out, int* G_out, size_t* smem_out, int* ctas_per_sm);
int k1_csr_window(int ldx);
cudaError_t k1_launch(const Problem* d_probs, int nprob, bool csr, int ldx, int has_bias, int ctas_per_problem,
                      int force_emit, cudaStream_t stream, int* launches, int csr_fx = 0, int nprob_dyn = 0, int mode = K1_GRAD);

// fused multi-lambda CSR K1 (k1_csr_fused.cu)
bool k1f_plan(long long n, int ldx, int L, int num_sms, int* S_out, int* rows_out, int* LP_out, size_t* smem_out);
cudaError_t k1f_build(long long n, int Dg, long long nnz, const long long* rowptr, const int* colidx, const float* vals, int S, int sg_rows, int* ngrp_out,
                      int** perm_out, int** depth_out, long long** goff_out, unsigned short** row16_out, float** val_out, long long* total_out,
                      unsigned short** col16_out, cudaStream_t st);
cudaError_t k1f_launch(const Problem* d_probs, int ngroups, int L, int S, int LP, size_t smem, int has_bias, int force_emit, cudaStream_t st, int* launches,
                       int mode = K1_GRAD);
// max over rows of sum_j |v_ij| (float bits, non-negative: order preserving) -> *out (k1_score_grad.cu)
cudaError_t csr_row_l1_max(long long n, const long long* rowptr, const float* vals, unsigned* out, cudaStream_t st);

// Newton state machine (newton.cu)
cudaError_t newton_begin(const Problem* d_probs, int nprob, double xtol, int max_newton, int hess_policy,
                         int invalidate_hess, int rebuild_is_expensive, cudaStream_t st, int* launches);
cudaError_t k1_reduce_decide(const Problem* d_probs, int nprob, int Dt, cudaStream_t st, int* launches, int spec = 0);
cudaError_t newton_solve(const Problem* d_probs, int nprob, int ldh, cudaStream_t st, int* launches, int group_L = 1);
// the two triangular GEMVs of the factored direction (ldh > 2048) alone, over the whole batch: dir = Y^T (Y qf), t in tf
cudaError_t newton_gemv_tri(const Problem* d_probs, int nprob, int ldh, int group_L, cudaStream_t st);
// matrix-free Newton-CG direction (newton.cu): begin (pick the problems that need a direction), the fixed-order reduction of the
// Hv / diagonal partials (out 0: g_t, 1: cg_Hp, 2: cg_diag), init (after the diagonal pass), one CG step (after an Hv pass), and
// the poll of the CG flags into *d_any (1 while a problem's CG still runs)
cudaError_t cg_begin(const Problem* d_probs, int nprob, cudaStream_t st, int* launches);
cudaError_t hv_reduce(const Problem* d_probs, int nprob, int Dt, int out, cudaStream_t st, int* launches);
cudaError_t cg_init(const Problem* d_probs, int nprob, int Dt, cudaStream_t st, int* launches);
cudaError_t cg_step(const Problem* d_probs, int nprob, int Dt, cudaStream_t st, int* launches);
cudaError_t cg_poll(const Problem* d_probs, int nprob, int* d_any, cudaStream_t st, int* launches);
// the direction bookkeeping of newton_solve alone (the direction is already in dir, no secant pairs)
cudaError_t newton_finish(const Problem* d_probs, int nprob, int Dt, cudaStream_t st, int* launches);

// K2 (k2_gram.cu)
int gram_make_tensor_map(void* out_map_host, const void* xt, long long n, int Dp);
int gram_tile_list(int Dp, short* bi_bj_pairs, int max_tiles, int csr_tiles = 0);
cudaError_t gram_launch_wgmma(const Problem* d_probs, int nprob, const void* d_tmaps, const void* d_tiles, int ntiles,
                              int nslices, int force, cudaStream_t st, int* launches, int share = 0);
cudaError_t gram_launch_csr_wgmma(const Problem* d_probs, int nprob, const void* d_tiles, int ntiles, int nslices, int force,
                                  cudaStream_t st, int* launches, int share = 0);
// the exact sparse CSR Gram of Dp x Dp problems (one slice), the largest partition (rows) and system (D') it accepts, and its
// column index, built once at upload: for column c < bias_col + 1 the positions pos[offs[c] .. offs[c + 1]) of its entries in
// the row-order operand (row r at [rowptr[r] + r, rowptr[r + 1] + r], its intercept entry last)
cudaError_t gram_launch_csr_sparse(const Problem* d_probs, int nprob, int Dp, int force, cudaStream_t st, int* launches, int share = 0);
long long gram_sparse_max_rows();
int gram_sparse_max_cols();
cudaError_t csr_col_index(long long n, const long long* rowptr, const int* colidx, int bias_col, long long entries, uint32_t* offs,
                          uint32_t* pos, cudaStream_t st);
cudaError_t csr_bm_offsets(long long n, const long long* rowptr, const int* colidx, int bias_col, int nblk, long long ngroups, long long* offs,
                           cudaStream_t st);
cudaError_t csr_bm_fill(long long n, const long long* rowptr, const int* colidx, const float* vals, int bias_col, int nblk, long long ngroups,
                        const long long* offs, unsigned short* keys, float* bvals, cudaStream_t st);
cudaError_t gram_launch_simt(const Problem* d_probs, int nprob, int Dp, int force, cudaStream_t st, int* launches);

// K3 (k3_cholesky.cu)
cudaError_t cholesky_launch(const Problem* d_probs, int nprob, int ldh, cudaStream_t st, int* launches, int share = 0, int skip_prep = 0,
                            int want_hinv = 0);
// the first launch of cholesky_launch: Lc = sum of the Gram partials (the group leader's when share > 1) + diag(q), identity padding
cudaError_t cholesky_prep(const Problem* d_probs, int nprob, int ldh, int share, cudaStream_t st, int* launches);
// test support: the same fp64 products through DMMA m8n8k4 and m16n8k4 (k3_cholesky.cu, mlease_internal_dmma_shapes)
cudaError_t dmma_shapes(const double* A, const double* B, int n, int K, double* D8, double* D16, cudaStream_t st);
bool cholesky_factored_direction(int ldh);   // wide systems: Ysym holds Y = L^-1 (bf16, symmetric storage), the direction is Y^T (Y q)
cudaError_t cholesky_share_begin(const Problem* d_probs, int nprob, int share, cudaStream_t st, int* launches);
cudaError_t cholesky_share_end(const Problem* d_probs, int nprob, int share, cudaStream_t st, int* launches);
// before a rebuild slot of a wide batch whose followers may still read a shared cold-start factor: every follower whose owner
// refactorises in this slot (and which does not) copies the owner's Ysym into its own and points at it (d_probs: the whole batch)
cudaError_t cholesky_detach_followers(const Problem* d_probs, int nprob, int ldh, cudaStream_t st, int* launches);
// K4 (k4_consensus.cu)
cudaError_t admm_reset(const Problem* d_probs, int nprob, int L, double* d_z, int ldv, const double* d_rho_eff,
                       cudaStream_t st, int* launches);
cudaError_t admm_init(const Problem* d_probs, int nprob, const double* d_z, int ldv, cudaStream_t st, int* launches);
cudaError_t admm_pack(const Problem* d_probs, int nlocal_parts, int L, int Dt, double* d_exchange, cudaStream_t st,
                      int* launches);
cudaError_t admm_consensus(const Problem* d_probs, int nlocal_parts, int L, int Dt, int ldv, int P, const double* d_exchange_sum,
                           double* d_z, const double* d_wz, const double* d_rho_eff_next, double* d_diff, cudaStream_t st,
                           int* launches, const double* d_l1_thr = nullptr);

// posterior variance (k6_postvar.cu): exact fp64 Hessian diagonal / full Hessian into Lc
// rowweights / diag run over the problems d_probs[0 .. nprob): problem b owns rows [d_row_start[b], d_row_start[b+1]) of d_dvec
// (nrows = d_row_start[nprob]); d_dvec[r] = w_i p_i (1 - p_i) at the problem's beta; diag leaves q + sum_i d_i x_ik^2 in each g_t
cudaError_t postvar_rowweights(const Problem* d_probs, int nprob, const long long* d_row_start, long long nrows, int has_bias, double* d_dvec,
                               cudaStream_t st, int* launches);
cudaError_t postvar_diag(const Problem* d_probs, int nprob, const long long* d_row_start, long long nrows, const double* d_dvec, int has_bias,
                         cudaStream_t st, int* launches);
cudaError_t postvar_hessian(const Problem* d_prob, bool csr, int ldh, const double* d_dvec, const double* d_q, int has_bias, cudaStream_t st,
                            int* launches);
// the full Hessian of every problem d_probs[0 .. nprob) of a CSR batch (rows with strictly increasing column ids, width ldh) into its
// Lc, as chol_prep leaves it; deterministic (no atomics, every cell summed in row order)
cudaError_t postvar_hessian_batch(const Problem* d_probs, int nprob, int ldh, const long long* d_row_start, const double* d_dvec, int has_bias,
                                  cudaStream_t st, int* launches);
// the ADMM model's posterior (mlease_admm_posterior): every kernel is deterministic (fixed summation order, no atomics on values).
// rowof: rowof[q] = r for the n + nnz positions of the sparse Gram's row-order operand (row r at [rowptr[r] + r, rowptr[r + 1] + r]).
// hessian_csr_cols: H[c2][c1] += sum_i d_i x_{i,c1} x_{i,c2} (c2 >= c1, the intercept an implicit column Dt - 1, ld ldh) of one CSR
// partition with strictly increasing columns, from the column index offs [Dt + 1] / pos and rowof; hessian_dense_add: the same for the
// dense rows of d_prob[0] into its Lc (ld ldh); diag_*: diag[k] += sum_i d_i x_ik^2; lc: Lc = Hs + diag(q) as chol_prep leaves it;
// pack: the lower triangle of [0, Dt) to (unpack = 0) or from (1) Dt (Dt + 1) / 2 packed doubles
cudaError_t postvar_rowof(long long n, const long long* rowptr, uint32_t* rowof, cudaStream_t st);
cudaError_t postvar_hessian_csr_cols(long long n, const long long* rowptr, const int* colidx, const float* vals, const double* d_dvec,
                                     const uint32_t* offs, const uint32_t* pos, const uint32_t* rowof, int Dt, int ldh, double* H, cudaStream_t st);
cudaError_t postvar_hessian_dense_add(const Problem* d_prob, int ldh, const double* d_dvec, cudaStream_t st);
cudaError_t postvar_diag_csr_cols(const long long* rowptr, const float* vals, const double* d_dvec, const uint32_t* offs, const uint32_t* pos,
                                  const uint32_t* rowof, int Dt, double* diag, cudaStream_t st);
cudaError_t postvar_diag_dense(long long n, int Dt, const float* X, int ldx, const double* d_dvec, double* diag, cudaStream_t st);
cudaError_t postvar_lc(const double* Hs, const double* d_q, int Dt, int ldh, double* Lc, cudaStream_t st);
cudaError_t postvar_pack(double* H, int Dt, int ldh, double* packed, int unpack, cudaStream_t st);

}  // namespace mlease
