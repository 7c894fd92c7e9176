/*
 * mlease_internal.h -- the mlease_internal_* test hooks of libmlease_b200.so: exported for the tests and tools that drive single
 * kernels of a session's batches, not part of the C ABI (include/mlease_b200.h does not declare them).  Defined in test_hooks.cu,
 * bound for Python in mlease_b200/_hooks.py.
 *
 * A hook that runs kernels on the ADMM batch borrows it: it injects its state, launches, reads back, and on every return path parks
 * every problem's control block -- the block as it was before the hook, with done = 1, h0_scale = 1 and hess_valid, need_solve,
 * need_hess, have_dir, bfgs_count, skip_eval, refresh_next, cg_active, k1_chunks, fail = 0 (pointers and ysym_use untouched).  That
 * consumes the batch's x-update state: mlease_admm_local_step (iterate, run) refuses until mlease_admm_begin runs again.  Every
 * refusal of a hook returns before it touches the batch.
 */
#ifndef MLEASE_INTERNAL_H
#define MLEASE_INTERNAL_H

#include "../../include/mlease_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* mlease_internal_set_keyed_budget caps, process-wide, the device bytes the keyed calls (mlease_naive_train*,
 * mlease_item_model_train, mlease_score_keyed[_var]) and mlease_test_auc plan with (0 = the free memory only), so that small inputs
 * stream through many chunks.  mlease_internal_keyed_last_call reports the most recent keyed call of the process: the key
 * boundaries of its chunks (*count of them, the first 0 and the last K; for mlease_test_auc the set boundaries, the last num_sets;
 * up to cap are written), whether it streamed (mlease_test_auc: ran more than one chunk), and for a streamed call the host
 * milliseconds its rows took to stage (all chunks: a fit's copy into the pinned ring and H2D, on a staging thread; scoring's
 * direct copies, queued from the calling thread) and the milliseconds a fit waited for its staging thread (0 for scoring; both 0 for mlease_test_auc). */
int mlease_internal_set_keyed_budget(int64_t bytes);
int mlease_internal_keyed_last_call(int64_t* bounds, int32_t cap, int32_t* count, int32_t* streamed, double* stage_ms, double* wait_ms);

/* One Hv (mode 1) or Hessian-diagonal (mode 2) pass over the session's ADMM batch -- every (partition, lambda) problem at its own
 * point w[b] and vector v[b] (b = local partition * L + lambda, Dt entries each), through the kernels a matrix-free x-update runs
 * (fused multi-lambda or per-problem).  out[b] = the data term X^T D X v resp. sum_i d_i x_ic^2, without the prior.  Consumes the
 * batch's x-update state. */
int mlease_internal_batch_hv(mlease_session* s, int32_t mode, const double* w, const double* v, double* out);

/* One gradient pass over the session's ADMM batch (after begin()) through exactly the K1 kernels batch_k1 runs for it.  Problem b
 * (= local partition * L + lambda) is evaluated at float(w[b]) (Dt entries) when active[b] != 0; the others are marked done before
 * the launch, as problems that converged earlier are in an x-update.  skip_eval is cleared and the pass emits its Gram operand
 * (force_emit = 1).  The per-chunk partials are reduced by the fixed-order reduction of the solver.  Outputs (inactive problems:
 * NaN): f_out[b] = the loss (fpart summed in chunk order), g_out[b] (Dt) = the data-term gradient without the prior; if not NULL,
 * sd_out = sqrt(d_i) of every problem's rows, problem after problem (csr_fx batches: sdvec), and xt_out = the bf16 bits of the Xt
 * operand, n x Dp per problem (dense and general-CSR batches).  info (8 + nprob ints): [0] kernel kind (1 dense, 2 CSR fixed point,
 * 3 CSR fixed point with column windows, 4 general CSR, 5 fused multi-lambda CSR), [1] G (dense), LP (fused), beta in shared memory
 * (fixed point, general CSR), [2] k1_dyn, [3] k1_grid, [4] rows per thread RT (dense), rows per segment (fused), column window
 * width (windows), [5] row slices nsl (dense), [6] nprob, [7] 0, [8 + b] Ctrl::k1_chunks of an active problem (0 otherwise).
 * Consumes the batch's x-update state. */
int mlease_internal_batch_grad(mlease_session* s, const int32_t* active, const double* w, double* f_out, double* g_out, float* sd_out,
                               uint16_t* xt_out, int32_t* info);

/* One factorisation of the session's ADMM batch (after begin()) with an explicit inverse (ldh <= 2048), through batch_factor -- the
 * code of the solver's rebuild slot.  Problem b (= local partition * L + lambda):
 *   mode[b] = 0: done, no kernel may touch it;  1: Lc = H[b] (Dt x Dt row-major, lower triangle read) as chol_prep leaves it, then
 *   the factorisation without prep;  2: the fp32 Gram G[b] (Dt x Dt) goes into Hpart slice 0 (the other slices are zeroed), q[b]
 *   (Dt) into q, gram_unscale = 1, and chol_prep_kernel forms H with the batch's share.
 * order (norder entries, NULL: the batch order): the grids run over a device array of Problem copies in that order, as they run over
 * poll2_kernel's compacted array in batches of more than 64 problems.  share (0 or group_L > 1) and share_factor mirror the cold
 * start of a rebuild slot: share alone = distinct rho (every problem factorises the leader's Gram + its own q), share_factor too =
 * equal rho (the leaders factorise, chol_share_end_kernel and the Hinv copies serve the followers).  A batch mixing modes 1 and 2
 * runs chol_prep_kernel on its own first, with the mode-1 problems parked (need_hess = 0), then batch_factor without prep.  Before
 * the launch every problem's Lc, Ldiag, Ldinv, Yinv and Hinv are filled with a NaN sentinel (all bits set), except the strict upper
 * triangle of Yinv, which stays 0: the DMMA merges and Y^T Y of systems wider than 1000 read it as the zeros of a triangular matrix.
 * Outputs, each if not NULL: L_out (Dt x Dt), Y_out and Hinv_out (ldh x ldh), Ldinv_out (ldh x 32), ctrl_out (4 per problem: fail,
 * done, hess_valid, tot_hess as the kernels left them; the hook starts every problem from 0, 0/1, 0, 0).  Every argument is checked
 * before any launch.  gram_unscale and q are restored; the batch's x-update state is consumed. */
int mlease_internal_batch_factor(mlease_session* s, const int32_t* mode, const double* H, const float* G, const double* q,
                                 const int32_t* order, int32_t norder, int32_t share, int32_t share_factor, double* L_out,
                                 double* Y_out, double* Hinv_out, double* Ldinv_out, int32_t* ctrl_out);

/* The quasi-Newton direction on the explicit inverse (ldh <= 2048) of the problems with active[b] != 0, through the kernels of a
 * chord slot: k1_reduce_decide (its first L-BFGS loop) and newton_solve (newton_gemv_kernel, the second loop, h0_scale, the trial
 * point).  Run it after mlease_internal_batch_factor: it multiplies whatever Hinv holds.  Per active problem: the data-term gradient
 * g[b] (Dt), the secant ring S[b], Y[b] (BFGS_M x Dt each, slot-major), rho[b] (BFGS_M), count[b] = Ctrl::bfgs_count (>= 0; above
 * BFGS_M the ring has wrapped), h0[b] = Ctrl::h0_scale and the point beta[b] (Dt).  The decide kernel takes its accept path with no
 * pass over the rows: skip_eval = 1 (k1_partial_reduce_kernel leaves g_t alone, no loss partials: k1_chunks = 0), beta_t = m = beta
 * (the prior term is 0), have_dir = 0 (no line search, no new secant pair), hess_valid = 1, emit = 0 (no rebuild), newton_steps =
 * evals = 0 and max_newton >= 1 (no stop test can end the x-update).  Outputs, each if not NULL: dir_out (Dt per problem), phi0_out
 * = Ctrl::phi0, dirnorm_out = Ctrl::dirnorm, beta_t_out (Dt; float(beta + dir) as stored); an inactive problem's are NaN.  Checked
 * before any launch; consumes the batch's x-update state. */
int mlease_internal_direction(mlease_session* s, const int32_t* active, const double* g, const double* S, const double* Y,
                              const double* rho, const int32_t* count, const double* h0, const double* beta, double* dir_out,
                              double* phi0_out, double* dirnorm_out, double* beta_t_out);

/* The x-update fields of Ctrl as mlease_internal_newton_stage exchanges them, per problem: 23 ints and a pad, 14 reals, then the
 * cumulative counters (read back only).  The Ctrl pointers and ysym_use are never taken from the caller. */
#define STAGE_INTS(X)                                                                                                              \
  X(done) X(have_dir) X(need_solve) X(need_hess) X(emit) X(hess_valid) X(fail) X(newton_steps) X(evals) X(rejects) X(hess_builds) \
  X(stall) X(bfgs_count) X(k1_chunks) X(refresh_next) X(skip_eval) X(warm_used) X(build_step) X(max_newton) X(hess_policy)        \
  X(rebuild_is_expensive) X(cg_active) X(cg_iter)
#define STAGE_REALS(X) \
  X(h0_scale) X(worst_ratio) X(alpha) X(phi0) X(f_acc) X(f_t) X(gnorm) X(gnorm_prev) X(dirnorm) X(dirnorm_prev) X(xtol) X(cg_rz) X(cg_g2) X(hv_vinf)
#define STAGE_TOTALS(X) X(tot_evals) X(tot_newton) X(tot_rejects) X(tot_hess)
typedef struct StageCtrl {
#define X(f) int32_t f;
  STAGE_INTS(X)
#undef X
  int32_t pad_;
#define X(f) double f;
  STAGE_REALS(X)
  STAGE_TOTALS(X)
#undef X
} StageCtrl;

/* stages of mlease_internal_newton_stage and of mlease_internal_consensus */
enum { ST_BEGIN = 1, ST_DECIDE = 2, ST_SOLVE = 4, ST_FINISH = 8, ST_CG_BEGIN = 16, ST_CG_INIT = 32, ST_CG_STEP = 64, ST_CG_POLL = 128 };
enum { CS_RESET = 1, CS_INIT = 2, CS_PACK = 4, CS_CONSENSUS = 8 };

/* Injects an x-update state into every problem of the begun ADMM batch, runs the selected kernels of the Newton state machine
 * (newton.cu) once, each through the solver's own launcher, and reads the whole state back.
 *   stages: ST_BEGIN newton_begin(begin_args = {xtol, max_newton, policy, invalidate, rebuild_is_expensive}); ST_DECIDE
 *   k1_reduce_decide(spec) -- the fixed-order reduction of the partials and the decide kernel, no pass over the rows; ST_CG_BEGIN,
 *   ST_CG_INIT, ST_CG_STEP, ST_CG_POLL (matrix-free batches; *cg_any = the poll's flag) -- cg_init finds the diagonal's data term in
 *   cg_diag and cg_step finds X^T D X p in cg_Hp, as the reductions of their passes leave them; ST_SOLVE newton_solve (the GEMV on
 *   whatever Hinv / Ysym the batch holds, then newton_solve_kernel) or ST_FINISH newton_finish (newton_solve_kernel alone, on the r
 *   = H0^-1 q the caller put into dir).  They run in that order.  stages = 0 injects and runs nothing: info only.
 *   ctrl: nprob StageCtrl, in and out.  vec: nprob x 12 x ldx doubles (beta, beta_t, m, q, g_t, g_acc, dir, cg_r, cg_p, cg_z, cg_Hp,
 *   cg_diag; the last five only on a matrix-free batch), ring: nprob x (2 BFGS_M ldx + 2 BFGS_M) doubles (bfgs_S, bfgs_Y -- not on
 *   a matrix-free batch --, bfgs_rho, bfgs_alpha), fvec: nprob x 3 x ldx floats (beta_tf, qf = hv_vf, tf); all in and out, whole
 *   vectors, padding included, copied as bytes (a caller marks what no kernel may write with any pattern it likes).
 *   gpart (nprob x nct_cap x ldx doubles; stored as fp32 into gpart_f on a fused batch) and fpart (nprob x nct_cap), or both NULL
 *   when every k1_chunks is 0.
 *   info (12 ints): nprob, Dt, ldx, ldh, partial rows allocated per problem (k1_grid), fused K1, matrix-free, Ysym present,
 *   rebuild_is_expensive, group_L, 0, 0.
 * Refused before any launch: a state the kernels would index memory with (k1_chunks beyond the allocated rows or nct_cap,
 * bfgs_count < 0, a policy other than 2 or secant pairs on a matrix-free batch, which has no ring), ST_SOLVE on a batch that never
 * factorised (no batch_factor ran on it: mlease_internal_batch_factor or a rebuild slot), ST_SOLVE together with ST_FINISH, CG
 * stages on a batch without CG vectors.  With stages set, consumes the batch's x-update state. */
int mlease_internal_newton_stage(mlease_session* s, int32_t stages, int32_t spec, const double* begin_args, void* ctrl, double* vec,
                                 double* ring, float* fvec, const double* gpart, const double* fpart, int32_t nct_cap, int32_t* info,
                                 int32_t* cg_any);

/* One real x-update of the begun ADMM batch (at most 64 problems), slot by slot, through batch_slot -- the slot code batch_xupdate
 * runs: K1, the decide kernel, the Gram / Cholesky launches of a rebuild, the matrix-free direction, newton_solve / newton_finish.
 * args = {xtol (<= 0: the session's), max_newton (<= 0: the session's), policy, invalidate}; a matrix-free batch runs policy 2
 * whatever is asked, as in batch_xupdate.  newton_begin, then slots until every problem is done or max_slots have run.  spec[i] != 0
 * asks for slot i in speculative form (no rebuild launches); it is honoured as batch_xupdate would: only when, as of the state before
 * slot i - 1, every running problem had a valid factor and no rebuild was due.  A regular slot includes the rebuild launches iff a
 * running problem has emit set.  Refused before any launch: spec under a policy other than 0, spec for slot 0, a batch of more than
 * 64 problems (batch_xupdate never speculates there).  The trace has max_slots + 1 entries, entry 0 the state newton_begin left and
 * entry i + 1 the state after slot i, each in the layout of mlease_internal_newton_stage (ctrl: nprob StageCtrl; vec, ring, fvec);
 * slot_info (2 ints per slot): ran speculatively, included the rebuild launches; *nslots = slots run.  The batch is left as after an
 * x-update (beta = x): this hook does not consume its state. */
int mlease_internal_xupdate_trace(mlease_session* s, const double* args, const int32_t* spec, int32_t max_slots, void* ctrl_trace,
                                  double* vec_trace, double* ring_trace, float* fvec_trace, int32_t* slot_info, int32_t* nslots);

/* The factored direction of wide systems (ldh > 2048): each of the next four hooks refuses, before any launch, a batch that has no
 * Ysym (ldh <= 2048, or matrix-free), since the kernels they run dereference it.
 *
 * mlease_internal_factor: the caller's Dt x Dt H (row-major; its lower triangle is read) goes into the scratch problem's Lc of
 * partition pid as chol_prep leaves it (lower triangle, identity on the padding, zero above), then the factorisation the solver runs
 * for its direction: fp64 Cholesky, recursive inverse with TF32 merges, bf16 symmetric packing.  Read back, each if not NULL: Lc
 * (Dt x Dt), Yinv (ldh x ldh, whole) and the raw bits of Ysym (ldh x ldh).  The scratch problem's control block is cleared. */
int mlease_internal_factor(mlease_session* s, int32_t pid, const double* H, double* L_out, double* Y_out, uint16_t* ysym_out);

/* mlease_internal_factored_direction: on the ADMM batch (after begin() and at least one iterate()), the two triangular GEMV phases
 * of the direction for the problems with active[b] != 0, each on its q[b] (Dt entries; b = local partition * L + lambda), over the
 * whole problem array with the batch's group_L, exactly as newton_solve launches them.  t_out[b] / dir_out[b] (Dt entries each, if
 * not NULL) receive tf and dir; dir is filled with NaN beforehand, so an inactive problem keeps NaN.  Consumes the batch's x-update
 * state. */
int mlease_internal_factored_direction(mlease_session* s, const int32_t* active, const float* q, float* t_out, double* dir_out);

/* mlease_internal_ysym: the bytes problem b of the ADMM batch streams in its direction (Ctrl::ysym_use, else its own Ysym; ldh x ldh
 * bf16 bits), the index of the problem that owns them, and b's factorisation count (Ctrl::tot_hess).  Reads only. */
int mlease_internal_ysym(mlease_session* s, int32_t b, uint16_t* out, int32_t* owner, int32_t* tot_hess);

/* mlease_internal_request_refresh: problem b of the ADMM batch refactorises at the start point of its next x-update, as after a slow
 * x-update (Ctrl::refresh_next), whatever the other problems do.  Lets a test make one lambda rebuild on its own. */
int mlease_internal_request_refresh(mlease_session* s, int32_t b);

/* The CSR Gram kernel of the batches allocated from now on -- 0 = picked from the data, CSR_GRAM_WGMMA (1), CSR_GRAM_SPARSE (2).
 * Must be called before the ADMM batch exists; the one-problem scratch batch (objective, timing) is rebuilt with the new setting on
 * its next use.  The query returns the kind of the ADMM batch and of the scratch batch (0: no such batch, or no CSR Gram). */
int mlease_internal_set_csr_gram(mlease_session* s, int32_t kind);
int mlease_internal_csr_gram(mlease_session* s, int32_t* batch_kind, int32_t* scratch_kind);

/* On the current device, n 16x8 tiles D = A B^T (A: n x 16 x K, B: n x 8 x K, row-major, K a multiple of 4) accumulated as
 * dgemm_kernel accumulates, once through DMMA m8n8k4 (D8) and once through m16n8k4 (D16). */
int mlease_internal_dmma_shapes(const double* A, const double* B, int32_t n, int32_t K, double* D8, double* D16);

/* The consensus step (K4, k4_consensus.cu) of the begun ADMM batch on an injected state.
 *   stages: CS_RESET (d_rho = rho of iteration 1, then admm_reset, as begin() runs them), CS_INIT (admm_init on the injected z, as
 *   begin_initialized() runs it; not on an L1 session), CS_PACK (admm_pack into the session's exchange buffer), CS_CONSENSUS (the
 *   session's own consensus_enqueue on that buffer, one stream synchronisation, consensus_finish, with s->iter = args[0] >= 1 and
 *   s->liblinear_eps = (float)args[1]).  They run in that order.  stages = 0 injects and runs nothing: it reads the state back (or
 *   only info when vec is NULL).
 *   vec: nprob x 5 x ldx doubles (beta, m, q, g_t, x_d), fvec: nprob x 3 x ldx floats (u_f, uplusx_f, x_f), z: L x ldx, exch: L Dt + 1
 *   (the last slot is the failed-fit count), diff: L, ctrl: nprob x 3 ints (Ctrl::hess_valid, skip_eval, k1_chunks); all in and out,
 *   whole vectors, padding included, copied as bytes.  ctrl_raw (out, may be NULL): 2 x nprob x sizeof(Ctrl) bytes, every problem's
 *   Ctrl just before the first stage and after the last one, with the three fields of ctrl zeroed in both.  wz (L x ldx), l1thr (L;
 *   NULL on an L2 session) and rho (L): the z-weights, L1 thresholds and d_rho the kernels read, as the last stage left d_rho.
 *   res (3 doubles, CS_CONSENSUS): maxdiff, the session's mindiff, stop.
 *   info (12 ints): nprob, Dt, ldx, L, P, local partitions, CSR, fused K1 (gpart_f present), matrix-free, regularizer, k1_grid,
 *   sizeof(Ctrl).
 * Every kernel of K4 indexes by Dt, ldx, L and the problem count alone; k1_chunks is still refused beyond the partial rows the batch
 * allocated.  Refused before any launch: no begun batch, a stage mask outside [0, 15], CS_INIT on an L1 session, CS_CONSENSUS
 * without args or with args[0] < 1, a null array.  With stages set, consumes the batch's x-update state; s->iter, liblinear_eps,
 * mindiff and last_maxdiff are restored. */
int mlease_internal_consensus(mlease_session* s, int32_t stages, const double* args, double* vec, float* fvec, double* z, double* exch,
                              double* diff, int32_t* ctrl, uint8_t* ctrl_raw, double* wz, double* l1thr, double* rho, double* res,
                              int32_t* info);

/* Partition pid of the session as its upload left it, after the deferred CSR checks and lists are built (their refusal is returned).
 * Neither hook touches the ADMM batch.
 * mlease_internal_partition_info: out (PARTITION_INFO_LEN doubles, every value exact): [0] rows n, [1] stored entries (0 for a dense
 * partition), [2] CSR, [3] ldx (floats per dense row), [4] wmax (largest weight), [5] vmax (largest |stored value|), [6] rowl1 (largest
 * row sum of |stored value|), [7] gram_pairs (products of one sparse Gram build; 0 where no block-major list was built), [8] csr_unique,
 * [9] block-major Gram list built, [10] column index of the sparse Gram built, [11] fused-K1 segment lists built, [12] sg_S (their
 * segments, 0 without them).
 * mlease_internal_partition_data: the session's device copies, each to the host if not NULL: y (n int8, +1 / -1), w and o (n floats),
 * X_or_vals (a dense partition's X, n x ldx floats with the intercept column and the padding; a CSR partition's nnz stored values, as
 * binary.feature left them). */
#define PARTITION_INFO_LEN 13
int mlease_internal_partition_info(mlease_session* s, int32_t pid, double* out);
int mlease_internal_partition_data(mlease_session* s, int32_t pid, int8_t* y, float* w, float* o, float* X_or_vals);

#ifdef __cplusplus
}
#endif

#endif /* MLEASE_INTERNAL_H */
