/*
 * mlease_b200.h -- C ABI of the H100-native ADMM logistic-regression hot path.
 *
 * Drop-in boundary for ONE path of linkedin/ml-ease: the body of
 * RegressionAdmmTrain.run() (jobs/RegressionAdmmTrain.java:278-501), the reducer it drives
 * (AdmmReducer.reduce, :642-718 -> LibLinear.train, llf/LibLinear.java:200-208), the scoring
 * of RegressionTest/RegressionTestLoglik and the per-key fits of RegressionNaiveTrain.
 * The reference has no FFI seam (it is 100% Java); these are the entry points a JNI shim
 * (INTEGRATION.md) binds.  Paths cited below are relative to
 * /root/reference/src/main/java/com/linkedin/mlease/ unless they start with bw/ (= de/bwaldvogel/liblinear/).
 *
 * Conventions: every function returns 0 on success, non-zero on error (message via
 * mlease_last_error(), thread-local).  Plain pointers and sizes only.  "host-or-device"
 * pointers may be either (UVA); everything else says which.  Feature ids are the GLOBAL
 * dictionary 0..num_features-1; the intercept "(INTERCEPT)" is index num_features (last), the
 * bias column the reference appends to every row (regression/liblinearfunc/LibLinearDataset.java:592-614).
 * One host thread drives a session (the reference's driver and reducers are single threaded).
 * There is NO CPU fallback: without a CUDA device every compute entry point fails.
 */
#ifndef MLEASE_B200_H
#define MLEASE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct mlease_session mlease_session;
typedef struct mlease_comm mlease_comm;     /* one NCCL communicator rank (multi-GPU jobs) */
typedef struct mlease_world mlease_world;   /* N sessions on N GPUs of this process */

#define MLEASE_OK 0
#define MLEASE_ERR_INVALID 1   /* bad argument / config (reference: IOException in the job) */
#define MLEASE_ERR_CUDA 2      /* CUDA failure (reference: IOException("Model fitting error!"), jobs/RegressionAdmmTrain.java:713-716) */
#define MLEASE_ERR_NUMERIC 3   /* a fit did not converge / Hessian not SPD (same mapping) */
#define MLEASE_ERR_STATE 4     /* call order (e.g. partitions missing: RuntimeException("Some models failed!"), utils/LinearModelUtils.java:80-83) */

const char* mlease_last_error(void);
int mlease_abi_version(void);

/* ---------------------------------------------------------------------------------------
 * Session = one RegressionAdmmTrain job on one GPU (partitions are sharded over sessions; the
 * all-reduce between them is the library's, see "Multi-GPU" below, or a caller-supplied callback).
 * Config keys mirrored (jobs/RegressionAdmmTrain.java:78-122,138-185):
 *   num.blocks, lambda (list, Float.parseFloat), rho (list or NULL -> 1 if lambda<=100 else 10),
 *   regularizer (2 = L2 z-update :377-404, 1 = L1 thresholded z-update :406-451, anything else -> "Only L1 and L2
 *   regularization supported!" :144-147), penalize.intercept, epsilon, rho.adapt.coefficient,
 *   aggressive.liblinear.epsilon.decay (pure control: only moves the stop rule :493-496).
 * ------------------------------------------------------------------------------------- */
typedef struct {
  int32_t device;              /* CUDA ordinal */
  int32_t num_blocks;          /* P, partitions over ALL processes */
  int32_t num_features;        /* global dictionary size, intercept excluded */
  int32_t num_lambdas;         /* L */
  const float* lambdas;        /* [L] host */
  const float* rhos;           /* [L] host or NULL */
  const float* lambda_map;     /* [num_features] host or NULL; >0 entries override lambda per feature (:382-386) */
  int32_t regularizer;         /* 1 or 2 */
  int32_t penalize_intercept;  /* default 0 */
  int32_t aggressive_decay;    /* default 0 */
  int32_t binary_feature;      /* binary.feature: ignore values, use 1 (regression/liblinearfunc/LibLinearBinaryDataset.java) */
  double epsilon;              /* outer stop (:473); < 0 -> default 1e-4, 0 = never stop early */
  float rho_adapt_coefficient; /* default 0 (:323-327) */
  /* solver knobs (no reference equivalent: the inner solve is exact Newton, not TRON) */
  double newton_xtol;          /* stop when |dir|_inf <= xtol*max(|beta|_inf,1e-2); 0 -> 2e-7 (float32 lattice of the data path) */
  int32_t max_newton;          /* max accepted Newton steps per x-update; 0 -> 50 */
  int32_t hessian_policy;      /* Newton direction of the x-update.  0: Gram + Cholesky, adaptive chord (refactorise when the steps
                                  contract poorly, L-BFGS pairs on the stale factor); 1: Gram + Cholesky at every step; 2: matrix-free
                                  truncated Newton, preconditioned CG on Hessian-vector passes over the rows (CSR partitions with sorted
                                  unique rows only, MLEASE_ERR_INVALID otherwise): no D'^2 state, O(D') per problem.  Automatic rule:
                                  with 0 or 1, a CSR session whose Gram path would allocate more than the free device memory (~26 D'^2
                                  bytes per (partition, lambda)) is built matrix-free instead of failing.  A matrix-free session never
                                  forms H: with policy 2 (at any width) mlease_objective's H, mlease_posterior_variance(full = 1) and
                                  the Gram / Cholesky timings of mlease_time_kernel return MLEASE_ERR_INVALID, and the CSR upload
                                  builds no block-major Gram list. */
  void* stream;                /* cudaStream_t to run on (NULL = legacy default stream) */
} mlease_admm_config;

int mlease_session_create(const mlease_admm_config* cfg, mlease_session** out);
int mlease_session_destroy(mlease_session* s);

/* Replaces the per-iteration re-ingest LibLinearDataset.addInstanceAvro/finish
 * (regression/liblinearfunc/LibLinearDataset.java:413-484,586-658; jobs/RegressionAdmmTrain.java:677-690):
 * records are uploaded ONCE and stay resident in HBM.  Rows are RegressionPrepareOutput records
 * (src/main/avro/RegressionPrepareOutput.avsc): response in {1,0,-1} (0 -> -1), weight >= 0, float32
 * values.  Pointers are host-or-device; the library copies.
 * dense: X row-major [nrows x num_features], leading dimension ldx (floats).
 * csr:   rowptr [nrows+1] (int64), colidx (global ids, any order, duplicates add), vals.  The call returns when the arrays
 *        have been copied (the caller's buffers are free again); the checks on colidx and the derived lists of partition p
 *        are built while partition p+1 is being copied, so "partition <id>: feature index out of range" is reported by the
 *        NEXT call on the session (add_partition / begin / fit / objective).  response / weight errors are immediate. */
int mlease_add_partition_dense(mlease_session* s, int32_t partition_id, int64_t nrows, const float* X, int64_t ldx,
                               const int32_t* response, const float* weight, const float* offset);
int mlease_add_partition_csr(mlease_session* s, int32_t partition_id, int64_t nrows, const int64_t* rowptr,
                             const int32_t* colidx, const float* vals, const int32_t* response, const float* weight,
                             const float* offset);

/* ADMM loop, one iteration = jobs/RegressionAdmmTrain.java:281-497 :
 *   begin      : z = {}, u = {}  (:155-185, :312), schedule reset (:278-279)
 *   local_step : x-update of every local (partition, lambda) (AdmmReducer.reduce :642-718) and
 *                exchange[l][k] = sum over LOCAL partitions of float(x_p)[k] + u_p[k]   (device, double,
 *                [L][num_features+1]) -- the only data that crosses GPUs
 *   consensus  : given the exchange buffer summed over ALL processes (one all-reduce), the z-update
 *                (:362-404), convergence (:456-472), schedule + stop rule (:338-346,:493-496) and next u
 *                (computeU :736-765).  *stop is 1 when the reference would break.
 * mlease_admm_run drives these for a single-process job (allreduce == NULL) or with a caller-supplied
 * all-reduce (sum, double, in place on `buf` which is DEVICE memory, ordered on `stream`). */
typedef int (*mlease_allreduce_fn)(void* ctx, double* buf, size_t count, void* stream);
int mlease_admm_begin(mlease_session* s);
/* initialize.boost.rate > 0 (jobs/RegressionAdmmTrain.java:236-266, 313-316): the run starts from z0 ([num_lambdas][num_features+1]
 * doubles on the host, intercept last: the mean of per-partition RegressionNaiveTrain fits, which the caller obtains with
 * mlease_fit_partition) instead of z = {}, u is empty, and the reducers of ITERATION 1 use rho * boost_rate: the driver builds a
 * new JobConf every iteration (:286-291), so rho.adapt.rate is back at the reducers' default 1.0f (:621) from iteration 2 on
 * (or follows rho_adapt_coefficient, :323-327).  The factors built with the boosted rho are invalidated at iteration 2. */
int mlease_admm_begin_initialized(mlease_session* s, const double* z0, float boost_rate);
int mlease_admm_local_step(mlease_session* s, double* exchange_dev);
int mlease_admm_consensus(mlease_session* s, const double* exchange_sum_dev, double* maxdiff, int32_t* stop);
int mlease_admm_run(mlease_session* s, int32_t num_iters, mlease_allreduce_fn allreduce, void* ctx, int32_t* iters_done);
/* One iteration with the exchange inside the library: local_step, all-reduce over the attached communicator (none for a
 * single-process job holding all num_blocks partitions), consensus.  Lets a host job write the reference's iter-<i>/ files
 * between iterations.  A failed fit on any rank returns MLEASE_ERR_NUMERIC on every rank ("Model fitting error!", :713-716). */
int mlease_admm_iterate(mlease_session* s, double* maxdiff, int32_t* stop);

/* ---------------------------------------------------------------------------------------
 * Multi-GPU: the path shards exactly where ADMM does -- partitions are independent in the x-update and meet in ONE
 * all-reduce (sum, fp64, [L][num_features+1] (+1 failure counter)) per iteration, the mean the reference's driver takes over
 * the reducer outputs (:362-364, cons/MeanLinearModelConsumer.java:44-70).  NCCL is loaded at run time (libnccl.so.2).
 *  (a) one process per GPU: rank 0 calls mlease_comm_unique_id and ships the 128 bytes to the other ranks by any means;
 *      every rank creates its communicator, attaches it to its session (which holds the partitions p with p % nranks == rank)
 *      and calls mlease_admm_run(s, iters, NULL, NULL, &done): the whole RegressionAdmmTrain loop runs in C.
 *  (b) one process, several GPUs (a single-JVM driver, the C++ job layer): mlease_world_* below -- same calls as a session,
 *      partitions routed to GPU  partition_id % ndev, one worker thread per GPU, ncclCommInitAll inside.
 * ------------------------------------------------------------------------------------- */
#define MLEASE_COMM_ID_BYTES 128
int mlease_comm_unique_id(void* id128);
int mlease_comm_create(const void* id128, int32_t rank, int32_t nranks, int32_t device, mlease_comm** out);
int mlease_comm_destroy(mlease_comm* c);
int mlease_comm_info(const mlease_comm* c, int32_t* rank, int32_t* nranks, int32_t* nccl_version);
int mlease_session_set_comm(mlease_session* s, mlease_comm* comm);   /* not owned; NULL detaches */

int mlease_world_create(const mlease_admm_config* cfg /* .device/.stream ignored */, const int32_t* devices /* NULL = 0..ndev-1 */,
                        int32_t ndev, mlease_world** out);
int mlease_world_destroy(mlease_world* w);
int mlease_world_num_devices(const mlease_world* w);
int mlease_world_add_partition_dense(mlease_world* w, int32_t partition_id, int64_t nrows, const float* X, int64_t ldx,
                                     const int32_t* response, const float* weight, const float* offset);
int mlease_world_add_partition_csr(mlease_world* w, int32_t partition_id, int64_t nrows, const int64_t* rowptr, const int32_t* colidx,
                                   const float* vals, const int32_t* response, const float* weight, const float* offset);
int mlease_world_begin(mlease_world* w);
int mlease_world_begin_initialized(mlease_world* w, const double* z0, float boost_rate);
int mlease_world_iterate(mlease_world* w, double* maxdiff, int32_t* stop);
int mlease_world_run(mlease_world* w, int32_t num_iters, int32_t* iters_done);
int mlease_world_get_z(mlease_world* w, int32_t lambda_idx, double* out);
int mlease_world_get_final_model(mlease_world* w, int32_t lambda_idx, float* out);
int mlease_world_get_x(mlease_world* w, int32_t partition_id, int32_t lambda_idx, double* out);
int mlease_world_get_u(mlease_world* w, int32_t partition_id, int32_t lambda_idx, float* out);
int mlease_world_get_uplusx(mlease_world* w, int32_t partition_id, int32_t lambda_idx, float* out);
int mlease_world_fit_partition(mlease_world* w, int32_t partition_id, double* x, const double* m, const double* q, int32_t* newton_steps);

/* State readback (host buffers).  z: driver-side double z (:365-404); final model = float(z)
 * (models/LinearModel.java:697-720 toAvro).  After consensus of iteration i: x = the double x_p of iteration i
 * (float(x) is iter-<i>/model), uplusx = float(u+x) of iteration i (:706-711), u = float(uplusx - z), i.e. the
 * iter-<i+1>/u file computeU (:736-765) writes.  Length num_features+1, intercept last. */
int mlease_get_z(mlease_session* s, int32_t lambda_idx, double* out);
int mlease_get_final_model(mlease_session* s, int32_t lambda_idx, float* out);
int mlease_get_x(mlease_session* s, int32_t partition_id, int32_t lambda_idx, double* out);
int mlease_get_u(mlease_session* s, int32_t partition_id, int32_t lambda_idx, float* out);
int mlease_get_uplusx(mlease_session* s, int32_t partition_id, int32_t lambda_idx, float* out);

typedef struct {
  int64_t k1_passes;        /* fused score/reweight/gradient passes over X (all problems) */
  int64_t gram_builds;      /* Gram + Cholesky refreshes */
  int64_t newton_steps;     /* accepted Newton steps */
  int64_t rejected_steps;   /* line-search rejections */
  int64_t kernel_launches;  /* kernels launched by this session */
  int32_t not_converged;    /* x-updates that hit max_newton */
  int32_t last_iter_slots;  /* evaluation slots used by the last local_step */
  double last_maxdiff;
  float liblinear_epsilon;  /* schedule variable (:279,338-346), control only */
  int32_t k1_fused;         /* 1: the fused multi-lambda CSR K1 (csrc/k1_csr_fused.cu) serves this session's ADMM problems */
  double k1_shared_bytes;   /* CSR sessions: K1 bytes when the lambdas of a partition count as ONE read of its rows
                               (8*nnz + 9*n per partition pass + 8*n per lambda served); k1_bytes of mlease_profile counts every
                               (partition, lambda) pass separately, as SURVEY 8d defines the unit */
} mlease_stats;
int mlease_get_stats(mlease_session* s, mlease_stats* out);
int mlease_world_get_stats(mlease_world* w, mlease_stats* out);   /* counters summed over the devices */
/* Per-kernel device timing for roofline reporting (CUDA events on the session stream around every launch of
 * the Newton slot; categories: 0 = K1 fused pass, 1 = small kernels (reduce/decide, solve, poll), 2 = Hessian: Gram builds
 * (wgmma), or in a matrix-free session the diagonal pass + CG set-up and every Hv pass with its CG update, 3 = Cholesky).
 * gram_flops counts the Gram builds actually run (none in a matrix-free session, whose mlease_stats.gram_builds stays 0).  enable: 1 on, 0 off, 2 on + reset accumulators, -1 read only.  Outputs (any may be NULL) are the
 * accumulators BEFORE this call's reset: ms4[4], count4[4], and the algorithmic work done by the session so far:
 * k1_bytes (SURVEY 8d: dense n*(4*ldx+9) per pass), k1_emit_bytes (bf16 operand writes), gram_flops (n*D'*(D'+1)). */
int mlease_profile(mlease_session* s, int32_t enable, double* ms4, int64_t* count4, double* k1_bytes, double* k1_emit_bytes,
                   double* gram_flops);

/* ---------------------------------------------------------------------------------------
 * Function-level entry points (parity tests against the oracle's fun/grad/hessian):
 * LogisticRegressionL2.fun/grad/hessian (regression/liblinearfunc/LogisticRegressionL2.java:156-297)
 * evaluated on a resident partition at host vector w, prior mean m, prior precision q (=1/priorVar),
 * all of length num_features+1.  Any output may be NULL.  H is [Dt x Dt] row-major (full, symmetric).
 * tensor != 0 builds H with the wgmma Gram kernel (bf16 operands for dense partitions, e4m3 operands assembled from the rows
 * for CSR partitions with sorted unique rows), 0 with the fp32 SIMT debug kernel (dense bf16 operand only).
 * tensor == 2 returns in H the INVERSE the Newton direction is computed with (wgmma Gram + diag(q) -> fp64 blocked
 * Cholesky -> explicit inverse), so that tests can check H^-1 * H = I for every factorisation path.
 * ------------------------------------------------------------------------------------- */
int mlease_objective(mlease_session* s, int32_t partition_id, const double* w, const double* m, const double* q,
                     double* f, double* g, double* H, int32_t tensor);
/* LibLinear.train(dataset, init, priorMean, priorVar...) (regression/liblinearfunc/LibLinear.java:200-208) for one
 * resident partition: exact Newton solve of the same objective.  x: in = init, out = minimiser. */
int mlease_fit_partition(mlease_session* s, int32_t partition_id, double* x, const double* m, const double* q,
                         int32_t* newton_steps);
/* LogisticRegressionL2.Hv (regression/liblinearfunc/LogisticRegressionL2.java:231-248) on a resident CSR partition with sorted
 * unique rows: out = X^T D(w) X v + q .* v, D(w) = diag(weight_i p_i (1 - p_i)) at w, through the Hv mode of the CSR K1 kernels
 * (the pass matrix-free sessions run for every CG step).  All vectors have num_features+1 entries (host memory). */
int mlease_hessian_vector(mlease_session* s, int32_t partition_id, const double* w, const double* q, const double* v, double* out);

/* Posterior variance of the model w of one resident partition under prior precision q (= 1/priorVar), the
 * computePosteriorVar / computeFullPostVar tail of LibLinear.train (regression/liblinearfunc/LibLinear.java:315-334) that
 * ItemModelTrain reports as "posteriorVar" (jobs/ItemModelTrain.java:257-266):
 *   full = 0: var[k] = 1 / (q[k] + sum_i weight_i p_i (1-p_i) x_ik^2)         (hessianDiagonal, LogisticRegressionL2.java:304-327)
 *   full = 1: var = diag(H^-1), H = LogisticRegressionL2.hessian (:258-297) accumulated in fp64 (NOT the bf16 tensor-core
 *             Gram, which only preconditions), Cholesky + explicit inverse in fp64; cov (may be NULL) receives H^-1,
 *             [Dt x Dt] row-major.  Needs rows with strictly increasing column ids, as the reference's hessian() does (:277).
 * var has num_features+1 entries, intercept last; a feature absent from the partition gets its prior variance 1/q[k]
 * (the reference lists only the features present in the dataset). */
int mlease_posterior_variance(mlease_session* s, int32_t partition_id, const double* w, const double* q, int32_t full,
                              double* var, double* cov);

/* Posterior of the ADMM model: the Laplace posterior, at z, of the objective the z-update minimises
 * (jobs/RegressionAdmmTrain.java:377-404) over ALL partitions of the job, for lambda index lambda_index:
 *   H = sum over partitions, sum_i weight_i p_i (1-p_i) x~_i x~_i^T + diag(q),   x~_i = row i with the intercept entry 1,
 *   p_i at z with the row's offset, q[k] = lambda (lambda_map[k] where that is > 0), q[intercept] = lambda with
 *   penalize_intercept, else 0.
 * z (num_features+1 doubles, intercept last, host or device) or NULL for the session's consensus z of that lambda (after
 * mlease_admm_begin).  Every partition's H is exact fp64 from the fp32 rows (CSR: built column by column from the rows' suffixes,
 * no atomics; dense: tiled X^T D X), the partitions are summed in partition-id order whatever order they were uploaded in, and with
 * a communicator attached the ranks' sums go through one fp64 all-reduce: the call is then collective on every rank, and a
 * refusal on one rank is returned on all of them.  The result is bitwise repeatable.
 *   full = 0: var[k] = 1 / (q[k] + sum_i weight_i p_i (1-p_i) x~_ik^2)  -- any width, matrix-free sessions included
 *   full = 1: var = diag(H^-1), cov (may be NULL) = H^-1, [D+1][D+1] row-major host memory; Cholesky + explicit inverse in fp64 on
 *             buffers of the call's own (4 x 8 x ldh^2 bytes, ldh = round_up(D+1, 32), checked against the free device memory
 *             before anything is allocated).
 * The ADMM batch, its factors and its state are not touched: the session iterates on exactly as it would have.
 * MLEASE_ERR_INVALID: regularizer 1 (the L1 penalty has no Hessian), lambda_index out of range, CSR rows that are not strictly
 * increasing, a full posterior that does not fit the device; MLEASE_ERR_NUMERIC: H not positive definite. */
int mlease_admm_posterior(mlease_session* s, int32_t lambda_index, const double* z, int32_t full, double* var, double* cov);
/* the same over the devices of a world (collective over its NCCL communicator); var / cov from device 0 */
int mlease_world_admm_posterior(mlease_world* w, int32_t lambda_index, const double* z, int32_t full, double* var, double* cov);

/* ---------------------------------------------------------------------------------------
 * RegressionNaiveTrain (jobs/RegressionNaiveTrain.java:302-415): num_keys x num_lambdas independent fits ("lambda#key"
 * reducers, :228-241).  Key k owns rows [key_rowstart[k], key_rowstart[k+1]) of ONE matrix, uploaded once for all lambdas:
 *   CSR   (rowptr != NULL): rowptr [nrows+1] int64, colidx (global ids), vals -- the reference's per-key sparse datasets
 *         (:360-398).  A feature that no row of a key lists is not in that key's dataset, hence not in its model
 *         (regression/liblinearfunc/LibLinear.java:343-350): its output coefficient is 0, whatever prior.mean is.
 *         binary_feature: every listed feature counts as 1 (LibLinearBinaryDataset).
 *         Each key is solved in its own column space when that is narrower: with Dk the distinct columns its rows list, a key with
 *         round_up(Dk + 1, 32) < round_up(num_features + 1, 32) is fitted over those Dk columns and the intercept only, and its
 *         model is scattered back to the global columns.  Device memory then scales with each key's own width, not with
 *         num_features (a 200 000-feature dictionary whose keys list a few hundred features each fits easily); the dense host
 *         output, num_lambdas * num_keys * (num_features+1) doubles, is what remains proportional to the dictionary:
 *         mlease_naive_train_sparse below returns each key's listed columns only.  Which width a key runs at depends on its own
 *         rows alone.
 *   dense (rowptr == NULL): vals = X row-major [nrows x num_features], leading dimension ldx; every feature is present.
 * priorVar = 1/lambda, 1/lambda_map[k] for listed features (lambda_map [num_features] or NULL, entries > 0), intercept variance
 * 100000 unless penalize_intercept (:333-343), prior.mean, has.intercept, data.size.threshold (skipped keys -> skipped[k]=1,
 * model 0, :379-382).  out_model [num_lambdas][num_keys][num_features+1] double, intercept last.  All pointers host-or-device
 * except out_model / skipped (host).  A fit that does not converge -> MLEASE_ERR_NUMERIC ("Model fitting error!", :400-412).
 *
 * Inputs larger than the device: when the rows, labels and key boundaries do not fit next to the first chunk's solver state, the
 * keyed calls (mlease_naive_train, mlease_naive_train_dense, mlease_item_model_train, mlease_score_keyed[_var]) stream contiguous key
 * ranges through the device, the next range's rows copied while the current one is solved.  A key's fit then matches the resident
 * call's within the run-to-run spread of the CSR kernels (their gradient sums use float atomics); scores are bitwise the same.
 * In that mode "rows sorted and unique" (which selects the CSR kernels) is decided per key range, not per call, so one key with
 * unsorted rows changes the kernels of its range only.
 * Several devices: these four calls may run at the same time from several host threads, one device per thread (keys are
 * independent; a caller shards them into contiguous ranges, each with its own key_rowstart and rowptr from 0).
 * ------------------------------------------------------------------------------------- */
int mlease_naive_train(int32_t device, void* stream, int32_t num_keys, int32_t num_features, const int64_t* key_rowstart,
                       const int64_t* rowptr, const int32_t* colidx, const float* vals, int64_t ldx, const int32_t* response,
                       const float* weight, const float* offset, int32_t num_lambdas, const float* lambdas, const float* lambda_map,
                       float prior_mean, int32_t penalize_intercept, int32_t has_intercept, int32_t data_size_threshold,
                       int32_t binary_feature, double* out_model, int32_t* skipped);
/* single-lambda dense form of the above (kept from ABI version 1) */
int mlease_naive_train_dense(int32_t device, void* stream, int32_t num_keys, int32_t num_features,
                             const int64_t* key_rowstart, const float* X, int64_t ldx, const int32_t* response,
                             const float* weight, const float* offset, float lambda, const float* lambda_map,
                             float prior_mean, int32_t penalize_intercept, int32_t has_intercept,
                             int32_t data_size_threshold, double* out_model, int32_t* skipped);

/* ItemModelTrain (jobs/ItemModelTrain.java:226-276): num_keys x IL x DL independent fits on the CSR input of mlease_naive_train
 * (rowptr, colidx, vals, key_rowstart, response, weight, offset; binary_feature), always with an intercept and no size threshold.
 * Fit (a, b) of key k: priorVar = 1/lambda_map[j] for a listed feature (lambda_map [num_features] or NULL, entries > 0, 0 = none),
 * 1/intercept_lambdas[a] for the intercept, 1/default_lambdas[b] otherwise (every lambda > 0, checked, naming its list); prior mean
 * intercept_prior_mean[k] for the intercept, 0 otherwise; start 0.  out_model [IL][DL][num_keys][num_features+1] double, intercept
 * last, features absent from the key's rows 0.  compute_var: out_var of the same shape receives the diagonal posterior variance
 * 1 / (1/priorVar[j] + sum_i weight_i p_i (1-p_i) x_ij^2) at the fit (llf/LibLinear.java:328-333), 1/q = priorVar[j] for an absent
 * feature.  Each key is solved in its own column space when that is narrower, as mlease_naive_train's CSR keys are: device memory
 * scales with each key's own width, and the dense host outputs (IL * DL * num_keys * (num_features+1) doubles, twice with
 * compute_var) are what remains proportional to the dictionary (mlease_item_model_train_sparse below avoids them).  All inputs
 * host-or-device; intercept_prior_mean, out_model and out_var host.  With IL = DL = 1, intercept_lambdas[0] =
 * default_lambdas[0] and zero means the models are bitwise those of mlease_naive_train(prior_mean 0, penalize_intercept 1). */
int mlease_item_model_train(int32_t device, void* stream, int32_t num_keys, int32_t num_features, const int64_t* key_rowstart,
                            const int64_t* rowptr, const int32_t* colidx, const float* vals, const int32_t* response, const float* weight,
                            const float* offset, const double* intercept_prior_mean, int32_t num_intercept_lambdas,
                            const float* intercept_lambdas, int32_t num_default_lambdas, const float* default_lambdas,
                            const float* lambda_map, int32_t binary_feature, int32_t compute_var, double* out_model, double* out_var);

/* Sparse outputs of the two keyed CSR fits above: the same fits (same plan, kernels and priors), each key's model returned as the
 * columns its rows list instead of a num_features + 1 row.  Inputs, checks, errors, streaming, budgets and several-device use are
 * those of mlease_naive_train (CSR only: rowptr and colidx required) and mlease_item_model_train.
 *   lists:    key k's list is entries [out_key_ptr[k], out_key_ptr[k+1]) of out_col (out_key_ptr [num_keys+1], out_key_ptr[0] = 0):
 *             the distinct columns its rows list, ascending, then the intercept as column num_features (always for ItemModelTrain,
 *             for NaiveTrain when has_intercept), so strictly ascending as mlease_score_keyed requires.  A key that is not fitted
 *             (skipped by data_size_threshold, also flagged in skipped; or without rows) has an empty list.  A key's list is the
 *             same for every prior.
 *   values:   prior p's value of entry e is out_model[p * capacity + e] (out_var likewise with compute_var), priors in the dense
 *             calls' order (lambda; a * num_default_lambdas + b).  Each value is the one the dense call computes at that column
 *             (the same fit; for a one-row key in its own column space, bit for bit; otherwise within the run-to-run spread the
 *             dense call has from call to call); the variance is 1 / hessianDiagonal in fp64.  Unlisted features are not reported: their
 *             coefficient is 0 and their variance 1/q.
 *   capacity: the entries out_col holds (and each prior's stride in out_model / out_var).  Checked before any row is read against
 *             the bound sum over fitted keys of min(stored entries of the key, num_features) + 1 for the intercept (read from
 *             rowptr at the key boundaries); a smaller capacity is MLEASE_ERR_INVALID, the message giving the bound.  The lists hold
 *             out_key_ptr[num_keys] <= bound entries; nothing past them is written.
 * Host and device memory are proportional to the data (the lists, one chunk of keys at a time on the device), never to
 * num_keys * num_features.  out_key_ptr, out_col, out_model, out_var and skipped are host memory. */
int mlease_naive_train_sparse(int32_t device, void* stream, int32_t num_keys, int32_t num_features, const int64_t* key_rowstart,
                              const int64_t* rowptr, const int32_t* colidx, const float* vals, const int32_t* response,
                              const float* weight, const float* offset, int32_t num_lambdas, const float* lambdas,
                              const float* lambda_map, float prior_mean, int32_t penalize_intercept, int32_t has_intercept,
                              int32_t data_size_threshold, int32_t binary_feature,
                              int64_t capacity, int64_t* out_key_ptr, int32_t* out_col, double* out_model, int32_t* skipped);
int mlease_item_model_train_sparse(int32_t device, void* stream, int32_t num_keys, int32_t num_features, const int64_t* key_rowstart,
                                   const int64_t* rowptr, const int32_t* colidx, const float* vals, const int32_t* response,
                                   const float* weight, const float* offset, const double* intercept_prior_mean,
                                   int32_t num_intercept_lambdas, const float* intercept_lambdas, int32_t num_default_lambdas,
                                   const float* default_lambdas, const float* lambda_map, int32_t binary_feature, int32_t compute_var,
                                   int64_t capacity, int64_t* out_key_ptr, int32_t* out_col, double* out_model, double* out_var);

/* mlease_item_model_train_sparse with the full posterior of every fit (computeFullPostVar, llf/LibLinear.java:315-326): the same
 * inputs, plan, fits, lists and several-device use, the models bit for bit those of the sparse call for one-row keys in their own
 * column spaces (within its run-to-run spread otherwise).  At each fit, H = diag(q) + sum_i w_i p_i (1-p_i) x_i x_i^T is assembled
 * in fp64 on the device over the key's own columns (deterministically: Sigma depends on the key's rows and fit alone, not on the
 * chunking, the streaming or the other keys) and inverted by Cholesky (K3's fp64 factorisation and explicit inverse), Sigma = H^-1.
 *   out_var:  required; prior p's entry e is diag(Sigma) at the list's column, out_var[p * capacity + e], in place of the sparse call's
 *             1 / hessianDiagonal.  An unlisted feature is uncorrelated with the listed ones: its variance is 1/q.
 *   out_cov:  NULL (then cov_capacity and out_cov_ptr are ignored), or key k's block is entries [out_cov_ptr[k], out_cov_ptr[k+1])
 *             (out_cov_ptr [num_keys+1], out_cov_ptr[0] = 0): for a list of n_k entries, n_k (n_k + 1) / 2 values, the lower
 *             triangle of Sigma over the list's order, row-major -- entry (a, b), a >= b, at out_cov_ptr[k] + a (a+1) / 2 + b.  Prior
 *             p's values are at out_cov[p * cov_capacity + e].  Keys that are not fitted have empty blocks.  cov_capacity is checked
 *             chunk by chunk, once the chunk's list lengths are fixed and before it writes anything: a shortfall is
 *             MLEASE_ERR_INVALID, the message giving the entries needed up to that chunk's last key.
 * Refused with MLEASE_ERR_INVALID: rows whose columns are not strictly increasing (llf/LogisticRegressionL2.java:277), and a fitted
 * key whose system (its own column space, or num_features + 1 at the global width) is wider than 2048 columns -- the widest whose
 * explicit inverse K3 forms -- before that key's chunk is solved, the message naming the key and its width.  A Hessian that is not
 * positive definite is MLEASE_ERR_NUMERIC.  out_key_ptr, out_col, out_model, out_var, out_cov_ptr and out_cov are host memory. */
int mlease_item_model_train_cov(int32_t device, void* stream, int32_t num_keys, int32_t num_features, const int64_t* key_rowstart,
                                const int64_t* rowptr, const int32_t* colidx, const float* vals, const int32_t* response,
                                const float* weight, const float* offset, const double* intercept_prior_mean,
                                int32_t num_intercept_lambdas, const float* intercept_lambdas, int32_t num_default_lambdas,
                                const float* default_lambdas, const float* lambda_map, int32_t binary_feature, int64_t capacity,
                                int64_t* out_key_ptr, int32_t* out_col, double* out_model, double* out_var, int64_t cov_capacity,
                                int64_t* out_cov_ptr, double* out_cov);

/* ---------------------------------------------------------------------------------------
 * RegressionTest / RegressionTestLoglik.
 * score: pred = float(offset + interceptTerm + sum beta_k x_k), interceptTerm = -log(n-1+n*exp(-b)),
 *        n = num.click.replicates (models/LinearModel.java:241-257,491-554; jobs/RegressionTest.java:163).
 *        dense (colidx==NULL: X = vals, ld = ldx) or CSR.  All data pointers host-or-device; pred host-or-device.
 * test_loglik: mapper float cast, combiner partial sums cast to float per `combiner_block` records
 *        (<=0: no combiner), reducer float(sum/count) (jobs/RegressionTestLoglik.java:124-200).
 * ------------------------------------------------------------------------------------- */
int mlease_score(int32_t device, void* stream, int32_t num_features, int64_t nrows, const int64_t* rowptr,
                 const int32_t* colidx, const float* vals, int64_t ldx, const float* offset, const double* model,
                 int32_t num_click_replicates, int32_t binary_feature, float* pred);
/* score_var: score's pred, bit for bit, and each record's predictive variance under the posterior of the model,
 *        pred_var = float(g^T Sigma g) accumulated in fp64 in a fixed order: g holds the record's entries (1 with binary_feature)
 *        and, at the intercept, d pred / d b = n e^-b / (n - 1 + n e^-b) (1 for n = 1): the delta method through interceptTerm.
 *        Exactly one of var ([num_features+1], Sigma diagonal: sum_k var_k g_k^2) and cov ([num_features+1]^2 row-major, dense
 *        Sigma, its lower triangle read; mlease_admm_posterior's output) is given.  CSR rows only, strictly ascending columns
 *        (checked: MLEASE_ERR_INVALID).  All pointers host-or-device. */
int mlease_score_var(int32_t device, void* stream, int32_t num_features, int64_t nrows, const int64_t* rowptr,
                     const int32_t* colidx, const float* vals, const float* offset, const double* model,
                     int32_t num_click_replicates, int32_t binary_feature, const double* var, const double* cov, float* pred,
                     float* pred_var);
int mlease_test_loglik(int32_t device, void* stream, int64_t nrows, const int32_t* response, const float* pred,
                       const float* weight, int64_t combiner_block, float* out_loglik, double* out_count);

/* ItemModelTest (jobs/ItemModelTest.java:181-211): the rows of key k are [key_rowstart[k], key_rowstart[k+1]) of one CSR (rowptr
 * [nrows+1] int64, colidx < num_features, any order, repeats add; vals; offset [nrows] or NULL); key_rowstart[0] = 0 and
 * nrows = key_rowstart[num_keys].  Model m = l*num_keys + k is entries [model_ptr[m], model_ptr[m+1]) of model_col (strictly
 * ascending within a model, checked; num_features = the intercept) and model_val (float).  An empty model is the reference's empty
 * LinearModel: pred = float(offset).  binary_feature: every listed feature counts as 1.  pred [num_lambdas][nrows]; every pred is
 * bitwise what mlease_score gives on its key's rows with its key's model widened to double.  All pointers host-or-device. */
int mlease_score_keyed(int32_t device, void* stream, int32_t num_features, int32_t num_keys, const int64_t* key_rowstart,
                       const int64_t* rowptr, const int32_t* colidx, const float* vals, const float* offset, int32_t num_lambdas,
                       const int64_t* model_ptr, const int32_t* model_col, const float* model_val, int32_t binary_feature, float* pred);
/* mlease_score_keyed with each record's predictive variance under the diagonal posterior of its key's model (ItemModelTrain with
 * compute.var).  Rows, keys and models as in mlease_score_keyed, model m = g*num_keys + k for grid point g of
 * num_models_per_key; rows must list strictly ascending columns (checked).  Model m's variance list is entries
 * [var_ptr[m], var_ptr[m+1]) of var_col (strictly ascending, <= num_features = the intercept, checked) and var_val; var_default[m]
 * is the variance of every column the list does not name; every variance finite and >= 0 (checked).
 * pred [G][nrows] is bitwise mlease_score_keyed's; pred_var [G][nrows] = float(sum_e v(c_e) x_e^2 + v_b) accumulated in double,
 * x_e = 1 under binary_feature, v_b = the listed intercept variance or 0; a model with an empty variance list gives NaN (no
 * posterior).  All pointers host-or-device; streams over key ranges and runs on several devices like mlease_score_keyed. */
int mlease_score_keyed_var(int32_t device, void* stream, int32_t num_features, int32_t num_keys, const int64_t* key_rowstart,
                           const int64_t* rowptr, const int32_t* colidx, const float* vals, const float* offset,
                           int32_t num_models_per_key, const int64_t* model_ptr, const int32_t* model_col, const float* model_val,
                           const int64_t* var_ptr, const int32_t* var_col, const float* var_val, const float* var_default,
                           int32_t binary_feature, float* pred, float* pred_var);
/* mlease_score_keyed with each record's predictive variance under the FULL posterior of its key's model (mlease_item_model_train_cov's
 * blocks, ordered by keyed_cov_for_scoring / as the models).  Model m = g * num_keys + k; its covariance is cov_val[cov_ptr[m] ..
 * cov_ptr[m+1]) (cov_ptr [G * num_keys + 1], cov_ptr[0] = 0), the packed lower triangle of Sigma over model m's own model_col list,
 * row-major (entry (a, b), a >= b, at cov_ptr[m] + a(a+1)/2 + b), of n_m(n_m+1)/2 finite values for a list of n_m entries, or empty
 * (no posterior: pred_var is NaN); any other size is MLEASE_ERR_INVALID.  An unlisted column c has variance 1 / lambda_map[c] where
 * lambda_map ([num_features] or NULL) is > 0, else var_default[m] (ItemModelTrain's own prior).  pred [G][nrows] is bitwise
 * mlease_score_keyed's; pred_var [G][nrows] = float(x_L^T Sigma_m x_L + sum over unlisted columns of v_c x_c^2), x_L the record's
 * entries the list names plus the intercept at 1 when the list ends with it, in fp64 in a fixed order (bitwise repeatable, the same
 * streamed or resident).  Rows must list strictly ascending columns (checked); binary_feature makes every x 1.  Streaming, budgets
 * and several-device use are mlease_score_keyed's; the blocks are held on the device for the whole call.  All pointers
 * host-or-device. */
int mlease_score_keyed_cov(int32_t device, void* stream, int32_t num_features, int32_t num_keys, const int64_t* key_rowstart,
                           const int64_t* rowptr, const int32_t* colidx, const float* vals, const float* offset, int32_t num_models_per_key,
                           const int64_t* model_ptr, const int32_t* model_col, const float* model_val, const int64_t* cov_ptr,
                           const double* cov_val, const float* lambda_map, const float* var_default, int32_t binary_feature, float* pred,
                           float* pred_var);
/* ItemModelTestLoglik (jobs/ItemModelTestLoglik.java:60-142): entry e = one (record, pred-map key) pair: entry_key[e] in
 * [0, num_keys), entry_group[e] = combiner group (non-decreasing), the record's response (1, 0, -1) and weight (NULL = 1), pred[e].
 * out_loglik / out_count [num_keys] (host): reducer float(sum of float combiner partials / sum of counts), partials added in group
 * order; a key without entries gets count 0 and loglik NaN.  Deterministic. */
int mlease_test_loglik_keyed(int32_t device, void* stream, int64_t nentries, const int32_t* entry_key, const int32_t* entry_group,
                             const int32_t* response, const float* weight, const float* pred, int32_t num_keys,
                             float* out_loglik, double* out_count);
/* The weighted ROC AUC of held-out predictions: the exact Mann-Whitney statistic with weights, tied pairs counting 1/2.
 * pred [num_sets][nrows] (a set is a lambda or a grid point: the pred of mlease_score_keyed[_var|_cov]); response [nrows] (1
 * positive; 0 or -1 negative, ItemModelTestLoglik's labels) and weight [nrows] (NULL = 1) are shared by every set.  key_rowstart
 * [num_keys + 1] (NULL with num_keys = 0: no per-key results): key k owns rows [key_rowstart[k], key_rowstart[k+1]).  Input
 * pointers host-or-device.
 * A segment is a set, or a (set, key) pair.  Over its runs r of equal pred in ascending order (-0.0 and +0.0 tie; +-inf are
 * ordinary values), with P_r / N_r its positive / negative weight and Nb_r the negative weight of the runs below r, in fp64:
 * U = sum_r P_r (Nb_r + N_r / 2), P = sum P_r, N = sum N_r, auc = U / (P N), NaN when P or N is 0.
 * Outputs (host memory, each may be NULL, not both AUC outputs): out_auc [num_sets]; out_weight [2] = positive and negative weight
 * of all rows; out_key_auc [num_sets][num_keys]; out_key_weight [num_keys][2].
 * Every AUC is bitwise repeatable and depends only on its own segment's records in stable sorted order (ties in row order): a
 * key's or a set's AUC is the same computed alone or among others.  The call streams over chunks of sets within free device
 * memory; a set that does not fit is MLEASE_ERR_INVALID, with the bytes it needs.  MLEASE_ERR_INVALID, before any output is
 * written: nrows outside [1, 2^31 - 1], num_sets < 1, a NaN pred, a response other than 1, 0, -1, a negative or NaN weight,
 * key_rowstart not starting at 0, decreasing or not ending at nrows, both AUC outputs NULL. */
int mlease_test_auc(int32_t device, void* stream, int64_t nrows, int32_t num_sets, const float* pred, const int32_t* response,
                    const float* weight, int32_t num_keys, const int64_t* key_rowstart, double* out_auc, double* out_weight,
                    double* out_key_auc, double* out_key_weight);

/* Bench / profiling hooks (not part of the reference surface): time one fused K1 pass or one Gram build
 * on a resident partition with CUDA events on the session stream, `reps` launches, returns avg ms. */
int mlease_time_kernel(mlease_session* s, int32_t partition_id, int32_t which /*1=K1,2=Gram wgmma,3=cholesky,4=Hv pass*/,
                       int32_t reps, int32_t emit_scaled, float* avg_ms);

#ifdef __cplusplus
}
#endif
#endif /* MLEASE_B200_H */
