// session.cu -- the session C ABI of include/mlease_b200.h: partition upload, the ADMM iteration driver, the getters and
// instrumentation, and the function-level entry points on a one-problem scratch batch.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "host.cuh"

using namespace mlease;

namespace {
thread_local std::string g_err;
}  // namespace

int mlease::fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

int mlease::open_device(int device, int* num_sms) {
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(MLEASE_ERR_CUDA, std::string("no CUDA device: this library has no CPU fallback (") + cudaGetErrorString(e) + ")");
  if (device < 0 || device >= ndev) return fail(MLEASE_ERR_INVALID, "bad device ordinal");
  CK(cudaSetDevice(device));
  int major = 0, minor = 0;
  CK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
  CK(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device));
  if (major != 9) return fail(MLEASE_ERR_CUDA, "this build targets sm_90a (H100) only; found sm_" + std::to_string(major) + std::to_string(minor));
  if (num_sms) CK(cudaDeviceGetAttribute(num_sms, cudaDevAttrMultiProcessorCount, device));
  return 0;
}

extern "C" {
static int csr_flush_pending(mlease_session* s);   // builds the deferred lists of the last CSR partition
}

namespace {

int find_part(mlease_session* s, int pid) {
  for (size_t i = 0; i < s->parts.size(); i++)
    if (s->parts[i].pid == pid) return (int)i;
  return -1;
}

void fill_problem_data(Problem& p, const PartData& pd) {
  p = pd.data;
  p.gram_scale = 1.f; p.gram_unscale = 1.f;
  if (p.bm_offs) {
    // e4m3 operands of the CSR Gram: |sqrt(d) x| <= 0.5 sqrt(wmax) max(|x|max, 1); scale the largest to ~224 (e4m3 max 448)
    const float amax = 0.5f * std::sqrt(std::max(p.wmax, 1e-30f)) * std::max(p.vmax, 1.f);
    int e = 0;
    std::frexp(224.f / amax, &e);
    e = std::max(-60, std::min(60, e - 1));
    p.gram_scale = std::ldexp(1.f, e);
    p.gram_unscale = std::ldexp(1.f, -2 * e);
  }
}

int finalize(mlease_session* s) {
  if (s->batch) return 0;
  if (int rc = csr_flush_pending(s)) return rc;
  if (s->copy_stream) {   // hand the builders' cached temporaries back before the solver state is allocated
    cudaMemPool_t mp;
    if (cudaDeviceGetDefaultMemPool(&mp, s->cfg.device) == cudaSuccess) cudaMemPoolTrimTo(mp, 0);
  }
  if (s->parts.empty()) return fail(MLEASE_ERR_STATE, "no partitions were added to this session");
  if (s->any_csr && s->any_dense) return fail(MLEASE_ERR_INVALID, "a session must hold either dense or CSR partitions, not both");
  std::sort(s->parts.begin(), s->parts.end(), [](const PartData& a, const PartData& b) { return a.pid < b.pid; });
  Batch* B = new Batch();
  s->batch = B;
  B->nprob = (int)s->parts.size() * s->L;
  B->Dt = s->Dt; B->ldx = s->ldx; B->csr = s->any_csr; B->has_bias = 1;
  B->group_L = s->L;
  B->h.resize(B->nprob);
  for (size_t pi = 0; pi < s->parts.size(); pi++)
    for (int l = 0; l < s->L; l++) {
      Problem& p = B->h[pi * s->L + l];
      fill_problem_data(p, s->parts[pi]);
      p.lambda_idx = l; p.part_local = (int)pi;
    }
  if (int rc = batch_alloc(*B, s->num_sms, s->cfg.hessian_policy, s->csr_gram_force)) return rc;
  const size_t ldv = s->ldx;
  if (int rc = s->mem.get(&s->d_z, s->L * ldv, true)) return rc;
  if (int rc = s->mem.get(&s->d_wz, s->L * ldv, true)) return rc;
  if (int rc = s->mem.get(&s->d_rho, s->L, true)) return rc;
  if (int rc = s->mem.get(&s->d_diff, s->L, true)) return rc;
  if (int rc = s->mem.get(&s->d_exch, (size_t)s->L * s->Dt + 1, true)) return rc;
  // z-update weights (jobs/RegressionAdmmTrain.java:381-386,392-403), in the reference's mixed float/double arithmetic
  std::vector<double> wz(s->L * ldv, 0.0);
  for (int l = 0; l < s->L; l++) {
    const float lf = s->lambdas[l], rf = s->rhos[l];
    const float pr = (float)s->P * rf;
    const double weight = (double)(pr / (lf + pr));
    for (int k = 0; k < s->Dg; k++) {
      double w = weight;
      if (!s->lambda_map.empty() && s->lambda_map[k] > 0.f) w = (double)pr / ((double)(s->lambda_map[k] + pr) + 0.0);
      wz[l * ldv + k] = w;
    }
    wz[l * ldv + s->Dg] = s->cfg.penalize_intercept ? weight : 1.0;
  }
  CK(cudaMemcpy(s->d_wz, wz.data(), wz.size() * sizeof(double), cudaMemcpyHostToDevice));
  if (s->cfg.regularizer == 1) {
    // weight = l / (r * nblocks + 0.0) (jobs/RegressionAdmmTrain.java:409): float product, double division.  The weightmap
    // built from lambda.map (:411-415) is never used by the thresholding loop, so lambda_map has no effect under L1.
    std::vector<double> thr(s->L);
    for (int l = 0; l < s->L; l++) thr[l] = (double)s->lambdas[l] / ((double)(s->rhos[l] * (float)s->P) + 0.0);
    if (int rc = s->mem.get(&s->d_l1thr, s->L, true)) return rc;
    CK(cudaMemcpy(s->d_l1thr, thr.data(), thr.size() * sizeof(double), cudaMemcpyHostToDevice));
  }
  return 0;
}

int ensure_scratch(mlease_session* s, int part_idx) {
  if (s->scratch && s->scratch_part == part_idx) return 0;
  if (int rc = csr_flush_pending(s)) return rc;
  delete s->scratch;
  s->scratch = new Batch();
  Batch* B = s->scratch;
  B->nprob = 1; B->Dt = s->Dt; B->ldx = s->ldx; B->csr = s->parts[part_idx].csr; B->has_bias = 1;
  B->h.resize(1);
  fill_problem_data(B->h[0], s->parts[part_idx]);
  s->scratch_part = part_idx;
  return batch_alloc(*B, s->num_sms, s->cfg.hessian_policy, s->csr_gram_force);
}

}  // namespace

double mlease::rho_eff_for_iter(mlease_session* s, int l, int iter) {
  // reducer: rho = lambdaRho[lambda] (float -> double), times rho.adapt.rate if != 1 (jobs/RegressionAdmmTrain.java:652-658);
  // rate = (float) exp(-(i-1)*coef) for i > 1 (:323-327)
  double r = (double)s->rhos[l];
  // rho.adapt.rate is a key of the per-iteration JobConf, which the driver re-creates every iteration (:286-291 ->
  // com/linkedin/mapred/AbstractAvroJob.java:101-115): the boost is seen by the reducers of iteration 1 only (:313-316)
  float rate = (iter == 1 && s->boost_rate > 0.f) ? s->boost_rate : 1.0f;
  // the product is float (int times float), the exponential double (Math.exp): std::exp of the float would be expf, which rounds
  // differently for some arguments (coefficient 0.289 at iteration 2: 0.74901223f instead of 0.7490122f)
  if (iter > 1 && s->cfg.rho_adapt_coefficient > 0) rate = (float)std::exp((double)(-(iter - 1) * s->cfg.rho_adapt_coefficient));
  if (rate != 1.0f) r = r * (double)rate;
  return r;
}

int mlease::scratch_for(mlease_session* s, int pid, Batch** B) {
  CK(cudaSetDevice(s->cfg.device));
  const int pi = find_part(s, pid);
  if (pi < 0) return fail(MLEASE_ERR_INVALID, "partition not resident in this session");
  if (int rc = ensure_scratch(s, pi)) return rc;
  *B = s->scratch;
  return 0;
}

// the Hv pass multiplies the fp32 copy of v (hv_vf) and scales its fixed-point sums by max |v| (Ctrl::hv_vinf)
int mlease::load_hv(Batch& B, int b, const double* v, cudaStream_t st) {
  std::vector<float> vf(B.ldx, 0.f);
  float vinf = 0.f;
  for (int k = 0; k < B.Dt; k++) { vf[k] = (float)v[k]; vinf = std::max(vinf, std::fabs(vf[k])); }
  const int on = 1;
  CK(cudaMemcpyAsync(B.h[b].hv_vf, vf.data(), (size_t)B.ldx * sizeof(float), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(&B.d_ctrl[b].hv_vinf, &vinf, sizeof(float), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(&B.d_ctrl[b].cg_active, &on, sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaStreamSynchronize(st));   // the host values above are read by the copies before this returns
  return 0;
}

// the stale-factor bookkeeping of the problem no longer matches its Lc / Hinv: force a rebuild on its next use
int mlease::reset_ctrl(Batch& B) {
  Ctrl c; std::memset(&c, 0, sizeof(c));
  CK(cudaMemcpy(B.d_ctrl, &c, sizeof(Ctrl), cudaMemcpyHostToDevice));
  B.mirror.clear();
  return 0;
}

// ============================================================================================
extern "C" {

const char* mlease_last_error(void) { return g_err.c_str(); }
int mlease_abi_version(void) { return 2; }

int mlease_session_create(const mlease_admm_config* cfg, mlease_session** out) {
  if (!cfg || !out) return fail(MLEASE_ERR_INVALID, "null argument");
  if (cfg->regularizer != 1 && cfg->regularizer != 2) return fail(MLEASE_ERR_INVALID, "Only L1 and L2 regularization supported!");
  if (cfg->num_blocks <= 0 || cfg->num_features <= 0 || cfg->num_lambdas <= 0 || !cfg->lambdas)
    return fail(MLEASE_ERR_INVALID, "num.blocks, num_features and lambda must be set");
  int num_sms = 0;
  if (int rc = open_device(cfg->device, &num_sms)) return rc;
  mlease_session* s = new mlease_session();
  s->cfg = *cfg;
  s->L = cfg->num_lambdas; s->P = cfg->num_blocks; s->Dg = cfg->num_features; s->Dt = s->Dg + 1;
  s->ldx = round_up(s->Dt, 4);
  s->lambdas.assign(cfg->lambdas, cfg->lambdas + s->L);
  for (int a = 0; a < s->L; a++)
    for (int b = a + 1; b < s->L; b++)
      if (s->lambdas[a] == s->lambdas[b]) { delete s; return fail(MLEASE_ERR_INVALID, "duplicate lambda"); }
  s->rhos.resize(s->L);
  for (int l = 0; l < s->L; l++) s->rhos[l] = cfg->rhos ? cfg->rhos[l] : (s->lambdas[l] <= 100 ? 1.0f : 10.0f);
  if (cfg->lambda_map) s->lambda_map.assign(cfg->lambda_map, cfg->lambda_map + s->Dg);
  s->cfg.lambdas = nullptr; s->cfg.rhos = nullptr; s->cfg.lambda_map = nullptr;
  s->stream = reinterpret_cast<cudaStream_t>(cfg->stream);
  s->num_sms = num_sms;
  s->xtol = cfg->newton_xtol > 0 ? cfg->newton_xtol : 2e-7;
  s->max_newton = cfg->max_newton > 0 ? cfg->max_newton : 50;
  int rc = s->pinned.get(&s->h_flag, 16, false);   // 64 B each
  if (!rc) rc = s->mem.get(&s->d_flag, 16, false);
  if (!rc) rc = s->pinned.get(&s->h_small, (size_t)(8 * s->L + 8), false);
  if (rc) { delete s; return rc; }
  *out = s;
  return 0;
}

int mlease_session_destroy(mlease_session* s) {
  if (!s) return 0;
  cudaSetDevice(s->cfg.device);
  cudaDeviceSynchronize();
  delete s;
  return 0;
}

static int add_common(mlease_session* s, PartData& pd, const int32_t* response, const float* weight, const float* offset) {
  const long long n = pd.data.n;
  signed char* y; float *w, *o;
  if (int rc = s->mem.get(&y, n, true)) return rc;
  if (int rc = s->mem.get(&w, n, true)) return rc;
  if (int rc = s->mem.get(&o, n, true)) return rc;
  if (int rc = ingest_labels(s->stream, n, response, weight, offset, y, w, o, s->d_flag, s->h_flag, &pd.data.wmax)) return rc;
  pd.data.y = y; pd.data.w = w; pd.data.o = o;
  return 0;
}

int mlease_add_partition_dense(mlease_session* s, int32_t pid, int64_t nrows, const float* X, int64_t ldx_in, const int32_t* response,
                               const float* weight, const float* offset) {
  if (!s || !X || !response || nrows <= 0) return fail(MLEASE_ERR_INVALID, "bad argument (null pointer or empty partition)");
  if (s->batch) return fail(MLEASE_ERR_STATE, "partitions must be added before the first ADMM call");
  if (pid < 0 || pid >= s->P) return fail(MLEASE_ERR_INVALID, "Map key is wrong! key has to be in the range of [0,numPartitions-1].");
  if (find_part(s, pid) >= 0) return fail(MLEASE_ERR_INVALID, "partition added twice");
  if (s->cfg.binary_feature) return fail(MLEASE_ERR_INVALID, "binary.feature needs CSR input (every listed feature counts as 1)");
  if (ldx_in < s->Dg) return fail(MLEASE_ERR_INVALID, "ldx < num_features");
  CK(cudaSetDevice(s->cfg.device));
  PartData pd;
  pd.pid = pid; pd.data.n = nrows; pd.csr = false;
  float* x;
  if (int rc = s->mem.get(&x, (size_t)nrows * s->ldx, false)) return rc;
  pd.data.X = x;
  if (int rc = upload_dense_rows(x, s->ldx, X, ldx_in, nrows, s->Dg, 1, s->stream)) return rc;
  if (int rc = add_common(s, pd, response, weight, offset)) return rc;
  s->parts.push_back(pd);
  s->any_dense = true;
  return 0;
}

static int csr_flush_pending(mlease_session* s) {
  if (s->pending_csr < 0) return 0;
  const int idx = s->pending_csr;
  s->pending_csr = -1;
  return csr_build_layout(s, s->parts[idx]);
}

// The big arrays travel on copy_stream while the previous partition's lists are built on s->stream; a malformed colidx of
// partition p is therefore reported by the NEXT session call (add_partition / begin / fit), with the partition id in the message.
int mlease_add_partition_csr(mlease_session* s, int32_t pid, int64_t nrows, const int64_t* rowptr, const int32_t* colidx, const float* vals,
                             const int32_t* response, const float* weight, const float* offset) {
  if (!s || !rowptr || !response || nrows <= 0) return fail(MLEASE_ERR_INVALID, "bad argument (null pointer or empty partition)");
  if (s->batch) return fail(MLEASE_ERR_STATE, "partitions must be added before the first ADMM call");
  if (pid < 0 || pid >= s->P) return fail(MLEASE_ERR_INVALID, "Map key is wrong! key has to be in the range of [0,numPartitions-1].");
  if (find_part(s, pid) >= 0) return fail(MLEASE_ERR_INVALID, "partition added twice");
  CK(cudaSetDevice(s->cfg.device));
  if (!s->copy_stream) {
    CK(cudaStreamCreateWithFlags(&s->copy_stream, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&s->copy_ev, cudaEventDisableTiming));
    // the list builders take their temporaries from the device's stream-ordered pool: keep them cached between partitions
    cudaMemPool_t mp;
    if (cudaDeviceGetDefaultMemPool(&mp, s->cfg.device) == cudaSuccess) {
      unsigned long long keep = 8ULL << 30;
      cudaMemPoolSetAttribute(mp, cudaMemPoolAttrReleaseThreshold, &keep);
    }
  }
  // the inputs are ready in the order of the session stream (they may be device arrays a kernel on that stream is still writing)
  CK(cudaEventRecord(s->copy_ev, s->stream));
  CK(cudaStreamWaitEvent(s->copy_stream, s->copy_ev, 0));
  PartData pd;
  pd.pid = pid; pd.data.n = nrows; pd.csr = true;
  long long ends[2];
  CK(cudaMemcpyAsync(&ends[0], rowptr, 8, cudaMemcpyDefault, s->copy_stream));
  CK(cudaMemcpyAsync(&ends[1], rowptr + nrows, 8, cudaMemcpyDefault, s->copy_stream));
  CK(cudaStreamSynchronize(s->copy_stream));
  if (ends[0] != 0) return fail(MLEASE_ERR_INVALID, "rowptr[0] must be 0");
  if (ends[1] < 0) return fail(MLEASE_ERR_INVALID, "rowptr[nrows] < 0");
  const long long nnz = ends[1];
  pd.data.nnz_hint = nnz;
  if (nnz > 0 && (!colidx || !vals)) return fail(MLEASE_ERR_INVALID, "null colidx/vals");
  if (int rc = add_common(s, pd, response, weight, offset)) return rc;   // label checks first: nothing is in flight when they fail
  // not zero-filled: the copies write every byte, and a fill on the default stream would not be ordered before them
  long long* rp; int* ci; float* vv;
  if (int rc = s->mem.get(&rp, nrows + 1, false)) return rc;
  if (int rc = s->mem.get(&ci, nnz, false)) return rc;
  if (int rc = s->mem.get(&vv, nnz, false)) return rc;
  pd.data.rowptr = rp; pd.data.colidx = ci; pd.data.vals = vv;
  cudaError_t ce = cudaMemcpyAsync(rp, rowptr, (nrows + 1) * 8, cudaMemcpyDefault, s->copy_stream);
  if (ce == cudaSuccess && nnz > 0) ce = cudaMemcpyAsync(ci, colidx, nnz * 4, cudaMemcpyDefault, s->copy_stream);
  if (ce == cudaSuccess && nnz > 0) ce = cudaMemcpyAsync(vv, vals, nnz * 4, cudaMemcpyDefault, s->copy_stream);
  const int rc_prev = ce == cudaSuccess ? csr_flush_pending(s) : 0;      // overlaps the copies above
  const cudaError_t cs = cudaStreamSynchronize(s->copy_stream);          // the caller's buffers are free again on every return path
  CK(ce);
  CK(cs);
  if (rc_prev) return rc_prev;
  s->parts.push_back(pd);
  s->pending_csr = (int)s->parts.size() - 1;
  s->any_csr = true;
  return 0;
}

static int admm_begin_impl(mlease_session* s, const double* z0, float boost_rate) {
  if (!s) return fail(MLEASE_ERR_INVALID, "null session");
  CK(cudaSetDevice(s->cfg.device));
  if (int rc = finalize(s)) return rc;
  s->boost_rate = z0 ? boost_rate : 0.f;
  s->iter = 0; s->liblinear_eps = 0.01f; s->mindiff = 99999999; s->last_maxdiff = 0;
  for (int l = 0; l < s->L; l++) s->h_small[l] = rho_eff_for_iter(s, l, 1);
  CK(cudaMemcpyAsync(s->d_rho, s->h_small, s->L * sizeof(double), cudaMemcpyHostToDevice, s->stream));
  int launches = 0;
  CK(admm_reset(s->batch->d, s->batch->nprob, s->L, s->d_z, s->ldx, s->d_rho, s->stream, &launches));
  if (z0) {
    std::vector<double> zh((size_t)s->L * s->ldx, 0.0);
    for (int l = 0; l < s->L; l++) std::memcpy(&zh[(size_t)l * s->ldx], z0 + (size_t)l * s->Dt, (size_t)s->Dt * sizeof(double));
    CK(cudaMemcpyAsync(s->d_z, zh.data(), zh.size() * sizeof(double), cudaMemcpyHostToDevice, s->stream));
    CK(admm_init(s->batch->d, s->batch->nprob, s->d_z, s->ldx, s->stream, &launches));
    CK(cudaStreamSynchronize(s->stream));   // zh is a stack-lifetime buffer
  }
  CK(cudaStreamSynchronize(s->stream));
  s->cnt.launches += launches;
  s->rho_fact.assign(s->L, -1.0);
  s->begun = true;
  return 0;
}

int mlease_admm_begin(mlease_session* s) { return admm_begin_impl(s, nullptr, 0.f); }

int mlease_admm_begin_initialized(mlease_session* s, const double* z0, float boost_rate) {
  if (!z0) return fail(MLEASE_ERR_INVALID, "null z0");
  if (!(boost_rate > 0.f)) return fail(MLEASE_ERR_INVALID, "initialize.boost.rate must be > 0 to start from a model");
  if (s && s->cfg.regularizer != 2) return fail(MLEASE_ERR_INVALID, "mean-model initialization is an L2 feature (jobs/RegressionAdmmTrain.java:236)");
  return admm_begin_impl(s, z0, boost_rate);
}

int mlease_admm_local_step(mlease_session* s, double* exchange_dev) {
  if (!s || !exchange_dev) return fail(MLEASE_ERR_INVALID, "null argument");
  if (!s->begun) return fail(MLEASE_ERR_STATE, "mlease_admm_begin was not called");
  CK(cudaSetDevice(s->cfg.device));
  s->iter++;
  const int i = s->iter;
  // tolerance schedule: control only (jobs/RegressionAdmmTrain.java:338-346)
  if (i > 1 && s->mindiff < 0.001 && !s->cfg.aggressive_decay) s->liblinear_eps = s->liblinear_eps / 10;
  else if (s->cfg.aggressive_decay && i > 5) s->liblinear_eps = s->liblinear_eps / 10;
  int invalidate = 0;
  for (int l = 0; l < s->L; l++) {
    const double r = rho_eff_for_iter(s, l, i);
    if (r != s->rho_fact[l]) invalidate = 1;   // prior precision changed -> stale factors are for another H
    s->rho_fact[l] = r;
  }
  int same_rho = 1;   // cold start: equal rho across lambdas means equal Hessians (H = G + rho I at beta = 0)
  for (int l = 1; l < s->L; l++) if (s->rho_fact[l] != s->rho_fact[0]) same_rho = 0;
  const int nc_before = s->cnt.not_converged;
  if (int rc = batch_xupdate(*s->batch, s->stream, s->xtol, s->max_newton, s->cfg.hessian_policy, invalidate, s->h_flag, s->d_flag, s->cnt, &s->prof,
                             (i == 1 && s->L > 1 && s->boost_rate == 0.f) ? s->L : 0, same_rho)) return rc;   // sharing needs beta = 0 for every lambda
  // An x-update that ran out of Newton steps (or slots) is a failed fit: the reducer wraps any fit exception as
  // IOException("Model fitting error!") and the job dies (jobs/RegressionAdmmTrain.java:713-716); an unconverged x_p must not
  // be averaged into z silently.
  if (s->cnt.not_converged > nc_before)
    return fail(MLEASE_ERR_NUMERIC, "Model fitting error! (" + std::to_string(s->cnt.not_converged - nc_before) +
                                        " x-update(s) of iteration " + std::to_string(i) + " did not converge within max_newton = " +
                                        std::to_string(s->max_newton) + " steps)");
  int launches = 0;
  CK(admm_pack(s->batch->d, (int)s->parts.size(), s->L, s->Dt, exchange_dev, s->stream, &launches));
  s->cnt.launches += launches;
  return 0;
}

}  // extern "C"

// z/u update of the iteration: enqueue (kernel + read-back of the per-lambda |z - z_prev| into pinned memory), then, after the
// caller's ONE stream synchronisation, finish (convergence scalars, stop rule :493-496).
int mlease::consensus_enqueue(mlease_session* s, const double* exchange_sum_dev) {
  for (int l = 0; l < s->L; l++) s->h_small[l] = rho_eff_for_iter(s, l, s->iter + 1);
  CK(cudaMemcpyAsync(s->d_rho, s->h_small, s->L * sizeof(double), cudaMemcpyHostToDevice, s->stream));
  int launches = 0;
  CK(admm_consensus(s->batch->d, (int)s->parts.size(), s->L, s->Dt, s->ldx, s->P, exchange_sum_dev, s->d_z, s->d_wz, s->d_rho, s->d_diff, s->stream, &launches, s->d_l1thr));
  s->cnt.launches += launches;
  CK(cudaMemcpyAsync(s->h_small + s->L, s->d_diff, s->L * sizeof(double), cudaMemcpyDeviceToHost, s->stream));
  return 0;
}
void mlease::consensus_finish(mlease_session* s, double* maxdiff, int32_t* stop) {
  const double* hd = s->h_small + s->L;
  double mx = 0, mn = 99999999;
  for (int l = 0; l < s->L; l++) { mx = std::max(mx, hd[l]); mn = std::min(mn, hd[l]); }
  s->mindiff = mn; s->last_maxdiff = mx;
  if (maxdiff) *maxdiff = mx;
  const double eps = s->cfg.epsilon >= 0 ? s->cfg.epsilon : 0.0001;   // default 1e-4 (:473); 0 = never stop early
  if (stop) *stop = (mx < eps && s->liblinear_eps <= 0.00001) ? 1 : 0;   // :493-496
}

extern "C" {

int mlease_admm_consensus(mlease_session* s, const double* exchange_sum_dev, double* maxdiff, int32_t* stop) {
  if (!s || !exchange_sum_dev) return fail(MLEASE_ERR_INVALID, "null argument");
  if (!s->begun || s->iter < 1) return fail(MLEASE_ERR_STATE, "consensus before local_step");
  CK(cudaSetDevice(s->cfg.device));
  if (int rc = consensus_enqueue(s, exchange_sum_dev)) return rc;
  CK(cudaStreamSynchronize(s->stream));
  consensus_finish(s, maxdiff, stop);
  return 0;
}

int mlease_session_set_comm(mlease_session* s, mlease_comm* comm) {
  if (!s) return fail(MLEASE_ERR_INVALID, "null session");
  s->comm = comm;
  return 0;
}

// One iteration with the exchange inside: local x-updates, all-reduce (NCCL communicator, caller's callback, or nothing for
// a single-process job), z/u update.  A rank whose fit failed still enters the collective -- with its failure counted in the
// extra last element of the buffer -- so that every rank leaves with the same error instead of the others hanging in NCCL
// (the reference: one failed reducer fails the whole iteration job, jobs/RegressionAdmmTrain.java:713-716).
static int admm_iterate_impl(mlease_session* s, mlease_allreduce_fn allreduce, void* ctx, double* maxdiff, int32_t* stop) {
  const size_t cnt = (size_t)s->L * s->Dt;
  int rc_local = mlease_admm_local_step(s, s->d_exch);
  std::string local_msg;
  if (rc_local == MLEASE_ERR_NUMERIC) local_msg = g_err;
  else if (rc_local) return rc_local;                      // CUDA / state errors are not recoverable: no collective
  const bool multi = s->comm != nullptr || allreduce != nullptr;
  if (multi) {
    // all-reduce, z/u update and both read-backs are enqueued back to back; ONE synchronisation per iteration.  (If a fit
    // failed somewhere the z/u update has run on a meaningless sum, but the job is over: every rank returns the error.)
    double* h_flag = s->h_small + 3 * s->L + 1;   // pinned
    *h_flag = rc_local ? 1.0 : 0.0;
    CK(cudaMemcpyAsync(s->d_exch + cnt, h_flag, sizeof(double), cudaMemcpyHostToDevice, s->stream));
    if (s->comm) { if (int rc = comm_allreduce(s->comm, s->d_exch, cnt + 1, s->stream)) return rc; }
    else if (allreduce(ctx, s->d_exch, cnt + 1, (void*)s->stream) != 0) return fail(MLEASE_ERR_CUDA, "all-reduce callback failed");
    double* h_failed = s->h_small + 3 * s->L + 2;
    CK(cudaMemcpyAsync(h_failed, s->d_exch + cnt, sizeof(double), cudaMemcpyDeviceToHost, s->stream));
    if (int rc = consensus_enqueue(s, s->d_exch)) return rc;
    CK(cudaStreamSynchronize(s->stream));
    if (rc_local) return fail(rc_local, local_msg);
    if (*h_failed > 0) return fail(MLEASE_ERR_NUMERIC, "Model fitting error! (the x-update failed on " + std::to_string((int)*h_failed) + " other rank(s))");
    consensus_finish(s, maxdiff, stop);
    return 0;
  } else if (rc_local) {
    return fail(rc_local, local_msg);
  }
  return mlease_admm_consensus(s, s->d_exch, maxdiff, stop);
}

static int check_partitions_present(mlease_session* s, bool multi) {
  if (!multi && (int)s->parts.size() != s->P)
    return fail(MLEASE_ERR_STATE, "Some models failed! (" + std::to_string(s->parts.size()) + " of " + std::to_string(s->P) +
                                      " partitions present and neither a communicator nor an all-reduce was given)");
  return 0;
}

int mlease_admm_run(mlease_session* s, int32_t num_iters, mlease_allreduce_fn allreduce, void* ctx, int32_t* iters_done) {
  if (!s) return fail(MLEASE_ERR_INVALID, "null session");
  if (int rc = mlease_admm_begin(s)) return rc;
  if (int rc = check_partitions_present(s, s->comm != nullptr || allreduce != nullptr)) return rc;
  int done = 0;
  for (int i = 1; i <= num_iters; i++) {
    double md; int32_t stop;
    if (int rc = admm_iterate_impl(s, allreduce, ctx, &md, &stop)) return rc;
    done = i;
    if (stop) break;
  }
  if (iters_done) *iters_done = done;
  return 0;
}

int mlease_admm_iterate(mlease_session* s, double* maxdiff, int32_t* stop) {
  if (!s) return fail(MLEASE_ERR_INVALID, "null session");
  if (!s->begun) return fail(MLEASE_ERR_STATE, "mlease_admm_begin was not called");
  if (int rc = check_partitions_present(s, s->comm != nullptr)) return rc;
  return admm_iterate_impl(s, nullptr, nullptr, maxdiff, stop);
}

int mlease_get_z(mlease_session* s, int32_t l, double* out) {
  if (!s || !out || l < 0 || l >= s->L || !s->batch) return fail(MLEASE_ERR_INVALID, "bad argument");
  CK(cudaSetDevice(s->cfg.device));
  CK(cudaMemcpyAsync(out, s->d_z + (size_t)l * s->ldx, s->Dt * sizeof(double), cudaMemcpyDeviceToHost, s->stream));
  CK(cudaStreamSynchronize(s->stream));
  return 0;
}
int mlease_get_final_model(mlease_session* s, int32_t l, float* out) {
  std::vector<double> z(s ? s->Dt : 0);
  if (int rc = mlease_get_z(s, l, z.data())) return rc;
  for (int k = 0; k < s->Dt; k++) out[k] = (float)z[k];   // models/LinearModel.java:703,716
  return 0;
}
static int get_vec(mlease_session* s, int pid, int l, int which, void* out) {
  if (!s || !out || l < 0 || l >= s->L || !s->batch) return fail(MLEASE_ERR_INVALID, "bad argument");
  const int pi = find_part(s, pid);
  if (pi < 0) return fail(MLEASE_ERR_INVALID, "partition not resident in this session");
  CK(cudaSetDevice(s->cfg.device));
  const Problem& p = s->batch->h[pi * s->L + l];
  const void* src = which == 0 ? (const void*)p.x_d : which == 1 ? (const void*)p.u_f : (const void*)p.uplusx_f;
  CK(cudaMemcpyAsync(out, src, s->Dt * (which == 0 ? 8 : 4), cudaMemcpyDeviceToHost, s->stream));
  CK(cudaStreamSynchronize(s->stream));
  return 0;
}
int mlease_get_x(mlease_session* s, int32_t pid, int32_t l, double* out) { return get_vec(s, pid, l, 0, out); }
int mlease_get_u(mlease_session* s, int32_t pid, int32_t l, float* out) { return get_vec(s, pid, l, 1, out); }
int mlease_get_uplusx(mlease_session* s, int32_t pid, int32_t l, float* out) { return get_vec(s, pid, l, 2, out); }

int mlease_profile(mlease_session* s, int32_t enable, double* ms4, int64_t* count4, double* k1_bytes, double* k1_emit_bytes, double* gram_flops) {
  if (!s) return fail(MLEASE_ERR_INVALID, "null session");
  if (ms4) for (int i = 0; i < 4; i++) ms4[i] = s->prof.ms[i];
  if (count4) for (int i = 0; i < 4; i++) count4[i] = s->prof.n[i];
  if (k1_bytes) *k1_bytes = s->cnt.k1_bytes;
  if (k1_emit_bytes) *k1_emit_bytes = s->cnt.k1_emit_bytes;
  if (gram_flops) *gram_flops = s->cnt.gram_flops;
  if (enable >= 0) {
    s->prof.on = enable != 0;
    if (enable == 2) { for (int i = 0; i < 4; i++) { s->prof.ms[i] = 0; s->prof.n[i] = 0; } s->cnt.k1_bytes = s->cnt.k1_emit_bytes = s->cnt.gram_flops = 0; }
  }
  return 0;
}

int mlease_get_stats(mlease_session* s, mlease_stats* out) {
  if (!s || !out) return fail(MLEASE_ERR_INVALID, "null argument");
  out->k1_passes = s->cnt.k1_passes; out->gram_builds = s->cnt.gram_builds; out->newton_steps = s->cnt.newton_steps;
  out->rejected_steps = s->cnt.rejected; out->kernel_launches = s->cnt.launches; out->not_converged = s->cnt.not_converged;
  out->last_iter_slots = s->cnt.last_slots; out->last_maxdiff = s->last_maxdiff; out->liblinear_epsilon = s->liblinear_eps;
  out->k1_shared_bytes = s->cnt.k1_shared_bytes;
  out->k1_fused = (s->batch && s->batch->k1_fused) ? 1 : 0;
  return 0;
}

// ------------------------------------------------------------------------------------------
// function-level entry points on the scratch problem
// ------------------------------------------------------------------------------------------
static int scratch_set(mlease_session* s, const double* w, const double* m, const double* q) {
  Batch* B = s->scratch;
  const Problem& p = B->h[0];
  std::vector<double> buf(3 * (size_t)s->ldx, 0.0);
  for (int k = 0; k < s->Dt; k++) { buf[k] = w[k]; buf[s->ldx + k] = m[k]; buf[2 * s->ldx + k] = q[k]; }
  for (int k = s->Dt; k < s->ldx; k++) buf[2 * s->ldx + k] = 1.0;
  CK(cudaMemcpyAsync(p.beta, buf.data(), s->ldx * 8, cudaMemcpyHostToDevice, s->stream));
  CK(cudaMemcpyAsync(p.m, buf.data() + s->ldx, s->ldx * 8, cudaMemcpyHostToDevice, s->stream));
  CK(cudaMemcpyAsync(p.q, buf.data() + 2 * s->ldx, s->ldx * 8, cudaMemcpyHostToDevice, s->stream));
  CK(cudaStreamSynchronize(s->stream));
  return 0;
}

int mlease_objective(mlease_session* s, int32_t pid, const double* w, const double* m, const double* q, double* f, double* g, double* H,
                     int32_t tensor) {
  if (!s || !w || !m || !q) return fail(MLEASE_ERR_INVALID, "null argument");
  Batch* B;
  if (int rc = scratch_for(s, pid, &B)) return rc;
  if (int rc = scratch_set(s, w, m, q)) return rc;
  int launches = 0;
  CK(newton_begin(B->d, 1, 1e-8, 1, 1, 1, 0, s->stream, &launches));
  CK(batch_k1(*B, H ? 1 : 0, s->stream, &launches));
  CK(k1_reduce_decide(B->d, 1, B->Dt, s->stream, &launches));
  const Problem& p = B->h[0];
  Ctrl c;
  CK(cudaMemcpyAsync(&c, B->d_ctrl, sizeof(Ctrl), cudaMemcpyDeviceToHost, s->stream));
  if (g) CK(cudaMemcpyAsync(g, p.g_acc, s->Dt * 8, cudaMemcpyDeviceToHost, s->stream));   // first evaluation is always accepted: g_acc = gradient at w
  CK(cudaStreamSynchronize(s->stream));
  if (f) *f = c.f_t;
  if (H) {
    if (B->matfree) return fail(MLEASE_ERR_INVALID, "this session's problems are matrix-free (hessian_policy 2, or a Hessian too large for the device): use mlease_hessian_vector");
    if (!tensor && B->gram_from_csr) return fail(MLEASE_ERR_INVALID, "the SIMT debug Gram needs the dense bf16 operand, which CSR partitions with sorted unique rows do not materialise");
    if (tensor) CK(batch_gram(*B, B->d, 1, 1, s->stream, &launches));
    else CK(gram_launch_simt(B->d, 1, B->Dp, 1, s->stream, &launches));
    if (tensor == 2) {
      // the inverse the Newton direction uses: split-K Gram partials + diag(q) -> fp64 Cholesky -> explicit inverse
      Ctrl c2; std::memset(&c2, 0, sizeof(c2)); c2.need_hess = 1;
      CK(cudaMemcpyAsync(B->d_ctrl, &c2, sizeof(Ctrl), cudaMemcpyHostToDevice, s->stream));
      CK(cholesky_launch(B->d, 1, B->ldh, s->stream, &launches, 0, 0, 1));
      std::vector<double> hi((size_t)B->ldh * B->ldh);
      CK(cudaMemcpyAsync(hi.data(), p.Hinv, hi.size() * 8, cudaMemcpyDeviceToHost, s->stream));
      CK(cudaMemcpyAsync(&c2, B->d_ctrl, sizeof(Ctrl), cudaMemcpyDeviceToHost, s->stream));
      CK(cudaStreamSynchronize(s->stream));
      s->cnt.launches += launches;
      if (c2.fail) return fail(MLEASE_ERR_NUMERIC, "Hessian not positive definite");
      for (int i = 0; i < s->Dt; i++)
        for (int j = 0; j < s->Dt; j++) H[(size_t)i * s->Dt + j] = hi[(size_t)i * B->ldh + j];
      return 0;
    }
    const size_t per = (size_t)B->Dp * B->Dp;
    std::vector<float> hp(per * B->gram_slices);
    CK(cudaMemcpyAsync(hp.data(), p.Hpart, hp.size() * 4, cudaMemcpyDeviceToHost, s->stream));
    CK(cudaStreamSynchronize(s->stream));
    const int Dt = s->Dt;
    for (int i = 0; i < Dt; i++)
      for (int j = 0; j <= i; j++) {
        double a = 0;
        for (int t = 0; t < B->gram_slices; t++) a += (double)hp[t * per + (size_t)i * B->Dp + j];
        if (B->gram_from_csr) a *= (double)p.gram_unscale;
        if (i == j) a += q[i];
        H[(size_t)i * Dt + j] = a;
        H[(size_t)j * Dt + i] = a;
      }
  }
  s->cnt.launches += launches;
  return 0;
}

int mlease_fit_partition(mlease_session* s, int32_t pid, double* x, const double* m, const double* q, int32_t* newton_steps) {
  if (!s || !x || !m || !q) return fail(MLEASE_ERR_INVALID, "null argument");
  Batch* B;
  if (int rc = scratch_for(s, pid, &B)) return rc;
  if (int rc = scratch_set(s, x, m, q)) return rc;
  Counters c;
  if (int rc = batch_xupdate(*B, s->stream, s->xtol, s->max_newton, s->cfg.hessian_policy, 1, s->h_flag, s->d_flag, c)) return rc;
  s->cnt.launches += c.launches; s->cnt.k1_passes += c.k1_passes; s->cnt.gram_builds += c.gram_builds;
  s->cnt.newton_steps += c.newton_steps; s->cnt.rejected += c.rejected; s->cnt.not_converged += c.not_converged;
  CK(cudaMemcpyAsync(x, B->h[0].beta, s->Dt * 8, cudaMemcpyDeviceToHost, s->stream));
  CK(cudaStreamSynchronize(s->stream));
  if (newton_steps) *newton_steps = (int)c.newton_steps;
  if (c.not_converged) return fail(MLEASE_ERR_NUMERIC, "Model fitting error! (Newton did not converge within max_newton steps)");
  return 0;
}

int mlease_posterior_variance(mlease_session* s, int32_t pid, const double* w, const double* q, int32_t full, double* var, double* cov) {
  if (!s || !w || !q || !var) return fail(MLEASE_ERR_INVALID, "null argument");
  if (cov && !full) return fail(MLEASE_ERR_INVALID, "the covariance matrix is only available with full = 1 (computeFullPostVar)");
  Batch* B;
  if (int rc = scratch_for(s, pid, &B)) return rc;
  const Problem& p = B->h[0];
  if (full && B->matfree) return fail(MLEASE_ERR_INVALID, "the full posterior variance needs the Hessian matrix, which a matrix-free session does not form");
  if (full && B->csr && !p.csr_unique)
    return fail(MLEASE_ERR_INVALID, "the full Hessian needs rows with strictly increasing column ids (llf/LogisticRegressionL2.java:277)");
  std::vector<double> zero(s->Dt, 0.0);
  if (int rc = scratch_set(s, w, zero.data(), q)) return rc;          // beta = w, q = prior precision (1 on the padding)
  DevMem t;
  double* dvec; long long* drs;
  if (int rc = t.get(&dvec, (size_t)p.n, false)) return rc;
  if (int rc = t.get(&drs, 2, false)) return rc;
  const long long rs[2] = {0, p.n};   // the batch kernels over one problem
  CK(cudaMemcpyAsync(drs, rs, sizeof(rs), cudaMemcpyHostToDevice, s->stream));
  int launches = 0;
  CK(postvar_rowweights(B->d, 1, drs, p.n, 1, dvec, s->stream, &launches));
  if (!full) {
    // H[k] = 1/priorVar[k] + sum_i weight_i p_i (1-p_i) x_ik^2, postVar = 1/H (llf/LibLinear.java:330-333)
    CK(postvar_diag(B->d, 1, drs, p.n, dvec, 1, s->stream, &launches));
    CK(cudaMemcpyAsync(var, p.g_t, (size_t)s->Dt * sizeof(double), cudaMemcpyDeviceToHost, s->stream));
    CK(cudaStreamSynchronize(s->stream));
    for (int k = 0; k < s->Dt; k++) var[k] = 1.0 / var[k];
    s->cnt.launches += launches;
    return 0;
  }
  // exact fp64 Hessian -> K3's factorisation and explicit inverse (llf/LibLinear.java:318-326)
  CK(postvar_hessian(B->d, B->csr, B->ldh, dvec, p.q, 1, s->stream, &launches));
  Ctrl c; std::memset(&c, 0, sizeof(c)); c.need_hess = 1;
  CK(cudaMemcpyAsync(B->d_ctrl, &c, sizeof(Ctrl), cudaMemcpyHostToDevice, s->stream));
  CK(cholesky_launch(B->d, 1, B->ldh, s->stream, &launches, 0, 1, 1));
  std::vector<double> hi((size_t)B->ldh * B->ldh);
  CK(cudaMemcpyAsync(hi.data(), p.Hinv, hi.size() * sizeof(double), cudaMemcpyDeviceToHost, s->stream));
  CK(cudaMemcpyAsync(&c, B->d_ctrl, sizeof(Ctrl), cudaMemcpyDeviceToHost, s->stream));
  CK(cudaStreamSynchronize(s->stream));
  s->cnt.launches += launches;
  if (c.fail) return fail(MLEASE_ERR_NUMERIC, "Model fitting error! (Hessian not positive definite)");
  for (int i = 0; i < s->Dt; i++) {
    var[i] = hi[(size_t)i * B->ldh + i];
    if (cov) for (int j = 0; j < s->Dt; j++) cov[(size_t)i * s->Dt + j] = hi[(size_t)i * B->ldh + j];
  }
  return reset_ctrl(*B);
}

int mlease_hessian_vector(mlease_session* s, int32_t pid, const double* w, const double* q, const double* v, double* out) {
  if (!s || !w || !q || !v || !out) return fail(MLEASE_ERR_INVALID, "null argument");
  Batch* B;
  if (int rc = scratch_for(s, pid, &B)) return rc;
  if (!(B->csr && B->csr_fx)) return fail(MLEASE_ERR_INVALID, "Hessian-vector products need CSR rows with strictly increasing column ids");
  std::vector<double> zero(s->Dt, 0.0);
  if (int rc = scratch_set(s, w, zero.data(), q)) return rc;
  const Problem& p = B->h[0];
  int launches = 0;
  // one gradient pass at w leaves sqrt(d) in sdvec; the Hv pass multiplies the fp32 copy of v (hv_vf) with X^T D X
  CK(newton_begin(B->d, 1, 1e-8, 1, 1, 1, 0, s->stream, &launches));
  CK(batch_k1(*B, 1, s->stream, &launches));
  if (int rc = load_hv(*B, 0, v, s->stream)) return rc;
  const int off = 0;
  CK(batch_k1(*B, 0, s->stream, &launches, K1_HV));
  CK(hv_reduce(B->d, 1, B->Dt, 0, s->stream, &launches));
  CK(cudaMemcpyAsync(&B->d_ctrl->cg_active, &off, sizeof(int), cudaMemcpyHostToDevice, s->stream));
  CK(cudaMemcpyAsync(out, p.g_t, (size_t)s->Dt * sizeof(double), cudaMemcpyDeviceToHost, s->stream));
  CK(cudaStreamSynchronize(s->stream));   // (the stack values above are read by the copies before this returns)
  for (int k = 0; k < s->Dt; k++) out[k] += q[k] * v[k];   // prior term s / priorVar (llf/LogisticRegressionL2.java:246)
  s->cnt.launches += launches;
  return 0;
}
int mlease_time_kernel(mlease_session* s, int32_t pid, int32_t which, int32_t reps, int32_t emit_scaled, float* avg_ms) {
  if (!s || !avg_ms || reps <= 0) return fail(MLEASE_ERR_INVALID, "bad argument");
  Batch* B;
  if (int rc = scratch_for(s, pid, &B)) return rc;
  if ((which == 2 || which == 3) && B->matfree) return fail(MLEASE_ERR_INVALID, "a matrix-free session builds no Gram and no factor");
  if (which == 4 && !(B->csr && B->csr_fx)) return fail(MLEASE_ERR_INVALID, "Hessian-vector passes need CSR rows with strictly increasing column ids");
  std::vector<double> zero(s->Dt, 0.0), one(s->Dt, 1.0);
  if (int rc = scratch_set(s, zero.data(), zero.data(), one.data())) return rc;
  int launches = 0;
  CK(newton_begin(B->d, 1, 1e-8, 1, 1, 1, 0, s->stream, &launches));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  // warm-up launch (also produces the scaled copy the Gram needs)
  CK(batch_k1(*B, 1, s->stream, &launches));
  if (which == 3) {
    CK(batch_gram(*B, B->d, 1, 1, s->stream, &launches));
    Ctrl c; std::memset(&c, 0, sizeof(c)); c.need_hess = 1;
    CK(cudaMemcpyAsync(B->d_ctrl, &c, sizeof(Ctrl), cudaMemcpyHostToDevice, s->stream));
  }
  const int off = 0;
  if (which == 4)   // Hv pass at beta = 0 (d from the warm-up pass) of v = 1
    if (int rc = load_hv(*B, 0, one.data(), s->stream)) return rc;
  CK(cudaStreamSynchronize(s->stream));
  CK(cudaEventRecord(e0, s->stream));
  for (int r = 0; r < reps; r++) {
    if (which == 1) CK(batch_k1(*B, emit_scaled ? 1 : 0, s->stream, &launches));
    else if (which == 2) CK(batch_gram(*B, B->d, 1, 1, s->stream, &launches));
    else if (which == 3) CK(cholesky_launch(B->d, 1, B->ldh, s->stream, &launches));
    else if (which == 4) { CK(batch_k1(*B, 0, s->stream, &launches, K1_HV)); CK(hv_reduce(B->d, 1, B->Dt, 0, s->stream, &launches)); }
    else return fail(MLEASE_ERR_INVALID, "which must be 1, 2, 3 or 4");
  }
  CK(cudaEventRecord(e1, s->stream));
  CK(cudaEventSynchronize(e1));
  if (which == 4) CK(cudaMemcpy(&B->d_ctrl->cg_active, &off, sizeof(int), cudaMemcpyHostToDevice));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  *avg_ms = ms / reps;
  s->cnt.launches += launches;
  return 0;
}

}  // extern "C"
