// keyed_fit.cu -- K independent fits per prior over one upload of the rows: RegressionNaiveTrain (mlease_naive_train,
// mlease_naive_train_dense) and ItemModelTrain (mlease_item_model_train).
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
__global__ void gather_i64_kernel(const long long* src, const long long* idx, int n, long long* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = src[idx[i]];
}
// One prior of a keyed fit: precision q and mean m of every coefficient ([ldx], the intercept at Dg, 1 / 0 on the padding)
struct KeyedPrior { std::vector<double> q, m; };

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
// callers run keyed_fit_check first
int keyed_fit(int num_sms, cudaStream_t st, int32_t K, int32_t Dg, const int64_t* key_rowstart, const int64_t* rowptr, const int32_t* colidx,
              const float* vals, int64_t ldx_in, const int32_t* response, const float* weight, const float* offset, bool has_intercept,
              int32_t data_size_threshold, int32_t binary_feature, const std::vector<KeyedPrior>& priors, const double* intercept_mean,
              double* out_model, double* out_var, int32_t* skipped) {
  const bool csr = rowptr != nullptr;
  const int L = (int)priors.size();
  const int Dt = Dg + 1, ldx = round_up(Dt, 4);
  std::vector<long long> krs(K + 1);
  CK(cudaMemcpy(krs.data(), key_rowstart, (size_t)(K + 1) * 8, cudaMemcpyDefault));
  const long long ntot = krs[K];
  for (int k = 0; k < K; k++) if (krs[k + 1] < krs[k]) return fail(MLEASE_ERR_INVALID, "key_rowstart must be non-decreasing");
  DevMem t;
  PinnedMem pinned;
  float* dX = nullptr; signed char* dy; float *dw, *dofs; int* dflag; int* hflag;
  const long long* d_rp = nullptr; const int* d_ci = nullptr; float* d_v = nullptr;
  std::vector<long long> key_nnz0(K + 1, 0);   // CSR: rowptr at the key boundaries
  int csr_unique = 0;
  if (int rc = t.get(&dy, (size_t)ntot, false)) return rc;
  if (int rc = t.get(&dw, (size_t)ntot, false)) return rc;
  if (int rc = t.get(&dofs, (size_t)ntot, false)) return rc;
  if (int rc = t.get(&dflag, 16, false)) return rc;
  if (int rc = pinned.get(&hflag, 16, false)) return rc;
  if (!csr) {
    if (int rc = t.get(&dX, (size_t)ntot * ldx, false)) return rc;
    if (int rc = upload_dense_rows(dX, ldx, vals, ldx_in, ntot, Dg, has_intercept ? 1 : 0, st)) return rc;
  } else {
    if (int rc = to_device(t, (const long long*)rowptr, (size_t)ntot + 1, &d_rp, st)) return rc;
    long long nnz = 0, first = 0;
    CK(cudaMemcpyAsync(&nnz, d_rp + ntot, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&first, d_rp, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (first != 0) return fail(MLEASE_ERR_INVALID, "rowptr[0] must be 0");
    if (int rc = to_device(t, colidx, (size_t)nnz, &d_ci, st)) return rc;
    // values are copied even when they already live on the device: binary.feature rewrites them
    if (int rc = t.get(&d_v, (size_t)nnz, false)) return rc;
    CK(cudaMemcpyAsync(d_v, vals, (size_t)nnz * 4, cudaMemcpyDefault, st));
    CK(cudaMemsetAsync(dflag, 0, 8, st));
    check_csr(st, ntot, nnz, d_rp, d_ci, d_v, Dg, binary_feature, dflag);
    CK(cudaMemcpyAsync(hflag, dflag, 8, cudaMemcpyDeviceToHost, st));
    // rowptr at the key boundaries (nnz per key for the cost model and the byte accounting)
    long long* d_kn; long long* d_krs;
    if (int rc = t.get(&d_kn, (size_t)K + 1, false)) return rc;
    if (int rc = t.get(&d_krs, (size_t)K + 1, false)) return rc;
    CK(cudaMemcpyAsync(d_krs, krs.data(), (size_t)(K + 1) * 8, cudaMemcpyHostToDevice, st));
    gather_i64_kernel<<<(K + 256) / 256, 256, 0, st>>>(d_rp, d_krs, K + 1, d_kn);
    CK(cudaMemcpyAsync(key_nnz0.data(), d_kn, (size_t)(K + 1) * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (hflag[0]) return fail(MLEASE_ERR_INVALID, "feature index out of range");
    csr_unique = hflag[1] ? 0 : 1;
  }
  if (int rc = ingest_labels(st, ntot, response, weight, offset, dy, dw, dofs, dflag, hflag, nullptr)) return rc;
  for (size_t e = 0; e < (size_t)L * K * Dt; e++) out_model[e] = 0.0;
  std::vector<int> todo;
  for (int k = 0; k < K; k++) {
    const long long nk = krs[k + 1] - krs[k];
    if (skipped) skipped[k] = 0;
    if (nk < data_size_threshold || nk <= 0) { if (skipped) skipped[k] = 1; }   // "data size < threshold": no model (:379-382)
    else todo.push_back(k);
  }
  if (out_var)   // a key without rows has no fit: every variance is the prior's
    for (int l = 0; l < L; l++)
      for (int k = 0; k < K; k++)
        for (int j = 0; j < Dt; j++) out_var[((size_t)l * K + k) * Dt + j] = 1.0 / priors[l].q[j];
  // chunk size bounded by memory: Xt (n*Dp*2) + Hpart + Lc per problem (+ the row weights of the variance)
  const int Dp = round_up(ldx, 128), ldh = round_up(Dt, 32);
  size_t free_b, total_b;
  CK(cudaMemGetInfo(&free_b, &total_b));
  Counters cnt;
  size_t pos = 0;
  while (pos < todo.size()) {
    size_t bytes = 0;
    size_t end = pos;
    while (end < todo.size() && end - pos < 16384) {
      const long long nk = krs[todo[end] + 1] - krs[todo[end]];
      const size_t need = (size_t)nk * Dp * 2 + (size_t)Dp * Dp * 4 + 3 * (size_t)ldh * ldh * 8 + 2 * (size_t)ldh * 32 * 8 + 64 * (size_t)ldx +
                          (out_var ? (size_t)nk * 8 : 0);
      if (end > pos && bytes + need > free_b / 2) break;
      bytes += need;
      end++;
    }
    Batch B;
    B.nprob = (int)(end - pos); B.Dt = Dt; B.ldx = ldx; B.csr = csr; B.has_bias = has_intercept ? 1 : 0;
    B.h.resize(B.nprob);
    std::vector<long long> row_start(B.nprob + 1, 0);   // the chunk's rows numbered across its problems (batched variance)
    for (int b = 0; b < B.nprob; b++) {
      const int k = todo[pos + b];
      Problem& p = B.h[b];
      std::memset(&p, 0, sizeof(Problem));
      p.n = krs[k + 1] - krs[k];
      p.y = dy + krs[k]; p.w = dw + krs[k]; p.o = dofs + krs[k];
      if (csr) {
        // a key = a row range of the one CSR: the row pointers keep their absolute offsets into colidx / vals
        p.rowptr = d_rp + krs[k]; p.colidx = d_ci; p.vals = d_v; p.nnz_hint = key_nnz0[k + 1] - key_nnz0[k]; p.csr_unique = csr_unique;
      } else {
        p.X = dX + (size_t)krs[k] * ldx;
      }
      row_start[b + 1] = row_start[b] + p.n;
    }
    if (int rc = batch_alloc(B, num_sms, 0)) return rc;
    DevMem ct;   // the chunk's temporaries: freed with the chunk, before the next chunk's batch_alloc
    double *dm, *dq, *dout, *dim = nullptr, *dvec = nullptr; long long* drs = nullptr; unsigned char* dmask = nullptr;
    if (int rc = ct.get(&dm, (size_t)ldx, false)) return rc;
    if (int rc = ct.get(&dq, (size_t)ldx, false)) return rc;
    if (int rc = ct.get(&dout, (size_t)B.nprob * Dt, false)) return rc;
    if (intercept_mean) {
      std::vector<double> im(B.nprob);
      for (int b = 0; b < B.nprob; b++) im[b] = intercept_mean[todo[pos + b]];
      if (int rc = ct.get(&dim, (size_t)B.nprob, false)) return rc;
      CK(cudaMemcpyAsync(dim, im.data(), im.size() * 8, cudaMemcpyHostToDevice, st));
      CK(cudaStreamSynchronize(st));   // im is released here
    }
    if (out_var) {
      if (int rc = ct.get(&dvec, (size_t)row_start[B.nprob], false)) return rc;
      if (int rc = ct.get(&drs, row_start.size(), false)) return rc;
      CK(cudaMemcpyAsync(drs, row_start.data(), row_start.size() * 8, cudaMemcpyHostToDevice, st));
    }
    if (csr) {
      // features absent from a key's rows are not part of its dataset, hence not of its model (llf/LibLinear.java:343-350; the only
      // prior mean a caller may set per key is the intercept's, which every dataset holds, so :374-383 adds nothing): mask them out
      if (int rc = ct.get(&dmask, (size_t)B.nprob * Dt, false)) return rc;
      CK(cudaMemsetAsync(dmask, 0, (size_t)B.nprob * Dt, st));
      naive_present_kernel<<<B.nprob, 256, 0, st>>>(B.d, Dt, has_intercept ? 1 : 0, dmask);
    }
    std::vector<double> xs((size_t)B.nprob * Dt);
    for (int l = 0; l < L; l++) {
      CK(cudaMemcpyAsync(dm, priors[l].m.data(), ldx * 8, cudaMemcpyHostToDevice, st));
      CK(cudaMemcpyAsync(dq, priors[l].q.data(), ldx * 8, cudaMemcpyHostToDevice, st));
      CK(cudaStreamSynchronize(st));   // dq / dm are reused by the next prior
      naive_init_kernel<<<B.nprob, 128, 0, st>>>(B.d, dm, dq, dim);
      B.mirror.clear();                // the factors of the previous prior belong to another prior
      if (int rc = batch_xupdate(B, st, 2e-7, 100, 0, 1, hflag, dflag, cnt)) return rc;
      gather_beta_kernel<<<B.nprob, 128, 0, st>>>(B.d, Dt, dout, dmask, 0);
      CK(cudaMemcpyAsync(xs.data(), dout, xs.size() * 8, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      for (int b = 0; b < B.nprob; b++) {
        double* dst = out_model + ((size_t)l * K + todo[pos + b]) * Dt;
        std::memcpy(dst, xs.data() + (size_t)b * Dt, Dt * 8);
        if (!has_intercept) dst[Dg] = 0.0;
      }
      if (out_var) {
        // posteriorVar, diagonal (llf/LibLinear.java:328-333): one pass over the chunk's rows for all of its keys
        CK(postvar_rowweights(B.d, B.nprob, drs, row_start[B.nprob], B.has_bias, dvec, st, nullptr));
        CK(postvar_diag(B.d, B.nprob, drs, row_start[B.nprob], dvec, B.has_bias, st, nullptr));
        gather_beta_kernel<<<B.nprob, 128, 0, st>>>(B.d, Dt, dout, nullptr, 1);
        CK(cudaMemcpyAsync(xs.data(), dout, xs.size() * 8, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        for (int b = 0; b < B.nprob; b++) {
          double* dst = out_var + ((size_t)l * K + todo[pos + b]) * Dt;
          for (int j = 0; j < Dt; j++) dst[j] = 1.0 / xs[(size_t)b * Dt + j];
        }
      }
    }
    pos = end;
  }
  if (cnt.not_converged) return fail(MLEASE_ERR_NUMERIC, "Model fitting error! (" + std::to_string(cnt.not_converged) + " fits did not converge)");
  return 0;
}
// host copy of a host-or-device array (NULL -> empty)
template <class T> int host_copy(const T* in, size_t count, std::vector<T>& out) {
  out.clear();
  if (!in) return 0;
  out.resize(count);
  CK(cudaMemcpy(out.data(), in, count * sizeof(T), cudaMemcpyDefault));
  return 0;
}
}  // namespace

extern "C" {

// ------------------------------------------------------------------------------------------
// RegressionNaiveTrain: K independent fits per lambda (keyed_fit)
// ------------------------------------------------------------------------------------------
int mlease_naive_train(int32_t device, void* stream, int32_t K, int32_t Dg, const int64_t* key_rowstart, const int64_t* rowptr,
                       const int32_t* colidx, const float* vals, int64_t ldx_in, const int32_t* response, const float* weight,
                       const float* offset, int32_t L, const float* lambdas, const float* lambda_map, float prior_mean,
                       int32_t penalize_intercept, int32_t has_intercept, int32_t data_size_threshold, int32_t binary_feature,
                       double* out_model, int32_t* skipped) {
  if (K <= 0 || Dg <= 0 || L <= 0 || !lambdas || !key_rowstart || !vals || !response || !out_model) return fail(MLEASE_ERR_INVALID, "bad argument");
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
                   data_size_threshold, binary_feature, priors, nullptr, out_model, nullptr, skipped);
}

// ------------------------------------------------------------------------------------------
// ItemModelTrain (jobs/ItemModelTrain.java:226-276): per key, one fit per (intercept lambda, default lambda) in config order, the
// intercept's prior mean the key's own; diagonal posterior variance on request
// ------------------------------------------------------------------------------------------
int mlease_item_model_train(int32_t device, void* stream, int32_t K, int32_t Dg, const int64_t* key_rowstart, const int64_t* rowptr,
                            const int32_t* colidx, const float* vals, const int32_t* response, const float* weight, const float* offset,
                            const double* intercept_prior_mean, int32_t IL, const float* intercept_lambdas, int32_t DL,
                            const float* default_lambdas, const float* lambda_map, int32_t binary_feature, int32_t compute_var,
                            double* out_model, double* out_var) {
  if (K <= 0 || Dg <= 0 || IL <= 0 || DL <= 0 || !intercept_lambdas || !default_lambdas || !key_rowstart || !rowptr || !vals || !response ||
      !intercept_prior_mean || !out_model || (compute_var && !out_var))
    return fail(MLEASE_ERR_INVALID, "bad argument");
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
                   priors, im.data(), out_model, compute_var ? out_var : nullptr, nullptr);
}

int mlease_naive_train_dense(int32_t device, void* stream, int32_t K, int32_t Dg, const int64_t* key_rowstart, const float* X, int64_t ldx_in,
                             const int32_t* response, const float* weight, const float* offset, float lambda, const float* lambda_map,
                             float prior_mean, int32_t penalize_intercept, int32_t has_intercept, int32_t data_size_threshold,
                             double* out_model, int32_t* skipped) {
  return mlease_naive_train(device, stream, K, Dg, key_rowstart, nullptr, nullptr, X, ldx_in, response, weight, offset, 1, &lambda, lambda_map,
                            prior_mean, penalize_intercept, has_intercept, data_size_threshold, 0, out_model, skipped);
}

}  // extern "C"
