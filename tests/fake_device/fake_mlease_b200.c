/* TEST DOUBLE of libmlease_b200.so for the CPU tests of the host job layer (tests/test_host_jobs_fake_device_cpu.py).
 * It COMPUTES NOTHING: every entry point the job layer calls returns canned numbers that are a deterministic function of what
 * was passed in (partition contents are folded into a checksum, so a job that uploads different rows gets different "models").
 * Its only purpose is to let RegressionAdmmTrain / RegressionTest / RegressionTestLoglik / RegressionNaiveTrain run end to end
 * without a GPU, so that their orchestration and file output can be compared between the plan-walker and the generic avro
 * paths and run under sanitizers.  It is not part of the product and is never linked into it: the product library refuses to
 * run without an sm_90 device (tests/test_abi.py). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/mlease_b200.h"

struct mlease_world {
  int P, D, L, iter, initialized;
  float lambdas[16];
  double* sum;   /* [P] checksum of the uploaded rows */
  double z0sum;
};
struct mlease_session { int unused; };

const char* mlease_last_error(void) { return "fake device"; }
int mlease_session_destroy(mlease_session* s) { (void)s; return 0; }

static double mix(double a, double b) { return fmod(a * 1.0000001 + b * 0.6180339887 + 0.1234567, 97.0); }

int mlease_world_create(const mlease_admm_config* cfg, const int32_t* devices, int32_t ndev, mlease_world** out) {
  (void)devices; (void)ndev;
  mlease_world* w = (mlease_world*)calloc(1, sizeof(*w));
  w->P = cfg->num_blocks; w->D = cfg->num_features; w->L = cfg->num_lambdas;
  for (int l = 0; l < w->L && l < 16; l++) w->lambdas[l] = cfg->lambdas[l];
  w->sum = (double*)calloc((size_t)w->P, sizeof(double));
  *out = w;
  return 0;
}
int mlease_world_destroy(mlease_world* w) { if (w) { free(w->sum); free(w); } return 0; }
int mlease_world_add_partition_csr(mlease_world* w, int32_t p, int64_t n, const int64_t* rowptr, const int32_t* colidx, const float* vals,
                                   const int32_t* response, const float* weight, const float* offset) {
  double s = 0;
  for (int64_t i = 0; i < n; i++) {
    s = mix(s, (double)response[i] + (weight ? weight[i] : 1.0) * 3.0 + (offset ? offset[i] : 0.0) * 7.0 + (double)(rowptr[i + 1] - rowptr[i]));
    for (int64_t j = rowptr[i]; j < rowptr[i + 1]; j++) s = mix(s, (double)colidx[j] * 0.01 + (double)vals[j]);
  }
  w->sum[p] = s;
  return 0;
}
int mlease_world_begin(mlease_world* w) { w->iter = 0; w->initialized = 0; return 0; }
int mlease_world_begin_initialized(mlease_world* w, const double* z0, float boost) {
  w->iter = 0; w->initialized = 1; w->z0sum = boost;
  for (int k = 0; k < w->L * (w->D + 1); k++) w->z0sum = mix(w->z0sum, z0[k]);
  return 0;
}
int mlease_world_iterate(mlease_world* w, double* maxdiff, int32_t* stop) {
  w->iter++;
  *maxdiff = 1.0 / w->iter;
  *stop = w->iter >= 6;
  return 0;
}
static double coef(const mlease_world* w, int p, int l, int k, int what) {
  return sin(w->sum[p < 0 ? 0 : p] + 0.37 * l + 0.011 * k + 1.7 * w->iter + what + (w->initialized ? w->z0sum : 0.0)) * (1.0 + w->lambdas[l]);
}
int mlease_world_get_z(mlease_world* w, int32_t l, double* out) {
  for (int k = 0; k <= w->D; k++) { double s = 0; for (int p = 0; p < w->P; p++) s += coef(w, p, l, k, 0); out[k] = s / w->P; }
  return 0;
}
int mlease_world_get_x(mlease_world* w, int32_t p, int32_t l, double* out) { for (int k = 0; k <= w->D; k++) out[k] = coef(w, p, l, k, 1); return 0; }
int mlease_world_get_u(mlease_world* w, int32_t p, int32_t l, float* out) { for (int k = 0; k <= w->D; k++) out[k] = (float)coef(w, p, l, k, 2); return 0; }
int mlease_world_get_uplusx(mlease_world* w, int32_t p, int32_t l, float* out) { for (int k = 0; k <= w->D; k++) out[k] = (float)coef(w, p, l, k, 3); return 0; }
int mlease_world_fit_partition(mlease_world* w, int32_t p, double* x, const double* m, const double* q, int32_t* steps) {
  for (int k = 0; k <= w->D; k++) x[k] = sin(w->sum[p] + 0.02 * k + q[k]) + m[k];
  if (steps) *steps = 3;
  return 0;
}
int mlease_score(int32_t device, void* stream, int32_t D, int64_t n, const int64_t* rowptr, const int32_t* colidx, const float* vals, int64_t ldx,
                 const float* offset, const double* model, int32_t reps, int32_t binary, float* pred) {
  (void)device; (void)stream; (void)ldx; (void)reps; (void)binary;
  for (int64_t i = 0; i < n; i++) {
    double s = model[D] + (offset ? offset[i] : 0.0);
    for (int64_t j = rowptr[i]; j < rowptr[i + 1]; j++) s += 0.001 * colidx[j] + 0.01 * vals[j] * model[colidx[j]];
    pred[i] = (float)s;
  }
  return 0;
}
int mlease_test_loglik(int32_t device, void* stream, int64_t n, const int32_t* response, const float* pred, const float* weight, int64_t block,
                       float* ll, double* cnt) {
  (void)device; (void)stream; (void)block;
  double s = 0, c = 0;
  for (int64_t i = 0; i < n; i++) { s += (response[i] == 1 ? 1.0 : -1.0) * pred[i] * weight[i]; c += weight[i]; }
  *ll = (float)(s / c); *cnt = c;
  return 0;
}
int mlease_naive_train(int32_t device, void* stream, int32_t K, int32_t D, const int64_t* krs, const int64_t* rowptr, const int32_t* colidx, const float* vals,
                       int64_t ldx, const int32_t* response, const float* weight, const float* offset, int32_t L, const float* lambdas, const float* lambda_map,
                       float prior_mean, int32_t pen, int32_t has_icpt, int32_t threshold, int32_t binary, double* out, int32_t* skipped) {
  (void)device; (void)stream; (void)ldx; (void)weight; (void)offset; (void)pen; (void)has_icpt; (void)binary;
  for (int k = 0; k < K; k++) {
    double s = 0;
    for (int64_t i = krs[k]; i < krs[k + 1]; i++) { s = mix(s, response[i]); for (int64_t j = rowptr[i]; j < rowptr[i + 1]; j++) s = mix(s, colidx[j] * 0.01 + vals[j]); }
    skipped[k] = (krs[k + 1] - krs[k]) < threshold;
    for (int l = 0; l < L; l++)
      for (int j = 0; j <= D; j++)
        out[((size_t)l * K + k) * (D + 1) + j] = sin(s + 0.3 * l + 0.05 * j) / (1.0 + lambdas[l]) + prior_mean + (lambda_map && j < D ? lambda_map[j] : 0.0);
  }
  return 0;
}
