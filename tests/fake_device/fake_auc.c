/* TEST DOUBLE of mlease_test_auc for the CPU tests of the RegressionTestAuc / ItemModelGridTestAuc jobs (tests/test_auc_jobs_cpu.py),
 * linked together with fake_mlease_b200.c.  It COMPUTES NO AUC: a segment's "auc" is a hash of its own rows (position in the
 * segment, response, weight, pred), NaN where the segment has no positive or no negative weight as the real call gives; the
 * weights are the exact positive / negative sums in row order.  So the jobs' layout, order and keyAuc arithmetic can be checked
 * without a GPU.  Never part of the product. */
#include <math.h>
#include <stdint.h>

#include "../../include/mlease_b200.h"

static double mix(double a, double b) { return fmod(a * 1.0000001 + b * 0.6180339887 + 0.1234567, 97.0); }

/* hash of rows [a, b) of one set, and their positive / negative weight */
static double segment(int64_t a, int64_t b, const float* pred, const int32_t* response, const float* weight, double* pw, double* nw) {
  double h = 0.0, p = 0.0, n = 0.0;
  for (int64_t i = a; i < b; i++) {
    const double w = weight ? weight[i] : 1.0;
    h = mix(h, (double)(i - a) + 0.5 * response[i] + 0.25 * w + pred[i]);
    if (response[i] == 1) p += w; else n += w;
  }
  if (pw) *pw = p;
  if (nw) *nw = n;
  return p > 0.0 && n > 0.0 ? h / 97.0 : NAN;
}

int mlease_test_auc(int32_t device, void* stream, int64_t n, int32_t S, const float* pred, const int32_t* response, const float* weight,
                    int32_t K, const int64_t* krs, double* out_auc, double* out_weight, double* out_key_auc, double* out_key_weight) {
  (void)device; (void)stream;
  for (int32_t s = 0; s < S; s++) {
    const float* ps = pred + (size_t)s * n;
    if (out_auc) out_auc[s] = segment(0, n, ps, response, weight, s == 0 && out_weight ? &out_weight[0] : 0, s == 0 && out_weight ? &out_weight[1] : 0);
    for (int32_t k = 0; k < K; k++) {
      double pw, nw;
      const double h = segment(krs[k], krs[k + 1], ps, response, weight, &pw, &nw);
      if (out_key_auc) out_key_auc[(size_t)s * K + k] = h;
      if (s == 0 && out_key_weight) { out_key_weight[2 * k] = pw; out_key_weight[2 * k + 1] = nw; }
    }
  }
  return 0;
}
