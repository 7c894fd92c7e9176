/* TEST DOUBLE of the keyed entry points of libmlease_b200.so (mlease_score_keyed, mlease_test_loglik_keyed) for the CPU tests of the
 * ItemModelTest / ItemModelTestLoglik jobs (tests/test_item_model_cpu.py), linked together with fake_mlease_b200.c.  Like that file
 * it COMPUTES NOTHING: the numbers are a deterministic function of the inputs, so that the jobs' orchestration and file output can
 * be checked without a GPU.  Never part of the product. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include "../../include/mlease_b200.h"

static double mix(double a, double b) { return fmod(a * 1.0000001 + b * 0.6180339887 + 0.1234567, 97.0); }

int mlease_score_keyed(int32_t device, void* stream, int32_t D, int32_t K, const int64_t* krs, const int64_t* rowptr, const int32_t* colidx,
                       const float* vals, const float* offset, int32_t L, const int64_t* mp, const int32_t* mc, const float* mv, int32_t binary, float* pred) {
  (void)device; (void)stream; (void)binary;
  const int64_t n = krs[K];
  for (int l = 0; l < L; l++)
    for (int k = 0; k < K; k++) {
      const int64_t m = (int64_t)l * K + k;
      double s = 0;
      for (int64_t e = mp[m]; e < mp[m + 1]; e++) s = mix(s, mc[e] * 0.01 + mv[e] + (mc[e] == D));
      for (int64_t i = krs[k]; i < krs[k + 1]; i++) {
        double t = s + (offset ? offset[i] : 0.0);
        for (int64_t j = rowptr[i]; j < rowptr[i + 1]; j++) t += 0.001 * colidx[j] + 0.01 * vals[j];
        pred[(size_t)l * n + i] = (float)t;
      }
    }
  return 0;
}

int mlease_test_loglik_keyed(int32_t device, void* stream, int64_t n, const int32_t* key, const int32_t* group, const int32_t* response,
                             const float* weight, const float* pred, int32_t K, float* ll, double* cnt) {
  (void)device; (void)stream;
  for (int k = 0; k < K; k++) { ll[k] = 0; cnt[k] = 0; }
  for (int64_t e = 0; e < n; e++) {
    const double w = weight ? weight[e] : 1.0;
    ll[key[e]] += (float)((response[e] == 1 ? 1.0 : -1.0) * pred[e] * w + 0.5 * group[e]);
    cnt[key[e]] += w;
  }
  return 0;
}
