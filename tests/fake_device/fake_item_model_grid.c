/* TEST DOUBLE of mlease_score_keyed_var of libmlease_b200.so for the CPU tests of the ItemModelGridTest job
 * (tests/test_item_model_grid_cpu.py), linked together with fake_mlease_b200.c and fake_item_model.c.  Like them it COMPUTES
 * NOTHING: pred and pred_var are deterministic hashes of each key's own rows and of its model and variance list, so that the job's
 * orchestration and file output (layout, order, schema, sharding) can be checked without a GPU.  Never part of the product. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include "../../include/mlease_b200.h"

static double mix(double a, double b) { return fmod(a * 1.0000001 + b * 0.6180339887 + 0.1234567, 97.0); }

int mlease_score_keyed_var(int32_t device, void* stream, int32_t D, int32_t K, const int64_t* krs, const int64_t* rowptr, const int32_t* colidx,
                           const float* vals, const float* offset, int32_t G, const int64_t* mp, const int32_t* mc, const float* mv,
                           const int64_t* vp, const int32_t* vc, const float* vv, const float* vdef, int32_t binary, float* pred, float* pred_var) {
  (void)device; (void)stream; (void)binary;
  const int64_t n = krs[K];
  for (int g = 0; g < G; g++)
    for (int k = 0; k < K; k++) {
      const int64_t m = (int64_t)g * K + k;
      double s = 0, u = vdef[m];
      for (int64_t e = mp[m]; e < mp[m + 1]; e++) s = mix(s, mc[e] * 0.01 + mv[e] + (mc[e] == D));
      for (int64_t e = vp[m]; e < vp[m + 1]; e++) u = mix(u, vc[e] * 0.02 + vv[e]);
      for (int64_t i = krs[k]; i < krs[k + 1]; i++) {
        double t = s + (offset ? offset[i] : 0.0), w = u;
        for (int64_t j = rowptr[i]; j < rowptr[i + 1]; j++) { t += 0.001 * colidx[j] + 0.01 * vals[j]; w += 0.003 * colidx[j]; }
        pred[(size_t)g * n + i] = (float)t;
        pred_var[(size_t)g * n + i] = vp[m + 1] > vp[m] ? (float)w : NAN;
      }
    }
  return 0;
}
