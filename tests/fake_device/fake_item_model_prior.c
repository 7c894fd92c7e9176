/* TEST DOUBLE of mlease_item_model_train_prior for the CPU tests of ItemModelTrain with prior.model.path
 * (tests/test_item_model_prior_cpu.py), linked together with fake_mlease_b200.c and fake_item_model_train.c.  It COMPUTES NO FIT: it
 * builds each key's list as the library does (the distinct columns its rows list united with its prior-only columns, ascending, then
 * the intercept) and fills it with canned numbers that show which input each value came from:
 *   a column the rows list:  model 10 a + b + 0.001 j, var 1 / (1 + j + a + b); with a prior entry: model mean + 0.5, var the entry's
 *                            variance when > 0
 *   a prior-only column:     model = the entry's mean, var = its variance, or -1 where that is 0
 *   the intercept:           model = its entry's mean, else intercept_prior_mean[k]; var = its entry's variance, else 7 */
#include <stdint.h>
#include <stdlib.h>

#include "../../include/mlease_b200.h"

static int cmp_i32(const void* a, const void* b) { return *(const int32_t*)a < *(const int32_t*)b ? -1 : *(const int32_t*)a > *(const int32_t*)b; }

/* index of x in p[0 .. n) (ascending), or -1 */
static int64_t find(const int32_t* p, int64_t n, int32_t x) {
  for (int64_t i = 0; i < n; i++) if (p[i] == x) return i;
  return -1;
}

int mlease_item_model_train_prior(int32_t device, void* stream, int32_t K, int32_t D, const int64_t* krs, const int64_t* rowptr,
                                  const int32_t* colidx, const float* vals, const int32_t* response, const float* weight, const float* offset,
                                  const double* mean, int32_t IL, const float* il, int32_t DL, const float* dl, const float* lambda_map,
                                  int32_t binary, int32_t compute_var, int64_t capacity, int64_t* key_ptr, int32_t* out_col, double* out_model,
                                  double* out_var, const int64_t* pp, const int32_t* pc, const double* pm, const double* pv) {
  (void)device; (void)stream; (void)vals; (void)response; (void)weight; (void)offset; (void)il; (void)dl; (void)lambda_map; (void)binary;
  int64_t n = 0;
  key_ptr[0] = 0;
  for (int k = 0; k < K; k++) {
    const int64_t z0 = rowptr[krs[k]], z1 = rowptr[krs[k + 1]];
    int32_t* c = (int32_t*)malloc(sizeof(int32_t) * (size_t)(z1 - z0 + pp[k + 1] - pp[k] + 1));
    int64_t m = 0;
    for (int64_t z = z0; z < z1; z++) c[m++] = colidx[z];
    const int64_t listed = m;
    for (int64_t e = pp[k]; e < pp[k + 1]; e++)
      if (pc[e] != D && find(c, listed, pc[e]) < 0) c[m++] = pc[e];
    qsort(c, (size_t)m, sizeof(int32_t), cmp_i32);
    int64_t u = 0;
    for (int64_t i = 0; i < m; i++) if (u == 0 || c[i] != c[u - 1]) c[u++] = c[i];
    if (krs[k + 1] > krs[k]) c[u++] = D;
    else u = 0;
    if (n + u > capacity) { free(c); return MLEASE_ERR_INVALID; }
    for (int64_t i = 0; i < u; i++) {
      const int32_t j = c[i];
      const int64_t e = find(pc + pp[k], pp[k + 1] - pp[k], j);
      const int data = j == D || find(colidx + z0, z1 - z0, j) >= 0;
      out_col[n + i] = j;
      for (int a = 0; a < IL; a++)
        for (int b = 0; b < DL; b++) {
          const size_t at = (size_t)(a * DL + b) * (size_t)capacity + (size_t)(n + i);
          double mv, vv;
          if (j == D) { mv = e >= 0 ? pm[pp[k] + e] : mean[k]; vv = e >= 0 ? pv[pp[k] + e] : 7.0; }
          else if (!data) { mv = pm[pp[k] + e]; vv = pv[pp[k] + e] > 0 ? pv[pp[k] + e] : -1.0; }
          else if (e >= 0) { mv = pm[pp[k] + e] + 0.5; vv = pv[pp[k] + e] > 0 ? pv[pp[k] + e] : 1.0 / (1.0 + j + a + b); }
          else { mv = 10.0 * a + b + 0.001 * j; vv = 1.0 / (1.0 + j + a + b); }
          out_model[at] = mv;
          if (compute_var) out_var[at] = vv;
        }
    }
    n += u;
    key_ptr[k + 1] = n;
    free(c);
  }
  return 0;
}
