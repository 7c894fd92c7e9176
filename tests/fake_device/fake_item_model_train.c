/* TEST DOUBLE of mlease_item_model_train for the CPU tests of the ItemModelTrain job (tests/test_item_model_train_cpu.py), linked
 * together with fake_mlease_b200.c.  It COMPUTES NOTHING: the numbers are canned so that the job's orchestration and file output can
 * be checked without a GPU.  Never part of the product.
 *   model[a][b][k][j] = 10 a + b + 0.001 j (j < num_features); the intercept = intercept_prior_mean[k]
 *   var[a][b][k][j]   = 1 / (1 + j + a + b); the intercept = 1e9 * (mean - (double)(float)mean), which shows whether the job passed
 *                       a double or a float-rounded mean */
#include <stdint.h>

#include "../../include/mlease_b200.h"

int mlease_item_model_train(int32_t device, void* stream, int32_t K, int32_t D, const int64_t* krs, const int64_t* rowptr, const int32_t* colidx,
                            const float* vals, const int32_t* response, const float* weight, const float* offset, const double* mean, int32_t IL,
                            const float* il, int32_t DL, const float* dl, const float* lambda_map, int32_t binary, int32_t compute_var,
                            double* out_model, double* out_var) {
  (void)device; (void)stream; (void)krs; (void)rowptr; (void)colidx; (void)vals; (void)response; (void)weight; (void)offset; (void)il; (void)dl;
  (void)lambda_map; (void)binary;
  for (int a = 0; a < IL; a++)
    for (int b = 0; b < DL; b++)
      for (int k = 0; k < K; k++) {
        const size_t base = (((size_t)a * DL + b) * K + k) * (size_t)(D + 1);
        for (int j = 0; j < D; j++) {
          out_model[base + j] = 10.0 * a + b + 0.001 * j;
          if (compute_var) out_var[base + j] = 1.0 / (1.0 + j + a + b);
        }
        out_model[base + D] = mean[k];
        if (compute_var) out_var[base + D] = 1e9 * (mean[k] - (double)(float)mean[k]);
      }
  return 0;
}
