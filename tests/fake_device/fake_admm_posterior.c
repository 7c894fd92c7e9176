/* TEST DOUBLE of mlease_world_admm_posterior for the CPU tests of the RegressionPosterior job (tests/test_regression_posterior_cpu.py),
 * linked together with fake_mlease_b200.c.  It COMPUTES NOTHING: the numbers are canned so that the job's orchestration and file
 * output can be checked without a GPU.  Never part of the product.
 *   var[k] = 1 / (1 + k + 10 l) + (full ? 1000 : 0) + z[k] / 1024, so the output shows which lambda, which mode and which z the job
 *   passed; mlease_world's leading fields are those of fake_mlease_b200.c's (P, D, L). */
#include <stdint.h>

#include "../../include/mlease_b200.h"

struct fake_world_head { int P, D, L; };

int mlease_world_admm_posterior(mlease_world* w, int32_t l, const double* z, int32_t full, double* var, double* cov) {
  const struct fake_world_head* h = (const struct fake_world_head*)w;
  (void)cov;
  for (int k = 0; k <= h->D; k++) var[k] = 1.0 / (1.0 + k + 10.0 * l) + (full ? 1000.0 : 0.0) + z[k] / 1024.0;
  return 0;
}
