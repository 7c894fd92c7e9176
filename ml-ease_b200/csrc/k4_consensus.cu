// k4_consensus.cu -- K4: the consensus step of one ADMM iteration, fused around the single all-reduce.
//
//   admm_pack      (before the all-reduce)  per local problem: x_f = float(x), uplusx_f = float(u + x)
//                  (jobs/RegressionAdmmTrain.java:706-711, models/LinearModel.java:703,716) and the local
//                  exchange vector  S_local[l][k] = sum_p float(x_p)[k] + u_p[k]  in double.
//   admm_consensus (after the all-reduce)   z = wz * S / P   (L2, :362-404; L1: thresholded mean, :406-451; wz = P rho/(lambda+P rho) computed on
//                  the host in the reference's float arithmetic :381, 1 for the unpenalised intercept :392-403,
//                  per-feature lambda.map weights :382-386), |z - z_prev|_inf (:456-472), and the NEXT
//                  iteration's reducer inputs: u = float(uplusx - z) (computeU :736-765), z as float (:330-331),
//                  prior mean m = z_f - u (:695-698), prior precision rho_eff (:652-658,705); the warm start is the previous x_p
//                  (the reference's init = z_f, :692-693, only seeds TRON; the minimiser is the same).
//
// Latency-bound, O(P_local * L * D') work: one CTA per lambda.
#include "kernels.cuh"

namespace mlease {

__global__ void admm_reset_kernel(const Problem* __restrict__ probs, int L, double* __restrict__ z, int ldv,
                                  const double* __restrict__ rho_eff) {
  const Problem& pb = probs[blockIdx.x];
  const int l = pb.lambda_idx;
  for (int k = threadIdx.x; k < ldv; k += blockDim.x) {
    pb.u_f[k] = 0.f; pb.uplusx_f[k] = 0.f; pb.x_f[k] = 0.f; pb.x_d[k] = 0.0;
    pb.m[k] = 0.0;                       // z - u with both maps empty (:155-185, :312)
    pb.beta[k] = 0.0;                    // init = z = {}
    pb.q[k] = k < pb.Dt ? rho_eff[l] : 1.0;
    if (pb.part_local == 0) z[(size_t)l * ldv + k] = 0.0;
  }
  if (threadIdx.x == 0) { pb.ctrl->hess_valid = 0; pb.ctrl->skip_eval = 0; }
}

// Start from a given z (initialize.boost.rate): the reducers read z as float from the init-value file
// (jobs/RegressionAdmmTrain.java:330-331, models/LinearModel.java:716); u is the empty map, so priorMean = z - u = float(z).
__global__ void admm_init_kernel(const Problem* __restrict__ probs, const double* __restrict__ z, int ldv) {
  const Problem& pb = probs[blockIdx.x];
  const int l = pb.lambda_idx;
  for (int k = threadIdx.x; k < pb.Dt; k += blockDim.x) {
    const double zf = (double)(float)z[(size_t)l * ldv + k];
    pb.m[k] = zf;
    pb.beta[k] = zf;   // init = z (:692-693)
  }
}

__global__ void admm_pack_kernel(const Problem* __restrict__ probs, int nparts, int L, int Dt, double* __restrict__ exch) {
  const int l = blockIdx.y;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= Dt) return;
  double s = 0.0;
  for (int p = 0; p < nparts; p++) {
    const Problem& pb = probs[p * L + l];
    const double x = pb.beta[k];
    const float xf = (float)x;
    const float uf = pb.u_f[k];
    pb.x_f[k] = xf;
    pb.x_d[k] = x;
    pb.uplusx_f[k] = (float)(1.0 * (double)uf + 1.0 * x);
    s += (double)xf + (double)uf;
  }
  exch[(size_t)l * Dt + k] = s;
}

__global__ void __launch_bounds__(256) admm_consensus_kernel(const Problem* __restrict__ probs, int nparts, int L, int Dt, int ldv,
                                                             int P, const double* __restrict__ exch, double* __restrict__ z,
                                                             const double* __restrict__ wz, const double* __restrict__ rho_next,
                                                             double* __restrict__ diff, const double* __restrict__ l1_thr) {
  const int l = blockIdx.y;
  __shared__ double sc[8];
  double dmax = 0.0;
  const double invP = 1.0 / (double)P;
  // regularizer = 1 (l1_thr != NULL): z = xbar + ubar, then the reference's "iterative thresholding" of the coefficients
  // (jobs/RegressionAdmmTrain.java:406-437): val > t -> val - t, val < -t -> val + t, values inside [-t, t] stay as they are
  // (the reference does not zero them); the intercept (not in getCoefficients()) is the plain mean (:438-449).  Column Dt - 1 IS
  // the intercept in every batch this kernel sees: a session's batches are built with has_bias = 1 and Dt = num_features + 1
  // (session.cu), there is no ADMM session without an intercept column, so k == Dt - 1 needs no flag.
  const double thr = l1_thr ? l1_thr[l] : 0.0;
  for (int k = blockIdx.x * 256 + threadIdx.x; k < Dt; k += gridDim.x * 256) {   // one element per thread: the grid covers Dt
    double zn;
    if (l1_thr) {
      zn = exch[(size_t)l * Dt + k] * invP;
      if (k < Dt - 1) {
        if (zn > thr) zn -= thr;
        else if (zn < -thr) zn += thr;
      }
    } else {
      zn = wz[(size_t)l * ldv + k] * (exch[(size_t)l * Dt + k] * invP);
    }
    const double zo = z[(size_t)l * ldv + k];
    const double dk = fabs(zo - zn);
    dmax = fmax(dmax, dk);
    // LinearModel.maxAbsValue (models/LinearModel.java:728-740) starts from |intercept diff| and skips a NaN coefficient diff
    // (`maxabs < v` is false), as fmax does; a NaN at the intercept is the lambda's diff whatever follows.  fabs leaves a positive
    // NaN, whose bit pattern orders above every other non-negative double in the atomicMax below.
    if (k == Dt - 1 && dk != dk) atomicMax(reinterpret_cast<unsigned long long*>(diff + l), (unsigned long long)__double_as_longlong(dk));
    z[(size_t)l * ldv + k] = zn;
    const float zf = (float)zn;
    for (int p = 0; p < nparts; p++) {
      const Problem& pb = probs[p * L + l];
      const float un = (float)((double)pb.uplusx_f[k] - zn);
      pb.u_f[k] = un;
      // Gradient at the warm start without a pass over the rows.  x_p minimised  data(x) + q/2 |x - m_old|^2  up to the solver's
      // tolerance, so the data-term gradient there is  -q_old (x_p - m_old)  (to first order in the last, unevaluated Newton
      // correction); the next x-update starts AT x_p with a new prior, and its first direction can be taken from this estimate.
      // Every later point -- including the one the stop test is taken at -- is evaluated exactly by K1 (newton_solve_kernel
      // does not let an x-update end before its first exact evaluation), so the fixed point is untouched; what is saved is the
      // start-point pass of every warm x-update, about a third of all passes.  Only where the fused CSR K1 runs (gpart_f).
      if (pb.gpart_f) pb.g_t[k] = -pb.q[k] * (pb.x_d[k] - pb.m[k]);
      pb.m[k] = -1.0 * (double)un + 1.0 * (double)zf;
      // Warm start of the next x-update.  The reference starts TRON at z (:692-693) because its reducers are stateless;
      // the minimiser does not depend on the start, and with the state resident the previous x_p is far closer to it:
      // the optimality conditions of two consecutive x-updates give H (x_new - x_old) = -rho ((x_old - z) - (z - z_prev)),
      // i.e. a move of order (rho / lambda_min(H)) * primal residual, while |z - x_new| is of the order of the residual itself.
      pb.beta[k] = pb.x_d[k];
      pb.q[k] = rho_next[l];
    }
  }
  if (threadIdx.x == 0 && blockIdx.x == 0)
    for (int p = 0; p < nparts; p++) {
      const Problem& pb = probs[p * L + l];
      if (pb.gpart_f) { pb.ctrl->skip_eval = 1; pb.ctrl->k1_chunks = 0; }
    }
  dmax = warp_max(dmax);
  if ((threadIdx.x & 31) == 0) sc[threadIdx.x >> 5] = dmax;
  __syncthreads();
  if (threadIdx.x == 0) {
    double d = 0.0;
    for (int w = 0; w < 8; w++) d = fmax(d, sc[w]);
    // max over the CTAs of this lambda: non-negative doubles order like their bit patterns (diff[] is zeroed before the launch)
    atomicMax(reinterpret_cast<unsigned long long*>(diff + l), (unsigned long long)__double_as_longlong(d));
  }
}

cudaError_t admm_reset(const Problem* d_probs, int nprob, int L, double* d_z, int ldv, const double* d_rho_eff, cudaStream_t st,
                       int* launches) {
  admm_reset_kernel<<<nprob, 256, 0, st>>>(d_probs, L, d_z, ldv, d_rho_eff);
  if (launches) *launches += 1;
  return cudaGetLastError();
}
cudaError_t admm_init(const Problem* d_probs, int nprob, const double* d_z, int ldv, cudaStream_t st, int* launches) {
  admm_init_kernel<<<nprob, 256, 0, st>>>(d_probs, d_z, ldv);
  if (launches) *launches += 1;
  return cudaGetLastError();
}
cudaError_t admm_pack(const Problem* d_probs, int nlocal_parts, int L, int Dt, double* d_exchange, cudaStream_t st, int* launches) {
  admm_pack_kernel<<<dim3((Dt + 255) / 256, L), 256, 0, st>>>(d_probs, nlocal_parts, L, Dt, d_exchange);
  if (launches) *launches += 1;
  return cudaGetLastError();
}
cudaError_t admm_consensus(const Problem* d_probs, int nlocal_parts, int L, int Dt, int ldv, int P, const double* d_exchange_sum,
                           double* d_z, const double* d_wz, const double* d_rho_eff_next, double* d_diff, cudaStream_t st,
                           int* launches, const double* d_l1_thr) {
  cudaError_t e = cudaMemsetAsync(d_diff, 0, (size_t)L * sizeof(double), st);
  if (e != cudaSuccess) return e;
  admm_consensus_kernel<<<dim3((Dt + 255) / 256, L), 256, 0, st>>>(d_probs, nlocal_parts, L, Dt, ldv, P, d_exchange_sum, d_z, d_wz, d_rho_eff_next, d_diff,
                                                                  d_l1_thr);
  if (launches) *launches += 1;
  return cudaGetLastError();
}

}  // namespace mlease
