// test_hooks.cu -- the mlease_internal_* test hooks: not part of the C ABI (include/mlease_b200.h does not declare them), exported
// for the tests and tools that drive single kernels of a session's batches.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <mutex>
#include <vector>

#include "host.cuh"

using namespace mlease;

namespace {
std::atomic<unsigned long long> g_keyed_budget{0};
std::mutex g_keyed_mu;   // the keyed calls of several host threads (one device each) record here
std::vector<long long> g_keyed_bounds;
bool g_keyed_streamed = false;
double g_keyed_stage_ms = 0, g_keyed_wait_ms = 0;
}  // namespace

namespace mlease {
size_t keyed_budget(size_t free_b) {
  const unsigned long long cap = g_keyed_budget.load();
  return cap ? std::min<size_t>(free_b, (size_t)cap) : free_b;
}
void keyed_record(const std::vector<long long>& bounds, bool streamed, double stage_ms, double wait_ms) {
  std::lock_guard<std::mutex> g(g_keyed_mu);
  g_keyed_bounds = bounds;
  g_keyed_streamed = streamed;
  g_keyed_stage_ms = stage_ms;
  g_keyed_wait_ms = wait_ms;
}
}  // namespace mlease

extern "C" {

// Test hooks, not part of the C ABI: mlease_internal_set_keyed_budget caps, process-wide, the device bytes the keyed calls
// (mlease_naive_train*, mlease_item_model_train, mlease_score_keyed[_var]) plan with (0 = the free memory only), so that small inputs stream
// through many chunks.  mlease_internal_keyed_last_call reports the most recent keyed call of the process: the key boundaries of its
// chunks (*count of them, the first 0 and the last K; up to cap are written), whether it streamed, and for a streamed fit the host
// milliseconds its rows took to stage (copy into the pinned ring and H2D, all chunks) and the milliseconds the solve waited for them.
int mlease_internal_set_keyed_budget(int64_t bytes) {
  if (bytes < 0) return fail(MLEASE_ERR_INVALID, "bad argument");
  g_keyed_budget.store((unsigned long long)bytes);
  return 0;
}

int mlease_internal_keyed_last_call(int64_t* bounds, int32_t cap, int32_t* count, int32_t* streamed, double* stage_ms, double* wait_ms) {
  if (!count || cap < 0 || (cap > 0 && !bounds)) return fail(MLEASE_ERR_INVALID, "bad argument");
  std::lock_guard<std::mutex> g(g_keyed_mu);
  *count = (int32_t)g_keyed_bounds.size();
  for (size_t i = 0; i < g_keyed_bounds.size() && (int)i < cap; i++) bounds[i] = g_keyed_bounds[i];
  if (streamed) *streamed = g_keyed_streamed ? 1 : 0;
  if (stage_ms) *stage_ms = g_keyed_stage_ms;
  if (wait_ms) *wait_ms = g_keyed_wait_ms;
  return 0;
}

// Test hook, not part of the C ABI (include/mlease_b200.h does not declare it): one Hv (mode 1) or Hessian-diagonal (mode 2) pass
// over the session's ADMM batch -- every (partition, lambda) problem at its own point w[b] and vector v[b] (b = local partition * L
// + lambda, Dt entries each), through the kernels a matrix-free x-update runs (fused multi-lambda or per-problem).  out[b] = the data
// term X^T D X v resp. sum_i d_i x_ic^2, without the prior.  The batch's x-update state is consumed: begin() again before iterating.
int mlease_internal_batch_hv(mlease_session* s, int32_t mode, const double* w, const double* v, double* out) {
  if (!s || !w || !v || !out || (mode != K1_HV && mode != K1_DIAG)) return fail(MLEASE_ERR_INVALID, "bad argument");
  if (!s->batch) return fail(MLEASE_ERR_STATE, "mlease_admm_begin was not called");
  CK(cudaSetDevice(s->cfg.device));
  Batch& B = *s->batch;
  if (!(B.csr && B.csr_fx)) return fail(MLEASE_ERR_INVALID, "Hessian-vector passes need CSR rows with strictly increasing column ids");
  const int nprob = B.nprob, ldx = s->ldx, Dt = s->Dt;
  std::vector<Ctrl> c(nprob);
  auto set_ctrl = [&](int skip_clear, int active) -> int {
    CK(cudaMemcpy(c.data(), B.d_ctrl, (size_t)nprob * sizeof(Ctrl), cudaMemcpyDeviceToHost));
    for (auto& x : c) { if (skip_clear) x.skip_eval = 0; x.cg_active = active; if (active < 0) { x.cg_active = 0; x.done = 1; } }
    CK(cudaMemcpy(B.d_ctrl, c.data(), (size_t)nprob * sizeof(Ctrl), cudaMemcpyHostToDevice));
    return 0;
  };
  std::vector<double> wb(ldx, 0.0);
  for (int b = 0; b < nprob; b++) {
    std::memcpy(wb.data(), w + (size_t)b * Dt, (size_t)Dt * sizeof(double));
    CK(cudaMemcpy(B.h[b].beta, wb.data(), (size_t)ldx * sizeof(double), cudaMemcpyHostToDevice));
  }
  if (int rc = set_ctrl(1, 0)) return rc;
  int launches = 0;
  CK(newton_begin(B.d, nprob, 1e-8, 1, 2, 1, 0, s->stream, &launches));   // beta_t = float(w), every problem running
  CK(batch_k1(B, 1, s->stream, &launches));                               // sqrt(d) at w
  CK(cudaStreamSynchronize(s->stream));
  for (int b = 0; b < nprob; b++)
    if (int rc = load_hv(B, b, v + (size_t)b * Dt, s->stream)) return rc;
  CK(batch_k1(B, 0, s->stream, &launches, mode));
  CK(hv_reduce(B.d, nprob, Dt, 0, s->stream, &launches));
  CK(cudaStreamSynchronize(s->stream));
  for (int b = 0; b < nprob; b++) CK(cudaMemcpy(out + (size_t)b * Dt, B.h[b].g_t, (size_t)Dt * sizeof(double), cudaMemcpyDeviceToHost));
  if (int rc = set_ctrl(0, -1)) return rc;
  B.mirror.clear();
  s->cnt.launches += launches;
  return 0;
}

// Test hook, not part of the C ABI: one gradient pass over the session's ADMM batch (after begin()) through exactly the K1 kernels
// batch_k1 runs for it.  Problem b (= local partition * L + lambda) is evaluated at float(w[b]) (Dt entries) when active[b] != 0; the
// others are marked done before the launch, as problems that converged earlier are in an x-update.  skip_eval is cleared and the
// pass emits its Gram operand (force_emit = 1).  The per-chunk partials are reduced by the fixed-order reduction of the solver.
// Outputs (inactive problems: NaN): f_out[b] = the loss (fpart summed in chunk order), g_out[b] (Dt) = the data-term gradient without
// the prior; if not NULL, sd_out = sqrt(d_i) of every problem's rows, problem after problem (csr_fx batches: sdvec), and xt_out = the
// bf16 bits of the Xt operand, n x Dp per problem (dense and general-CSR batches).  info (8 + nprob ints): [0] kernel kind
// (1 dense, 2 CSR fixed point, 3 CSR fixed point with column windows, 4 general CSR, 5 fused multi-lambda CSR), [1] G (dense), LP
// (fused), beta in shared memory (fixed point, general CSR), [2] k1_dyn, [3] k1_grid, [4] rows per thread RT (dense), rows per
// segment (fused), column window width (windows), [5] row slices nsl (dense), [6] nprob, [7] 0, [8 + b] Ctrl::k1_chunks of an
// active problem (0 otherwise).  The batch's x-update state is consumed (every problem is left done): begin() again before iterating.
int mlease_internal_batch_grad(mlease_session* s, const int32_t* active, const double* w, double* f_out, double* g_out, float* sd_out,
                               uint16_t* xt_out, int32_t* info) {
  if (!s || !active || !w || !f_out || !g_out || !info) return fail(MLEASE_ERR_INVALID, "null argument");
  if (!s->batch || !s->begun) return fail(MLEASE_ERR_STATE, "mlease_admm_begin was not called");
  Batch& B = *s->batch;
  if (sd_out && !(B.csr && B.csr_fx)) return fail(MLEASE_ERR_INVALID, "sqrt(d) goes to sdvec only on CSR batches with sorted unique rows");
  if (xt_out && B.csr && B.csr_fx) return fail(MLEASE_ERR_INVALID, "this batch emits no Xt operand (its Gram reads sdvec)");
  CK(cudaSetDevice(s->cfg.device));
  const int nprob = B.nprob, ldx = s->ldx, Dt = s->Dt;
  std::vector<int32_t> inf(8 + (size_t)nprob, 0);
  inf[2] = B.k1_dyn; inf[3] = B.k1_grid; inf[6] = nprob;
  if (B.k1_fused) {
    inf[0] = 5; inf[1] = B.k1f_LP; inf[4] = B.h[0].sg_rows;
  } else if (B.csr && B.csr_fx) {
    const int W = k1_csr_window(ldx);
    inf[0] = W > 0 ? 3 : 2;
    inf[1] = (W == 0 && (size_t)2 * (ldx + 32) * 4 + (size_t)ldx * 4 <= 220 * 1024) ? 1 : 0;   // as k1_csr_fx_launch decides
    inf[4] = W;
  } else if (B.csr) {
    inf[0] = 4; inf[1] = (size_t)2 * ldx * 4 <= 200 * 1024 ? 1 : 0;   // as k1_launch decides
  } else {
    int R, S, G, cps; size_t smem;
    if (!k1_dense_plan(ldx, &R, &S, &G, &smem, &cps)) return fail(MLEASE_ERR_INVALID, "no dense K1 plan for this width");
    inf[0] = 1; inf[1] = G; inf[4] = G == 4 ? 4 : 8; inf[5] = R / inf[4];
  }
  std::vector<float> bf(ldx, 0.f);
  for (int b = 0; b < nprob; b++) {
    for (int k = 0; k < Dt; k++) bf[k] = (float)w[(size_t)b * Dt + k];
    CK(cudaMemcpy(B.h[b].beta_tf, bf.data(), (size_t)ldx * sizeof(float), cudaMemcpyHostToDevice));
  }
  std::vector<Ctrl> c(nprob);
  CK(cudaMemcpy(c.data(), B.d_ctrl, (size_t)nprob * sizeof(Ctrl), cudaMemcpyDeviceToHost));
  for (int b = 0; b < nprob; b++) { c[b].done = active[b] ? 0 : 1; c[b].skip_eval = 0; c[b].cg_active = active[b] ? 1 : 0; c[b].k1_chunks = 0; }
  CK(cudaMemcpy(B.d_ctrl, c.data(), (size_t)nprob * sizeof(Ctrl), cudaMemcpyHostToDevice));
  int launches = 0;
  CK(batch_k1(B, 1, s->stream, &launches));
  CK(hv_reduce(B.d, nprob, Dt, 0, s->stream, &launches));
  CK(cudaStreamSynchronize(s->stream));
  CK(cudaMemcpy(c.data(), B.d_ctrl, (size_t)nprob * sizeof(Ctrl), cudaMemcpyDeviceToHost));
  const double nan = std::nan("");
  std::vector<double> fp;
  size_t row0 = 0;
  for (int b = 0; b < nprob; b++) {
    const Problem& p = B.h[b];
    const size_t n = (size_t)p.n;
    if (active[b]) {
      inf[8 + b] = c[b].k1_chunks;
      fp.resize(std::max(1, c[b].k1_chunks));
      CK(cudaMemcpy(fp.data(), p.fpart, (size_t)c[b].k1_chunks * sizeof(double), cudaMemcpyDeviceToHost));
      double f = 0.0;
      for (int t = 0; t < c[b].k1_chunks; t++) f += fp[t];
      f_out[b] = f;
      CK(cudaMemcpy(g_out + (size_t)b * Dt, p.g_t, (size_t)Dt * sizeof(double), cudaMemcpyDeviceToHost));
      if (sd_out) CK(cudaMemcpy(sd_out + row0, p.sdvec, n * sizeof(float), cudaMemcpyDeviceToHost));
      if (xt_out) CK(cudaMemcpy(xt_out + row0 * B.Dp, p.Xt, n * B.Dp * sizeof(uint16_t), cudaMemcpyDeviceToHost));
    } else {
      f_out[b] = nan;
      std::fill(g_out + (size_t)b * Dt, g_out + (size_t)(b + 1) * Dt, nan);
      if (sd_out) std::fill(sd_out + row0, sd_out + row0 + n, std::nanf(""));
      if (xt_out) std::fill(xt_out + row0 * B.Dp, xt_out + (row0 + n) * B.Dp, (uint16_t)0x7FC0);   // bf16 NaN
    }
    row0 += n;
  }
  for (auto& x : c) { x.done = 1; x.cg_active = 0; }
  CK(cudaMemcpy(B.d_ctrl, c.data(), (size_t)nprob * sizeof(Ctrl), cudaMemcpyHostToDevice));
  B.mirror.clear();
  s->cnt.launches += launches;
  std::copy(inf.begin(), inf.end(), info);
  return 0;
}

// Test hook, not part of the C ABI: one factorisation of the session's ADMM batch (after begin()) with an explicit inverse (ldh
// <= 2048), through batch_factor -- the code of the solver's rebuild slot.  Problem b (= local partition * L + lambda):
//   mode[b] = 0: done, no kernel may touch it;  1: Lc = H[b] (Dt x Dt row-major, lower triangle read) as chol_prep leaves it,
//   then the factorisation without prep;  2: the fp32 Gram G[b] (Dt x Dt) goes into Hpart slice 0 (the other slices are zeroed),
//   q[b] (Dt) into q, gram_unscale = 1, and chol_prep_kernel forms H with the batch's share.
// order (norder entries, NULL: the batch order): the grids run over a device array of Problem copies in that order, as they run
// over poll2_kernel's compacted array in batches of more than 64 problems.  share (0 or group_L > 1) and share_factor mirror the
// cold start of a rebuild slot: share alone = distinct rho (every problem factorises the leader's Gram + its own q), share_factor
// too = equal rho (the leaders factorise, chol_share_end_kernel and the Hinv copies serve the followers).  A batch mixing modes 1
// and 2 runs chol_prep_kernel on its own first, with the mode-1 problems parked (need_hess = 0), then batch_factor without prep.
// Before the launch every problem's Lc, Ldiag, Ldinv, Yinv and Hinv are filled with a NaN sentinel (all bits set), except the
// strict upper triangle of Yinv, which stays 0: the DMMA merges and Y^T Y of systems wider than 1000 read it as the zeros of a
// triangular matrix.  Outputs, each if not NULL: L_out (Dt x Dt), Y_out and Hinv_out (ldh x ldh), Ldinv_out (ldh x 32), ctrl_out
// (4 per problem: fail, done, hess_valid, tot_hess as the kernels left them; the hook starts every problem from 0, 0/1, 0, 0).
// Every argument is checked before any launch.  gram_unscale and q are restored; the batch's x-update state is consumed (every
// problem is left done without a factor): begin() again before iterating.
int mlease_internal_batch_factor(mlease_session* s, const int32_t* mode, const double* H, const float* G, const double* q,
                                 const int32_t* order, int32_t norder, int32_t share, int32_t share_factor, double* L_out,
                                 double* Y_out, double* Hinv_out, double* Ldinv_out, int32_t* ctrl_out) {
  if (!s || !mode) return fail(MLEASE_ERR_INVALID, "null argument");
  if (!s->batch || !s->begun) return fail(MLEASE_ERR_STATE, "mlease_admm_begin was not called");
  Batch& B = *s->batch;
  if (B.matfree || !B.h[0].Hinv) return fail(MLEASE_ERR_INVALID, "a matrix-free session forms no factor");
  if (cholesky_factored_direction(B.ldh)) return fail(MLEASE_ERR_INVALID, "only systems up to 2048 (ldh) form the explicit inverse");
  const int nprob = B.nprob, Dt = s->Dt, ldh = B.ldh, Dp = B.Dp;
  bool any1 = false, any2 = false, any0 = false;
  for (int b = 0; b < nprob; b++) {
    if (mode[b] < 0 || mode[b] > 2) return fail(MLEASE_ERR_INVALID, "mode must be 0, 1 or 2");
    any0 |= mode[b] == 0; any1 |= mode[b] == 1; any2 |= mode[b] == 2;
  }
  if (any1 && !H) return fail(MLEASE_ERR_INVALID, "mode 1 needs H");
  if (any2 && (!G || !q)) return fail(MLEASE_ERR_INVALID, "mode 2 needs G and q");
  if (order) {
    if (norder < 0 || norder > nprob) return fail(MLEASE_ERR_INVALID, "launch order longer than the batch");
    std::vector<char> seen(nprob, 0);
    for (int i = 0; i < norder; i++) {
      if (order[i] < 0 || order[i] >= nprob) return fail(MLEASE_ERR_INVALID, "launch order leaves the batch");
      if (seen[order[i]]++) return fail(MLEASE_ERR_INVALID, "launch order repeats a problem");
    }
  }
  if (share != 0 && !(share > 1 && share == B.group_L)) return fail(MLEASE_ERR_INVALID, "share must be 0 or the batch's group_L (> 1)");
  if (share && order) return fail(MLEASE_ERR_INVALID, "a shared cold start runs over the batch order");
  if (share_factor && !share) return fail(MLEASE_ERR_INVALID, "share_factor needs share");
  if (share_factor && (any0 || (any1 && any2))) return fail(MLEASE_ERR_INVALID, "share_factor needs every problem in one mode, 1 or 2");
  if (share)
    for (int b = 0; b < nprob; b++)
      if (mode[b] != mode[b - b % share]) return fail(MLEASE_ERR_INVALID, "with share, every problem of a group has its leader's mode");
  CK(cudaSetDevice(s->cfg.device));
  const size_t hh = (size_t)ldh * ldh;
  std::vector<Ctrl> c0(nprob), c(nprob);
  CK(cudaMemcpy(c0.data(), B.d_ctrl, (size_t)nprob * sizeof(Ctrl), cudaMemcpyDeviceToHost));
  std::vector<double> qsave((size_t)nprob * Dt);
  // sentinel: all bits set (a NaN) everywhere, but 0 in the strict upper triangle of Yinv
  std::vector<double> ypat(hh);
  {
    double nan; std::memset(&nan, 0xFF, sizeof(nan));
    for (int i = 0; i < ldh; i++)
      for (int j = 0; j < ldh; j++) ypat[(size_t)i * ldh + j] = j > i ? 0.0 : nan;
  }
  std::vector<double> lc(hh);
  std::vector<float> gp((size_t)Dp * Dp, 0.f);
  std::vector<Problem> ph = B.h;
  for (int b = 0; b < nprob; b++) {
    const Problem& p = B.h[b];
    CK(cudaMemset(p.Lc, 0xFF, hh * sizeof(double)));
    CK(cudaMemset(p.Hinv, 0xFF, hh * sizeof(double)));
    CK(cudaMemset(p.Ldiag, 0xFF, (size_t)ldh * 32 * sizeof(double)));
    CK(cudaMemset(p.Ldinv, 0xFF, (size_t)ldh * 32 * sizeof(double)));
    CK(cudaMemcpy(p.Yinv, ypat.data(), hh * sizeof(double), cudaMemcpyHostToDevice));
    if (mode[b] == 1) {
      const double* h = H + (size_t)b * Dt * Dt;
      std::fill(lc.begin(), lc.end(), 0.0);
      for (int i = 0; i < ldh; i++)
        for (int j = 0; j <= i; j++) lc[(size_t)i * ldh + j] = i < Dt ? h[(size_t)i * Dt + j] : (i == j ? 1.0 : 0.0);
      CK(cudaMemcpy(p.Lc, lc.data(), hh * sizeof(double), cudaMemcpyHostToDevice));
    } else if (mode[b] == 2) {
      const float* g = G + (size_t)b * Dt * Dt;
      for (int i = 0; i < Dt; i++) std::memcpy(&gp[(size_t)i * Dp], g + (size_t)i * Dt, (size_t)Dt * sizeof(float));
      CK(cudaMemset(p.Hpart, 0, (size_t)B.gram_slices * Dp * Dp * sizeof(float)));
      CK(cudaMemcpy(p.Hpart, gp.data(), gp.size() * sizeof(float), cudaMemcpyHostToDevice));
      CK(cudaMemcpy(&qsave[(size_t)b * Dt], p.q, (size_t)Dt * sizeof(double), cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(p.q, q + (size_t)b * Dt, (size_t)Dt * sizeof(double), cudaMemcpyHostToDevice));
      ph[b].gram_unscale = 1.f;
    }
    c[b] = c0[b];
    c[b].done = mode[b] ? 0 : 1; c[b].need_hess = 1; c[b].fail = 0; c[b].hess_valid = 0; c[b].tot_hess = 0;
  }
  CK(cudaMemcpy(B.d, ph.data(), (size_t)nprob * sizeof(Problem), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(B.d_ctrl, c.data(), (size_t)nprob * sizeof(Ctrl), cudaMemcpyHostToDevice));
  Problem* d_ord = nullptr;
  int launches = 0;
  auto run = [&]() -> int {
    const Problem* d_hess = B.d;
    int n_hess = nprob;
    if (order) {
      std::vector<Problem> po(std::max(1, (int)norder));
      for (int i = 0; i < norder; i++) po[i] = ph[order[i]];
      CK(cudaMalloc(&d_ord, po.size() * sizeof(Problem)));
      CK(cudaMemcpy(d_ord, po.data(), (size_t)norder * sizeof(Problem), cudaMemcpyHostToDevice));
      d_hess = d_ord; n_hess = norder;
    }
    int skip_prep = any2 ? 0 : 1;
    if (any1 && any2 && n_hess > 0) {
      std::vector<Ctrl> cp = c;
      for (int b = 0; b < nprob; b++) if (mode[b] == 1) cp[b].need_hess = 0;
      CK(cudaMemcpy(B.d_ctrl, cp.data(), (size_t)nprob * sizeof(Ctrl), cudaMemcpyHostToDevice));
      CK(cholesky_prep(d_hess, n_hess, ldh, share, s->stream, &launches));
      CK(cudaStreamSynchronize(s->stream));
      CK(cudaMemcpy(B.d_ctrl, c.data(), (size_t)nprob * sizeof(Ctrl), cudaMemcpyHostToDevice));
      skip_prep = 1;
    }
    if (n_hess > 0)
      if (int rc = batch_factor(B, d_hess, n_hess, share, share_factor != 0, skip_prep, s->stream, &launches)) return rc;
    CK(cudaStreamSynchronize(s->stream));
    return 0;
  };
  // read back, then restore q, gram_unscale and Ctrl (also after a failed launch)
  auto read = [&]() -> int {
    if (int rc = run()) return rc;
    CK(cudaMemcpy(c.data(), B.d_ctrl, (size_t)nprob * sizeof(Ctrl), cudaMemcpyDeviceToHost));
    for (int b = 0; b < nprob; b++) {
    const Problem& p = B.h[b];
    if (L_out) {
      CK(cudaMemcpy(lc.data(), p.Lc, hh * sizeof(double), cudaMemcpyDeviceToHost));
      for (int i = 0; i < Dt; i++) std::memcpy(L_out + (size_t)b * Dt * Dt + (size_t)i * Dt, &lc[(size_t)i * ldh], (size_t)Dt * sizeof(double));
    }
    if (Y_out) CK(cudaMemcpy(Y_out + (size_t)b * hh, p.Yinv, hh * sizeof(double), cudaMemcpyDeviceToHost));
    if (Hinv_out) CK(cudaMemcpy(Hinv_out + (size_t)b * hh, p.Hinv, hh * sizeof(double), cudaMemcpyDeviceToHost));
    if (Ldinv_out) CK(cudaMemcpy(Ldinv_out + (size_t)b * ldh * 32, p.Ldinv, (size_t)ldh * 32 * sizeof(double), cudaMemcpyDeviceToHost));
    if (ctrl_out) {
      int32_t* o = ctrl_out + 4 * (size_t)b;
      o[0] = c[b].fail; o[1] = c[b].done; o[2] = c[b].hess_valid; o[3] = (int32_t)c[b].tot_hess;
    }
    }
    return 0;
  };
  const int rc = read();
  if (d_ord) cudaFree(d_ord);
  cudaStreamSynchronize(s->stream);
  for (int b = 0; b < nprob; b++)
    if (mode[b] == 2) CK(cudaMemcpy(B.h[b].q, &qsave[(size_t)b * Dt], (size_t)Dt * sizeof(double), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(B.d, B.h.data(), (size_t)nprob * sizeof(Problem), cudaMemcpyHostToDevice));
  for (int b = 0; b < nprob; b++) { c0[b].done = 1; c0[b].hess_valid = 0; c0[b].need_hess = 0; c0[b].fail = 0; }
  CK(cudaMemcpy(B.d_ctrl, c0.data(), (size_t)nprob * sizeof(Ctrl), cudaMemcpyHostToDevice));
  B.mirror.clear();
  s->cnt.launches += launches;
  return rc;
}

// Test hook, not part of the C ABI: the quasi-Newton direction on the explicit inverse (ldh <= 2048) of the problems with active[b]
// != 0, through the kernels of a chord slot: k1_reduce_decide (its first L-BFGS loop) and newton_solve (newton_gemv_kernel, the
// second loop, h0_scale, the trial point).  Run it after mlease_internal_batch_factor: it multiplies whatever Hinv holds.  Per
// active problem: the data-term gradient g[b] (Dt), the secant ring S[b], Y[b] (BFGS_M x Dt each, slot-major), rho[b] (BFGS_M),
// count[b] = Ctrl::bfgs_count (>= 0; above BFGS_M the ring has wrapped), h0[b] = Ctrl::h0_scale and the point beta[b] (Dt).
// The decide kernel takes its accept path with no pass over the rows: skip_eval = 1 (k1_partial_reduce_kernel leaves g_t alone,
// no loss partials: k1_chunks = 0), beta_t = m = beta (the prior term is 0), have_dir = 0 (no line search, no new secant pair),
// hess_valid = 1, emit = 0 (no rebuild), newton_steps = evals = 0 and max_newton >= 1 (no stop test can end the x-update).  Outputs, each if not NULL:
// dir_out (Dt per problem), phi0_out = Ctrl::phi0, dirnorm_out = Ctrl::dirnorm, beta_t_out (Dt; float(beta + dir) as stored);
// an inactive problem's are NaN.  Checked before any launch; the batch's x-update state is consumed: begin() again before iterating.
int mlease_internal_direction(mlease_session* s, const int32_t* active, const double* g, const double* S, const double* Y,
                              const double* rho, const int32_t* count, const double* h0, const double* beta, double* dir_out,
                              double* phi0_out, double* dirnorm_out, double* beta_t_out) {
  if (!s || !active || !g || !S || !Y || !rho || !count || !h0 || !beta) return fail(MLEASE_ERR_INVALID, "null argument");
  if (!s->batch || !s->begun) return fail(MLEASE_ERR_STATE, "mlease_admm_begin was not called");
  Batch& B = *s->batch;
  if (B.matfree || !B.h[0].Hinv) return fail(MLEASE_ERR_INVALID, "a matrix-free session forms no factor");
  if (cholesky_factored_direction(B.ldh)) return fail(MLEASE_ERR_INVALID, "only systems up to 2048 (ldh) form the explicit inverse");
  const int nprob = B.nprob, Dt = s->Dt, ldx = s->ldx;
  for (int b = 0; b < nprob; b++)
    if (active[b] && count[b] < 0) return fail(MLEASE_ERR_INVALID, "bfgs_count must be >= 0");
  CK(cudaSetDevice(s->cfg.device));
  std::vector<Ctrl> c(nprob);
  CK(cudaMemcpy(c.data(), B.d_ctrl, (size_t)nprob * sizeof(Ctrl), cudaMemcpyDeviceToHost));
  std::vector<double> v(ldx), ring((size_t)BFGS_M * ldx);
  for (int b = 0; b < nprob; b++) {
    Ctrl& x = c[b];
    x.done = active[b] ? 0 : 1;
    if (!active[b]) continue;
    const Problem& p = B.h[b];
    x.skip_eval = 1; x.k1_chunks = 0; x.have_dir = 0; x.hess_valid = 1; x.emit = 0; x.need_hess = 0; x.need_solve = 0;
    x.newton_steps = 0; x.evals = 0; x.fail = 0; x.bfgs_count = count[b]; x.h0_scale = h0[b];
    x.max_newton = std::max(1, s->max_newton);   // (a batch that never ran an x-update has 0: the decide kernel would stop it)
    std::fill(v.begin(), v.end(), 0.0);
    std::memcpy(v.data(), g + (size_t)b * Dt, (size_t)Dt * sizeof(double));
    CK(cudaMemcpy(p.g_t, v.data(), (size_t)ldx * sizeof(double), cudaMemcpyHostToDevice));
    std::memcpy(v.data(), beta + (size_t)b * Dt, (size_t)Dt * sizeof(double));
    CK(cudaMemcpy(p.beta_t, v.data(), (size_t)ldx * sizeof(double), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(p.m, v.data(), (size_t)ldx * sizeof(double), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(p.beta, v.data(), (size_t)ldx * sizeof(double), cudaMemcpyHostToDevice));
    std::fill(v.begin(), v.end(), std::nan(""));
    CK(cudaMemcpy(p.dir, v.data(), (size_t)ldx * sizeof(double), cudaMemcpyHostToDevice));
    for (int pass = 0; pass < 2; pass++) {
      const double* src = (pass ? Y : S) + (size_t)b * BFGS_M * Dt;
      std::fill(ring.begin(), ring.end(), 0.0);
      for (int j = 0; j < BFGS_M; j++) std::memcpy(&ring[(size_t)j * ldx], src + (size_t)j * Dt, (size_t)Dt * sizeof(double));
      CK(cudaMemcpy(pass ? p.bfgs_Y : p.bfgs_S, ring.data(), ring.size() * sizeof(double), cudaMemcpyHostToDevice));
    }
    CK(cudaMemcpy(p.bfgs_rho, rho + (size_t)b * BFGS_M, BFGS_M * sizeof(double), cudaMemcpyHostToDevice));
  }
  CK(cudaMemcpy(B.d_ctrl, c.data(), (size_t)nprob * sizeof(Ctrl), cudaMemcpyHostToDevice));
  int launches = 0;
  CK(k1_reduce_decide(B.d, nprob, Dt, s->stream, &launches, 0));
  CK(newton_solve(B.d, nprob, B.ldh, s->stream, &launches, B.group_L));
  CK(cudaStreamSynchronize(s->stream));
  CK(cudaMemcpy(c.data(), B.d_ctrl, (size_t)nprob * sizeof(Ctrl), cudaMemcpyDeviceToHost));
  const double nan = std::nan("");
  for (int b = 0; b < nprob; b++) {
    const Problem& p = B.h[b];
    if (dir_out) {
      if (active[b]) CK(cudaMemcpy(dir_out + (size_t)b * Dt, p.dir, (size_t)Dt * sizeof(double), cudaMemcpyDeviceToHost));
      else std::fill(dir_out + (size_t)b * Dt, dir_out + (size_t)(b + 1) * Dt, nan);
    }
    if (beta_t_out) {
      if (active[b]) CK(cudaMemcpy(beta_t_out + (size_t)b * Dt, p.beta_t, (size_t)Dt * sizeof(double), cudaMemcpyDeviceToHost));
      else std::fill(beta_t_out + (size_t)b * Dt, beta_t_out + (size_t)(b + 1) * Dt, nan);
    }
    if (phi0_out) phi0_out[b] = active[b] ? c[b].phi0 : nan;
    if (dirnorm_out) dirnorm_out[b] = active[b] ? c[b].dirnorm : nan;
  }
  for (auto& x : c) { x.done = 1; x.hess_valid = 0; x.need_solve = 0; x.need_hess = 0; x.have_dir = 0; x.bfgs_count = 0; x.h0_scale = 1.0; }
  CK(cudaMemcpy(B.d_ctrl, c.data(), (size_t)nprob * sizeof(Ctrl), cudaMemcpyHostToDevice));
  B.mirror.clear();
  s->cnt.launches += launches;
  return 0;
}

}  // extern "C"

namespace {
// The x-update fields of Ctrl as mlease_internal_newton_stage exchanges them, per problem: 24 ints, 14 reals, then the cumulative
// counters (read back only).  The Ctrl pointers and ysym_use are never taken from the caller.
#define STAGE_INTS(X)                                                                                                              \
  X(done) X(have_dir) X(need_solve) X(need_hess) X(emit) X(hess_valid) X(fail) X(newton_steps) X(evals) X(rejects) X(hess_builds) \
  X(stall) X(bfgs_count) X(k1_chunks) X(refresh_next) X(skip_eval) X(warm_used) X(build_step) X(max_newton) X(hess_policy)        \
  X(rebuild_is_expensive) X(cg_active) X(cg_iter)
#define STAGE_REALS(X) \
  X(h0_scale) X(worst_ratio) X(alpha) X(phi0) X(f_acc) X(f_t) X(gnorm) X(gnorm_prev) X(dirnorm) X(dirnorm_prev) X(xtol) X(cg_rz) X(cg_g2) X(hv_vinf)
#define STAGE_TOTALS(X) X(tot_evals) X(tot_newton) X(tot_rejects) X(tot_hess)
struct StageCtrl {
#define X(f) int32_t f;
  STAGE_INTS(X)
#undef X
  int32_t pad_;
#define X(f) double f;
  STAGE_REALS(X)
  STAGE_TOTALS(X)
#undef X
};
static_assert(sizeof(StageCtrl) == 24 * 4 + 18 * 8, "StageCtrl is packed: 24 ints, 18 doubles");
void stage_to_ctrl(const StageCtrl& a, Ctrl& c) {
#define X(f) c.f = (decltype(c.f))a.f;
  STAGE_INTS(X)
  STAGE_REALS(X)
#undef X
}
void ctrl_to_stage(const Ctrl& c, StageCtrl& a) {
#define X(f) a.f = c.f;
  STAGE_INTS(X)
#undef X
#define X(f) a.f = (double)c.f;
  STAGE_REALS(X)
  STAGE_TOTALS(X)
#undef X
  a.pad_ = 0;
}
enum { ST_BEGIN = 1, ST_DECIDE = 2, ST_SOLVE = 4, ST_FINISH = 8, ST_CG_BEGIN = 16, ST_CG_INIT = 32, ST_CG_STEP = 64, ST_CG_POLL = 128 };
constexpr int STAGE_NVEC = 12;
// Every problem's vectors, secant ring and fp32 vectors to the device (h2d) or back, in the layout of mlease_internal_newton_stage.
int stage_exchange(Batch& B, int ldx, bool h2d, double* vec, double* ring, float* fvec) {
  const size_t vb = (size_t)ldx * sizeof(double), ring_n = 2 * (size_t)BFGS_M * ldx + 2 * BFGS_M;
  const int nvec = B.matfree ? STAGE_NVEC : 7;
  auto cp = [&](void* dev, void* host, size_t bytes) {
    return h2d ? cudaMemcpy(dev, host, bytes, cudaMemcpyHostToDevice) : cudaMemcpy(host, dev, bytes, cudaMemcpyDeviceToHost);
  };
  for (int b = 0; b < B.nprob; b++) {
    const Problem& p = B.h[b];
    double* v[STAGE_NVEC] = {p.beta, p.beta_t, p.m, p.q, p.g_t, p.g_acc, p.dir, p.cg_r, p.cg_p, p.cg_z, p.cg_Hp, p.cg_diag};
    for (int i = 0; i < nvec; i++) CK(cp(v[i], vec + ((size_t)b * STAGE_NVEC + i) * ldx, vb));
    double* r = ring + (size_t)b * ring_n;
    if (!B.matfree) {
      CK(cp(p.bfgs_S, r, (size_t)BFGS_M * vb));
      CK(cp(p.bfgs_Y, r + (size_t)BFGS_M * ldx, (size_t)BFGS_M * vb));
    }
    CK(cp(p.bfgs_rho, r + 2 * (size_t)BFGS_M * ldx, BFGS_M * sizeof(double)));
    CK(cp(p.bfgs_alpha, r + 2 * (size_t)BFGS_M * ldx + BFGS_M, BFGS_M * sizeof(double)));
    float* f = fvec + (size_t)b * 3 * ldx;
    CK(cp(p.beta_tf, f, (size_t)ldx * sizeof(float)));
    CK(cp(p.qf, f + ldx, 2 * (size_t)ldx * sizeof(float)));   // qf and tf are adjacent
  }
  return 0;
}
}  // namespace

extern "C" {

// Test hook, not part of the C ABI: injects an x-update state into every problem of the begun ADMM batch, runs the selected kernels
// of the Newton state machine (newton.cu) once, each through the solver's own launcher, and reads the whole state back.
//   stages: ST_BEGIN newton_begin(begin_args = {xtol, max_newton, policy, invalidate, rebuild_is_expensive}); ST_DECIDE
//   k1_reduce_decide(spec) -- the fixed-order reduction of the partials and the decide kernel, no pass over the rows; ST_CG_BEGIN,
//   ST_CG_INIT, ST_CG_STEP, ST_CG_POLL (matrix-free batches; *cg_any = the poll's flag) -- cg_init finds the diagonal's data term in
//   cg_diag and cg_step finds X^T D X p in cg_Hp, as the reductions of their passes leave them; ST_SOLVE newton_solve (the GEMV on
//   whatever Hinv / Ysym the batch holds, then newton_solve_kernel) or ST_FINISH newton_finish (newton_solve_kernel alone, on the r
//   = H0^-1 q the caller put into dir).  They run in that order.  stages = 0 injects and runs nothing: info only.
//   ctrl: nprob StageCtrl, in and out.  vec: nprob x 12 x ldx doubles (beta, beta_t, m, q, g_t, g_acc, dir, cg_r, cg_p, cg_z, cg_Hp,
//   cg_diag; the last five only on a matrix-free batch), ring: nprob x (2 BFGS_M ldx + 2 BFGS_M) doubles (bfgs_S, bfgs_Y -- not on
//   a matrix-free batch --, bfgs_rho, bfgs_alpha), fvec: nprob x 3 x ldx floats (beta_tf, qf = hv_vf, tf); all in and out, whole
//   vectors, padding included, copied as bytes (a caller marks what no kernel may write with any pattern it likes).
//   gpart (nprob x nct_cap x ldx doubles; stored as fp32 into gpart_f on a fused batch) and fpart (nprob x nct_cap), or both NULL
//   when every k1_chunks is 0.
//   info (12 ints): nprob, Dt, ldx, ldh, partial rows allocated per problem (k1_grid), fused K1, matrix-free, Ysym present,
//   rebuild_is_expensive, group_L, 0, 0.
// Refused before any launch: a state the kernels would index memory with (k1_chunks beyond the allocated rows or nct_cap,
// bfgs_count < 0, a policy other than 2 or secant pairs on a matrix-free batch, which has no ring), ST_SOLVE on a batch that never
// factorised (no batch_factor ran on it: mlease_internal_batch_factor or a rebuild slot), ST_SOLVE together with ST_FINISH, CG stages on a batch without CG vectors.  The batch's x-update state is consumed
// (every problem is left done, without a factor or pairs): begin() again before iterating.
int mlease_internal_newton_stage(mlease_session* s, int32_t stages, int32_t spec, const double* begin_args, void* ctrl, double* vec,
                                 double* ring, float* fvec, const double* gpart, const double* fpart, int32_t nct_cap, int32_t* info,
                                 int32_t* cg_any) {
  if (!s || !info) return fail(MLEASE_ERR_INVALID, "null argument");
  if (!s->batch || !s->begun) return fail(MLEASE_ERR_STATE, "mlease_admm_begin was not called");
  Batch& B = *s->batch;
  const int nprob = B.nprob, Dt = s->Dt, ldx = s->ldx;
  const bool wide = cholesky_factored_direction(B.ldh);
  const int32_t inf[12] = {nprob, Dt, ldx, B.ldh, B.k1_grid, B.k1_fused, B.matfree, (!B.matfree && B.h[0].Ysym) ? 1 : 0,
                           B.rebuild_is_expensive, B.group_L, 0, 0};
  std::copy(inf, inf + 12, info);
  if (stages == 0) return 0;
  if (stages < 0 || stages > 255 || (spec != 0 && spec != 1)) return fail(MLEASE_ERR_INVALID, "stage mask or spec out of range");
  if (!ctrl || !vec || !ring || !fvec) return fail(MLEASE_ERR_INVALID, "null argument");
  if ((gpart == nullptr) != (fpart == nullptr) || nct_cap < 0) return fail(MLEASE_ERR_INVALID, "gpart and fpart come together");
  if ((stages & ST_SOLVE) && (stages & ST_FINISH)) return fail(MLEASE_ERR_INVALID, "newton_solve and newton_finish are alternatives");
  if ((stages & ST_SOLVE) && (B.matfree || !B.h[0].Hinv || (wide && !B.h[0].Ysym) || !B.has_factor))
    return fail(MLEASE_ERR_INVALID, "newton_solve needs a batch that has factorised (batch_factor ran; a matrix-free batch forms no factor)");
  if ((stages & (ST_CG_BEGIN | ST_CG_INIT | ST_CG_STEP | ST_CG_POLL)) && (!B.matfree || !B.h[0].cg_r))
    return fail(MLEASE_ERR_INVALID, "the CG kernels need a matrix-free batch");
  if ((stages & ST_CG_POLL) && !cg_any) return fail(MLEASE_ERR_INVALID, "cg_poll needs cg_any");
  if (stages & ST_BEGIN) {
    if (!begin_args) return fail(MLEASE_ERR_INVALID, "newton_begin needs its arguments");
    const double pol = begin_args[2];
    if (!(begin_args[0] >= 0.0) || !(begin_args[1] >= 0.0 && begin_args[1] <= 1e6) || !(pol == 0.0 || pol == 1.0 || pol == 2.0) ||
        (B.matfree && pol != 2.0))
      return fail(MLEASE_ERR_INVALID, "newton_begin arguments out of range (a matrix-free batch runs policy 2 only)");
  }
  const StageCtrl* in = static_cast<const StageCtrl*>(ctrl);
  for (int b = 0; b < nprob; b++) {
    const StageCtrl& a = in[b];
    if (a.k1_chunks < 0 || a.k1_chunks > B.k1_grid) return fail(MLEASE_ERR_INVALID, "k1_chunks beyond the partial rows the batch allocated");
    if (a.k1_chunks > (gpart ? nct_cap : 0)) return fail(MLEASE_ERR_INVALID, "k1_chunks beyond the partials passed");
    if (a.bfgs_count < 0 || a.bfgs_count > (1 << 20)) return fail(MLEASE_ERR_INVALID, "bfgs_count must be >= 0");
    if (a.hess_policy < 0 || a.hess_policy > 2 || a.max_newton < 0 || a.cg_iter < 0) return fail(MLEASE_ERR_INVALID, "policy, max_newton or cg_iter out of range");
    if (B.matfree && (a.hess_policy != 2 || a.bfgs_count != 0)) return fail(MLEASE_ERR_INVALID, "a matrix-free batch keeps no secant pairs: policy 2, bfgs_count 0");
  }
  CK(cudaSetDevice(s->cfg.device));
  std::vector<Ctrl> c0(nprob), c(nprob);
  CK(cudaMemcpy(c0.data(), B.d_ctrl, (size_t)nprob * sizeof(Ctrl), cudaMemcpyDeviceToHost));
  const size_t vb = (size_t)ldx * sizeof(double);
  if (int rc = stage_exchange(B, ldx, true, vec, ring, fvec)) return rc;
  if (gpart) {
    std::vector<float> gf;
    for (int b = 0; b < nprob; b++) {
      const Problem& p = B.h[b];
      const int nct = in[b].k1_chunks;
      if (nct == 0) continue;
      const double* src = gpart + (size_t)b * nct_cap * ldx;
      if (p.gpart_f) {
        gf.assign(src, src + (size_t)nct * ldx);
        CK(cudaMemcpy(p.gpart_f, gf.data(), gf.size() * sizeof(float), cudaMemcpyHostToDevice));
      } else {
        CK(cudaMemcpy(p.gpart, src, (size_t)nct * vb, cudaMemcpyHostToDevice));
      }
      CK(cudaMemcpy(p.fpart, fpart + (size_t)b * nct_cap, (size_t)nct * sizeof(double), cudaMemcpyHostToDevice));
    }
  }
  for (int b = 0; b < nprob; b++) { c[b] = c0[b]; stage_to_ctrl(in[b], c[b]); }
  CK(cudaMemcpy(B.d_ctrl, c.data(), (size_t)nprob * sizeof(Ctrl), cudaMemcpyHostToDevice));
  int launches = 0;
  auto run = [&]() -> int {
    if (stages & ST_BEGIN)
      CK(newton_begin(B.d, nprob, begin_args[0], (int)begin_args[1], (int)begin_args[2], begin_args[3] != 0.0, begin_args[4] != 0.0, s->stream, &launches));
    if (stages & ST_DECIDE) CK(k1_reduce_decide(B.d, nprob, Dt, s->stream, &launches, spec));
    if (stages & ST_CG_BEGIN) CK(cg_begin(B.d, nprob, s->stream, &launches));
    if (stages & ST_CG_INIT) CK(cg_init(B.d, nprob, Dt, s->stream, &launches));
    if (stages & ST_CG_STEP) CK(cg_step(B.d, nprob, Dt, s->stream, &launches));
    if (stages & ST_CG_POLL) {
      CK(cg_poll(B.d, nprob, s->d_flag + 2, s->stream, &launches));
      CK(cudaMemcpyAsync(s->h_flag + 2, s->d_flag + 2, sizeof(int), cudaMemcpyDeviceToHost, s->stream));
    }
    if (stages & ST_SOLVE) CK(newton_solve(B.d, nprob, B.ldh, s->stream, &launches, B.group_L));
    if (stages & ST_FINISH) CK(newton_finish(B.d, nprob, Dt, s->stream, &launches));
    CK(cudaStreamSynchronize(s->stream));
    if (stages & ST_CG_POLL) *cg_any = s->h_flag[2];
    CK(cudaMemcpy(c.data(), B.d_ctrl, (size_t)nprob * sizeof(Ctrl), cudaMemcpyDeviceToHost));
    StageCtrl* out = static_cast<StageCtrl*>(ctrl);
    for (int b = 0; b < nprob; b++) ctrl_to_stage(c[b], out[b]);
    return stage_exchange(B, ldx, false, vec, ring, fvec);
  };
  const int rc = run();
  cudaStreamSynchronize(s->stream);
  for (int b = 0; b < nprob; b++) {
    Ctrl& x = c0[b];
    x.done = 1; x.hess_valid = 0; x.need_solve = 0; x.need_hess = 0; x.have_dir = 0; x.bfgs_count = 0; x.h0_scale = 1.0;
    x.skip_eval = 0; x.refresh_next = 0; x.cg_active = 0; x.k1_chunks = 0; x.fail = 0;
  }
  CK(cudaMemcpy(B.d_ctrl, c0.data(), (size_t)nprob * sizeof(Ctrl), cudaMemcpyHostToDevice));
  B.mirror.clear();
  s->cnt.launches += launches;
  return rc;
}

// Test hook, not part of the C ABI: one real x-update of the begun ADMM batch (at most 64 problems), slot by slot, through batch_slot
// -- the slot code batch_xupdate runs: K1, the decide kernel, the Gram / Cholesky launches of a rebuild, the matrix-free direction,
// newton_solve / newton_finish.  args = {xtol (<= 0: the session's), max_newton (<= 0: the session's), policy, invalidate}; a
// matrix-free batch runs policy 2 whatever is asked, as in batch_xupdate.  newton_begin, then slots until every problem is done or
// max_slots have run.  spec[i] != 0 asks for slot i in speculative form (no rebuild launches); it is honoured as batch_xupdate
// would: only when, as of the state before slot i - 1, every running problem had a valid factor and no rebuild was due.  A regular
// slot includes the rebuild launches iff a running problem has emit set.  Refused before any launch: spec under a policy other than
// 0, spec for slot 0, a batch of more than 64 problems (batch_xupdate never speculates there).
// The trace has max_slots + 1 entries, entry 0 the state newton_begin left and entry i + 1 the state after slot i, each in the
// layout of mlease_internal_newton_stage (ctrl: nprob StageCtrl; vec, ring, fvec); slot_info (2 ints per slot): ran speculatively,
// included the rebuild launches; *nslots = slots run.  The batch is left as after an x-update (beta = x).
int mlease_internal_xupdate_trace(mlease_session* s, const double* args, const int32_t* spec, int32_t max_slots, void* ctrl_trace,
                                  double* vec_trace, double* ring_trace, float* fvec_trace, int32_t* slot_info, int32_t* nslots) {
  if (!s || !args || !spec || !ctrl_trace || !vec_trace || !ring_trace || !fvec_trace || !slot_info || !nslots) return fail(MLEASE_ERR_INVALID, "null argument");
  if (!s->batch || !s->begun) return fail(MLEASE_ERR_STATE, "mlease_admm_begin was not called");
  Batch& B = *s->batch;
  if (max_slots < 1 || max_slots > 400) return fail(MLEASE_ERR_INVALID, "max_slots out of range");
  if (B.nprob > 64) return fail(MLEASE_ERR_INVALID, "the slot trace follows batches of at most 64 problems");
  if (!(args[2] == 0.0 || args[2] == 1.0 || args[2] == 2.0)) return fail(MLEASE_ERR_INVALID, "policy must be 0, 1 or 2");
  const int policy = B.matfree ? 2 : (int)args[2];
  if (policy == 2 && !B.matfree) return fail(MLEASE_ERR_INVALID, "policy 2 needs a matrix-free batch");
  for (int i = 0; i < max_slots; i++)
    if (spec[i] && (policy != 0 || i == 0)) return fail(MLEASE_ERR_INVALID, "batch_xupdate speculates only under policy 0 and never on slot 0");
  CK(cudaSetDevice(s->cfg.device));
  const int nprob = B.nprob, ldx = s->ldx;
  const double xtol = args[0] > 0.0 ? args[0] : s->xtol;
  const int max_newton = args[1] > 0.0 ? (int)args[1] : s->max_newton;
  const size_t ring_n = 2 * (size_t)BFGS_M * ldx + 2 * BFGS_M;
  Profiler nop;
  int launches = 0;
  double shared_flops = 0;
  std::vector<Ctrl> c(nprob);
  auto record = [&](int entry) -> int {
    CK(cudaStreamSynchronize(s->stream));
    CK(cudaMemcpy(c.data(), B.d_ctrl, (size_t)nprob * sizeof(Ctrl), cudaMemcpyDeviceToHost));
    StageCtrl* out = static_cast<StageCtrl*>(ctrl_trace) + (size_t)entry * nprob;
    for (int b = 0; b < nprob; b++) ctrl_to_stage(c[b], out[b]);
    return stage_exchange(B, ldx, false, vec_trace + (size_t)entry * nprob * STAGE_NVEC * ldx, ring_trace + (size_t)entry * nprob * ring_n,
                          fvec_trace + (size_t)entry * nprob * 3 * ldx);
  };
  // flags of the read-back state: 1 a problem runs, 2 a rebuild is due; *valid: every running problem has a factor
  auto flags = [&](bool* valid) {
    int f = 0; *valid = true;
    for (int b = 0; b < nprob; b++) if (!c[b].done) { f |= 1; if (c[b].emit) f |= 2; if (!c[b].hess_valid) *valid = false; }
    return f;
  };
  CK(newton_begin(B.d, nprob, xtol, max_newton, policy, args[3] != 0.0, B.rebuild_is_expensive, s->stream, &launches));
  if (int rc = record(0)) return rc;
  bool valid_now, valid_before = false;
  int flag_now = flags(&valid_now), flag_before = 2;   // nothing is known before slot 0: no speculation on slot 1 unless slot 0's outcome allows it
  if (!B.matfree) { valid_before = valid_now; flag_before = flag_now; }   // (the host's prediction of slot 0 equals what newton_begin left)
  int slots = 0;
  while ((flag_now & 1) && slots < max_slots) {
    const bool sp = spec[slots] && valid_before && !(flag_before & 2);
    const bool with_hess = !sp && (flag_now & 2) && !B.matfree;
    const SlotCtx x{s->stream, &nop, &launches, B.d, nprob, 0, 0, &shared_flops, s->h_flag, s->d_flag, false};
    if (int rc = batch_slot(B, x, slots, with_hess, sp)) return rc;
    slot_info[2 * slots] = sp ? 1 : 0; slot_info[2 * slots + 1] = with_hess ? 1 : 0;
    valid_before = valid_now; flag_before = flag_now;
    if (int rc = record(slots + 1)) return rc;
    flag_now = flags(&valid_now);
    slots++;
  }
  *nslots = slots;
  B.mirror = c;
  s->cnt.launches += launches;
  return 0;
}

// Test hooks of the factored direction of wide systems (ldh > 2048), not part of the C ABI.  Each refuses, before any launch, a
// batch that has no Ysym (ldh <= 2048, or matrix-free), since the kernels they run dereference it.
//
// mlease_internal_factor: the caller's Dt x Dt H (row-major; its lower triangle is read) goes into the scratch problem's Lc of
// partition pid as chol_prep leaves it (lower triangle, identity on the padding, zero above), then the factorisation the solver
// runs for its direction: fp64 Cholesky, recursive inverse with TF32 merges, bf16 symmetric packing.  Read back, each if not NULL:
// Lc (Dt x Dt), Yinv (ldh x ldh, whole) and the raw bits of Ysym (ldh x ldh).  The scratch problem's x-update state is consumed.
int mlease_internal_factor(mlease_session* s, int32_t pid, const double* H, double* L_out, double* Y_out, uint16_t* ysym_out) {
  if (!s || !H) return fail(MLEASE_ERR_INVALID, "null argument");
  if (s->cfg.hessian_policy == 2) return fail(MLEASE_ERR_INVALID, "a matrix-free session forms no factor");
  if (!cholesky_factored_direction(round_up(s->Dt, 32))) return fail(MLEASE_ERR_INVALID, "only systems wider than 2048 (ldh) use the factored direction");
  Batch* B;
  if (int rc = scratch_for(s, pid, &B)) return rc;
  if (B->matfree) return fail(MLEASE_ERR_INVALID, "a matrix-free session forms no factor");   // (made so by the memory rule)
  if (!cholesky_factored_direction(B->ldh) || !B->h[0].Ysym) return fail(MLEASE_ERR_INVALID, "only systems wider than 2048 (ldh) use the factored direction");
  const Problem& p = B->h[0];
  const int Dt = s->Dt, ldh = B->ldh;
  const size_t hh = (size_t)ldh * ldh;
  std::vector<double> lc(hh, 0.0);
  for (int i = 0; i < ldh; i++)
    for (int j = 0; j <= i; j++) lc[(size_t)i * ldh + j] = i < Dt ? H[(size_t)i * Dt + j] : (i == j ? 1.0 : 0.0);
  CK(cudaMemcpy(p.Lc, lc.data(), hh * sizeof(double), cudaMemcpyHostToDevice));
  Ctrl c; std::memset(&c, 0, sizeof(c)); c.need_hess = 1;
  CK(cudaMemcpy(B->d_ctrl, &c, sizeof(Ctrl), cudaMemcpyHostToDevice));
  int launches = 0;
  CK(cholesky_launch(B->d, 1, ldh, s->stream, &launches, 0, 1, 0));
  CK(cudaStreamSynchronize(s->stream));
  CK(cudaMemcpy(&c, B->d_ctrl, sizeof(Ctrl), cudaMemcpyDeviceToHost));
  if (L_out) {
    CK(cudaMemcpy(lc.data(), p.Lc, hh * sizeof(double), cudaMemcpyDeviceToHost));
    for (int i = 0; i < Dt; i++) std::memcpy(L_out + (size_t)i * Dt, &lc[(size_t)i * ldh], (size_t)Dt * sizeof(double));
  }
  if (Y_out) CK(cudaMemcpy(Y_out, p.Yinv, hh * sizeof(double), cudaMemcpyDeviceToHost));
  if (ysym_out) CK(cudaMemcpy(ysym_out, p.Ysym, hh * sizeof(uint16_t), cudaMemcpyDeviceToHost));
  if (int rc = reset_ctrl(*B)) return rc;
  s->cnt.launches += launches;
  if (c.fail) return fail(MLEASE_ERR_NUMERIC, "Hessian not positive definite");
  return 0;
}

// mlease_internal_factored_direction: on the ADMM batch (after begin() and at least one iterate()), the two triangular GEMV phases of
// the direction for the problems with active[b] != 0, each on its q[b] (Dt entries; b = local partition * L + lambda), over the
// whole problem array with the batch's group_L, exactly as newton_solve launches them.  t_out[b] / dir_out[b] (Dt entries each, if
// not NULL) receive tf and dir; dir is filled with NaN beforehand, so an inactive problem keeps NaN.  The batch's x-update state
// is consumed (every problem is left done): begin() again before iterating.
int mlease_internal_factored_direction(mlease_session* s, const int32_t* active, const float* q, float* t_out, double* dir_out) {
  if (!s || !active || !q) return fail(MLEASE_ERR_INVALID, "null argument");
  if (!s->batch || !s->begun || s->iter < 1) return fail(MLEASE_ERR_STATE, "needs the ADMM batch after mlease_admm_begin and one iteration");
  CK(cudaSetDevice(s->cfg.device));
  Batch& B = *s->batch;
  if (B.matfree) return fail(MLEASE_ERR_INVALID, "a matrix-free session forms no factor");
  if (!cholesky_factored_direction(B.ldh) || !B.h[0].Ysym) return fail(MLEASE_ERR_INVALID, "only systems wider than 2048 (ldh) use the factored direction");
  const int nprob = B.nprob, ldx = s->ldx, Dt = s->Dt;
  std::vector<Ctrl> c(nprob);
  CK(cudaMemcpy(c.data(), B.d_ctrl, (size_t)nprob * sizeof(Ctrl), cudaMemcpyDeviceToHost));
  for (int b = 0; b < nprob; b++) { c[b].done = active[b] ? 0 : 1; c[b].need_solve = active[b] ? 1 : 0; }
  CK(cudaMemcpy(B.d_ctrl, c.data(), (size_t)nprob * sizeof(Ctrl), cudaMemcpyHostToDevice));
  std::vector<float> qt(2 * (size_t)ldx, 0.f);   // qf then tf: qf = float(q) on [0, Dt) and 0 on [Dt, ldx) (as the decide kernel leaves it)
  const std::vector<double> nan(ldx, std::nan(""));
  for (int b = 0; b < nprob; b++) {
    for (int k = 0; k < ldx; k++) { qt[k] = k < Dt ? q[(size_t)b * Dt + k] : 0.f; qt[ldx + k] = k < Dt ? std::nanf("") : 0.f; }
    CK(cudaMemcpy(B.h[b].qf, qt.data(), 2 * (size_t)ldx * sizeof(float), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(B.h[b].dir, nan.data(), (size_t)ldx * sizeof(double), cudaMemcpyHostToDevice));
  }
  CK(newton_gemv_tri(B.d, nprob, B.ldh, B.group_L, s->stream));
  CK(cudaStreamSynchronize(s->stream));
  for (int b = 0; b < nprob; b++) {
    if (t_out) CK(cudaMemcpy(t_out + (size_t)b * Dt, B.h[b].tf, (size_t)Dt * sizeof(float), cudaMemcpyDeviceToHost));
    if (dir_out) CK(cudaMemcpy(dir_out + (size_t)b * Dt, B.h[b].dir, (size_t)Dt * sizeof(double), cudaMemcpyDeviceToHost));
  }
  for (auto& x : c) { x.done = 1; x.need_solve = 0; }
  CK(cudaMemcpy(B.d_ctrl, c.data(), (size_t)nprob * sizeof(Ctrl), cudaMemcpyHostToDevice));
  B.mirror.clear();
  s->cnt.launches += 2;
  return 0;
}

// mlease_internal_ysym: the bytes problem b of the ADMM batch streams in its direction (Ctrl::ysym_use, else its own Ysym; ldh x ldh
// bf16 bits), the index of the problem that owns them, and b's factorisation count (Ctrl::tot_hess).  Reads only.
int mlease_internal_ysym(mlease_session* s, int32_t b, uint16_t* out, int32_t* owner, int32_t* tot_hess) {
  if (!s) return fail(MLEASE_ERR_INVALID, "null session");
  if (!s->batch) return fail(MLEASE_ERR_STATE, "mlease_admm_begin was not called");
  CK(cudaSetDevice(s->cfg.device));
  Batch& B = *s->batch;
  if (b < 0 || b >= B.nprob) return fail(MLEASE_ERR_INVALID, "problem index out of range");
  if (B.matfree) return fail(MLEASE_ERR_INVALID, "a matrix-free session forms no factor");
  if (!cholesky_factored_direction(B.ldh) || !B.h[0].Ysym) return fail(MLEASE_ERR_INVALID, "only systems wider than 2048 (ldh) use the factored direction");
  Ctrl c;
  CK(cudaMemcpy(&c, B.d_ctrl + b, sizeof(Ctrl), cudaMemcpyDeviceToHost));
  const void* use = c.ysym_use ? c.ysym_use : (const void*)B.h[b].Ysym;
  int own = -1;
  for (int j = 0; j < B.nprob; j++) if ((const void*)B.h[j].Ysym == use) own = j;
  if (own < 0) return fail(MLEASE_ERR_STATE, "problem's factor pointer matches no problem of the batch");
  if (out) CK(cudaMemcpy(out, use, (size_t)B.ldh * B.ldh * sizeof(uint16_t), cudaMemcpyDeviceToHost));
  if (owner) *owner = own;
  if (tot_hess) *tot_hess = (int32_t)c.tot_hess;
  return 0;
}

// mlease_internal_request_refresh: problem b of the ADMM batch refactorises at the start point of its next x-update, as after a
// slow x-update (Ctrl::refresh_next), whatever the other problems do.  Lets a test make one lambda rebuild on its own.
int mlease_internal_request_refresh(mlease_session* s, int32_t b) {
  if (!s) return fail(MLEASE_ERR_INVALID, "null session");
  if (!s->batch) return fail(MLEASE_ERR_STATE, "mlease_admm_begin was not called");
  Batch& B = *s->batch;
  if (b < 0 || b >= B.nprob) return fail(MLEASE_ERR_INVALID, "problem index out of range");
  CK(cudaSetDevice(s->cfg.device));
  const int one = 1;
  CK(cudaMemcpy(&B.d_ctrl[b].refresh_next, &one, sizeof(int), cudaMemcpyHostToDevice));
  if ((int)B.mirror.size() > b) B.mirror[b].refresh_next = 1;   // the host's prediction of slot 0: a rebuild is due
  return 0;
}

// Test hooks, not part of the C ABI: the CSR Gram kernel of the batches allocated from now on -- 0 = picked from the data,
// CSR_GRAM_WGMMA (1), CSR_GRAM_SPARSE (2).  Must be called before the ADMM batch exists; the one-problem scratch batch (objective,
// timing) is rebuilt with the new setting on its next use.  The query returns the kind of the ADMM batch and of the scratch batch
// (0: no such batch, or no CSR Gram).
int mlease_internal_set_csr_gram(mlease_session* s, int32_t kind) {
  if (!s || kind < 0 || kind > CSR_GRAM_SPARSE) return fail(MLEASE_ERR_INVALID, "bad argument");
  if (s->batch) return fail(MLEASE_ERR_STATE, "the CSR Gram kernel is chosen when the ADMM batch is allocated: set it before");
  s->csr_gram_force = kind;
  delete s->scratch;
  s->scratch = nullptr;
  s->scratch_part = -1;
  return 0;
}

int mlease_internal_csr_gram(mlease_session* s, int32_t* batch_kind, int32_t* scratch_kind) {
  if (!s || !batch_kind || !scratch_kind) return fail(MLEASE_ERR_INVALID, "null argument");
  *batch_kind = s->batch ? s->batch->csr_gram : 0;
  *scratch_kind = s->scratch ? s->scratch->csr_gram : 0;
  return 0;
}

// Test hook, not part of the C ABI: on the current device, n 16x8 tiles D = A B^T (A: n x 16 x K, B: n x 8 x K, row-major,
// K a multiple of 4) accumulated as dgemm_kernel accumulates, once through DMMA m8n8k4 (D8) and once through m16n8k4 (D16).
int mlease_internal_dmma_shapes(const double* A, const double* B, int32_t n, int32_t K, double* D8, double* D16) {
  if (!A || !B || !D8 || !D16 || n <= 0 || K <= 0 || K % 4) return fail(MLEASE_ERR_INVALID, "bad argument");
  const size_t na = (size_t)n * 16 * K, nb = (size_t)n * 8 * K, nd = (size_t)n * 128;
  double* d = nullptr;
  CK(cudaMalloc(&d, (na + nb + 2 * nd) * sizeof(double)));
  cudaError_t e = cudaMemcpy(d, A, na * sizeof(double), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(d + na, B, nb * sizeof(double), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = dmma_shapes(d, d + na, n, K, d + na + nb, d + na + nb + nd, 0);
  if (e == cudaSuccess) e = cudaMemcpy(D8, d + na + nb, nd * sizeof(double), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess) e = cudaMemcpy(D16, d + na + nb + nd, nd * sizeof(double), cudaMemcpyDeviceToHost);
  cudaFree(d);
  CK(e);
  return 0;
}

}  // extern "C"

namespace {
enum { CS_RESET = 1, CS_INIT = 2, CS_PACK = 4, CS_CONSENSUS = 8 };
constexpr int CS_NVEC = 5, CS_NFVEC = 3, CS_NCTRL = 3;
// Every problem's K4 vectors and the session's z / exchange / diff to the device (h2d) or back, in the layout of
// mlease_internal_consensus.
int consensus_exchange(mlease_session* s, bool h2d, double* vec, float* fvec, double* z, double* exch, double* diff) {
  Batch& B = *s->batch;
  const int ldx = s->ldx;
  auto cp = [&](void* dev, void* host, size_t bytes) {
    return h2d ? cudaMemcpy(dev, host, bytes, cudaMemcpyHostToDevice) : cudaMemcpy(host, dev, bytes, cudaMemcpyDeviceToHost);
  };
  for (int b = 0; b < B.nprob; b++) {
    const Problem& p = B.h[b];
    double* v[CS_NVEC] = {p.beta, p.m, p.q, p.g_t, p.x_d};
    float* f[CS_NFVEC] = {p.u_f, p.uplusx_f, p.x_f};
    for (int i = 0; i < CS_NVEC; i++) CK(cp(v[i], vec + ((size_t)b * CS_NVEC + i) * ldx, (size_t)ldx * sizeof(double)));
    for (int i = 0; i < CS_NFVEC; i++) CK(cp(f[i], fvec + ((size_t)b * CS_NFVEC + i) * ldx, (size_t)ldx * sizeof(float)));
  }
  CK(cp(s->d_z, z, (size_t)s->L * ldx * sizeof(double)));
  CK(cp(s->d_exch, exch, ((size_t)s->L * s->Dt + 1) * sizeof(double)));
  CK(cp(s->d_diff, diff, (size_t)s->L * sizeof(double)));
  return 0;
}
}  // namespace

extern "C" {

// Test hook, not part of the C ABI: the consensus step (K4, k4_consensus.cu) of the begun ADMM batch on an injected state.
//   stages: CS_RESET (d_rho = rho of iteration 1, then admm_reset, as begin() runs them), CS_INIT (admm_init on the injected z, as
//   begin_initialized() runs it; not on an L1 session), CS_PACK (admm_pack into the session's exchange buffer), CS_CONSENSUS (the
//   session's own consensus_enqueue on that buffer, one stream synchronisation, consensus_finish, with s->iter = args[0] >= 1 and
//   s->liblinear_eps = (float)args[1]).  They run in that order.  stages = 0 injects and runs nothing: it reads the state back
//   (or only info when vec is NULL).
//   vec: nprob x 5 x ldx doubles (beta, m, q, g_t, x_d), fvec: nprob x 3 x ldx floats (u_f, uplusx_f, x_f), z: L x ldx, exch: L Dt + 1
//   (the last slot is the failed-fit count), diff: L, ctrl: nprob x 3 ints (Ctrl::hess_valid, skip_eval, k1_chunks); all in and out,
//   whole vectors, padding included, copied as bytes.  ctrl_raw (out, may be NULL): 2 x nprob x sizeof(Ctrl) bytes, every problem's
//   Ctrl just before the first stage and after the last one, with the three fields of ctrl zeroed in both.  wz (L x ldx), l1thr (L;
//   NULL on an L2 session) and rho (L): the z-weights, L1 thresholds and d_rho the kernels read, as the last stage left d_rho.
//   res (3 doubles, CS_CONSENSUS): maxdiff, the session's mindiff, stop.
//   info (12 ints): nprob, Dt, ldx, L, P, local partitions, CSR, fused K1 (gpart_f present), matrix-free, regularizer, k1_grid,
//   sizeof(Ctrl).
// Every kernel of K4 indexes by Dt, ldx, L and the problem count alone; k1_chunks is still refused beyond the partial rows the batch
// allocated.  Refused before any launch: no begun batch, a stage mask outside [0, 15], CS_INIT on an L1 session, CS_CONSENSUS
// without args or with args[0] < 1, a null array.  With stages set, the batch's x-update state is consumed (every problem is left
// done, as by mlease_internal_newton_stage): begin() again before iterating; s->iter, liblinear_eps, mindiff and last_maxdiff are
// restored.
int mlease_internal_consensus(mlease_session* s, int32_t stages, const double* args, double* vec, float* fvec, double* z, double* exch,
                              double* diff, int32_t* ctrl, uint8_t* ctrl_raw, double* wz, double* l1thr, double* rho, double* res,
                              int32_t* info) {
  if (!s || !info) return fail(MLEASE_ERR_INVALID, "null argument");
  if (!s->batch || !s->begun) return fail(MLEASE_ERR_STATE, "mlease_admm_begin was not called");
  Batch& B = *s->batch;
  const int nprob = B.nprob, L = s->L, ldx = s->ldx;
  const int32_t inf[12] = {nprob, s->Dt, ldx, L, s->P, (int)s->parts.size(), B.csr ? 1 : 0, B.h[0].gpart_f ? 1 : 0, B.matfree,
                           s->cfg.regularizer, B.k1_grid, (int)sizeof(Ctrl)};
  std::copy(inf, inf + 12, info);
  if (stages < 0 || stages > 15) return fail(MLEASE_ERR_INVALID, "stage mask out of range");
  if (stages == 0 && !vec) return 0;
  if (!vec || !fvec || !z || !exch || !diff || !ctrl || !wz || !rho || !res || (s->cfg.regularizer == 1 && !l1thr))
    return fail(MLEASE_ERR_INVALID, "null argument");
  if ((stages & CS_INIT) && s->cfg.regularizer != 2) return fail(MLEASE_ERR_INVALID, "admm_init runs on L2 sessions only (begin_initialized)");
  if ((stages & CS_CONSENSUS) && (!args || !(args[0] >= 1.0 && args[0] <= 1e9)))
    return fail(MLEASE_ERR_INVALID, "the consensus step needs args = {iter >= 1, liblinear_eps}");
  if (stages)
    for (int b = 0; b < nprob; b++)
      if (ctrl[3 * b + 2] < 0 || ctrl[3 * b + 2] > B.k1_grid) return fail(MLEASE_ERR_INVALID, "k1_chunks beyond the partial rows the batch allocated");
  CK(cudaSetDevice(s->cfg.device));
  std::vector<Ctrl> c0(nprob), c(nprob);
  auto raw = [&](int which) {   // Ctrl bytes without the three fields the caller exchanges
    if (!ctrl_raw) return;
    for (int b = 0; b < nprob; b++) {
      Ctrl x = c[b];
      x.hess_valid = 0; x.skip_eval = 0; x.k1_chunks = 0;
      std::memcpy(ctrl_raw + ((size_t)which * nprob + b) * sizeof(Ctrl), &x, sizeof(Ctrl));
    }
  };
  CK(cudaStreamSynchronize(s->stream));
  CK(cudaMemcpy(c0.data(), B.d_ctrl, (size_t)nprob * sizeof(Ctrl), cudaMemcpyDeviceToHost));
  c = c0;
  const int iter0 = s->iter;
  const float eps0 = s->liblinear_eps;
  const double mindiff0 = s->mindiff, maxdiff0 = s->last_maxdiff;
  int launches = 0;
  auto run = [&]() -> int {
    if (stages) {
      if (int rc = consensus_exchange(s, true, vec, fvec, z, exch, diff)) return rc;
      for (int b = 0; b < nprob; b++) { c[b].hess_valid = ctrl[3 * b]; c[b].skip_eval = ctrl[3 * b + 1]; c[b].k1_chunks = ctrl[3 * b + 2]; }
      CK(cudaMemcpy(B.d_ctrl, c.data(), (size_t)nprob * sizeof(Ctrl), cudaMemcpyHostToDevice));
    }
    raw(0);
    if (stages & CS_RESET) {
      for (int l = 0; l < L; l++) s->h_small[l] = rho_eff_for_iter(s, l, 1);
      CK(cudaMemcpyAsync(s->d_rho, s->h_small, L * sizeof(double), cudaMemcpyHostToDevice, s->stream));
      CK(admm_reset(B.d, nprob, L, s->d_z, ldx, s->d_rho, s->stream, &launches));
      CK(cudaStreamSynchronize(s->stream));   // h_small is reused below
    }
    if (stages & CS_INIT) CK(admm_init(B.d, nprob, s->d_z, ldx, s->stream, &launches));
    if (stages & CS_PACK) CK(admm_pack(B.d, (int)s->parts.size(), L, s->Dt, s->d_exch, s->stream, &launches));
    if (stages & CS_CONSENSUS) {
      s->iter = (int)args[0];
      s->liblinear_eps = (float)args[1];
      double md = 0;
      int32_t stop = 0;
      if (int rc = consensus_enqueue(s, s->d_exch)) return rc;
      CK(cudaStreamSynchronize(s->stream));
      consensus_finish(s, &md, &stop);
      res[0] = md; res[1] = s->mindiff; res[2] = stop;
    }
    CK(cudaStreamSynchronize(s->stream));
    if (int rc = consensus_exchange(s, false, vec, fvec, z, exch, diff)) return rc;
    CK(cudaMemcpy(c.data(), B.d_ctrl, (size_t)nprob * sizeof(Ctrl), cudaMemcpyDeviceToHost));
    for (int b = 0; b < nprob; b++) { ctrl[3 * b] = c[b].hess_valid; ctrl[3 * b + 1] = c[b].skip_eval; ctrl[3 * b + 2] = c[b].k1_chunks; }
    raw(1);
    CK(cudaMemcpy(wz, s->d_wz, (size_t)L * ldx * sizeof(double), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(rho, s->d_rho, (size_t)L * sizeof(double), cudaMemcpyDeviceToHost));
    if (s->d_l1thr) CK(cudaMemcpy(l1thr, s->d_l1thr, (size_t)L * sizeof(double), cudaMemcpyDeviceToHost));
    return 0;
  };
  const int rc = run();
  cudaStreamSynchronize(s->stream);
  s->iter = iter0; s->liblinear_eps = eps0; s->mindiff = mindiff0; s->last_maxdiff = maxdiff0;
  s->cnt.launches += launches;
  if (!stages) return rc;
  for (int b = 0; b < nprob; b++) {
    Ctrl& x = c0[b];
    x.done = 1; x.hess_valid = 0; x.need_solve = 0; x.need_hess = 0; x.have_dir = 0; x.bfgs_count = 0; x.h0_scale = 1.0;
    x.skip_eval = 0; x.refresh_next = 0; x.cg_active = 0; x.k1_chunks = 0; x.fail = 0;
  }
  CK(cudaMemcpy(B.d_ctrl, c0.data(), (size_t)nprob * sizeof(Ctrl), cudaMemcpyHostToDevice));
  B.mirror.clear();
  return rc;
}

}  // extern "C"
