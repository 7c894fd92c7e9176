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
