// test_hooks.cu -- the mlease_internal_* test hooks declared in mlease_internal.h (not part of the C ABI), and the keyed-call
// budget and record that two of them expose.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <mutex>
#include <vector>

#include "mlease_internal.h"   // before host.cuh's hidden region: the hooks stay exported
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

namespace {

// The refusal of a hook on the ADMM batch: none yet, or (begun) one that mlease_admm_begin has not set up.
int need_batch(mlease_session* s, bool begun = true) {
  if (!s) return fail(MLEASE_ERR_INVALID, "null session");
  if (!s->batch || (begun && !s->begun)) return fail(MLEASE_ERR_STATE, "mlease_admm_begin was not called");
  return 0;
}

// The ADMM batch on loan to one hook; made after the hook's last refusal.  open(): the device made current, the stream drained and
// every problem's control block read into c0 (as before the hook) and c (the hook's working copy: pull / push).  From a successful
// open() on, every return path ends here: the stream synchronised, the launches counted and, when the hook consumes the x-update
// state, the batch parked as mlease_internal.h states (c0 with the fields below, mirror cleared, local_step refused until begin()).
// Raw CUDA calls only: the first error the hook recorded stays the one mlease_last_error reports.
class BatchLoan {
 public:
  BatchLoan(mlease_session* s, bool consume) : B(*s->batch), s_(s), consume_(consume) {}
  BatchLoan(const BatchLoan&) = delete;
  BatchLoan& operator=(const BatchLoan&) = delete;
  ~BatchLoan() {
    if (!open_) return;
    cudaStreamSynchronize(s_->stream);
    s_->cnt.launches += launches;
    if (!consume_) return;
    for (Ctrl& x : c0) {
      x.done = 1; x.hess_valid = 0; x.need_solve = 0; x.need_hess = 0; x.have_dir = 0; x.bfgs_count = 0; x.h0_scale = 1.0;
      x.skip_eval = 0; x.refresh_next = 0; x.cg_active = 0; x.k1_chunks = 0; x.fail = 0;
    }
    cudaMemcpy(B.d_ctrl, c0.data(), bytes(), cudaMemcpyHostToDevice);
    B.mirror.clear();
    s_->hook_consumed = true;
  }
  int open() {
    CK(cudaSetDevice(s_->cfg.device));
    CK(cudaStreamSynchronize(s_->stream));
    c0.resize(B.nprob);
    CK(cudaMemcpy(c0.data(), B.d_ctrl, bytes(), cudaMemcpyDeviceToHost));
    c = c0;
    open_ = true;
    return 0;
  }
  int pull() { CK(cudaMemcpy(c.data(), B.d_ctrl, bytes(), cudaMemcpyDeviceToHost)); return 0; }
  int push(const std::vector<Ctrl>& v) { CK(cudaMemcpy(B.d_ctrl, v.data(), bytes(), cudaMemcpyHostToDevice)); return 0; }
  int push() { return push(c); }

  Batch& B;
  std::vector<Ctrl> c0, c;
  int launches = 0;

 private:
  size_t bytes() const { return (size_t)B.nprob * sizeof(Ctrl); }
  mlease_session* s_;
  bool consume_, open_ = false;
};

// rows x Dt values of src (row-major), each row converted to T and zero-padded to ldx, to the device
template <class T, class S> int put_padded(T* dev, const S* src, int Dt, int ldx, int rows = 1) {
  std::vector<T> v((size_t)rows * ldx, T(0));
  for (int r = 0; r < rows; r++)
    for (int k = 0; k < Dt; k++) v[(size_t)r * ldx + k] = (T)src[(size_t)r * Dt + k];
  CK(cudaMemcpy(dev, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
  return 0;
}

// n values of a device array to out + off (out may be NULL: nothing), or n times `nan` for an inactive problem
template <class T> int get_or_nan(T* out, size_t off, const void* dev, size_t n, bool active, T nan) {
  if (!out) return 0;
  if (active) CK(cudaMemcpy(out + off, dev, n * sizeof(T), cudaMemcpyDeviceToHost));
  else std::fill(out + off, out + off + n, nan);
  return 0;
}

// a Dt x Dt H (row-major, lower triangle read) into an ldh x ldh Lc as chol_prep leaves it: lower triangle, identity on the
// padding, zero above
int put_lc(double* dev, const double* H, int Dt, int ldh) {
  std::vector<double> lc((size_t)ldh * ldh, 0.0);
  for (int i = 0; i < ldh; i++)
    for (int j = 0; j <= i; j++) lc[(size_t)i * ldh + j] = i < Dt ? H[(size_t)i * Dt + j] : (i == j ? 1.0 : 0.0);
  CK(cudaMemcpy(dev, lc.data(), lc.size() * sizeof(double), cudaMemcpyHostToDevice));
  return 0;
}

// the leading Dt x Dt block of an ldh x ldh Lc
int get_lc(double* out, const double* dev, int Dt, int ldh) {
  std::vector<double> lc((size_t)ldh * ldh);
  CK(cudaMemcpy(lc.data(), dev, lc.size() * sizeof(double), cudaMemcpyDeviceToHost));
  for (int i = 0; i < Dt; i++) std::memcpy(out + (size_t)i * Dt, &lc[(size_t)i * ldh], (size_t)Dt * sizeof(double));
  return 0;
}

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

constexpr int CS_NVEC = 5, CS_NFVEC = 3;
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

int mlease_internal_batch_hv(mlease_session* s, int32_t mode, const double* w, const double* v, double* out) {
  if (!s || !w || !v || !out || (mode != K1_HV && mode != K1_DIAG)) return fail(MLEASE_ERR_INVALID, "bad argument");
  if (int rc = need_batch(s, false)) return rc;
  Batch& B = *s->batch;
  if (!(B.csr && B.csr_fx)) return fail(MLEASE_ERR_INVALID, "Hessian-vector passes need CSR rows with strictly increasing column ids");
  const int nprob = B.nprob, ldx = s->ldx, Dt = s->Dt;
  BatchLoan loan(s, true);
  if (int rc = loan.open()) return rc;
  for (int b = 0; b < nprob; b++)
    if (int rc = put_padded(B.h[b].beta, w + (size_t)b * Dt, Dt, ldx)) return rc;
  for (Ctrl& x : loan.c) { x.skip_eval = 0; x.cg_active = 0; }
  if (int rc = loan.push()) return rc;
  CK(newton_begin(B.d, nprob, 1e-8, 1, 2, 1, 0, s->stream, &loan.launches));   // beta_t = float(w), every problem running
  CK(batch_k1(B, 1, s->stream, &loan.launches));                               // sqrt(d) at w
  CK(cudaStreamSynchronize(s->stream));
  for (int b = 0; b < nprob; b++)
    if (int rc = load_hv(B, b, v + (size_t)b * Dt, s->stream)) return rc;
  CK(batch_k1(B, 0, s->stream, &loan.launches, mode));
  CK(hv_reduce(B.d, nprob, Dt, 0, s->stream, &loan.launches));
  CK(cudaStreamSynchronize(s->stream));
  for (int b = 0; b < nprob; b++) CK(cudaMemcpy(out + (size_t)b * Dt, B.h[b].g_t, (size_t)Dt * sizeof(double), cudaMemcpyDeviceToHost));
  return 0;
}

int mlease_internal_batch_grad(mlease_session* s, const int32_t* active, const double* w, double* f_out, double* g_out, float* sd_out,
                               uint16_t* xt_out, int32_t* info) {
  if (!s || !active || !w || !f_out || !g_out || !info) return fail(MLEASE_ERR_INVALID, "null argument");
  if (int rc = need_batch(s)) return rc;
  Batch& B = *s->batch;
  if (sd_out && !(B.csr && B.csr_fx)) return fail(MLEASE_ERR_INVALID, "sqrt(d) goes to sdvec only on CSR batches with sorted unique rows");
  if (xt_out && B.csr && B.csr_fx) return fail(MLEASE_ERR_INVALID, "this batch emits no Xt operand (its Gram reads sdvec)");
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
  BatchLoan loan(s, true);
  if (int rc = loan.open()) return rc;
  for (int b = 0; b < nprob; b++)
    if (int rc = put_padded(B.h[b].beta_tf, w + (size_t)b * Dt, Dt, ldx)) return rc;
  for (int b = 0; b < nprob; b++) {
    Ctrl& x = loan.c[b];
    x.done = active[b] ? 0 : 1; x.skip_eval = 0; x.cg_active = active[b] ? 1 : 0; x.k1_chunks = 0;
  }
  if (int rc = loan.push()) return rc;
  CK(batch_k1(B, 1, s->stream, &loan.launches));
  CK(hv_reduce(B.d, nprob, Dt, 0, s->stream, &loan.launches));
  CK(cudaStreamSynchronize(s->stream));
  if (int rc = loan.pull()) return rc;
  const double nan = std::nan("");
  std::vector<double> fp;
  size_t row0 = 0;
  for (int b = 0; b < nprob; b++) {
    const Problem& p = B.h[b];
    const size_t n = (size_t)p.n;
    const int nct = loan.c[b].k1_chunks;
    f_out[b] = nan;
    if (active[b]) {
      inf[8 + b] = nct;
      fp.resize(std::max(1, nct));
      CK(cudaMemcpy(fp.data(), p.fpart, (size_t)nct * sizeof(double), cudaMemcpyDeviceToHost));
      double f = 0.0;
      for (int t = 0; t < nct; t++) f += fp[t];
      f_out[b] = f;
    }
    if (int rc = get_or_nan(g_out, (size_t)b * Dt, p.g_t, Dt, active[b], nan)) return rc;
    if (int rc = get_or_nan(sd_out, row0, p.sdvec, n, active[b], std::nanf(""))) return rc;
    if (int rc = get_or_nan(xt_out, row0 * B.Dp, p.Xt, n * B.Dp, active[b], (uint16_t)0x7FC0)) return rc;   // bf16 NaN
    row0 += n;
  }
  std::copy(inf.begin(), inf.end(), info);
  return 0;
}

int mlease_internal_batch_factor(mlease_session* s, const int32_t* mode, const double* H, const float* G, const double* q,
                                 const int32_t* order, int32_t norder, int32_t share, int32_t share_factor, double* L_out,
                                 double* Y_out, double* Hinv_out, double* Ldinv_out, int32_t* ctrl_out) {
  if (!s || !mode) return fail(MLEASE_ERR_INVALID, "null argument");
  if (int rc = need_batch(s)) return rc;
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
  const size_t hh = (size_t)ldh * ldh;
  BatchLoan loan(s, true);
  if (int rc = loan.open()) return rc;
  std::vector<double> qsave((size_t)nprob * Dt);
  for (int b = 0; b < nprob; b++)
    if (mode[b] == 2) CK(cudaMemcpy(&qsave[(size_t)b * Dt], B.h[b].q, (size_t)Dt * sizeof(double), cudaMemcpyDeviceToHost));
  DevMem ord_mem;
  auto run = [&]() -> int {
    // sentinel: all bits set (a NaN) everywhere, but 0 in the strict upper triangle of Yinv
    std::vector<double> ypat(hh);
    double nan; std::memset(&nan, 0xFF, sizeof(nan));
    for (int i = 0; i < ldh; i++)
      for (int j = 0; j < ldh; j++) ypat[(size_t)i * ldh + j] = j > i ? 0.0 : nan;
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
        if (int rc = put_lc(p.Lc, H + (size_t)b * Dt * Dt, Dt, ldh)) return rc;
      } else if (mode[b] == 2) {
        const float* g = G + (size_t)b * Dt * Dt;
        for (int i = 0; i < Dt; i++) std::memcpy(&gp[(size_t)i * Dp], g + (size_t)i * Dt, (size_t)Dt * sizeof(float));
        CK(cudaMemset(p.Hpart, 0, (size_t)B.gram_slices * Dp * Dp * sizeof(float)));
        CK(cudaMemcpy(p.Hpart, gp.data(), gp.size() * sizeof(float), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(p.q, q + (size_t)b * Dt, (size_t)Dt * sizeof(double), cudaMemcpyHostToDevice));
        ph[b].gram_unscale = 1.f;
      }
      Ctrl& x = loan.c[b];
      x.done = mode[b] ? 0 : 1; x.need_hess = 1; x.fail = 0; x.hess_valid = 0; x.tot_hess = 0;
    }
    CK(cudaMemcpy(B.d, ph.data(), (size_t)nprob * sizeof(Problem), cudaMemcpyHostToDevice));
    if (int rc = loan.push()) return rc;
    const Problem* d_hess = B.d;
    int n_hess = nprob;
    if (order) {
      std::vector<Problem> po(std::max(1, (int)norder));
      for (int i = 0; i < norder; i++) po[i] = ph[order[i]];
      Problem* d_ord;
      if (int rc = ord_mem.get(&d_ord, po.size(), false)) return rc;
      CK(cudaMemcpy(d_ord, po.data(), (size_t)norder * sizeof(Problem), cudaMemcpyHostToDevice));
      d_hess = d_ord; n_hess = norder;
    }
    int skip_prep = any2 ? 0 : 1;
    if (any1 && any2 && n_hess > 0) {
      std::vector<Ctrl> cp = loan.c;
      for (int b = 0; b < nprob; b++) if (mode[b] == 1) cp[b].need_hess = 0;
      if (int rc = loan.push(cp)) return rc;
      CK(cholesky_prep(d_hess, n_hess, ldh, share, s->stream, &loan.launches));
      CK(cudaStreamSynchronize(s->stream));
      if (int rc = loan.push()) return rc;
      skip_prep = 1;
    }
    if (n_hess > 0)
      if (int rc = batch_factor(B, d_hess, n_hess, share, share_factor != 0, skip_prep, s->stream, &loan.launches)) return rc;
    CK(cudaStreamSynchronize(s->stream));
    if (int rc = loan.pull()) return rc;
    for (int b = 0; b < nprob; b++) {
      const Problem& p = B.h[b];
      if (L_out)
        if (int rc = get_lc(L_out + (size_t)b * Dt * Dt, p.Lc, Dt, ldh)) return rc;
      if (Y_out) CK(cudaMemcpy(Y_out + (size_t)b * hh, p.Yinv, hh * sizeof(double), cudaMemcpyDeviceToHost));
      if (Hinv_out) CK(cudaMemcpy(Hinv_out + (size_t)b * hh, p.Hinv, hh * sizeof(double), cudaMemcpyDeviceToHost));
      if (Ldinv_out) CK(cudaMemcpy(Ldinv_out + (size_t)b * ldh * 32, p.Ldinv, (size_t)ldh * 32 * sizeof(double), cudaMemcpyDeviceToHost));
      if (ctrl_out) {
        int32_t* o = ctrl_out + 4 * (size_t)b;
        o[0] = loan.c[b].fail; o[1] = loan.c[b].done; o[2] = loan.c[b].hess_valid; o[3] = (int32_t)loan.c[b].tot_hess;
      }
    }
    return 0;
  };
  const int rc = run();
  // q and gram_unscale (the device Problem array) come back on every path, once the kernels are done
  cudaError_t e = cudaStreamSynchronize(s->stream);
  for (int b = 0; b < nprob; b++)
    if (mode[b] == 2 && e == cudaSuccess) e = cudaMemcpy(B.h[b].q, &qsave[(size_t)b * Dt], (size_t)Dt * sizeof(double), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(B.d, B.h.data(), (size_t)nprob * sizeof(Problem), cudaMemcpyHostToDevice);
  if (rc) return rc;
  CK(e);
  return 0;
}

int mlease_internal_direction(mlease_session* s, const int32_t* active, const double* g, const double* S, const double* Y,
                              const double* rho, const int32_t* count, const double* h0, const double* beta, double* dir_out,
                              double* phi0_out, double* dirnorm_out, double* beta_t_out) {
  if (!s || !active || !g || !S || !Y || !rho || !count || !h0 || !beta) return fail(MLEASE_ERR_INVALID, "null argument");
  if (int rc = need_batch(s)) return rc;
  Batch& B = *s->batch;
  if (B.matfree || !B.h[0].Hinv) return fail(MLEASE_ERR_INVALID, "a matrix-free session forms no factor");
  if (cholesky_factored_direction(B.ldh)) return fail(MLEASE_ERR_INVALID, "only systems up to 2048 (ldh) form the explicit inverse");
  const int nprob = B.nprob, Dt = s->Dt, ldx = s->ldx;
  for (int b = 0; b < nprob; b++)
    if (active[b] && count[b] < 0) return fail(MLEASE_ERR_INVALID, "bfgs_count must be >= 0");
  BatchLoan loan(s, true);
  if (int rc = loan.open()) return rc;
  const std::vector<double> nanv(ldx, std::nan(""));
  for (int b = 0; b < nprob; b++) {
    Ctrl& x = loan.c[b];
    x.done = active[b] ? 0 : 1;
    if (!active[b]) continue;
    const Problem& p = B.h[b];
    x.skip_eval = 1; x.k1_chunks = 0; x.have_dir = 0; x.hess_valid = 1; x.emit = 0; x.need_hess = 0; x.need_solve = 0;
    x.newton_steps = 0; x.evals = 0; x.fail = 0; x.bfgs_count = count[b]; x.h0_scale = h0[b];
    x.max_newton = std::max(1, s->max_newton);   // (a batch that never ran an x-update has 0: the decide kernel would stop it)
    if (int rc = put_padded(p.g_t, g + (size_t)b * Dt, Dt, ldx)) return rc;
    for (double* d : {p.beta_t, p.m, p.beta})
      if (int rc = put_padded(d, beta + (size_t)b * Dt, Dt, ldx)) return rc;
    CK(cudaMemcpy(p.dir, nanv.data(), (size_t)ldx * sizeof(double), cudaMemcpyHostToDevice));
    if (int rc = put_padded(p.bfgs_S, S + (size_t)b * BFGS_M * Dt, Dt, ldx, BFGS_M)) return rc;
    if (int rc = put_padded(p.bfgs_Y, Y + (size_t)b * BFGS_M * Dt, Dt, ldx, BFGS_M)) return rc;
    CK(cudaMemcpy(p.bfgs_rho, rho + (size_t)b * BFGS_M, BFGS_M * sizeof(double), cudaMemcpyHostToDevice));
  }
  if (int rc = loan.push()) return rc;
  CK(k1_reduce_decide(B.d, nprob, Dt, s->stream, &loan.launches, 0));
  CK(newton_solve(B.d, nprob, B.ldh, s->stream, &loan.launches, B.group_L));
  CK(cudaStreamSynchronize(s->stream));
  if (int rc = loan.pull()) return rc;
  const double nan = std::nan("");
  for (int b = 0; b < nprob; b++) {
    const Problem& p = B.h[b];
    if (int rc = get_or_nan(dir_out, (size_t)b * Dt, p.dir, Dt, active[b], nan)) return rc;
    if (int rc = get_or_nan(beta_t_out, (size_t)b * Dt, p.beta_t, Dt, active[b], nan)) return rc;
    if (phi0_out) phi0_out[b] = active[b] ? loan.c[b].phi0 : nan;
    if (dirnorm_out) dirnorm_out[b] = active[b] ? loan.c[b].dirnorm : nan;
  }
  return 0;
}

int mlease_internal_newton_stage(mlease_session* s, int32_t stages, int32_t spec, const double* begin_args, void* ctrl, double* vec,
                                 double* ring, float* fvec, const double* gpart, const double* fpart, int32_t nct_cap, int32_t* info,
                                 int32_t* cg_any) {
  if (!s || !info) return fail(MLEASE_ERR_INVALID, "null argument");
  if (int rc = need_batch(s)) return rc;
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
  BatchLoan loan(s, true);
  if (int rc = loan.open()) return rc;
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
        CK(cudaMemcpy(p.gpart, src, (size_t)nct * ldx * sizeof(double), cudaMemcpyHostToDevice));
      }
      CK(cudaMemcpy(p.fpart, fpart + (size_t)b * nct_cap, (size_t)nct * sizeof(double), cudaMemcpyHostToDevice));
    }
  }
  for (int b = 0; b < nprob; b++) stage_to_ctrl(in[b], loan.c[b]);
  if (int rc = loan.push()) return rc;
  int* launches = &loan.launches;
  if (stages & ST_BEGIN)
    CK(newton_begin(B.d, nprob, begin_args[0], (int)begin_args[1], (int)begin_args[2], begin_args[3] != 0.0, begin_args[4] != 0.0, s->stream, launches));
  if (stages & ST_DECIDE) CK(k1_reduce_decide(B.d, nprob, Dt, s->stream, launches, spec));
  if (stages & ST_CG_BEGIN) CK(cg_begin(B.d, nprob, s->stream, launches));
  if (stages & ST_CG_INIT) CK(cg_init(B.d, nprob, Dt, s->stream, launches));
  if (stages & ST_CG_STEP) CK(cg_step(B.d, nprob, Dt, s->stream, launches));
  if (stages & ST_CG_POLL) {
    CK(cg_poll(B.d, nprob, s->d_flag + 2, s->stream, launches));
    CK(cudaMemcpyAsync(s->h_flag + 2, s->d_flag + 2, sizeof(int), cudaMemcpyDeviceToHost, s->stream));
  }
  if (stages & ST_SOLVE) CK(newton_solve(B.d, nprob, B.ldh, s->stream, launches, B.group_L));
  if (stages & ST_FINISH) CK(newton_finish(B.d, nprob, Dt, s->stream, launches));
  CK(cudaStreamSynchronize(s->stream));
  if (stages & ST_CG_POLL) *cg_any = s->h_flag[2];
  if (int rc = loan.pull()) return rc;
  StageCtrl* out = static_cast<StageCtrl*>(ctrl);
  for (int b = 0; b < nprob; b++) ctrl_to_stage(loan.c[b], out[b]);
  return stage_exchange(B, ldx, false, vec, ring, fvec);
}

int mlease_internal_xupdate_trace(mlease_session* s, const double* args, const int32_t* spec, int32_t max_slots, void* ctrl_trace,
                                  double* vec_trace, double* ring_trace, float* fvec_trace, int32_t* slot_info, int32_t* nslots) {
  if (!s || !args || !spec || !ctrl_trace || !vec_trace || !ring_trace || !fvec_trace || !slot_info || !nslots) return fail(MLEASE_ERR_INVALID, "null argument");
  if (int rc = need_batch(s)) return rc;
  Batch& B = *s->batch;
  if (max_slots < 1 || max_slots > 400) return fail(MLEASE_ERR_INVALID, "max_slots out of range");
  if (B.nprob > 64) return fail(MLEASE_ERR_INVALID, "the slot trace follows batches of at most 64 problems");
  if (!(args[2] == 0.0 || args[2] == 1.0 || args[2] == 2.0)) return fail(MLEASE_ERR_INVALID, "policy must be 0, 1 or 2");
  const int policy = B.matfree ? 2 : (int)args[2];
  if (policy == 2 && !B.matfree) return fail(MLEASE_ERR_INVALID, "policy 2 needs a matrix-free batch");
  for (int i = 0; i < max_slots; i++)
    if (spec[i] && (policy != 0 || i == 0)) return fail(MLEASE_ERR_INVALID, "batch_xupdate speculates only under policy 0 and never on slot 0");
  const int nprob = B.nprob, ldx = s->ldx;
  const double xtol = args[0] > 0.0 ? args[0] : s->xtol;
  const int max_newton = args[1] > 0.0 ? (int)args[1] : s->max_newton;
  const size_t ring_n = 2 * (size_t)BFGS_M * ldx + 2 * BFGS_M;
  BatchLoan loan(s, false);   // the batch is left as after an x-update
  if (int rc = loan.open()) return rc;
  const std::vector<Ctrl>& c = loan.c;
  Profiler nop;
  double shared_flops = 0;
  auto record = [&](int entry) -> int {
    CK(cudaStreamSynchronize(s->stream));
    if (int rc = loan.pull()) return rc;
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
  CK(newton_begin(B.d, nprob, xtol, max_newton, policy, args[3] != 0.0, B.rebuild_is_expensive, s->stream, &loan.launches));
  if (int rc = record(0)) return rc;
  bool valid_now, valid_before = false;
  int flag_now = flags(&valid_now), flag_before = 2;   // nothing is known before slot 0: no speculation on slot 1 unless slot 0's outcome allows it
  if (!B.matfree) { valid_before = valid_now; flag_before = flag_now; }   // (the host's prediction of slot 0 equals what newton_begin left)
  int slots = 0;
  while ((flag_now & 1) && slots < max_slots) {
    const bool sp = spec[slots] && valid_before && !(flag_before & 2);
    const bool with_hess = !sp && (flag_now & 2) && !B.matfree;
    const SlotCtx x{s->stream, &nop, &loan.launches, B.d, nprob, 0, 0, &shared_flops, s->h_flag, s->d_flag, false};
    if (int rc = batch_slot(B, x, slots, with_hess, sp)) return rc;
    slot_info[2 * slots] = sp ? 1 : 0; slot_info[2 * slots + 1] = with_hess ? 1 : 0;
    valid_before = valid_now; flag_before = flag_now;
    if (int rc = record(slots + 1)) return rc;
    flag_now = flags(&valid_now);
    slots++;
  }
  *nslots = slots;
  B.mirror = c;
  return 0;
}

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
  if (int rc = put_lc(p.Lc, H, Dt, ldh)) return rc;
  Ctrl c; std::memset(&c, 0, sizeof(c)); c.need_hess = 1;
  CK(cudaMemcpy(B->d_ctrl, &c, sizeof(Ctrl), cudaMemcpyHostToDevice));
  int launches = 0;
  CK(cholesky_launch(B->d, 1, ldh, s->stream, &launches, 0, 1, 0));
  CK(cudaStreamSynchronize(s->stream));
  CK(cudaMemcpy(&c, B->d_ctrl, sizeof(Ctrl), cudaMemcpyDeviceToHost));
  if (L_out)
    if (int rc = get_lc(L_out, p.Lc, Dt, ldh)) return rc;
  if (Y_out) CK(cudaMemcpy(Y_out, p.Yinv, hh * sizeof(double), cudaMemcpyDeviceToHost));
  if (ysym_out) CK(cudaMemcpy(ysym_out, p.Ysym, hh * sizeof(uint16_t), cudaMemcpyDeviceToHost));
  if (int rc = reset_ctrl(*B)) return rc;
  s->cnt.launches += launches;
  if (c.fail) return fail(MLEASE_ERR_NUMERIC, "Hessian not positive definite");
  return 0;
}

int mlease_internal_factored_direction(mlease_session* s, const int32_t* active, const float* q, float* t_out, double* dir_out) {
  if (!s || !active || !q) return fail(MLEASE_ERR_INVALID, "null argument");
  if (!s->batch || !s->begun || s->iter < 1) return fail(MLEASE_ERR_STATE, "needs the ADMM batch after mlease_admm_begin and one iteration");
  Batch& B = *s->batch;
  if (B.matfree) return fail(MLEASE_ERR_INVALID, "a matrix-free session forms no factor");
  if (!cholesky_factored_direction(B.ldh) || !B.h[0].Ysym) return fail(MLEASE_ERR_INVALID, "only systems wider than 2048 (ldh) use the factored direction");
  const int nprob = B.nprob, ldx = s->ldx, Dt = s->Dt;
  BatchLoan loan(s, true);
  if (int rc = loan.open()) return rc;
  for (int b = 0; b < nprob; b++) { loan.c[b].done = active[b] ? 0 : 1; loan.c[b].need_solve = active[b] ? 1 : 0; }
  if (int rc = loan.push()) return rc;
  // qf = float(q) on [0, Dt) and 0 on the padding (as the decide kernel leaves it); tf NaN on [0, Dt); dir NaN
  const std::vector<float> tnan(Dt, std::nanf(""));
  const std::vector<double> dnan(ldx, std::nan(""));
  for (int b = 0; b < nprob; b++) {
    if (int rc = put_padded(B.h[b].qf, q + (size_t)b * Dt, Dt, ldx)) return rc;
    if (int rc = put_padded(B.h[b].tf, tnan.data(), Dt, ldx)) return rc;
    CK(cudaMemcpy(B.h[b].dir, dnan.data(), (size_t)ldx * sizeof(double), cudaMemcpyHostToDevice));
  }
  CK(newton_gemv_tri(B.d, nprob, B.ldh, B.group_L, s->stream));
  loan.launches += 2;   // its two phases
  CK(cudaStreamSynchronize(s->stream));
  for (int b = 0; b < nprob; b++) {
    if (t_out) CK(cudaMemcpy(t_out + (size_t)b * Dt, B.h[b].tf, (size_t)Dt * sizeof(float), cudaMemcpyDeviceToHost));
    if (dir_out) CK(cudaMemcpy(dir_out + (size_t)b * Dt, B.h[b].dir, (size_t)Dt * sizeof(double), cudaMemcpyDeviceToHost));
  }
  return 0;
}

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

int mlease_internal_partition_info(mlease_session* s, int32_t pid, double* out) {
  if (!s || !out) return fail(MLEASE_ERR_INVALID, "null argument");
  const PartData* pd;
  if (int rc = resident_part(s, pid, &pd)) return rc;
  const Problem& d = pd->data;
  const double v[PARTITION_INFO_LEN] = {(double)d.n, pd->csr ? (double)d.nnz_hint : 0.0, pd->csr ? 1.0 : 0.0, (double)s->ldx, (double)d.wmax,
                                        (double)d.vmax, (double)d.rowl1, d.gram_pairs, (double)d.csr_unique, d.bm_offs ? 1.0 : 0.0,
                                        d.gc_offs ? 1.0 : 0.0, d.sg_perm ? 1.0 : 0.0, (double)d.sg_S};
  std::copy(v, v + PARTITION_INFO_LEN, out);
  return 0;
}

int mlease_internal_partition_data(mlease_session* s, int32_t pid, int8_t* y, float* w, float* o, float* X_or_vals) {
  if (!s) return fail(MLEASE_ERR_INVALID, "null session");
  const PartData* pd;
  if (int rc = resident_part(s, pid, &pd)) return rc;
  const Problem& d = pd->data;
  CK(cudaStreamSynchronize(s->stream));
  const size_t n = (size_t)d.n;
  if (y) CK(cudaMemcpy(y, d.y, n, cudaMemcpyDeviceToHost));
  if (w) CK(cudaMemcpy(w, d.w, n * sizeof(float), cudaMemcpyDeviceToHost));
  if (o) CK(cudaMemcpy(o, d.o, n * sizeof(float), cudaMemcpyDeviceToHost));
  if (X_or_vals && pd->csr && d.nnz_hint > 0) CK(cudaMemcpy(X_or_vals, d.vals, (size_t)d.nnz_hint * sizeof(float), cudaMemcpyDeviceToHost));
  if (X_or_vals && !pd->csr) CK(cudaMemcpy(X_or_vals, d.X, n * s->ldx * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}

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

int mlease_internal_consensus(mlease_session* s, int32_t stages, const double* args, double* vec, float* fvec, double* z, double* exch,
                              double* diff, int32_t* ctrl, uint8_t* ctrl_raw, double* wz, double* l1thr, double* rho, double* res,
                              int32_t* info) {
  if (!s || !info) return fail(MLEASE_ERR_INVALID, "null argument");
  if (int rc = need_batch(s)) return rc;
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
  BatchLoan loan(s, stages != 0);   // stages = 0 reads only
  if (int rc = loan.open()) return rc;
  std::vector<Ctrl>& c = loan.c;
  auto raw = [&](int which) {   // Ctrl bytes without the three fields the caller exchanges
    if (!ctrl_raw) return;
    for (int b = 0; b < nprob; b++) {
      Ctrl x = c[b];
      x.hess_valid = 0; x.skip_eval = 0; x.k1_chunks = 0;
      std::memcpy(ctrl_raw + ((size_t)which * nprob + b) * sizeof(Ctrl), &x, sizeof(Ctrl));
    }
  };
  const int iter0 = s->iter;
  const float eps0 = s->liblinear_eps;
  const double mindiff0 = s->mindiff, maxdiff0 = s->last_maxdiff;
  auto run = [&]() -> int {
    if (stages) {
      if (int rc = consensus_exchange(s, true, vec, fvec, z, exch, diff)) return rc;
      for (int b = 0; b < nprob; b++) { c[b].hess_valid = ctrl[3 * b]; c[b].skip_eval = ctrl[3 * b + 1]; c[b].k1_chunks = ctrl[3 * b + 2]; }
      if (int rc = loan.push()) return rc;
    }
    raw(0);
    if (stages & CS_RESET) {
      for (int l = 0; l < L; l++) s->h_small[l] = rho_eff_for_iter(s, l, 1);
      CK(cudaMemcpyAsync(s->d_rho, s->h_small, L * sizeof(double), cudaMemcpyHostToDevice, s->stream));
      CK(admm_reset(B.d, nprob, L, s->d_z, ldx, s->d_rho, s->stream, &loan.launches));
      CK(cudaStreamSynchronize(s->stream));   // h_small is reused below
    }
    if (stages & CS_INIT) CK(admm_init(B.d, nprob, s->d_z, ldx, s->stream, &loan.launches));
    if (stages & CS_PACK) CK(admm_pack(B.d, (int)s->parts.size(), L, s->Dt, s->d_exch, s->stream, &loan.launches));
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
    if (int rc = loan.pull()) return rc;
    for (int b = 0; b < nprob; b++) { ctrl[3 * b] = c[b].hess_valid; ctrl[3 * b + 1] = c[b].skip_eval; ctrl[3 * b + 2] = c[b].k1_chunks; }
    raw(1);
    CK(cudaMemcpy(wz, s->d_wz, (size_t)L * ldx * sizeof(double), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(rho, s->d_rho, (size_t)L * sizeof(double), cudaMemcpyDeviceToHost));
    if (s->d_l1thr) CK(cudaMemcpy(l1thr, s->d_l1thr, (size_t)L * sizeof(double), cudaMemcpyDeviceToHost));
    return 0;
  };
  const int rc = run();
  s->iter = iter0; s->liblinear_eps = eps0; s->mindiff = mindiff0; s->last_maxdiff = maxdiff0;
  return rc;
}

}  // extern "C"
