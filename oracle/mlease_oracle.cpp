// =====================================================================================
// mlease_oracle.cpp -- TEST INFRASTRUCTURE ONLY (never linked into, imported by or
// executed from the product path; see DESIGN.md "Oracle").
//
// A CPU restatement, in plain C++17 / double precision, of the ONE path of
// linkedin/ml-ease that this repo accelerates: the per-partition L2 logistic-regression
// x-update (TRON), the consensus z/u update of RegressionAdmmTrain, RegressionTest /
// RegressionTestLoglik scoring, RegressionNaiveTrain and the deterministic branches of
// RegressionPrepare / PartitionIdAssigner.  Every function cites the reference
// file:line it follows (paths relative to /root/reference/src/main/java/):
//   bw/    = de/bwaldvogel/liblinear/
//   llf/   = com/linkedin/mlease/regression/liblinearfunc/
//   jobs/  = com/linkedin/mlease/regression/jobs/
//   cons/  = com/linkedin/mlease/regression/consumers/
//   models/= com/linkedin/mlease/models/
//   utils/ = com/linkedin/mlease/utils/
//
// PARITY PINNING -- "parity unpinned" by the reference: it ships no golden vectors, known-answer tests or expected outputs,
// and cannot be built or run here (no JVM, see DESIGN.md).  This oracle is pinned by (1) finite differences of fun/grad/Hv/hessian,
// (2) scikit-learn's independent solver at the ADMM fixed point on the reference's only
// fixture (examples/sample-data.avro, decoded into tests/golden/), and (3) frozen outputs
// in tests/golden/.  It is therefore "pinned by independent implementation", not by
// reference-produced vectors -- stated in DESIGN.md.
//
// Two modes:  faithful = the reference's tolerance schedule (liblinearEpsilon 0.01f ...)
//             exact    = same flow and the same float32 rounding points, but TRON is run
//                        to machine precision (eps 1e-14), which is what the GPU path
//                        (exact Newton) is gated against.
// =====================================================================================
#include <algorithm>
#include <atomic>
#include <charconv>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

namespace {

using vecd = std::vector<double>;

thread_local std::string g_err;

// ---------------------------------------------------------------------------------------
// One partition's dataset, as LibLinearDataset holds it after finish()
// (llf/LibLinearDataset.java:413-484 addInstanceAvro, :586-658 finish):
//   * rows of (index,value) nodes sorted by index, value widened float->double (:461)
//   * response 0 -> -1 (:421-422); weight<0 rejected (:428-429)
//   * a bias node (index n, value bias=1.0) appended to every row when bias>0 (:592-614)
// Local feature indices: the reference numbers features in first-seen order (:467-479);
// here the locally PRESENT global features are numbered in ascending global id.  Only the
// summation order inside dot products differs (rounding-level; documented in DESIGN.md).
// ---------------------------------------------------------------------------------------
struct Dataset {
  int64_t l = 0;            // instances
  int n = 0;                // features incl. bias column if has_bias
  bool has_bias = true;
  std::vector<int64_t> rp;  // row pointers (l+1)
  std::vector<int32_t> ci;  // 0-based local feature index
  vecd v;                   // values
  std::vector<int> y;       // +1 / -1
  vecd weight, offset;
  std::vector<int32_t> local2global;  // size n (bias -> Dg)
};

// llf/LogisticRegressionL2.java:72-113 (constructor), Cp = positive_weight, Cn = 1
struct LrL2 {
  const Dataset& d;
  vecd weight, z, D;
  const double* priorMean;
  vecd priorVar_inv;
  double multiplier;
  int64_t passes = 0;  // sparse passes over X (cost model, SURVEY 8a)

  LrL2(const Dataset& ds, const double* pm, const double* pv, double mult, double Cp, double Cn)
      : d(ds), weight(ds.l), z(ds.l), D(ds.l), priorMean(pm), priorVar_inv(ds.n), multiplier(mult) {
    for (int64_t i = 0; i < d.l; i++) weight[i] = (d.y[i] == 1 ? Cp : Cn) * d.weight[i];
    for (int k = 0; k < d.n; k++) priorVar_inv[k] = 1.0 / pv[k];
  }
  // llf/LogisticRegressionL2.java:115-129
  void Xv(const double* v, double* out) {
    passes++;
    for (int64_t i = 0; i < d.l; i++) {
      double a = 0;
      for (int64_t j = d.rp[i]; j < d.rp[i + 1]; j++) a += v[d.ci[j]] * d.v[j];
      out[i] = a;
    }
  }
  // llf/LogisticRegressionL2.java:131-150
  void XTv(const double* v, double* out) {
    passes++;
    for (int k = 0; k < d.n; k++) out[k] = 0;
    for (int64_t i = 0; i < d.l; i++)
      for (int64_t j = d.rp[i]; j < d.rp[i + 1]; j++) out[d.ci[j]] += v[i] * d.v[j];
  }
  // llf/LogisticRegressionL2.java:156-193
  double fun(const double* w) {
    double f = 0;
    Xv(w, z.data());
    for (int64_t i = 0; i < d.l; i++) {
      z[i] += d.offset[i];
      double yz = d.y[i] * z[i];
      if (yz >= 0) f += weight[i] * std::log1p(std::exp(-yz));
      else f += weight[i] * (-yz + std::log1p(std::exp(yz)));
    }
    f = 2.0 * f;
    for (int k = 0; k < d.n; k++) {
      double t = w[k] - priorMean[k];
      f += t * t * priorVar_inv[k];
    }
    f /= 2.0;
    return multiplier * f;
  }
  // llf/LogisticRegressionL2.java:199-225 (consumes the scores fun() left in z[])
  void grad(const double* w, double* g) {
    for (int64_t i = 0; i < d.l; i++) {
      z[i] = 1 / (1 + std::exp(-d.y[i] * z[i]));
      D[i] = z[i] * (1 - z[i]);
      z[i] = weight[i] * (z[i] - 1) * d.y[i];
    }
    XTv(z.data(), g);
    for (int k = 0; k < d.n; k++) g[k] = ((w[k] - priorMean[k]) * priorVar_inv[k] + g[k]) * multiplier;
  }
  // llf/LogisticRegressionL2.java:231-248
  void Hv(const double* s, double* Hs) {
    vecd wa(d.l);
    Xv(s, wa.data());
    for (int64_t i = 0; i < d.l; i++) wa[i] = weight[i] * D[i] * wa[i];
    XTv(wa.data(), Hs);
    for (int k = 0; k < d.n; k++) Hs[k] = (s[k] * priorVar_inv[k] + Hs[k]) * multiplier;
  }
  // llf/LogisticRegressionL2.java:258-297 ; H is row-major n x n.  Returns false if a row
  // is not strictly sorted by index (the reference throws RuntimeException, :277).
  bool hessian(const double* w, double* H) {
    const int n = d.n;
    for (int k = 0; k < n; k++) H[(size_t)k * n + k] = priorVar_inv[k];
    for (int64_t i = 0; i < d.l; i++) {
      double score = 0;
      for (int64_t j = d.rp[i]; j < d.rp[i + 1]; j++) score += w[d.ci[j]] * d.v[j];
      score += d.offset[i];
      double p = 1.0 / (1.0 + std::exp(-d.y[i] * score));
      double Dii = weight[i] * p * (1 - p);
      int prev = INT32_MIN;
      for (int64_t a = d.rp[i]; a < d.rp[i + 1]; a++) {
        int m = d.ci[a];
        if (m <= prev) return false;
        prev = m;
        for (int64_t b = d.rp[i]; b < d.rp[i + 1]; b++) {
          int nn = d.ci[b];
          H[(size_t)m * n + nn] += Dii * d.v[a] * d.v[b];
          if (m == nn) break;
        }
      }
    }
    for (int m = 0; m < n; m++)
      for (int nn = m + 1; nn < n; nn++) H[(size_t)m * n + nn] = H[(size_t)nn * n + m];
    return true;
  }
  // llf/LogisticRegressionL2.java:304-327
  void hessianDiagonal(const double* w, double* H) {
    for (int k = 0; k < d.n; k++) H[k] = priorVar_inv[k];
    for (int64_t i = 0; i < d.l; i++) {
      double score = 0;
      for (int64_t j = d.rp[i]; j < d.rp[i + 1]; j++) score += w[d.ci[j]] * d.v[j];
      score += d.offset[i];
      double p = 1.0 / (1.0 + std::exp(-d.y[i] * score));
      double q = weight[i] * p * (1 - p);
      for (int64_t j = d.rp[i]; j < d.rp[i + 1]; j++) H[d.ci[j]] += q * d.v[j] * d.v[j];
    }
  }
};

// ---------------------------------------------------------------------------------------
// TRON, bw/Tron.java:30-252, including the LinkedIn change at :47-60 (w is NOT zeroed and
// the stopping reference gnorm1 is |grad f(0)|, not |grad f(w0)|).
// ---------------------------------------------------------------------------------------
// bw/Tron.java:220-252 (scaled 2-norm)
double euclid_norm(const vecd& x) {
  size_t n = x.size();
  if (n < 1) return 0;
  if (n == 1) return std::fabs(x[0]);
  double scale = 0, sum = 1;
  for (size_t i = 0; i < n; i++) {
    if (x[i] != 0) {
      double a = std::fabs(x[i]);
      if (scale < a) { double t = scale / a; sum = 1 + sum * (t * t); scale = a; }
      else { double t = a / scale; sum += t * t; }
    }
  }
  return scale * std::sqrt(sum);
}
double dot(const vecd& a, const vecd& b) { double p = 0; for (size_t i = 0; i < a.size(); i++) p += a[i] * b[i]; return p; }
void daxpy(double c, const vecd& x, vecd& y) { if (c == 0) return; for (size_t i = 0; i < x.size(); i++) y[i] += c * x[i]; }
void scal(double c, vecd& x) { if (c == 1.0) return; for (auto& e : x) e *= c; }

struct TronStats { int outer = 0; int cg_total = 0; double gnorm = 0, gnorm1 = 0, f = 0; };

// bw/Tron.java:126-179
int trcg(LrL2& fn, double delta, const vecd& g, vecd& s, vecd& r) {
  size_t n = g.size();
  vecd d(n), Hd(n);
  for (size_t i = 0; i < n; i++) { s[i] = 0; r[i] = -g[i]; d[i] = r[i]; }
  double cgtol = 0.1 * euclid_norm(g);
  int cg_iter = 0;
  double rTr = dot(r, r);
  while (true) {
    if (euclid_norm(r) <= cgtol) break;
    cg_iter++;
    fn.Hv(d.data(), Hd.data());
    double alpha = rTr / dot(d, Hd);
    daxpy(alpha, d, s);
    if (euclid_norm(s) > delta) {
      alpha = -alpha;
      daxpy(alpha, d, s);
      double std_ = dot(s, d), sts = dot(s, s), dtd = dot(d, d), dsq = delta * delta;
      double rad = std::sqrt(std_ * std_ + dtd * (dsq - sts));
      if (std_ >= 0) alpha = (dsq - sts) / (std_ + rad);
      else alpha = (rad - std_) / dtd;
      daxpy(alpha, d, s);
      alpha = -alpha;
      daxpy(alpha, Hd, r);
      break;
    }
    alpha = -alpha;
    daxpy(alpha, Hd, r);
    double rnew = dot(r, r);
    double beta = rnew / rTr;
    scal(beta, d);
    daxpy(1.0, r, d);
    rTr = rnew;
  }
  return cg_iter;
}

// bw/Tron.java:30-124
void tron(LrL2& fn, double eps, int max_iter, vecd& w, TronStats* st) {
  const double eta0 = 1e-4, eta1 = 0.25, eta2 = 0.75;
  const double sigma1 = 0.25, sigma2 = 0.5, sigma3 = 4;
  size_t n = w.size();
  double delta, snorm, alpha, f, fnew, prered, actred, gs;
  int search = 1, iter = 1;
  vecd s(n, 0.0), r(n), w_new(n), g(n);
  f = fn.fun(s.data());               // :51-54  gradient norm at w = 0
  fn.grad(s.data(), g.data());
  double gnorm1 = euclid_norm(g);
  f = fn.fun(w.data());               // :56-59  warm start kept
  fn.grad(w.data(), g.data());
  delta = euclid_norm(g);
  double gnorm = delta;
  if (gnorm <= eps * gnorm1) search = 0;
  iter = 1;
  int cg_total = 0;
  while (iter <= max_iter && search != 0) {
    int cg = trcg(fn, delta, g, s, r);
    cg_total += cg;
    w_new = w;
    daxpy(1.0, s, w_new);
    gs = dot(g, s);
    prered = -0.5 * (gs - dot(s, r));
    fnew = fn.fun(w_new.data());
    actred = f - fnew;
    snorm = euclid_norm(s);
    if (iter == 1) delta = std::min(delta, snorm);
    if (fnew - f - gs <= 0) alpha = sigma3;
    else alpha = std::max(sigma1, -0.5 * (gs / (fnew - f - gs)));
    if (actred < eta0 * prered) delta = std::min(std::max(alpha, sigma1) * snorm, sigma2 * delta);
    else if (actred < eta1 * prered) delta = std::max(sigma1 * delta, std::min(alpha * snorm, sigma2 * delta));
    else if (actred < eta2 * prered) delta = std::max(sigma1 * delta, std::min(alpha * snorm, sigma3 * delta));
    else delta = std::max(delta, std::min(alpha * snorm, sigma3 * delta));
    if (actred > eta0 * prered) {
      iter++;
      w = w_new;
      f = fnew;
      fn.grad(w.data(), g.data());
      gnorm = euclid_norm(g);
      if (gnorm <= eps * gnorm1) break;
    }
    if (f < -1.0e+32) break;
    if (std::fabs(actred) <= 0 && prered <= 0) break;
    if (std::fabs(actred) <= 1.0e-12 * std::fabs(f) && std::fabs(prered) <= 1.0e-12 * std::fabs(f)) break;
  }
  if (st) { st->outer = iter - 1; st->cg_total = cg_total; st->gnorm = gnorm; st->gnorm1 = gnorm1; st->f = f; }
}

// ---------------------------------------------------------------------------------------
// LibLinear.train, llf/LibLinear.java:221-312: pos/neg counts (:272-276) and
// Tron(func, epsilon*min(pos,neg)/nInstances, max_iter=10000) (:310-312, :97).
// param/priorMean/priorVar are already the dense local arrays initSetup (:476-497) builds.
// ---------------------------------------------------------------------------------------
// EXACT-mode only (not in the reference): TRON's own safeguards (bw/Tron.java:116-123) stop
// it once the predicted/actual reduction falls under 1e-12*|f|, which can leave |grad| at
// ~1e-7.  The exact oracle is meant to be the mathematical minimiser of the same
// sub-problem (what TRON converges to as eps -> 0), so it is polished with a few full
// Newton steps, each solved by plain CG on the reference's own Hv until |grad| stalls.
void newton_cg_polish(LrL2& fn, vecd& w) {
  size_t n = w.size();
  vecd g(n), s(n), r(n), d(n), Hd(n), wt(n);
  fn.fun(w.data()); fn.grad(w.data(), g.data());
  double gn = std::sqrt(dot(g, g));
  for (int it = 0; it < 6 && gn > 0; it++) {
    for (size_t i = 0; i < n; i++) { s[i] = 0; r[i] = -g[i]; d[i] = r[i]; }
    double rTr = dot(r, r), r0 = rTr;
    for (int k = 0; k < 2 * (int)n + 50 && rTr > 1e-22 * r0; k++) {
      fn.Hv(d.data(), Hd.data());
      double a = rTr / dot(d, Hd);
      daxpy(a, d, s); daxpy(-a, Hd, r);
      double rn = dot(r, r);
      scal(rn / rTr, d); daxpy(1.0, r, d);
      rTr = rn;
    }
    wt = w; daxpy(1.0, s, wt);
    vecd gt(n);
    fn.fun(wt.data()); fn.grad(wt.data(), gt.data());
    double gnt = std::sqrt(dot(gt, gt));
    if (!(gnt < gn)) { fn.fun(w.data()); fn.grad(w.data(), g.data()); break; }
    bool tiny = gnt > 0.5 * gn;
    w = wt; g = gt; gn = gnt;
    if (tiny) break;
  }
}

void liblinear_train(const Dataset& ds, vecd& param, const vecd& priorMean, const vecd& priorVar,
                     double epsilon, int max_iter, TronStats* st, int64_t* passes, bool polish = false) {
  int pos = 0;
  for (int64_t i = 0; i < ds.l; i++) if (ds.y[i] == 1) pos++;
  int neg = (int)ds.l - pos;
  LrL2 fn(ds, priorMean.data(), priorVar.data(), 1.0, 1.0, 1.0);
  double eps = epsilon * std::min(pos, neg) / (double)ds.l;
  tron(fn, eps, max_iter, param, st);
  if (polish) newton_cg_polish(fn, param);
  if (passes) *passes += fn.passes;
}

// Build one partition's Dataset from global CSR slices (float32 inputs as in
// RegressionPrepareOutput.avsc:28,31,32).  Returns false (g_err set) on the inputs the
// reference rejects with IOException (llf/LibLinearDataset.java:419-420, :428-429).
bool build_dataset(Dataset& ds, int Dg, int64_t r0, int64_t r1, const int64_t* rowptr, const int32_t* colidx,
                   const float* val, const int32_t* response, const float* weight, const float* offset,
                   bool has_bias, bool binary_feature) {
  ds.l = r1 - r0;
  ds.has_bias = has_bias;
  std::vector<int32_t> g2l(Dg, -1);
  std::vector<char> present(Dg, 0);
  for (int64_t i = r0; i < r1; i++)
    for (int64_t j = rowptr[i]; j < rowptr[i + 1]; j++) {
      if (colidx[j] < 0 || colidx[j] >= Dg) { g_err = "feature index out of range"; return false; }
      present[colidx[j]] = 1;
    }
  ds.local2global.clear();
  for (int k = 0; k < Dg; k++) if (present[k]) { g2l[k] = (int)ds.local2global.size(); ds.local2global.push_back(k); }
  int nfeat = (int)ds.local2global.size();
  ds.n = nfeat + (has_bias ? 1 : 0);
  if (has_bias) ds.local2global.push_back(Dg);
  ds.rp.assign(ds.l + 1, 0);
  ds.y.resize(ds.l); ds.weight.resize(ds.l); ds.offset.resize(ds.l);
  int64_t nnz = rowptr[r1] - rowptr[r0] + (has_bias ? ds.l : 0);
  ds.ci.resize(nnz); ds.v.resize(nnz);
  int64_t o = 0;
  std::vector<std::pair<int32_t, double>> row;
  for (int64_t i = r0; i < r1; i++) {
    int resp = response[i];
    if (resp != 1 && resp != 0 && resp != -1) { g_err = "response = " + std::to_string(resp) + " (only 1, 0, -1 are allowed)"; return false; }
    if (resp == 0) resp = -1;
    ds.y[i - r0] = resp;
    double w = weight ? (double)weight[i] : 1.0;
    if (w < 0) { g_err = "weight cannot < 0"; return false; }
    ds.weight[i - r0] = w;
    ds.offset[i - r0] = offset ? (double)offset[i] : 0.0;
    row.clear();
    for (int64_t j = rowptr[i]; j < rowptr[i + 1]; j++)
      row.emplace_back(g2l[colidx[j]], binary_feature ? 1.0 : (double)val[j]);
    std::stable_sort(row.begin(), row.end(), [](auto& a, auto& b) { return a.first < b.first; });  // :481-482
    for (auto& e : row) { ds.ci[o] = e.first; ds.v[o] = e.second; o++; }
    if (has_bias) { ds.ci[o] = nfeat; ds.v[o] = 1.0; o++; }
    ds.rp[i - r0 + 1] = o;
  }
  return true;
}

// Java's Float.toString / String.valueOf(float) (shortest round-trip digits, Java layout):
// used for model keys "1.0#3" (jobs/RegressionAdmmTrain.java:184,650) and for the
// "epsilon=<float>" option string (:702) that LibLinear re-parses as a double
// (llf/LibLinear.java:127 via utils/Util.java:147-157).
std::string java_float_to_string(float f) {
  if (std::isnan(f)) return "NaN";
  if (std::isinf(f)) return f > 0 ? "Infinity" : "-Infinity";
  if (f == 0) return std::signbit(f) ? "-0.0" : "0.0";
  char buf[64];
  auto res = std::to_chars(buf, buf + sizeof(buf), f, std::chars_format::scientific);
  std::string s(buf, res.ptr);  // d.ddddde[+-]xx
  bool negv = s[0] == '-';
  if (negv) s = s.substr(1);
  size_t epos = s.find('e');
  std::string mant = s.substr(0, epos);
  int ex = std::atoi(s.c_str() + epos + 1);
  std::string digits;
  for (char c : mant) if (c != '.') digits.push_back(c);
  std::string out;
  if (ex >= -3 && ex < 7) {
    if (ex >= 0) {
      std::string ip = digits.substr(0, std::min<size_t>(digits.size(), ex + 1));
      while ((int)ip.size() < ex + 1) ip.push_back('0');
      std::string fp = digits.size() > (size_t)ex + 1 ? digits.substr(ex + 1) : "0";
      out = ip + "." + fp;
    } else {
      out = "0." + std::string(-ex - 1, '0') + digits;
    }
  } else {
    std::string fp = digits.size() > 1 ? digits.substr(1) : "0";
    out = digits.substr(0, 1) + "." + fp + "E" + std::to_string(ex);
  }
  return negv ? "-" + out : out;
}
double java_float_via_string_to_double(float f) { return std::strtod(java_float_to_string(f).c_str(), nullptr); }

// Java String.hashCode over UTF-16 code units (ASCII keys here).
int32_t java_string_hash(const std::string& s) {
  uint32_t h = 0;
  for (unsigned char c : s) h = 31u * h + c;
  return (int32_t)h;
}

void parallel_for(int ntasks, int nthreads, const std::function<void(int)>& fn) {
  if (nthreads <= 1 || ntasks <= 1) { for (int t = 0; t < ntasks; t++) fn(t); return; }
  std::atomic<int> next{0};
  std::vector<std::thread> th;
  int nt = std::min(nthreads, ntasks);
  for (int k = 0; k < nt; k++) th.emplace_back([&] { for (int t; (t = next.fetch_add(1)) < ntasks;) fn(t); });
  for (auto& t : th) t.join();
}
}  // namespace

extern "C" {

const char* orc_last_error() { return g_err.c_str(); }

// ---- objective-level entry points (one partition; all local features present) -----------
// mode: 0 fun, 1 grad, 2 Hv (vec = direction), 3 hessian (out n*n), 4 hessianDiagonal.
// w/priorMean/priorVar are dense over the Dg+bias GLOBAL index space; features absent from
// the data are dropped exactly as initSetup does (llf/LibLinear.java:491-493) and the
// outputs for them are left 0 (grad/Hv) -- callers test with all features present.
int orc_objective(int mode, int Dg, int64_t nrows, const int64_t* rowptr, const int32_t* colidx, const float* val,
                  const int32_t* response, const float* weight, const float* offset, int has_bias,
                  const double* w, const double* priorMean, const double* priorVar, const double* vec,
                  double* out_scalar, double* out_vec) {
  Dataset ds;
  if (!build_dataset(ds, Dg, 0, nrows, rowptr, colidx, val, response, weight, offset, has_bias != 0, false)) return 1;
  int n = ds.n;
  vecd lw(n), lm(n), lv(n), lvec(n);
  for (int k = 0; k < n; k++) {
    int g = ds.local2global[k];
    lw[k] = w[g]; lm[k] = priorMean[g]; lv[k] = priorVar[g]; if (vec) lvec[k] = vec[g];
  }
  LrL2 fn(ds, lm.data(), lv.data(), 1.0, 1.0, 1.0);
  int Dt = Dg + (has_bias ? 1 : 0);
  if (mode == 0) { *out_scalar = fn.fun(lw.data()); return 0; }
  if (mode == 1) {
    vecd g(n);
    *out_scalar = fn.fun(lw.data());
    fn.grad(lw.data(), g.data());
    for (int k = 0; k < Dt; k++) out_vec[k] = 0;
    for (int k = 0; k < n; k++) out_vec[ds.local2global[k]] = g[k];
    return 0;
  }
  if (mode == 2) {
    vecd g(n), hs(n);
    fn.fun(lw.data()); fn.grad(lw.data(), g.data());
    fn.Hv(lvec.data(), hs.data());
    for (int k = 0; k < Dt; k++) out_vec[k] = 0;
    for (int k = 0; k < n; k++) out_vec[ds.local2global[k]] = hs[k];
    return 0;
  }
  if (mode == 3) {
    vecd H((size_t)n * n, 0.0);
    if (!fn.hessian(lw.data(), H.data())) { g_err = "The input features are not sorted by feature index values"; return 2; }
    for (size_t k = 0; k < (size_t)Dt * Dt; k++) out_vec[k] = 0;
    for (int a = 0; a < n; a++)
      for (int b = 0; b < n; b++) out_vec[(size_t)ds.local2global[a] * Dt + ds.local2global[b]] = H[(size_t)a * n + b];
    return 0;
  }
  if (mode == 4) {
    vecd H(n);
    fn.hessianDiagonal(lw.data(), H.data());
    for (int k = 0; k < Dt; k++) out_vec[k] = 0;
    for (int k = 0; k < n; k++) out_vec[ds.local2global[k]] = H[k];
    return 0;
  }
  g_err = "bad mode";
  return 3;
}

// ---- LibLinear.train for one partition (llf/LibLinear.java:221-383) ---------------------
// param in/out, priorMean, priorVar: dense over Dg+bias global index space.  Features of the
// global space absent from this partition get coeff = priorMean (llf/LibLinear.java:374-383)
// when prior_mean_has_key != 0 for them (NULL = all keys present in the priorMean map).
int orc_liblinear_train(int Dg, int64_t nrows, const int64_t* rowptr, const int32_t* colidx, const float* val,
                        const int32_t* response, const float* weight, const float* offset, int has_bias,
                        double* param, const double* priorMean, const double* priorVar, double epsilon, int max_iter,
                        int* out_outer, int* out_cg, double* out_gnorm, int64_t* out_passes) {
  Dataset ds;
  if (!build_dataset(ds, Dg, 0, nrows, rowptr, colidx, val, response, weight, offset, has_bias != 0, false)) return 1;
  int n = ds.n;
  vecd lw(n), lm(n), lv(n);
  for (int k = 0; k < n; k++) { int g = ds.local2global[k]; lw[k] = param[g]; lm[k] = priorMean[g]; lv[k] = priorVar[g]; }
  TronStats st; int64_t passes = 0;
  liblinear_train(ds, lw, lm, lv, epsilon, max_iter, &st, &passes, epsilon <= 1e-13);
  int Dt = Dg + (has_bias ? 1 : 0);
  std::vector<char> have(Dt, 0);
  for (int k = 0; k < n; k++) { param[ds.local2global[k]] = lw[k]; have[ds.local2global[k]] = 1; }
  for (int k = 0; k < Dt; k++) if (!have[k]) param[k] = priorMean[k];
  if (out_outer) *out_outer = st.outer;
  if (out_cg) *out_cg = st.cg_total;
  if (out_gnorm) *out_gnorm = st.gnorm;
  if (out_passes) *out_passes = passes;
  return 0;
}

// ---- RegressionAdmmTrain.run (jobs/RegressionAdmmTrain.java:130-522), L2 branch ----------
// Inputs are PREPARED records (RegressionPrepareOutput): partition p owns rows
// [part_rowstart[p], part_rowstart[p+1]).  Feature ids are global 0..Dg-1, intercept = Dg.
// lambdas/rhos: as parsed by Float.parseFloat (:166,170); rhos==NULL -> defaults (:174-181).
// mode 0 = faithful tolerance schedule (:279,338-346); 1 = exact (TRON eps 1e-14).
// Outputs (any may be NULL):
//   z_hist  [niters][L][Dg+1]  driver-side double z after each iteration (:365-404)
//   diff_hist [niters][L]      |z - z_prev|_inf per lambda (:456-472)
//   eps_hist [niters]          liblinearEpsilon used (:338-346)
//   x_last [P][L][Dg+1] double x of the last executed iteration; u_last [P][L][Dg+1] the
//   float u that iteration used; uplusx_last [P][L][Dg+1] float(u+x) it emitted (:709-711)
//   iters_done, passes (total sparse passes over X, all solves), inner_outer/inner_cg totals
// lambda order in outputs = the caller's order (the reducers' ascending sort :636-638 only
// decides which reducer gets which lambda).
int orc_admm_run(int P, int Dg, const int64_t* part_rowstart, const int64_t* rowptr, const int32_t* colidx,
                 const float* val, const int32_t* response, const float* weight, const float* offset, int L,
                 const float* lambdas, const float* rhos, int niters, double epsilon, int mode, int penalize_intercept,
                 int aggressive_decay, float rho_adapt_coefficient, int binary_feature, int nthreads, double* z_hist,
                 double* diff_hist, float* eps_hist, double* x_last, float* u_last, float* uplusx_last,
                 int* iters_done, int64_t* passes_out, int64_t* tron_outer_out, int64_t* tron_cg_out,
                 float initialize_boost_rate, float init_liblinear_epsilon, int regularizer, const float* lambda_map) {
  // regularizer: 2 = L2 z-update (:377-404), 1 = L1 "iterative thresholding" z-update (:406-451); anything else is the
  // driver's IOException (:144-147).  lambda_map: [Dg] or NULL, entries > 0 = the features listed in the lambda.map file
  // (ReadLambdaMapConsumer, cons/ReadLambdaMapConsumer.java:33-52; :186-196).  It only enters the L2 z-update weights
  // (:382-386) and the NaiveTrain fits of the initialize.boost.rate start (:248); the L1 branch builds a weightmap
  // (:411-415) but never uses it.
  if (regularizer != 1 && regularizer != 2) { g_err = "Only L1 and L2 regularization supported!"; return 1; }
  const int Dt = Dg + 1;
  for (int a = 0; a < L; a++)
    for (int b = a + 1; b < L; b++)
      if (lambdas[a] == lambdas[b]) { g_err = "duplicate lambda (HashMap<Float,Float> would collapse them)"; return 1; }
  std::vector<float> rho(L);
  for (int j = 0; j < L; j++) rho[j] = rhos ? rhos[j] : (lambdas[j] <= 100 ? 1.0f : 10.0f);  // :174-181
  std::vector<Dataset> ds(P);
  {
    std::atomic<int> bad{0};
    std::string err;
    std::mutex mu;
    parallel_for(P, nthreads, [&](int p) {
      if (!build_dataset(ds[p], Dg, part_rowstart[p], part_rowstart[p + 1], rowptr, colidx, val, response, weight, offset, true, binary_feature != 0)) {
        std::lock_guard<std::mutex> lk(mu); err = g_err; bad = 1;
      }
    });
    if (bad) { g_err = err; return 1; }
  }
  // key-presence of the String-keyed maps: a feature exists in z/u only once some
  // partition emitted it (iteration 1: z,u are empty maps, :155-185,:312)
  std::vector<char> in_any(Dt, 0);
  for (int p = 0; p < P; p++) for (int g : ds[p].local2global) in_any[g] = 1;
  std::vector<vecd> z(L, vecd(Dt, 0.0));                     // driver z, double (:155,365-404)
  std::vector<std::vector<float>> uplusx(P * L, std::vector<float>(Dt, 0.f));
  std::vector<std::vector<float>> u(P * L, std::vector<float>(Dt, 0.f));
  std::vector<vecd> x(P * L, vecd(Dt, 0.0));
  bool z_has_keys = false;                                   // false while z is the empty map
  double mindiff = 99999999;                                 // :278
  float liblinearEpsilon = 0.01f;                            // :279
  int64_t passes = 0, touter = 0, tcg = 0;
  std::mutex stat_mu;
  int i;
  int done = 0;
  // initialize.boost.rate > 0 (:236-266): z starts at the mean of per-partition RegressionNaiveTrain fits (prior variance
  // 1/lambda, intercept variance 100000 unless penalize.intercept, prior mean 0, init 0, liblinear.epsilon 0.01 unless the
  // job sets one: jobs/RegressionNaiveTrain.java:333-343,395), averaged by MeanLinearModelConsumer over the float models.
  if (initialize_boost_rate > 0 && regularizer == 2) {       // `initializeBoostRate > 0 && reg==2` (:236)
    std::vector<vecd> xi(P * L, vecd(Dt, 0.0));
    parallel_for(P * L, nthreads, [&](int t) {
      int p = t / L, l = t % L;
      const Dataset& d = ds[p];
      int n = d.n;
      vecd param(n, 0.0), pm(n, 0.0), pv(n, 1.0 / (double)lambdas[l]);
      for (int k = 0; k < n; k++) {
        const int g = d.local2global[k];
        if (g == Dg) { if (!penalize_intercept) pv[k] = 100000.0; }
        else if (lambda_map && lambda_map[g] > 0) pv[k] = 1.0 / (double)lambda_map[g];   // propsIni.put(LAMBDA_MAP, ...) (:248)
      }
      double eps = mode == 0 ? java_float_via_string_to_double(init_liblinear_epsilon) : 1e-14;
      TronStats st; int64_t ps = 0;
      liblinear_train(d, param, pm, pv, eps, mode == 0 ? 10000 : 100000, &st, &ps, mode != 0);
      for (int k = 0; k < n; k++) xi[t][d.local2global[k]] = param[k];
      std::lock_guard<std::mutex> lk(stat_mu);
      passes += ps; touter += st.outer; tcg += st.cg_total;
    });
    for (int l = 0; l < L; l++)
      for (int p = 0; p < P; p++)
        for (int k = 0; k < Dt; k++) z[l][k] = 1.0 * z[l][k] + (1.0 / P) * (double)(float)xi[p * L + l][k];
    z_has_keys = true;
  }
  for (i = 1; i <= niters; i++) {
    // rho.adapt.rate lives in the per-iteration JobConf: `conf = createJobConf(...)` (:286-291) builds a NEW JobConf every
    // iteration (com/linkedin/mapred/AbstractAvroJob.java:101-115), so the reducers' default 1.0f (:621) is back unless this
    // iteration sets it: the boost reaches the reducers of iteration 1 only (:313-316), rho.adapt.coefficient those of i > 1 (:323-327).
    float rhoAdaptRate = 1.0f;
    if (i == 1 && initialize_boost_rate > 0 && regularizer == 2) rhoAdaptRate = initialize_boost_rate;   // :313-316
    // u = float(uplusx) - z, written as float (:736-765, models/LinearModel.java:716)
    if (i == 1) {
      for (auto& uu : u) std::fill(uu.begin(), uu.end(), 0.f);   // empty map (:312)
    } else {
      for (int p = 0; p < P; p++)
        for (int l = 0; l < L; l++)
          for (int k = 0; k < Dt; k++) u[p * L + l][k] = (float)((double)uplusx[p * L + l][k] + (-1.0) * z[l][k]);
      if (rho_adapt_coefficient > 0) rhoAdaptRate = (float)std::exp((double)(-(i - 1) * rho_adapt_coefficient));  // :323-327 (Math.exp: double)
    }
    // z as the reducers see it: float (:330-331)
    std::vector<std::vector<float>> zf(L, std::vector<float>(Dt));
    for (int l = 0; l < L; l++) for (int k = 0; k < Dt; k++) zf[l][k] = (float)z[l][k];
    if (i > 1 && mindiff < 0.001 && !aggressive_decay) liblinearEpsilon = liblinearEpsilon / 10;  // :338-341
    else if (aggressive_decay && i > 5) liblinearEpsilon = liblinearEpsilon / 10;                 // :342-345
    if (eps_hist) eps_hist[i - 1] = liblinearEpsilon;
    double eps_option = (mode == 0) ? java_float_via_string_to_double(liblinearEpsilon) : 1e-14;  // :702
    int max_iter = (mode == 0) ? 10000 : 100000;
    const bool has_keys = z_has_keys;
    // reducers, one per (partition, lambda) (:642-718)
    parallel_for(P * L, nthreads, [&](int t) {
      int p = t / L, l = t % L;
      const Dataset& d = ds[p];
      double r = (double)rho[l];
      if (rhoAdaptRate != 1.0) r = r * (double)rhoAdaptRate;   // :653-658
      int n = d.n;
      vecd param(n), pm(n), pv(n, 1.0 / r);                     // priorVar == 1/rho for ALL incl. intercept (:705)
      for (int k = 0; k < n; k++) {
        int g = d.local2global[k];
        param[k] = (double)zf[l][g];                            // init = z (:692-693)
        pm[k] = -1.0 * (double)u[t][g] + 1.0 * (double)zf[l][g];  // z - u (:695-698)
      }
      TronStats st; int64_t ps = 0;
      liblinear_train(d, param, pm, pv, eps_option, max_iter, &st, &ps, mode != 0);
      vecd& xo = x[t];
      // coeff for features absent from this partition = priorMean if the key exists in
      // the priorMean map (llf/LibLinear.java:374-383); absent key -> not in model (0).
      for (int g = 0; g < Dt; g++) xo[g] = (has_keys && in_any[g]) ? (-1.0 * (double)u[t][g] + 1.0 * (double)zf[l][g]) : 0.0;
      for (int k = 0; k < n; k++) xo[d.local2global[k]] = param[k];
      for (int g = 0; g < Dt; g++) uplusx[t][g] = (float)(1.0 * (double)u[t][g] + 1.0 * xo[g]);  // :709-711
      std::lock_guard<std::mutex> lk(stat_mu);
      passes += ps; touter += st.outer; tcg += st.cg_total;
    });
    // driver: xbar, ubar (cons/MeanLinearModelConsumer.java:44-70 -- model += (1/nblocks)*new, in file order)
    double maxdiff = 0;
    mindiff = 99999999;
    for (int l = 0; l < L; l++) {
      vecd xbar(Dt, 0.0), ubar(Dt, 0.0);
      for (int p = 0; p < P; p++)
        for (int k = 0; k < Dt; k++) {
          xbar[k] = 1.0 * xbar[k] + (1.0 / P) * (double)(float)x[p * L + l][k];   // model read back as float (:708)
          ubar[k] = 1.0 * ubar[k] + (1.0 / P) * (double)u[p * L + l][k];
        }
      bool ubar_empty = (i == 1);                                                 // u file is empty at i==1
      float lf = lambdas[l], rf = rho[l];
      vecd lastz = z[l];
      vecd& zz = z[l];
      if (regularizer == 2) {
        double weight = (double)((float)(P * rf) / (lf + (float)(P * rf)));        // :381 -- float arithmetic
        for (int k = 0; k < Dg; k++) {
          double wk = weight;
          // weightmap.put(k, nblocks * r / (lambdaMap.get(k) + nblocks * r + 0.0)) (:384): float sum, then double division
          if (lambda_map && lambda_map[k] > 0) wk = (double)(float)(P * rf) / ((double)(lambda_map[k] + (float)(P * rf)) + 0.0);
          double vv = 0 + wk * xbar[k];                                            // :387 (z cleared :373)
          if (!ubar_empty) vv = 1.0 * vv + wk * ubar[k];                          // :388-391
          zz[k] = vv;
        }
        double ic = 1.0 * 0.0 + weight * xbar[Dg];
        if (!ubar_empty) ic = 1.0 * ic + weight * ubar[Dg];
        if (!penalize_intercept) ic = ubar_empty ? xbar[Dg] : xbar[Dg] + ubar[Dg];  // :392-403
        zz[Dg] = ic;
      } else {
        // L1 (:406-451): z = xbar (+ ubar), then "iterative thresholding" of the coefficients (the intercept is not in
        // getCoefficients()): val > t -> val - t, val < -t -> val + t, and -- as written in the reference -- values inside
        // [-t, t] are LEFT UNCHANGED (no zeroing).  t = l / (r * nblocks + 0.0): float product, double division (:409).
        const double thr = (double)lf / ((double)(rf * (float)P) + 0.0);
        for (int k = 0; k < Dg; k++) {
          double vv = 1.0 * 0.0 + 1.0 * xbar[k];
          if (!ubar_empty) vv = 1.0 * vv + 1.0 * ubar[k];
          if (vv > thr) vv = vv - thr;
          else if (vv < -thr) vv = vv + thr;
          zz[k] = vv;
        }
        double ic = 1.0 * 0.0 + 1.0 * xbar[Dg];
        if (!ubar_empty) ic = 1.0 * ic + 1.0 * ubar[Dg];
        if (!penalize_intercept) ic = ubar_empty ? xbar[Dg] : xbar[Dg] + ubar[Dg];  // :438-449 (the same value either way)
        zz[Dg] = ic;
      }
      double diff = 0;
      for (int k = 0; k < Dt; k++) diff = std::max(diff, std::fabs(1 * lastz[k] + (-1) * zz[k]));  // :463-464
      if (diff_hist) diff_hist[(size_t)(i - 1) * L + l] = diff;
      if (mindiff > diff) mindiff = diff;
      if (maxdiff < diff) maxdiff = diff;
      if (z_hist) std::memcpy(z_hist + ((size_t)(i - 1) * L + l) * Dt, zz.data(), sizeof(double) * Dt);
    }
    z_has_keys = true;
    done = i;
    if (maxdiff < epsilon && liblinearEpsilon <= 0.00001) break;                    // :493-496
  }
  for (int t = 0; t < P * L; t++) {
    if (x_last) std::memcpy(x_last + (size_t)t * Dt, x[t].data(), sizeof(double) * Dt);
    if (u_last) std::memcpy(u_last + (size_t)t * Dt, u[t].data(), sizeof(float) * Dt);
    if (uplusx_last) std::memcpy(uplusx_last + (size_t)t * Dt, uplusx[t].data(), sizeof(float) * Dt);
  }
  if (iters_done) *iters_done = done;
  if (passes_out) *passes_out = passes;
  if (tron_outer_out) *tron_outer_out = touter;
  if (tron_cg_out) *tron_cg_out = tcg;
  return 0;
}

// ---- RegressionNaiveTrain reducer (jobs/RegressionNaiveTrain.java:302-415) ---------------
// One independent fit per key.  keys own rows [key_rowstart[k], key_rowstart[k+1]).
// priorVar[k] = 1/lambdaMap[k] if given (lambda_map[g] > 0), intercept variance 100000
// unless penalize_intercept (:333-343), default variance 1/lambda, default mean prior_mean
// (:395); init = 0; epsilon default 0.001 (:149); bias = has_intercept (:360-364); keys with
// fewer rows than data_size_threshold are skipped (:379-382) -> skipped[k]=1, model 0.
// out_model [K][Dg+1] double (intercept last; 0 if !has_intercept).
int orc_naive_train(int K, int Dg, const int64_t* key_rowstart, const int64_t* rowptr, const int32_t* colidx,
                    const float* val, const int32_t* response, const float* weight, const float* offset, float lambda,
                    const float* lambda_map, float prior_mean, int penalize_intercept, int has_intercept,
                    float liblinear_epsilon, int data_size_threshold, int mode, int nthreads, double* out_model,
                    int* skipped, int64_t* passes_out) {
  const int Dt = Dg + 1;
  std::atomic<int> bad{0};
  std::string err; std::mutex mu;
  int64_t passes = 0;
  parallel_for(K, nthreads, [&](int k) {
    Dataset d;
    if (!build_dataset(d, Dg, key_rowstart[k], key_rowstart[k + 1], rowptr, colidx, val, response, weight, offset, has_intercept != 0, false)) {
      std::lock_guard<std::mutex> lk(mu); err = g_err; bad = 1; return;
    }
    double* out = out_model + (size_t)k * Dt;
    for (int g = 0; g < Dt; g++) out[g] = 0;
    if (d.l < data_size_threshold) { if (skipped) skipped[k] = 1; return; }
    if (skipped) skipped[k] = 0;
    int n = d.n;
    vecd param(n, 0.0), pm(n, (double)prior_mean), pv(n, 1.0 / (double)lambda);
    for (int j = 0; j < n; j++) {
      int g = d.local2global[j];
      if (g == Dg) { if (!penalize_intercept) pv[j] = 100000.0; }
      else if (lambda_map && lambda_map[g] > 0) pv[j] = 1.0 / (double)lambda_map[g];
    }
    double eps = mode == 0 ? java_float_via_string_to_double(liblinear_epsilon) : 1e-14;
    TronStats st; int64_t ps = 0;
    liblinear_train(d, param, pm, pv, eps, mode == 0 ? 10000 : 100000, &st, &ps, mode != 0);
    for (int j = 0; j < n; j++) out[d.local2global[j]] = param[j];
    std::lock_guard<std::mutex> lk(mu); passes += ps;
  });
  if (bad) { g_err = err; return 1; }
  if (passes_out) *passes_out = passes;
  return 0;
}

// ---- scoring: LinearModel.evalInstanceAvro(loglik=false) + RegressionTest (float cast) ---
// models/LinearModel.java:241-257 (eval: intercept term -log(n-1+n*exp(-b)), n = num_click_replicates),
// :491-554; jobs/RegressionTest.java:163 casts to float.  model: [Dg+1] double, intercept last.
int orc_score(int Dg, int64_t nrows, const int64_t* rowptr, const int32_t* colidx, const float* val, const float* offset,
              const double* model, int num_click_replicates, int binary_feature, float* pred) {
  for (int64_t i = 0; i < nrows; i++) {
    double result = -std::log(num_click_replicates - 1 + num_click_replicates * std::exp(-model[Dg]));
    for (int64_t j = rowptr[i]; j < rowptr[i + 1]; j++) result += model[colidx[j]] * (binary_feature ? 1.0 : (double)val[j]);
    double o = offset ? (double)offset[i] : 0.0;
    pred[i] = (float)(o + result);
  }
  return 0;
}

// ---- RegressionTestLoglik (jobs/RegressionTestLoglik.java:124-200) -----------------------
// mapper: per record loglik = -log1p(exp(-/+pred))*weight cast to float (:140-148);
// combiner: sums floats in double, casts the partial sum to float (:182-200), one combiner
// call per block of `combiner_block` records (<=0: no combiner); reducer: float(sum/n) (:158-176).
int orc_test_loglik(int64_t nrows, const int32_t* response, const float* pred, const float* weight,
                    int64_t combiner_block, float* out_loglik, double* out_count) {
  double sum = 0, n = 0;
  auto rec = [&](int64_t i) -> float {
    int r = response[i];
    double w = weight ? (double)weight[i] : 1.0, p = (double)pred[i];
    double ll = (r == 1) ? -std::log1p(std::exp(-p)) * w : -std::log1p(std::exp(p)) * w;
    return (float)ll;
  };
  for (int64_t i = 0; i < nrows; i++)
    if (response[i] != 1 && response[i] != 0 && response[i] != -1) { g_err = "response should be 1,0 or -1!"; return 1; }
  if (combiner_block <= 0) {
    for (int64_t i = 0; i < nrows; i++) { sum += rec(i); n += weight ? (double)weight[i] : 1.0; }
  } else {
    for (int64_t b = 0; b < nrows; b += combiner_block) {
      double s = 0, c = 0;
      for (int64_t i = b; i < std::min(nrows, b + combiner_block); i++) { s += rec(i); c += weight ? (double)weight[i] : 1.0; }
      sum += (float)s; n += c;
    }
  }
  *out_loglik = (float)(sum / n);
  *out_count = n;
  return 0;
}

// ---- driver-side per-iteration test loglik (jobs/RegressionAdmmTrain.java:766-811) -------
// double throughout, at most MAX_NTEST_EVENTS=1e6 records (:122,799), divides by sum(weight).
int orc_sample_test_loglik(int Dg, int64_t nrows, const int64_t* rowptr, const int32_t* colidx, const float* val,
                           const int32_t* response, const float* weight, const float* offset, const double* model,
                           int binary_feature, double* out) {
  double ll = 0, n = 0;
  int64_t nrec = 0;
  for (int64_t i = 0; i < nrows; i++) {
    double xb = -std::log(1 - 1 + 1 * std::exp(-model[Dg]));
    for (int64_t j = rowptr[i]; j < rowptr[i + 1]; j++) xb += model[colidx[j]] * (binary_feature ? 1.0 : (double)val[j]);
    xb += offset ? (double)offset[i] : 0.0;
    double w = weight ? (double)weight[i] : 1.0;
    ll += (response[i] == 1) ? -std::log1p(std::exp(-xb)) * w : -std::log1p(std::exp(xb)) * w;  // models/LinearModel.java:541-553
    n += w; nrec++;
    if (nrec >= 1000000) break;
  }
  *out = ll / n;
  return 0;
}

// ---- RegressionPrepare deterministic branches (jobs/RegressionPrepare.java:95-191) -------
// For record i with base key k0 (either the map.key field parsed as int, or an externally
// supplied draw of floor(random*nblocks) -- the reference's Math.random() at :112 is
// unseeded and cannot be reproduced): emits the list of partition ids and the prepared
// weight.  random_key_mode=1 and response==1 -> num_click_replicates copies on consecutive
// partitions mod nblocks (:172-186).  weight: positives (field `response`==1, :159) are
// divided by num_click_replicates, then cast to float (:163).
// out_keys must hold num_click_replicates ints per record; out_nkeys[i] = count.
int orc_prepare(int64_t nrows, const int32_t* base_key, const int32_t* response, const double* weight_in,
                int nblocks, int num_click_replicates, int random_key_mode, int32_t* out_keys, int32_t* out_nkeys,
                float* out_weight) {
  for (int64_t i = 0; i < nrows; i++) {
    double w = weight_in ? weight_in[i] : 1.0;
    if (response[i] == 1) w = w / num_click_replicates;
    out_weight[i] = (float)w;
    int32_t* ok = out_keys + i * num_click_replicates;
    if (random_key_mode && response[i] == 1) {
      int pid = base_key[i];
      for (int c = 0; c < num_click_replicates; c++) {
        if (pid >= nblocks) pid = pid - nblocks;
        ok[c] = pid;
        pid++;
      }
      out_nkeys[i] = num_click_replicates;
    } else {
      ok[0] = base_key[i];
      out_nkeys[i] = 1;
    }
  }
  return 0;
}

// ---- PartitionIdAssigner + NaivePartitioner ---------------------------------------------
// jobs/PartitionIdAssigner.java:62-88: distinct "<lambda>#<key>" strings get sequential ids
// in reducer arrival order = sorted Utf8 byte order (single reducer,
// jobs/RegressionNaiveTrain.java:121).  jobs/RegressionNaiveTrain.java:269-283: partition =
// id % R if mapped else abs(String.hashCode()) % R.
// keys: nkeys NUL-terminated strings packed back to back.  out_ids[i] = id of keys[i].
int orc_partition_ids(int nkeys, const char* keys_packed, const float* lambdas, int L, int num_reducers,
                      int32_t* out_ids /*[L][nkeys]*/, int32_t* out_partition /*[L][nkeys]*/,
                      int32_t* out_hash_partition /*[L][nkeys]*/) {
  std::vector<std::string> keys;
  const char* p = keys_packed;
  for (int i = 0; i < nkeys; i++) { keys.emplace_back(p); p += keys.back().size() + 1; }
  std::map<std::string, int> ids;  // std::map orders by unsigned byte compare == Utf8 order
  for (int l = 0; l < L; l++)
    for (auto& k : keys) ids[java_float_to_string(lambdas[l]) + "#" + k] = 0;
  int next = 0;
  for (auto& kv : ids) kv.second = next++;
  for (int l = 0; l < L; l++)
    for (int i = 0; i < nkeys; i++) {
      std::string full = java_float_to_string(lambdas[l]) + "#" + keys[i];
      int id = ids[full];
      out_ids[(size_t)l * nkeys + i] = id;
      if (out_partition) out_partition[(size_t)l * nkeys + i] = id % num_reducers;
      if (out_hash_partition) {
        int32_t h = java_string_hash(full);
        int32_t a = (h == INT32_MIN) ? h : std::abs(h);   // Math.abs(Integer.MIN_VALUE) stays negative
        out_hash_partition[(size_t)l * nkeys + i] = a % num_reducers;
      }
    }
  return 0;
}

// helpers exposed for tests
int orc_java_float_to_string(float f, char* buf, int buflen) {
  std::string s = java_float_to_string(f);
  if ((int)s.size() + 1 > buflen) return 1;
  std::memcpy(buf, s.c_str(), s.size() + 1);
  return 0;
}
int32_t orc_java_string_hash(const char* s) { return java_string_hash(s); }

}  // extern "C"
