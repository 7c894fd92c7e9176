// jobs_common.hpp -- what the job translation units of the host layer share: the job config, the record containers, the
// readers and writers of regression_jobs.cpp that other jobs reuse, and the registry through which jobs defined outside
// regression_jobs.cpp are reached by mlease_job_run.
#pragma once
#include <algorithm>
#include <atomic>
#include <exception>
#include <fstream>
#include <map>
#include <stdexcept>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/mlease_b200.h"
#include "avro_io.hpp"
#include "avro_walk.hpp"

namespace mlease_jobs {
using namespace mlease_host;

struct JobError : std::runtime_error { using std::runtime_error::runtime_error; };
[[noreturn]] void io_error(const std::string& m);
void ck(int rc);   // non-zero status of the device library -> JobError with its message

// ------------------------------------------------------------------------------------------ JobConfig
struct JobConfig {
  std::map<std::string, std::string> kv;
  static std::string trim(const std::string& s) {
    size_t a = s.find_first_not_of(" \t\r\n"), b = s.find_last_not_of(" \t\r\n");
    return a == std::string::npos ? "" : s.substr(a, b - a + 1);
  }
  // java.util.Properties subset: key=value | key:value | key value, '#'/'!' comments, trailing '\' continuation
  static JobConfig load(const std::string& file) {
    std::ifstream f(file);
    if (!f) io_error("cannot open job config " + file);
    JobConfig c;
    std::string line, acc;
    while (std::getline(f, line)) {
      std::string t = trim(line);
      if (acc.empty() && (t.empty() || t[0] == '#' || t[0] == '!')) continue;
      if (!t.empty() && t.back() == '\\') { acc += t.substr(0, t.size() - 1); continue; }
      acc += t;
      size_t p = acc.find_first_of("=: \t");
      std::string k = p == std::string::npos ? acc : acc.substr(0, p);
      std::string v = p == std::string::npos ? "" : acc.substr(p);
      size_t q = v.find_first_not_of(" \t");
      if (q != std::string::npos && (v[q] == '=' || v[q] == ':')) v = v.substr(q + 1);
      c.kv[trim(k)] = trim(v);
      acc.clear();
    }
    return c;
  }
  bool has(const std::string& k) const { return kv.count(k) > 0; }
  std::string get(const std::string& k) const {
    auto it = kv.find(k);
    if (it == kv.end()) io_error("Key " + k + " is not in the job config");   // JobConfig.getString(key) on a missing key
    return it->second;
  }
  std::string get(const std::string& k, const std::string& d) const { auto it = kv.find(k); return it == kv.end() ? d : it->second; }
  int get_int(const std::string& k) const { return std::stoi(get(k)); }
  int get_int(const std::string& k, int d) const { return has(k) ? std::stoi(get(k)) : d; }
  double get_double(const std::string& k, double d) const { return has(k) ? std::stod(get(k)) : d; }
  float get_float(const std::string& k, float d) const { return has(k) ? std::stof(get(k)) : d; }
  bool get_bool(const std::string& k, bool d) const {
    if (!has(k)) return d;
    std::string v = get(k);
    std::transform(v.begin(), v.end(), v.begin(), ::tolower);
    return v == "true" || v == "1";
  }
  std::vector<std::string> get_list(const std::string& k, const std::string& sep = ",") const {
    std::vector<std::string> out;
    std::string v = get(k);
    size_t st = 0;
    while (true) {
      size_t p = v.find(sep, st);
      std::string tok = trim(v.substr(st, p == std::string::npos ? std::string::npos : p - st));
      if (!tok.empty()) out.push_back(tok);
      if (p == std::string::npos) break;
      st = p + sep.size();
    }
    return out;
  }
};

struct Dictionary {
  std::unordered_map<std::string, int> idx;
  std::vector<std::string> names;
  int add(const std::string& n) { auto it = idx.find(n); if (it != idx.end()) return it->second; int i = (int)names.size(); idx.emplace(n, i); names.push_back(n); return i; }
  int find(const std::string& n) const { auto it = idx.find(n); return it == idx.end() ? -1 : it->second; }
};

// one prepared record stream in CSR form (global dictionary ids)
struct Rows {
  std::vector<std::string> key;
  std::vector<int32_t> response;
  std::vector<float> weight, offset;
  std::vector<int64_t> rowptr{0};
  std::vector<int32_t> colidx;
  std::vector<float> vals;
  size_t n() const { return response.size(); }
};

inline const std::string INTERCEPT = "(INTERCEPT)";

// Avro binary primitives for the writers that encode records directly (no Value tree)
inline void put_long(std::string& o, int64_t v) {
  uint64_t z = ((uint64_t)v << 1) ^ (uint64_t)(v >> 63);
  while (z & ~0x7FULL) { o.push_back((char)((z & 0x7F) | 0x80)); z >>= 7; }
  o.push_back((char)z);
}
inline void put_str(std::string& o, const char* p, size_t n) { put_long(o, (int64_t)n); o.append(p, n); }
inline void put_float(std::string& o, float f) { o.append(reinterpret_cast<const char*>(&f), 4); }

// the (name, term) strings of a feature key (name, or name\u0001term)
inline void put_feature_key(std::string& o, const std::string& key) {
  const size_t p = key.find('\x01');
  if (p == std::string::npos) { put_str(o, key.data(), key.size()); put_long(o, 0); }
  else { put_str(o, key.data(), p); put_str(o, key.data() + p + 1, key.size() - p - 1); }
}

// The (name, term) part of every feature record of a model list in Avro binary, intercept first (models/LinearModel.java:697-720):
// built once per file, after which a model is a run of [prefix, 4-byte float] appends instead of a Value tree per feature.
struct FeaturePrefix {
  std::string bytes;
  std::vector<size_t> off;   // [D + 2]: entry 0 = intercept, entry k + 1 = dictionary feature k
  explicit FeaturePrefix(const Dictionary& dict) {
    off.push_back(bytes.size()); put_feature_key(bytes, INTERCEPT);
    for (auto& n : dict.names) { off.push_back(bytes.size()); put_feature_key(bytes, n); }
    off.push_back(bytes.size());
  }
  // one model list: coef[D] (intercept) first, then coef[0..D)
  void encode(std::string& o, const float* coef) const {
    const size_t D = off.size() - 2;
    put_long(o, (int64_t)(D + 1));
    o.append(bytes, off[0], off[1] - off[0]); put_float(o, coef[D]);
    for (size_t k = 0; k < D; k++) { o.append(bytes, off[k + 1], off[k + 2] - off[k + 1]); put_float(o, coef[k]); }
    put_long(o, 0);
  }
  // the intercept and the listed features only (a NaiveTrain model holds the features its key's rows list, llf/LibLinear.java:343-350)
  void encode_subset(std::string& o, const float* coef, const std::vector<int32_t>& subset) const {
    const size_t D = off.size() - 2;
    put_long(o, (int64_t)(subset.size() + 1));
    o.append(bytes, off[0], off[1] - off[0]); put_float(o, coef[D]);
    for (int32_t k : subset) { o.append(bytes, off[(size_t)k + 1], off[(size_t)k + 2] - off[(size_t)k + 1]); put_float(o, coef[k]); }
    put_long(o, 0);
  }
};
extern const char* SCHEMA_TEST_LOGLIK;
extern const char* SCHEMA_MODEL_WITH_VAR;

// regression_jobs.cpp
std::string java_float_to_string(float f);
double num_of(const Value& v);
const Value* field(const Value& rec, const Schema& s, const std::string& name);
const Schema& rec_schema(const SchemaP& s);
bool host_generic_ingest();
// raw (unprepared) records of one file -> rows; item_key non-empty: rows.key = data.get(item_key).toString()
void read_raw(const std::string& file, Dictionary& dict, Rows& rows, bool binary_feature, const std::string& item_key = "");
// prepared records (RegressionPrepareOutput) of every file under path -> rows (appended), global dictionary ids
void read_prepared(const std::string& path, Dictionary& dict, Rows& rows, bool binary_feature);
std::vector<std::pair<std::string, float>> read_lambda_map_entries(const std::string& path);
// {name, term, value} feature record of a model list (Value tree), value cast to float
Value feature_value(const std::string& key, float v);
std::map<std::string, std::unordered_map<std::string, double>> read_linear_models(const std::string& path, bool last_wins = false);
// RegressionTest-style output schema: input fields with unions removed + pred:float (+ predVar:float)
std::string test_output_schema(const SchemaP& in, const char* name = "AdmmTestOutput", const char* ns = nullptr, bool pred_var = false);
// (response, pred, weight) of the scored records of one file (RegressionTest / ItemModelGridTest output), appended; weight 1 when
// absent
void read_scored(const std::string& f, std::vector<int32_t>& resp, std::vector<float>& pred, std::vector<float>& weight);
// a record's bytes with the union branch indices dropped; throws NotPlain when the record is not plain
struct NotPlain {};
void transcode_plain(const Plan& pl, const uint8_t*& p, const uint8_t* e, std::string& o);

// gpu.devices = 0,1,2,...  (falls back to the single gpu.device, default 0)
std::vector<int32_t> gpu_devices(const JobConfig& c);
// Integer.parseInt; RegressionAdmmTrain's lambda list (Float.parseFloat); lambda.map as a dense [D] vector over dict (0 = not listed)
int java_parse_int(const std::string& s);
std::vector<float> parse_lambdas(const JobConfig& c);
std::vector<float> read_lambda_map(const std::string& path, const Dictionary& dict);

// ------------------------------------------------------------------------------------------ keyed jobs on several GPUs
// Keys are independent, so a keyed job (NaiveTrain, ItemModelTrain, ItemModelTest, ItemModelGridTest) cuts them into one contiguous range per device,
// runs the single-device library call of each range on its own thread, and writes the results into disjoint slices of its output.
//
// shard_keys: cuts[s] .. cuts[s + 1] is shard s's key range, balanced by the estimated cost of a key, rows * (D + 1)^2 + nnz (a
// shard's cost exceeds the mean by less than the largest key's).  Ranges may be empty when there are more shards than keys.
inline std::vector<int> shard_keys(const std::vector<int64_t>& krs, const std::vector<int64_t>& rowptr, int D, int nshards) {
  const int K = (int)krs.size() - 1;
  const double d2 = (double)(D + 1) * (double)(D + 1);
  std::vector<double> pre(K + 1, 0.0);
  for (int k = 0; k < K; k++)
    pre[k + 1] = pre[k] + (double)(krs[k + 1] - krs[k]) * d2 + (double)(rowptr[krs[k + 1]] - rowptr[krs[k]]);
  std::vector<int> cuts{0};
  int k = 0;
  for (int s = 1; s < nshards; s++) {
    const double target = pre[K] * s / nshards;
    while (k < K && pre[k] < target) k++;   // the key that crosses the target closes the shard
    cuts.push_back(k);
  }
  cuts.push_back(K);
  return cuts;
}

// The rows of keys [k0, k1) of a CSR grouped by key: their own key_rowstart and rowptr (both from 0); row0 / nz0 locate the
// range's rows and entries in the arrays of the whole job.
struct KeySlice {
  std::vector<int64_t> krs, rowptr;
  int64_t row0 = 0, nz0 = 0;
  KeySlice(const std::vector<int64_t>& krs_all, const std::vector<int64_t>& rp_all, int k0, int k1) {
    row0 = krs_all[k0]; nz0 = rp_all[row0];
    for (int k = k0; k <= k1; k++) krs.push_back(krs_all[k] - row0);
    for (int64_t i = row0; i <= krs_all[k1]; i++) rowptr.push_back(rp_all[i] - nz0);
  }
};

// fn(device, k0, k1) for every non-empty shard of cuts, one thread per device (on the calling thread when there is one device).
// Every thread is joined; the first failing shard's error (in shard order) is the job's.
template <class F> void run_shards(const std::vector<int32_t>& devs, const std::vector<int>& cuts, F fn) {
  if (devs.size() == 1) { fn(devs[0], cuts[0], cuts[1]); return; }
  std::vector<std::exception_ptr> err(devs.size());
  std::vector<std::thread> ts;
  for (size_t s = 0; s < devs.size(); s++) {
    if (cuts[s] == cuts[s + 1]) continue;
    try {
      ts.emplace_back([&, s] { try { fn(devs[s], cuts[s], cuts[s + 1]); } catch (...) { err[s] = std::current_exception(); } });
    } catch (...) {   // no thread for this shard: the job fails, after the running shards are joined
      err[s] = std::current_exception();
      break;
    }
  }
  for (auto& t : ts) t.join();
  for (auto& e : err) if (e) std::rethrow_exception(e);
}

// ------------------------------------------------------------------------------------------ ItemModelTest and ItemModelGridTest
// The records of one file as union-free bytes (transcode_plain), one string per record.  False when the schema or a record is
// not plain; the generic encoder then writes the job's output.
inline bool plain_records(const std::string& file, std::vector<std::string>& out) {
  AvroFile af(file);
  Plan plan;
  try { plan = plan_build(*af.schema()); } catch (const std::exception&) { return false; }
  {
    const Plan* p = &plan;
    while (p->type == Schema::Union) { const Plan* nx = nullptr; for (auto& k : p->kids) if (k.type != Schema::Null) { nx = &k; break; } if (!nx) return false; p = nx; }
    if (p->type != Schema::Record) return false;
  }
  const size_t nb = af.num_blocks();
  std::vector<std::vector<std::string>> parts(nb);
  std::atomic<bool> plain{true};
  parallel_blocks(nb, host_threads(), [&](size_t b) {
    if (!plain.load()) return;
    const std::string data = af.block_data(b);
    const uint8_t* p = reinterpret_cast<const uint8_t*>(data.data());
    const uint8_t* e = p + data.size();
    try {
      for (int64_t q = 0; q < af.block_records(b); q++) { std::string o; transcode_plain(plan, p, e, o); parts[b].push_back(std::move(o)); }
    } catch (const NotPlain&) { plain.store(false); }
  });
  if (!plain.load()) return false;
  for (auto& v : parts) for (auto& r : v) out.push_back(std::move(r));
  return true;
}

// Records grouped by item key in Avro string order (unsigned bytes), input order inside a key (jobs/ItemModelTest.java:65-248):
// position q holds record order[q]; keys knames with their rows [krs[k], krs[k+1]) of the CSR (rp, ci, vv) and offsets oo.
struct KeyedRows {
  std::vector<size_t> order;
  std::vector<std::string> knames;
  std::vector<int64_t> krs{0}, rp{0};
  std::vector<int32_t> ci;
  std::vector<float> vv, oo;
  explicit KeyedRows(const Rows& rows) {
    const size_t n = rows.n();
    order.resize(n);
    for (size_t i = 0; i < n; i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return rows.key[a] < rows.key[b]; });
    for (size_t q = 0; q < n; q++) {
      const size_t i = order[q];
      if (q > 0 && rows.key[i] != rows.key[order[q - 1]]) krs.push_back((int64_t)q);
      if (q == 0 || rows.key[i] != rows.key[order[q - 1]]) knames.push_back(rows.key[i]);
      for (int64_t j = rows.rowptr[i]; j < rows.rowptr[i + 1]; j++) { ci.push_back(rows.colidx[j]); vv.push_back(rows.vals[j]); }
      rp.push_back((int64_t)ci.size());
      oo.push_back(rows.offset[i]);
    }
    if (n) krs.push_back((int64_t)n);
  }
};

// Lists of L x K models as a CSR over (l, key), m = l*K + k: the lists of keys [k0, k1) of every l, as their own CSR.
inline void slice_model_lists(const std::vector<int64_t>& mp, const std::vector<int32_t>& mc, const std::vector<float>& mv, int L, int K,
                              int k0, int k1, std::vector<int64_t>& smp, std::vector<int32_t>& smc, std::vector<float>& smv) {
  smp.assign(1, 0); smc.clear(); smv.clear();
  for (int l = 0; l < L; l++)
    for (int k = k0; k < k1; k++) {
      const size_t m = (size_t)l * K + k;
      smc.insert(smc.end(), mc.begin() + mp[m], mc.begin() + mp[m + 1]);
      smv.insert(smv.end(), mv.begin() + mp[m], mv.begin() + mp[m + 1]);
      smp.push_back((int64_t)smc.size());
    }
}

// intercept.lambdas / default.lambdas of ItemModelTrain: Float.parseFloat of the comma list, in order, repeats kept
// (jobs/ItemModelTrain.java:313-321).  The reference divides by every lambda (:262), so a lambda <= 0 or NaN is refused instead of
// producing infinite prior variances.
inline std::vector<float> lambda_list(const JobConfig& c, const std::string& key) {
  std::vector<float> out;
  for (auto& t : c.get_list(key)) {
    const float v = std::stof(t);
    if (!(v > 0.f)) io_error(key + ": every lambda must be > 0 (got " + t + ")");
    out.push_back(v);
  }
  if (out.empty()) io_error(key + ": no lambda given");
  return out;
}

// job_class -> job for mlease_job_run; returns true (for use in a namespace-scope initializer)
using JobFn = void (*)(const JobConfig&);
bool register_job(const std::string& job_class, JobFn run);

}  // namespace mlease_jobs
