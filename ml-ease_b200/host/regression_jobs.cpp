// regression_jobs.cpp -- host-side mirror of the reference's job layer for the accelerated path, in C++ because
// the reference's host language (Java) has no toolchain in this image.  Same job classes, same config keys, same
// output directory layout and avro schemas; the arithmetic goes through the C ABI of include/mlease_b200.h.
//
//   Regression            jobs/Regression.java:37-80         Prepare -> AdmmTrain -> Test -> TestLoglik
//   RegressionPrepare     jobs/RegressionPrepare.java:58-191
//   RegressionAdmmTrain   jobs/RegressionAdmmTrain.java:130-522 (L2 and L1 z-updates, lambda.map, initialize.boost.rate; gpu.devices = several GPUs)
//   RegressionTest        jobs/RegressionTest.java:65-170
//   RegressionTestLoglik  jobs/RegressionTestLoglik.java:57-201
//   RegressionNaiveTrain  jobs/RegressionNaiveTrain.java:99-415 (+ jobs/PartitionIdAssigner.java:41-101)
//   ItemModelTest, ItemModelTestLoglik: item_model_jobs.cpp
//   ItemModelTrain: item_model_train_job.cpp
//   ItemModelGridTest (scores ItemModelTrain's grid models with their posterior variance): item_model_grid_test_job.cpp
//   JobConfig             com/linkedin/mapred/JobConfig.java:50-224 (java .properties file)
// Not mirrored: Hadoop job submission, HDFS, DistributedCache (local files only; is.local is implied).
#include <algorithm>
#include <charconv>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <map>
#include <set>
#include <sstream>
#include <unordered_map>

#include "../../include/mlease_b200.h"
#include "jobs_common.hpp"

namespace mlease_jobs {

thread_local std::string g_job_err;

[[noreturn]] void io_error(const std::string& m) { throw JobError(m); }
void ck(int rc) { if (rc != 0) io_error(std::string(mlease_last_error())); }


// ------------------------------------------------------------------------------------------ Java string semantics
// Float.toString / String.valueOf(float): model keys "1.0", "1.0#3" (jobs/RegressionAdmmTrain.java:184,650)
std::string java_float_to_string(float f) {
  if (std::isnan(f)) return "NaN";
  if (std::isinf(f)) return f > 0 ? "Infinity" : "-Infinity";
  if (f == 0) return std::signbit(f) ? "-0.0" : "0.0";
  char buf[64];
  auto res = std::to_chars(buf, buf + sizeof(buf), f, std::chars_format::scientific);
  std::string s(buf, res.ptr);
  bool neg = s[0] == '-';
  if (neg) s = s.substr(1);
  size_t e = s.find('e');
  std::string digits;
  for (char c : s.substr(0, e)) if (c != '.') digits.push_back(c);
  int ex = std::atoi(s.c_str() + e + 1);
  std::string out;
  if (ex >= -3 && ex < 7) {
    if (ex >= 0) {
      std::string ip = digits.substr(0, std::min<size_t>(digits.size(), ex + 1));
      while ((int)ip.size() < ex + 1) ip.push_back('0');
      out = ip + "." + (digits.size() > (size_t)ex + 1 ? digits.substr(ex + 1) : "0");
    } else out = "0." + std::string(-ex - 1, '0') + digits;
  } else out = digits.substr(0, 1) + "." + (digits.size() > 1 ? digits.substr(1) : "0") + "E" + std::to_string(ex);
  return neg ? "-" + out : out;
}
// Double.toString: same shortest-repr rule as Float.toString on the double's own digits
std::string java_double_to_string(double f) {
  if (std::isnan(f)) return "NaN";
  if (std::isinf(f)) return f > 0 ? "Infinity" : "-Infinity";
  if (f == 0) return std::signbit(f) ? "-0.0" : "0.0";
  char buf[64];
  auto res = std::to_chars(buf, buf + sizeof(buf), f, std::chars_format::scientific);
  std::string s(buf, res.ptr);
  bool neg = s[0] == '-';
  if (neg) s = s.substr(1);
  size_t e = s.find('e');
  std::string digits;
  for (char c : s.substr(0, e)) if (c != '.') digits.push_back(c);
  int ex = std::atoi(s.c_str() + e + 1);
  std::string out;
  if (ex >= -3 && ex < 7) {
    if (ex >= 0) {
      std::string ip = digits.substr(0, std::min<size_t>(digits.size(), ex + 1));
      while ((int)ip.size() < ex + 1) ip.push_back('0');
      out = ip + "." + (digits.size() > (size_t)ex + 1 ? digits.substr(ex + 1) : "0");
    } else out = "0." + std::string(-ex - 1, '0') + digits;
  } else out = digits.substr(0, 1) + "." + (digits.size() > 1 ? digits.substr(1) : "0") + "E" + std::to_string(ex);
  return neg ? "-" + out : out;
}
// Integer.parseInt: optional sign, decimal digits only, the whole string, 32-bit range; anything else is a NumberFormatException
int java_parse_int(const std::string& s) {
  size_t i = 0;
  bool neg = false;
  if (!s.empty() && (s[0] == '-' || s[0] == '+')) { neg = s[0] == '-'; i = 1; }
  if (i >= s.size()) io_error("For input string: \"" + s + "\"");
  long long v = 0;
  for (; i < s.size(); i++) {
    if (s[i] < '0' || s[i] > '9') io_error("For input string: \"" + s + "\"");
    v = v * 10 + (s[i] - '0');
    if (v > 2147483648LL) io_error("For input string: \"" + s + "\"");
  }
  if (neg) v = -v;
  if (v > 2147483647LL) io_error("For input string: \"" + s + "\"");
  return (int)v;
}
int32_t java_string_hash(const std::string& s) { uint32_t h = 0; for (unsigned char c : s) h = 31u * h + c; return (int32_t)h; }

// ------------------------------------------------------------------------------------------ schemas (src/main/avro/*.avsc)
const char* FEATURE_FIELDS = "[{\"name\":\"name\",\"type\":\"string\"},{\"name\":\"term\",\"type\":\"string\"},{\"name\":\"value\",\"type\":\"float\"}]";
std::string schema_prepare_output() {
  return std::string("{\"type\":\"record\",\"name\":\"RegressionPrepareOutput\",\"namespace\":\"com.linkedin.mlease.regression.avro\",\"fields\":["
                     "{\"name\":\"key\",\"type\":\"string\"},{\"name\":\"response\",\"type\":\"int\"},{\"name\":\"features\",\"type\":{\"type\":\"array\",\"items\":"
                     "{\"type\":\"record\",\"name\":\"feature\",\"fields\":") + FEATURE_FIELDS + "}}},{\"name\":\"weight\",\"type\":\"float\"},{\"name\":\"offset\",\"type\":\"float\"}]}";
}
std::string schema_linear_model() {
  return std::string("{\"type\":\"record\",\"name\":\"LinearModelAvro\",\"namespace\":\"com.linkedin.mlease.avro\",\"fields\":[{\"name\":\"key\",\"type\":\"string\"},"
                     "{\"name\":\"model\",\"type\":{\"type\":\"array\",\"items\":{\"type\":\"record\",\"name\":\"feature\",\"fields\":") + FEATURE_FIELDS + "}}}]}";
}
std::string schema_train_output() {
  return std::string("{\"type\":\"record\",\"name\":\"RegressionTrainOutput\",\"namespace\":\"com.linkedin.mlease.regression.avro\",\"fields\":[{\"name\":\"key\",\"type\":\"string\"},"
                     "{\"name\":\"model\",\"type\":{\"type\":\"array\",\"items\":{\"type\":\"record\",\"name\":\"feature\",\"fields\":") + FEATURE_FIELDS + "}}},"
                     "{\"name\":\"uplusx\",\"type\":{\"type\":\"array\",\"items\":{\"type\":\"record\",\"name\":\"feature1\",\"fields\":" + FEATURE_FIELDS + "}}}]}";
}
const char* SCHEMA_LAMBDA_RHO = "{\"type\":\"record\",\"name\":\"LambdaRhoMap\",\"namespace\":\"com.linkedin.mlease.regression.avro\",\"fields\":[{\"name\":\"lambda\",\"type\":\"float\"},{\"name\":\"rho\",\"type\":\"float\"}]}";
const char* SCHEMA_SAMPLE_LOGLIK = "{\"type\":\"record\",\"name\":\"SampleTestLoglik\",\"namespace\":\"com.linkedin.mlease.regression.avro\",\"fields\":[{\"name\":\"lambda\",\"type\":\"string\"},{\"name\":\"iter\",\"type\":\"int\"},{\"name\":\"testLoglik\",\"type\":\"float\"}]}";
// LinearModelWithVarAvro (ItemModelTrain, RegressionPosterior)
const char* SCHEMA_MODEL_WITH_VAR =
    "{\"type\":\"record\",\"name\":\"LinearModelWithVarAvro\",\"namespace\":\"com.linkedin.mlease.avro\",\"doc\":\"Linear Model with posterior variance in Avro\","
    "\"fields\":[{\"name\":\"key\",\"type\":\"string\"},"
    "{\"name\":\"model\",\"type\":{\"type\":\"array\",\"items\":{\"type\":\"record\",\"name\":\"feature\",\"fields\":["
    "{\"name\":\"name\",\"type\":\"string\"},{\"name\":\"term\",\"type\":\"string\"},{\"name\":\"value\",\"type\":\"float\"}]}}},"
    "{\"name\":\"posteriorVar\",\"type\":{\"type\":\"array\",\"items\":{\"type\":\"record\",\"name\":\"featureVar\",\"fields\":["
    "{\"name\":\"name\",\"type\":\"string\"},{\"name\":\"term\",\"type\":\"string\"},{\"name\":\"value\",\"type\":\"float\"}]}}}]}";
const char* SCHEMA_TEST_LOGLIK = "{\"type\":\"record\",\"name\":\"RegressionTestLoglikOutput\",\"namespace\":\"com.linkedin.mlease.regression.avro\",\"fields\":[{\"name\":\"key\",\"type\":\"string\"},{\"name\":\"testLoglik\",\"type\":\"float\"},{\"name\":\"count\",\"type\":\"double\"}]}";
const char* SCHEMA_PARTITION_ID = "{\"type\":\"record\",\"name\":\"Pair\",\"namespace\":\"org.apache.avro.mapred\",\"fields\":[{\"name\":\"key\",\"type\":\"string\"},{\"name\":\"value\",\"type\":\"int\"}]}";

// ------------------------------------------------------------------------------------------ generic record access
double num_of(const Value& v) { return (v.type == Schema::Float || v.type == Schema::Double) ? v.d : (double)v.i; }
const Value* field(const Value& rec, const Schema& s, const std::string& name) {
  int i = s.field_index(name);
  if (i < 0 || rec.items[i].is_null()) return nullptr;
  return &rec.items[i];
}
// resolves the record schema behind unions
const Schema& rec_schema(const SchemaP& s) {
  const Schema* p = s.get();
  while (p->type == Schema::Union) { const Schema* nx = nullptr; for (auto& b : p->branches) if (b->type != Schema::Null) { nx = b.get(); break; } p = nx; }
  return *p;
}
const Schema& items_schema(const Schema& arr_field) {
  const Schema* p = &arr_field;
  while (p->type == Schema::Union) { const Schema* nx = nullptr; for (auto& b : p->branches) if (b->type != Schema::Null) { nx = b.get(); break; } p = nx; }
  if (p->type != Schema::Array) io_error("features is not a list");
  return rec_schema(p->items);
}
// utils/Util.java:309-337 getResponseAvro: click, then response, then label override; Boolean or Integer only
int get_response(const Value& rec, const Schema& s) {
  const Value* r = nullptr;
  if (auto v = field(rec, s, "click")) r = v;
  if (auto v = field(rec, s, "response")) r = v;
  if (auto v = field(rec, s, "label")) r = v;
  if (!r) io_error("Data should contain one field of the three: response, click or label!");
  if (r->type == Schema::Boolean) return r->i ? 1 : 0;
  if (r->type == Schema::Int) return (int)r->i;
  io_error("Response/Click/Label column should be either boolean or int32!");
}
std::string feature_key(const std::string& name, const std::string& term) { return term.empty() ? name : name + "\x01" + term; }


// generic (Value-tree) reader: the reference implementation of read_prepared, and its fallback for unusual schemas
void read_prepared_generic(const std::string& path, Dictionary& dict, Rows& rows, bool binary_feature) {
  auto files = list_avro_files(path);
  if (files.empty()) io_error("no input files under " + path);
  for (auto& f : files) {
    AvroReader rd(f);
    const Schema& s = rec_schema(rd.schema());
    int fi = s.field_index("features");
    if (fi < 0) io_error("features is null");
    const Schema& fs = items_schema(*s.fields[fi].second);
    int ni = fs.field_index("name"), ti = fs.field_index("term"), vi = fs.field_index("value");
    Value rec;
    while (rd.next(rec)) {
      const Value* k = field(rec, s, "key");
      rows.key.push_back(k ? (k->type == Schema::String ? k->s : std::to_string(k->i)) : "");
      int resp = get_response(rec, s);
      if (resp != 1 && resp != 0 && resp != -1) io_error("response = " + std::to_string(resp) + " (only 1, 0, -1 are allowed)");
      rows.response.push_back(resp);
      const Value* w = field(rec, s, "weight"); const Value* o = field(rec, s, "offset");
      rows.weight.push_back(w ? (float)num_of(*w) : 1.0f);
      rows.offset.push_back(o ? (float)num_of(*o) : 0.0f);
      const Value& feats = rec.items[fi];
      for (auto& fv : feats.items) {
        const std::string& nm = fv.items[ni].s;
        std::string tm = (ti >= 0 && !fv.items[ti].is_null()) ? fv.items[ti].s : "";
        if (nm == INTERCEPT && tm.empty()) io_error("feature name cannot be (INTERCEPT)");
        rows.colidx.push_back(dict.add(feature_key(nm, tm)));
        rows.vals.push_back(binary_feature ? 1.0f : (float)num_of(fv.items[vi]));
      }
      rows.rowptr.push_back((int64_t)rows.colidx.size());
    }
  }
}



// ------------------------------------------------------------------------------------------ block-parallel ingest (avro_walk.hpp)
// Slots of the record plan.  The per-record logic below restates the generic readers field by field (same defaults, same casts,
// same error texts, same order of checks); tests/test_host_cpu.py compares the two on the fixture and on randomised schemas.
enum { S_KEY = 0, S_CLICK, S_RESPONSE, S_LABEL, S_WEIGHT, S_OFFSET, S_NAME, S_TERM, S_VALUE, S_MAPKEY, S_FEATNULL, S_COUNT };
constexpr int EV_FEATURES = 0;
constexpr unsigned K_NULL = 1u << Schema::Null, K_BOOL = 1u << Schema::Boolean, K_INT = 1u << Schema::Int, K_LONG = 1u << Schema::Long,
                   K_FLOAT = 1u << Schema::Float, K_DOUBLE = 1u << Schema::Double, K_STR = 1u << Schema::String;

struct RecPlan {
  Plan plan;
  int mapkey_slot = -1;   // slot the map.key field is read from (-1: no map.key, or the record has no such field)
};
// leaf types behind the unions of a plan node, as a bit mask (bit 31: something that is not a scalar)
unsigned plan_kinds(const Plan& p) {
  if (p.type == Schema::Union) { unsigned m = 0; for (auto& k : p.kids) m |= plan_kinds(k); return m; }
  return plan_is_scalar(p.type) ? 1u << p.type : 1u << 31;
}
// Tags record field `name` with `slot` if its leaf types are within `allowed`.  0: no such field, 1: tagged, -1: outside `allowed`.
int tag_field(Plan& rp, const Schema& rs, const std::string& name, int slot, unsigned allowed) {
  const int i = rs.field_index(name);
  if (i < 0) return 0;
  if (plan_kinds(rp.kids[i]) & ~allowed) return -1;
  return plan_tag_scalar(rp.kids[i], slot) ? 1 : -1;
}
// false: this schema is left to the generic reader (recursive type, non-scalar or oddly typed field, features not array<record>)
bool build_rec_plan(const SchemaP& schema, const std::string& mapkey, RecPlan& out) {
  try { out.plan = plan_build(*schema); } catch (const std::exception&) { return false; }
  Plan* p = &out.plan;
  const Schema* s = schema.get();
  if (!plan_resolve(p, s, Schema::Record)) return false;
  const unsigned any_scalar = ~(1u << 31);
  const unsigned numeric = K_NULL | K_INT | K_LONG | K_FLOAT | K_DOUBLE;
  static const struct { const char* name; int slot; unsigned allowed; } F[] = {
      {"key", S_KEY, K_NULL | K_STR | K_INT | K_LONG}, {"click", S_CLICK, any_scalar}, {"response", S_RESPONSE, any_scalar}, {"label", S_LABEL, any_scalar},
      {"weight", S_WEIGHT, numeric}, {"offset", S_OFFSET, numeric}};
  for (auto& f : F) if (tag_field(*p, *s, f.name, f.slot, f.name == mapkey ? any_scalar : f.allowed) < 0) return false;
  if (!mapkey.empty()) {
    out.mapkey_slot = -1;
    for (auto& f : F) if (mapkey == f.name && s->field_index(mapkey) >= 0) out.mapkey_slot = f.slot;   // map.key names a field read anyway
    if (out.mapkey_slot < 0) {
      if (mapkey == "features") return false;
      const int r = tag_field(*p, *s, mapkey, S_MAPKEY, K_NULL | K_BOOL | K_INT | K_LONG | K_FLOAT | K_DOUBLE | K_STR);
      if (r < 0) return false;
      if (r > 0) out.mapkey_slot = S_MAPKEY;
    }
  }
  const int fi = s->field_index("features");
  if (fi < 0) return false;
  Plan* fp = &p->kids[fi];
  const Schema* fs = s->fields[fi].second.get();
  // a null `features` (union branch) is reported through S_FEATNULL
  if (fp->type == Schema::Union) for (auto& k : fp->kids) if (k.type == Schema::Null) k.tag = S_FEATNULL;
  if (!plan_resolve(fp, fs, Schema::Array)) return false;
  fp->tag = EV_FEATURES;
  Plan* ip = &fp->kids[0];
  const Schema* is = fs->items.get();
  if (!plan_resolve(ip, is, Schema::Record)) return false;
  if (tag_field(*ip, *is, "name", S_NAME, K_NULL | K_STR) != 1) return false;
  if (tag_field(*ip, *is, "term", S_TERM, K_NULL | K_STR) < 0) return false;
  if (tag_field(*ip, *is, "value", S_VALUE, numeric) != 1) return false;
  return true;
}
struct FeatSink {
  struct F { Slot name, term, value; };
  std::vector<F> feats;
  void begin_item(int, Slot* s) {
    s[S_NAME].kind = Slot::Unset;
    s[S_TERM] = Slot();
    s[S_VALUE] = Slot(); s[S_VALUE].kind = Slot::Unset;
  }
  void item(int, Slot* s) {
    if (s[S_NAME].kind == Slot::Unset || s[S_VALUE].kind == Slot::Unset) throw std::runtime_error("avro: a feature is not a record (null element in the features list)");
    feats.push_back(F{s[S_NAME], s[S_TERM], s[S_VALUE]});
  }
};
// utils/Util.java:309-337 getResponseAvro on slots (see get_response)
int get_response_slots(const Slot* sl) {
  const Slot* r = nullptr;
  if (!sl[S_CLICK].is_null()) r = &sl[S_CLICK];
  if (!sl[S_RESPONSE].is_null()) r = &sl[S_RESPONSE];
  if (!sl[S_LABEL].is_null()) r = &sl[S_LABEL];
  if (!r) io_error("Data should contain one field of the three: response, click or label!");
  if (r->kind == Slot::Bool) return r->i ? 1 : 0;
  if (r->kind == Slot::Int) return (int)r->i;
  io_error("Response/Click/Label column should be either boolean or int32!");
}
void reset_record_slots(Slot* sl) {
  for (int k = 0; k < S_COUNT; k++) sl[k] = Slot();
  sl[S_FEATNULL].kind = Slot::Unset;
}
thread_local bool g_force_generic = false;   // tests: compare the two readers in one process
bool host_generic_ingest() { if (g_force_generic) return true; const char* e = getenv("MLEASE_HOST_GENERIC_INGEST"); return e && atoi(e); }

void read_raw_generic(const std::string& file, Dictionary& dict, Rows& rows, bool binary_feature, const std::string& item_key = "");

// rows of one block with block-local feature ids
struct BlockRows {
  Rows rows;
  StrTable names;
};
// One file -> rows (appended) with global dictionary ids, decoded block-parallel.  mode 0: prepared records (read_prepared), 1: raw
// records (read_raw); item_key (mode 1 only): rows.key = that column rendered as item_key_string() does.  Returns false (nothing
// touched) when the schema is left to the generic reader.
bool read_rows_fast(const std::string& file, Dictionary& dict, Rows& rows, bool binary_feature, int mode, const std::string& item_key = "") {
  if (host_generic_ingest()) return false;
  AvroFile af(file);
  RecPlan rp;
  if (!build_rec_plan(af.schema(), item_key, rp)) return false;
  const size_t nb = af.num_blocks();
  std::vector<BlockRows> outs(nb);
  parallel_blocks(nb, host_threads(), [&](size_t b) {
    const std::string data = af.block_data(b);
    const uint8_t* p = reinterpret_cast<const uint8_t*>(data.data());
    const uint8_t* e = p + data.size();
    BlockRows& o = outs[b];
    Rows& r = o.rows;
    Slot sl[S_COUNT];
    FeatSink sink;
    std::string scratch;
    const int64_t nrec = af.block_records(b);
    for (int64_t q = 0; q < nrec; q++) {
      reset_record_slots(sl);
      sink.feats.clear();
      plan_walk(rp.plan, p, e, sl, sink);
      if (mode == 0) {
        const Slot& k = sl[S_KEY];
        r.key.push_back(k.is_null() ? std::string() : (k.kind == Slot::Str ? std::string(k.p, k.n) : std::to_string(k.i)));
      }
      if (mode == 1) {
        if (item_key.empty()) r.key.push_back("");
        else {
          if (rp.mapkey_slot < 0 || sl[rp.mapkey_slot].is_null()) io_error("data does not contain the column" + item_key);   // jobs/ItemModelTest.java:109-114
          const Slot& k = sl[rp.mapkey_slot];
          r.key.push_back(k.kind == Slot::Str ? std::string(k.p, k.n)
                          : k.kind == Slot::Float ? java_float_to_string((float)k.d)
                          : k.kind == Slot::Double ? java_double_to_string(k.d)
                          : k.kind == Slot::Bool ? (k.i ? "true" : "false") : std::to_string(k.i));
        }
      }
      const int resp = get_response_slots(sl);
      if (resp != 1 && resp != 0 && resp != -1) io_error(mode == 0 ? "response = " + std::to_string(resp) + " (only 1, 0, -1 are allowed)" : "response = " + std::to_string(resp));
      r.response.push_back(resp);
      r.weight.push_back(sl[S_WEIGHT].is_null() ? 1.0f : (float)sl[S_WEIGHT].num());
      r.offset.push_back(sl[S_OFFSET].is_null() ? 0.0f : (float)sl[S_OFFSET].num());
      if (mode == 1 && sl[S_FEATNULL].kind == Slot::Null) io_error("features is null");
      for (auto& f : sink.feats) {
        if (mode == 1 && f.name.is_null()) io_error("name is null");
        const char* np = f.name.is_null() ? "" : f.name.p;
        const size_t nn = f.name.is_null() ? 0 : f.name.n;
        const bool has_term = !f.term.is_null() && f.term.n > 0;
        if (mode == 0 && !has_term && nn == INTERCEPT.size() && std::memcmp(np, INTERCEPT.data(), nn) == 0) io_error("feature name cannot be (INTERCEPT)");
        int id;
        if (!has_term) id = o.names.find_or_add(np, nn);
        else {
          scratch.assign(np, nn); scratch.push_back('\x01'); scratch.append(f.term.p, f.term.n);   // feature_key()
          id = o.names.find_or_add(scratch.data(), scratch.size());
        }
        r.colidx.push_back(id);
        r.vals.push_back(binary_feature ? 1.0f : (float)f.value.num());
      }
      r.rowptr.push_back((int64_t)r.colidx.size());
    }
  });
  // merge in block order: global ids in first-seen order of the record stream, exactly as a sequential read assigns them
  size_t add_rows = 0, add_nnz = 0;
  for (auto& o : outs) { add_rows += o.rows.n(); add_nnz += o.rows.colidx.size(); }
  rows.key.reserve(rows.key.size() + add_rows); rows.response.reserve(rows.response.size() + add_rows);
  rows.weight.reserve(rows.weight.size() + add_rows); rows.offset.reserve(rows.offset.size() + add_rows);
  rows.rowptr.reserve(rows.rowptr.size() + add_rows); rows.colidx.reserve(rows.colidx.size() + add_nnz); rows.vals.reserve(rows.vals.size() + add_nnz);
  std::vector<int32_t> gmap;
  for (auto& o : outs) {
    gmap.resize(o.names.size());
    for (size_t l = 0; l < o.names.size(); l++) gmap[l] = dict.add(std::string(o.names.data((int)l), o.names.length((int)l)));
    Rows& r = o.rows;
    const int64_t base = (int64_t)rows.colidx.size();
    for (auto& k : r.key) rows.key.push_back(std::move(k));
    rows.response.insert(rows.response.end(), r.response.begin(), r.response.end());
    rows.weight.insert(rows.weight.end(), r.weight.begin(), r.weight.end());
    rows.offset.insert(rows.offset.end(), r.offset.begin(), r.offset.end());
    for (size_t i = 1; i < r.rowptr.size(); i++) rows.rowptr.push_back(base + r.rowptr[i]);
    for (int32_t c : r.colidx) rows.colidx.push_back(gmap[c]);
    rows.vals.insert(rows.vals.end(), r.vals.begin(), r.vals.end());
    o = BlockRows();   // release the block's memory as we go
  }
  return true;
}

void read_prepared(const std::string& path, Dictionary& dict, Rows& rows, bool binary_feature) {
  auto files = list_avro_files(path);
  if (files.empty()) io_error("no input files under " + path);
  for (auto& f : files) {
    if (read_rows_fast(f, dict, rows, binary_feature, 0)) continue;
    // the generic reader takes a directory or a file: hand it this one file
    read_prepared_generic(f, dict, rows, binary_feature);
  }
}
void read_raw(const std::string& file, Dictionary& dict, Rows& rows, bool binary_feature, const std::string& item_key) {
  if (read_rows_fast(file, dict, rows, binary_feature, 1, item_key)) return;
  read_raw_generic(file, dict, rows, binary_feature, item_key);
}

// ------------------------------------------------------------------------------------------ model files
Value feature_value(const std::string& key, float v) {
  Value r; r.type = Schema::Record; r.items.resize(3);
  size_t p = key.find('\x01');
  r.items[0] = Value::of_string(p == std::string::npos ? key : key.substr(0, p));
  r.items[1] = Value::of_string(p == std::string::npos ? "" : key.substr(p + 1));
  r.items[2] = Value::of_float(v);
  return r;
}
// models/LinearModel.java:697-720 toAvro: intercept first, every value cast to float
Value model_list(const Dictionary& dict, const float* coef /*[D+1], intercept last*/, const std::vector<int32_t>* subset = nullptr) {
  Value a; a.type = Schema::Array;
  const int D = (int)dict.names.size();
  a.items.push_back(feature_value(INTERCEPT, coef[D]));
  if (subset) { for (int32_t k : *subset) a.items.push_back(feature_value(dict.names[k], coef[k])); }
  else for (int k = 0; k < D; k++) a.items.push_back(feature_value(dict.names[k], coef[k]));
  return a;
}
// LinearModelAvro records {key, model}; with uplusx: RegressionTrainOutput records {key, model, uplusx} (:706-711).
// subsets (one entry per model, NULL = all features): the dictionary ids a model lists, ascending.
void write_model_records(const std::string& path, const Dictionary& dict, const std::vector<std::pair<std::string, std::vector<float>>>& models,
                         const std::vector<std::vector<float>>* uplusx = nullptr, const std::vector<const std::vector<int32_t>*>* subsets = nullptr) {
  AvroWriter w(path, uplusx ? schema_train_output() : schema_linear_model());
  if (host_generic_ingest()) {   // Value-tree encoder: the reference implementation the tests compare with
    for (size_t i = 0; i < models.size(); i++) {
      Value r; r.type = Schema::Record; r.items.resize(uplusx ? 3 : 2);
      r.items[0] = Value::of_string(models[i].first);
      const std::vector<int32_t>* sub = subsets ? (*subsets)[i] : nullptr;
      r.items[1] = model_list(dict, models[i].second.data(), sub);
      if (uplusx) r.items[2] = model_list(dict, (*uplusx)[i].data(), sub);
      w.append(r);
    }
  } else {
    const FeaturePrefix fp(dict);
    std::string rec;
    for (size_t i = 0; i < models.size(); i++) {
      rec.clear();
      put_str(rec, models[i].first.data(), models[i].first.size());
      const std::vector<int32_t>* sub = subsets ? (*subsets)[i] : nullptr;
      if (sub) fp.encode_subset(rec, models[i].second.data(), *sub); else fp.encode(rec, models[i].second.data());
      if (uplusx) { if (sub) fp.encode_subset(rec, (*uplusx)[i].data(), *sub); else fp.encode(rec, (*uplusx)[i].data()); }
      w.append_encoded(rec.data(), rec.size(), 1);
    }
  }
  w.close();
}
void write_linear_models(const std::string& path, const Dictionary& dict, const std::vector<std::pair<std::string, std::vector<float>>>& models) {
  write_model_records(path, dict, models);
}
// reads LinearModelAvro files -> key -> (feature key -> value), intercept under INTERCEPT
// last_wins: a repeated key keeps only its last record (HashMap.put, regression/consumers/ReadLinearModelConsumer.java:54-88)
std::map<std::string, std::unordered_map<std::string, double>> read_linear_models(const std::string& path, bool last_wins) {
  std::map<std::string, std::unordered_map<std::string, double>> out;
  for (auto& f : list_avro_files(path)) {
    AvroReader rd(f);
    const Schema& s = rec_schema(rd.schema());
    int ki = s.field_index("key"), mi = s.field_index("model");
    Value rec;
    while (rd.next(rec)) {
      auto& m = out[rec.items[ki].s];
      if (last_wins) m.clear();
      for (auto& fv : rec.items[mi].items) m[feature_key(fv.items[0].s, fv.items[1].s)] = fv.items[2].d;
    }
  }
  return out;
}

struct Session {
  mlease_session* s = nullptr;
  ~Session() { if (s) mlease_session_destroy(s); }
};
// N GPUs of this process behind the session calls (include/mlease_b200.h "Multi-GPU" (b)); N = 1 is a plain session
struct World {
  mlease_world* w = nullptr;
  ~World() { if (w) mlease_world_destroy(w); }
};
// gpu.devices = 0,1,2,...  (falls back to the single gpu.device, default 0).  Not a reference key: the reference's
// parallelism is Hadoop's (one reducer per (partition, lambda), jobs/RegressionAdmmTrain.java:355).
// The keyed jobs shard their keys over the same list (run_shards).
std::vector<int32_t> gpu_devices(const JobConfig& c) {
  std::vector<int32_t> d;
  if (c.has("gpu.devices")) for (auto& t : c.get_list("gpu.devices")) d.push_back(std::stoi(t));
  if (d.empty()) d.push_back(c.get_int("gpu.device", 0));
  return d;
}

// lambda.map file (ReadLambdaMapConsumer, regression/consumers/ReadLambdaMapConsumer.java:33-52; jobs/RegressionAdmmTrain.java:186-196,
// jobs/RegressionNaiveTrain.java:318-332, jobs/ItemModelTrain.java:194-212): records {name, term, value}; key = name or name\u0001term;
// value cast to float.  The map's keys in order of first appearance, a repeated key keeping its last value (HashMap.put).
std::vector<std::pair<std::string, float>> read_lambda_map_entries(const std::string& path) {
  std::vector<std::pair<std::string, float>> out;
  std::unordered_map<std::string, size_t> at;
  for (auto& f : list_avro_files(path)) {
    AvroReader rd(f);
    const Schema& s = rec_schema(rd.schema());
    Value rec;
    while (rd.next(rec)) {
      const Value* nm = field(rec, s, "name"); const Value* vl = field(rec, s, "value");
      if (!nm || !vl) continue;                                   // `record.get("name") != null && record.get("value") != null` (:36)
      const Value* tm = field(rec, s, "term");
      const float lam = (float)num_of(*vl);
      if (!(lam > 0.f)) io_error("lambda.map: lambda of feature " + nm->s + " must be > 0 (it becomes the prior variance 1/lambda)");
      const std::string key = feature_key(nm->s, tm ? tm->s : "");
      auto it = at.find(key);
      if (it != at.end()) out[it->second].second = lam;
      else { at.emplace(key, out.size()); out.emplace_back(key, lam); }
    }
  }
  return out;
}
// The same as a dense [D] vector over the job's feature dictionary, 0 = not listed (features outside the dictionary cannot occur in
// any model of the job and are dropped).
std::vector<float> read_lambda_map(const std::string& path, const Dictionary& dict) {
  std::vector<float> lm(dict.names.size(), 0.f);
  for (auto& e : read_lambda_map_entries(path)) {
    const int k = dict.find(e.first);
    if (k >= 0) lm[k] = e.second;
  }
  return lm;
}

std::vector<float> parse_lambdas(const JobConfig& c) {
  std::vector<float> l;
  for (auto& t : c.get_list("lambda")) l.push_back(std::stof(t));   // Float.parseFloat (:166)
  return l;
}

// driver-side per-iteration test log-likelihood (jobs/RegressionAdmmTrain.java:766-811): double throughout,
// first test file only, at most 1e6 records, divides by sum of weights
double sample_test_loglik(const Rows& t, const Dictionary& dict, const std::vector<int>& test2model, const std::vector<double>& z) {
  const int D = (int)dict.names.size();
  double ll = 0, n = 0;
  size_t lim = std::min<size_t>(t.n(), 1000000);
  // updateLogLikBestModel receives the job's num.click.replicates but evaluates with the constant 1 (:817: testloglik(conf, z, testPath,
  // 1, ignoreValue)), so the intercept term -log(n - 1 + n exp(-b)) (models/LinearModel.java:241-244) is b itself here
  for (size_t i = 0; i < lim; i++) {
    double xb = -std::log(1 - 1 + 1 * std::exp(-z[D]));
    for (int64_t j = t.rowptr[i]; j < t.rowptr[i + 1]; j++) { int m = test2model[t.colidx[j]]; if (m >= 0) xb += z[m] * (double)t.vals[j]; }
    xb += (double)t.offset[i];
    ll += (t.response[i] == 1) ? -std::log1p(std::exp(-xb)) * t.weight[i] : -std::log1p(std::exp(xb)) * t.weight[i];
    n += t.weight[i];
  }
  return ll / n;
}

// raw (unprepared) records -> Rows; used by Test and by the per-iteration loglik (generic reader / fallback)
void read_raw_generic(const std::string& file, Dictionary& dict, Rows& rows, bool binary_feature, const std::string& item_key) {
  AvroReader rd(file);
  const Schema& s = rec_schema(rd.schema());
  int fi = s.field_index("features");
  if (fi < 0) io_error("features is null");
  const Schema& fs = items_schema(*s.fields[fi].second);
  int ni = fs.field_index("name"), ti = fs.field_index("term"), vi = fs.field_index("value");
  Value rec;
  while (rd.next(rec)) {
    std::string key;
    if (!item_key.empty()) {   // data.get(item.key).toString() (jobs/ItemModelTest.java:109-114)
      const Value* k = field(rec, s, item_key);
      if (!k) io_error("data does not contain the column" + item_key);
      key = k->type == Schema::String ? k->s
            : k->type == Schema::Float ? java_float_to_string((float)k->d)
            : k->type == Schema::Double ? java_double_to_string(k->d)
            : k->type == Schema::Boolean ? (k->i ? "true" : "false") : std::to_string(k->i);
    }
    int resp = get_response(rec, s);
    if (resp != 1 && resp != 0 && resp != -1) io_error("response = " + std::to_string(resp));
    rows.key.push_back(key);
    rows.response.push_back(resp);
    const Value* w = field(rec, s, "weight"); const Value* o = field(rec, s, "offset");
    rows.weight.push_back(w ? (float)num_of(*w) : 1.0f);
    rows.offset.push_back(o ? (float)num_of(*o) : 0.0f);
    if (rec.items[fi].is_null()) io_error("features is null");
    for (auto& fv : rec.items[fi].items) {
      if (fv.items[ni].is_null()) io_error("name is null");
      std::string tm = (ti >= 0 && !fv.items[ti].is_null()) ? fv.items[ti].s : "";
      rows.colidx.push_back(dict.add(feature_key(fv.items[ni].s, tm)));
      rows.vals.push_back(binary_feature ? 1.0f : (float)num_of(fv.items[vi]));
    }
    rows.rowptr.push_back((int64_t)rows.colidx.size());
  }
}


// ------------------------------------------------------------------------------------------ RegressionTest output
// output = input fields (unions removed, utils/Util.java:377-417) + pred (jobs/RegressionTest.java:198-236)
std::string test_output_schema(const SchemaP& in, const char* name, const char* ns, bool pred_var) {
  SchemaP os = std::make_shared<Schema>(*schema_remove_union(in));
  os->name = name;
  auto pf = std::make_shared<Schema>(); pf->type = Schema::Float;
  os->fields.emplace_back("pred", pf);
  if (pred_var) os->fields.emplace_back("predVar", pf);
  std::map<std::string, bool> em;
  Json j = schema_to_json(os, em);
  if (ns) {
    Json v; v.kind = Json::Str; v.str = ns;
    j.obj.insert(j.obj.begin() + 1, {"namespace", v});
  }
  return json_dump(j);
}
void write_test_output_generic(const std::string& in_file, const std::string& out_file, const std::vector<float>& pred) {
  AvroReader rd(in_file);
  AvroWriter w(out_file, test_output_schema(rd.schema()));
  Value rec; size_t i = 0;
  while (rd.next(rec)) { rec.items.push_back(Value::of_float(pred[i++])); w.append(rec); }
  w.close();
}
// Record bytes with the union branch indices dropped -- what encoding the decoded record against the union-free schema gives when
// every union holds its first non-null branch.  Anything else (a null where the output schema has none, a second non-null branch,
// a union of nulls) throws NotPlain and the file goes through the generic path, which then behaves exactly as before.
void copy_varint(const uint8_t*& p, const uint8_t* e, std::string& o) {
  const uint8_t* q = p;
  walk_detail::rd_long(p, e);
  o.append(reinterpret_cast<const char*>(q), (size_t)(p - q));
}
void transcode_plain(const Plan& pl, const uint8_t*& p, const uint8_t* e, std::string& o) {
  using namespace walk_detail;
  switch (pl.type) {
    case Schema::Null: break;
    case Schema::Boolean: need(p, e, 1); o.push_back((char)*p++); break;
    case Schema::Int: case Schema::Long: case Schema::Enum: copy_varint(p, e, o); break;
    case Schema::Float: need(p, e, 4); o.append(reinterpret_cast<const char*>(p), 4); p += 4; break;
    case Schema::Double: need(p, e, 8); o.append(reinterpret_cast<const char*>(p), 8); p += 8; break;
    case Schema::String: case Schema::Bytes: {
      const uint8_t* q = p;
      const int64_t n = rd_long(p, e);
      need(p, e, n);
      p += n;
      o.append(reinterpret_cast<const char*>(q), (size_t)(p - q));
      break;
    }
    case Schema::Fixed: need(p, e, pl.fixed_size); o.append(reinterpret_cast<const char*>(p), (size_t)pl.fixed_size); p += pl.fixed_size; break;
    case Schema::Union: {
      const int64_t br = rd_long(p, e);
      if (br < 0 || br >= (int64_t)pl.kids.size()) throw std::runtime_error("avro: bad union branch");
      int fnn = -1;
      for (size_t k = 0; k < pl.kids.size(); k++) if (pl.kids[k].type != Schema::Null) { fnn = (int)k; break; }
      if (fnn < 0 || br != fnn) throw NotPlain();
      transcode_plain(pl.kids[(size_t)fnn], p, e, o);
      break;
    }
    case Schema::Record: for (auto& k : pl.kids) transcode_plain(k, p, e, o); break;
    case Schema::Array:
      while (true) {
        int64_t n = rd_long(p, e);
        if (n == 0) break;
        if (n < 0) { n = -n; rd_long(p, e); }
        put_long(o, n);
        for (int64_t k = 0; k < n; k++) transcode_plain(pl.kids[0], p, e, o);
      }
      put_long(o, 0);
      break;
    case Schema::Map:
      while (true) {
        int64_t n = rd_long(p, e);
        if (n == 0) break;
        if (n < 0) { n = -n; rd_long(p, e); }
        put_long(o, n);
        for (int64_t k = 0; k < n; k++) {
          const uint8_t* q = p;
          const int64_t l = rd_long(p, e);
          need(p, e, l);
          p += l;
          o.append(reinterpret_cast<const char*>(q), (size_t)(p - q));
          transcode_plain(pl.kids[0], p, e, o);
        }
      }
      put_long(o, 0);
      break;
  }
}
bool write_test_output_fast(const std::string& in_file, const std::string& out_file, const std::vector<float>& pred) {
  if (host_generic_ingest()) return false;
  AvroFile af(in_file);
  Plan plan;
  try { plan = plan_build(*af.schema()); } catch (const std::exception&) { return false; }
  {
    const Plan* p = &plan;   // the datum must be a record behind its unions, as schema_remove_union() + "AdmmTestOutput" assume
    while (p->type == Schema::Union) { const Plan* nx = nullptr; for (auto& k : p->kids) if (k.type != Schema::Null) { nx = &k; break; } if (!nx) return false; p = nx; }
    if (p->type != Schema::Record) return false;
  }
  if ((int64_t)pred.size() < af.num_records()) return false;
  const size_t nb = af.num_blocks();
  std::vector<std::string> outs(nb);
  std::atomic<bool> plain{true};
  parallel_blocks(nb, host_threads(), [&](size_t b) {
    if (!plain.load()) return;
    const std::string data = af.block_data(b);
    const uint8_t* p = reinterpret_cast<const uint8_t*>(data.data());
    const uint8_t* e = p + data.size();
    std::string& o = outs[b];
    o.reserve(data.size() + 4 * (size_t)af.block_records(b));
    const int64_t first = af.records_before(b), nrec = af.block_records(b);
    try {
      for (int64_t q = 0; q < nrec; q++) { transcode_plain(plan, p, e, o); put_float(o, pred[(size_t)(first + q)]); }
    } catch (const NotPlain&) { plain.store(false); }
  });
  if (!plain.load()) return false;
  AvroWriter w(out_file, test_output_schema(af.schema()));
  for (size_t b = 0; b < nb; b++) { w.append_encoded(outs[b].data(), outs[b].size(), af.block_records(b)); outs[b] = std::string(); }
  w.close();
  return true;
}
void write_test_output(const std::string& in_file, const std::string& out_file, const std::vector<float>& pred) {
  if (!write_test_output_fast(in_file, out_file, pred)) write_test_output_generic(in_file, out_file, pred);
}


// ------------------------------------------------------------------------------------------ RegressionTestLoglik input
// (response, pred, weight) of scored records (jobs/RegressionTestLoglik.java:124-151); everything else in a record is skipped.
void read_scored_generic(const std::string& f, std::vector<int32_t>& resp, std::vector<float>& pred, std::vector<float>& weight) {
  AvroReader rd(f);
  const Schema& s = rec_schema(rd.schema());
  Value rec;
  while (rd.next(rec)) {
    const Value* r = field(rec, s, "response"); const Value* p = field(rec, s, "pred"); const Value* w = field(rec, s, "weight");
    if (!r || !p) io_error("response/pred is null");
    resp.push_back((int)num_of(*r)); pred.push_back((float)num_of(*p)); weight.push_back(w ? (float)num_of(*w) : 1.0f);
  }
}
bool read_scored_fast(const std::string& f, std::vector<int32_t>& resp, std::vector<float>& pred, std::vector<float>& weight) {
  if (host_generic_ingest()) return false;
  AvroFile af(f);
  Plan plan;
  try { plan = plan_build(*af.schema()); } catch (const std::exception&) { return false; }
  Plan* p = &plan;
  const Schema* s = af.schema().get();
  if (!plan_resolve(p, s, Schema::Record)) return false;
  enum { R = 0, P = 1, W = 2 };
  const unsigned numeric = K_NULL | K_BOOL | K_INT | K_LONG | K_FLOAT | K_DOUBLE;
  if (tag_field(*p, *s, "response", R, numeric) < 0 || tag_field(*p, *s, "pred", P, numeric) < 0 || tag_field(*p, *s, "weight", W, numeric) < 0) return false;
  struct Part { std::vector<int32_t> r; std::vector<float> p, w; };
  struct NoSink { void begin_item(int, Slot*) {} void item(int, Slot*) {} };
  const size_t nb = af.num_blocks();
  std::vector<Part> parts(nb);
  parallel_blocks(nb, host_threads(), [&](size_t b) {
    const std::string data = af.block_data(b);
    const uint8_t* q = reinterpret_cast<const uint8_t*>(data.data());
    const uint8_t* e = q + data.size();
    Part& o = parts[b];
    NoSink sink;
    Slot sl[3];
    for (int64_t k = 0; k < af.block_records(b); k++) {
      sl[R] = Slot(); sl[P] = Slot(); sl[W] = Slot();
      plan_walk(plan, q, e, sl, sink);
      if (sl[R].is_null() || sl[P].is_null()) io_error("response/pred is null");
      o.r.push_back((int)sl[R].num()); o.p.push_back((float)sl[P].num()); o.w.push_back(sl[W].is_null() ? 1.0f : (float)sl[W].num());
    }
  });
  for (auto& o : parts) {
    resp.insert(resp.end(), o.r.begin(), o.r.end()); pred.insert(pred.end(), o.p.begin(), o.p.end()); weight.insert(weight.end(), o.w.begin(), o.w.end());
  }
  return true;
}
void read_scored(const std::string& f, std::vector<int32_t>& resp, std::vector<float>& pred, std::vector<float>& weight) {
  if (!read_scored_fast(f, resp, pred, weight)) read_scored_generic(f, resp, pred, weight);
}

// ============================================================================================ RegressionPrepare
// jobs/RegressionPrepare.java:95-191.  map.key set -> key = data[map.key].toString() (bit-exact); otherwise the reference
// draws floor(Math.random()*nblocks) from an UNSEEDED generator (:112) which cannot be reproduced: here a splitmix64 stream
// seeded by `random.seed` (default 0) plays that role, and positives are replicated onto consecutive partitions (:172-186).
struct SplitMix { uint64_t s; double next() { uint64_t z = (s += 0x9E3779B97F4A7C15ULL); z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL; z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL; z ^= z >> 31; return (z >> 11) * (1.0 / 9007199254740992.0); } };

struct PrepareCfg {
  std::string mapkey;
  int nblocks = 0, reps = 1;
  bool ignore_value = false;
};
// one input file through the generic (Value-tree) decoder: the reference implementation / fallback of prepare_file_fast
void prepare_file_generic(const std::string& f, const PrepareCfg& pc, SplitMix& rng, AvroWriter& w) {
  const std::string& mapkey = pc.mapkey;
  const int nblocks = pc.nblocks, reps = pc.reps;
  const bool ignore_value = pc.ignore_value;
  {
    AvroReader rd(f);
    const Schema& s = rec_schema(rd.schema());
    int fi = s.field_index("features");
    Value rec;
    while (rd.next(rec)) {
      std::string key;
      if (!mapkey.empty()) {
        const Value* k = field(rec, s, mapkey);
        if (!k) io_error("map.key is wrongly specified! No such key exists in some lines of the data!");
        // data.get(map.key).toString() (:107): Float / Double print as Java does ("1.0", not "1.000000"), Boolean as true / false
        key = k->type == Schema::String ? k->s
              : k->type == Schema::Float ? java_float_to_string((float)k->d)
              : k->type == Schema::Double ? java_double_to_string(k->d)
              : k->type == Schema::Boolean ? (k->i ? "true" : "false") : std::to_string(k->i);
      } else {
        key = std::to_string((int)std::floor(rng.next() * nblocks));
      }
      const int response = get_response(rec, s);
      if (fi < 0 || rec.items[fi].is_null()) io_error("features is null");
      const Schema& fs = items_schema(*s.fields[fi].second);
      int ni = fs.field_index("name"), ti = fs.field_index("term"), vi = fs.field_index("value");
      Value feats; feats.type = Schema::Array;
      for (auto& fv : rec.items[fi].items) {
        if (ni < 0 || fv.items[ni].is_null()) io_error("name is null");
        Value r; r.type = Schema::Record; r.items.resize(3);
        r.items[0] = Value::of_string(fv.items[ni].s);
        r.items[1] = Value::of_string((ti >= 0 && !fv.items[ti].is_null()) ? fv.items[ti].s : "");
        r.items[2] = Value::of_float(ignore_value ? 1.0f : (float)num_of(fv.items[vi]));   // :142-146
        feats.items.push_back(r);
      }
      double weight = 1.0;
      if (auto wv = field(rec, s, "weight")) weight = num_of(*wv);
      {
        // Util.getIntAvro(data, "response") (:159, utils/Util.java:55-63): the field must exist and be an Integer, even when the
        // response itself was taken from click / label
        const Value* rv = field(rec, s, "response");
        if (!rv) io_error("response is null");
        if (rv->type != Schema::Int) io_error("response=" + std::string(rv->type == Schema::Boolean ? (rv->i ? "true" : "false") : "?") + " is not an integer");
        if (rv->i == 1) weight = weight / reps;
      }
      double offset = 0.0;
      if (auto ov = field(rec, s, "offset")) offset = num_of(*ov);
      Value o; o.type = Schema::Record; o.items.resize(5);
      o.items[1] = Value::of_int(response); o.items[2] = feats;
      o.items[3] = Value::of_float((float)weight); o.items[4] = Value::of_float((float)offset);
      if (mapkey.empty() && response == 1) {
        int pid = java_parse_int(key);
        for (int i = 0; i < reps; i++) {
          if (pid >= nblocks) pid -= nblocks;
          o.items[0] = Value::of_string(std::to_string(pid));
          w.append(o);
          pid++;
        }
      } else {
        o.items[0] = Value::of_string(key);
        w.append(o);
      }
    }
  }
}

// The same job on the plan walker, block-parallel: every input block is decoded and re-encoded on a worker thread, the main
// thread appends the encoded records in block order.  rng_state0 = state of the key stream before this file's first record: the
// stream is a counter (SplitMix), one draw per record, so a block starts at rng_state0 + gamma * (records before the block).
// Returns false (nothing written) when the schema is left to the generic decoder.
bool prepare_file_fast(const std::string& f, const PrepareCfg& pc, uint64_t rng_state0, AvroWriter& w, int64_t* nrecords) {
  if (host_generic_ingest()) return false;
  AvroFile af(f);
  RecPlan rp;
  if (!build_rec_plan(af.schema(), pc.mapkey, rp)) return false;
  const size_t nb = af.num_blocks();
  struct Out { std::string bytes; int64_t n = 0; };
  std::vector<Out> outs(nb);
  // blocks are handed out in waves so that the encoded output of at most a few blocks per thread is alive at a time
  const size_t wave = (size_t)std::max(1, host_threads()) * 4;
  for (size_t b0 = 0; b0 < nb; b0 += wave) {
    const size_t b1 = std::min(nb, b0 + wave);
    parallel_blocks(b1 - b0, host_threads(), [&](size_t bi) {
      const size_t b = b0 + bi;
      const std::string data = af.block_data(b);
      const uint8_t* p = reinterpret_cast<const uint8_t*>(data.data());
      const uint8_t* e = p + data.size();
      Out& o = outs[b];
      o.bytes.reserve(data.size() + data.size() / 8);
      SplitMix rng{rng_state0 + 0x9E3779B97F4A7C15ULL * (uint64_t)af.records_before(b)};
      Slot sl[S_COUNT];
      FeatSink sink;
      std::string key, body;
      const int64_t nrec = af.block_records(b);
      for (int64_t q = 0; q < nrec; q++) {
        reset_record_slots(sl);
        sink.feats.clear();
        plan_walk(rp.plan, p, e, sl, sink);
        if (!pc.mapkey.empty()) {
          if (rp.mapkey_slot < 0 || sl[rp.mapkey_slot].is_null()) io_error("map.key is wrongly specified! No such key exists in some lines of the data!");
          const Slot& k = sl[rp.mapkey_slot];
          key = k.kind == Slot::Str ? std::string(k.p, k.n)
                : k.kind == Slot::Float ? java_float_to_string((float)k.d)
                : k.kind == Slot::Double ? java_double_to_string(k.d)
                : k.kind == Slot::Bool ? (k.i ? "true" : "false") : std::to_string(k.i);
        } else {
          key = std::to_string((int)std::floor(rng.next() * pc.nblocks));
        }
        const int response = get_response_slots(sl);
        if (sl[S_FEATNULL].kind == Slot::Null) io_error("features is null");
        // everything after the key: response, features, weight, offset
        body.clear();
        put_long(body, response);
        if (!sink.feats.empty()) put_long(body, (int64_t)sink.feats.size());
        for (auto& fv : sink.feats) {
          if (fv.name.is_null()) io_error("name is null");
          put_str(body, fv.name.p, fv.name.n);
          if (fv.term.is_null()) put_long(body, 0); else put_str(body, fv.term.p, fv.term.n);
          put_float(body, pc.ignore_value ? 1.0f : (float)fv.value.num());   // :142-146
        }
        put_long(body, 0);
        double weight = 1.0;
        if (!sl[S_WEIGHT].is_null()) weight = sl[S_WEIGHT].num();
        {
          // Util.getIntAvro(data, "response") (:159, utils/Util.java:55-63)
          const Slot& rv = sl[S_RESPONSE];
          if (rv.is_null()) io_error("response is null");
          if (rv.kind != Slot::Int) io_error("response=" + std::string(rv.kind == Slot::Bool ? (rv.i ? "true" : "false") : "?") + " is not an integer");
          if (rv.i == 1) weight = weight / pc.reps;
        }
        double offset = 0.0;
        if (!sl[S_OFFSET].is_null()) offset = sl[S_OFFSET].num();
        put_float(body, (float)weight);
        put_float(body, (float)offset);
        if (pc.mapkey.empty() && response == 1) {
          int pid = java_parse_int(key);
          for (int i = 0; i < pc.reps; i++) {
            if (pid >= pc.nblocks) pid -= pc.nblocks;
            const std::string ks = std::to_string(pid);
            put_str(o.bytes, ks.data(), ks.size());
            o.bytes += body;
            o.n++;
            pid++;
          }
        } else {
          put_str(o.bytes, key.data(), key.size());
          o.bytes += body;
          o.n++;
        }
      }
    });
    for (size_t b = b0; b < b1; b++) {
      w.append_encoded(outs[b].bytes.data(), outs[b].bytes.size(), outs[b].n);
      outs[b] = Out();
    }
  }
  if (nrecords) *nrecords = af.num_records();
  return true;
}

void run_prepare(const JobConfig& c) {
  PrepareCfg pc;
  pc.mapkey = c.get("map.key", "");
  pc.nblocks = c.get_int("num.blocks", 0);
  pc.reps = c.get_int("num.click.replicates", 1);
  pc.ignore_value = c.get_bool("binary.feature", false);
  const std::string out = c.get("output.path");
  uint64_t rng_state = (uint64_t)c.get_double("random.seed", 0);
  auto files = list_avro_files(c.get("input.paths"));
  if (files.empty()) io_error("no input under " + c.get("input.paths"));
  AvroWriter w(out + "/part-00000.avro", schema_prepare_output());
  for (auto& f : files) {
    int64_t n = 0;
    if (prepare_file_fast(f, pc, rng_state, w, &n)) {
      if (pc.mapkey.empty()) rng_state += 0x9E3779B97F4A7C15ULL * (uint64_t)n;   // one draw per record
      continue;
    }
    SplitMix rng{rng_state};
    prepare_file_generic(f, pc, rng, w);
    rng_state = rng.s;
  }
  w.close();
}

// ============================================================================================ RegressionAdmmTrain
void run_admm_train(const JobConfig& c) {
  const std::string out = c.get("output.base.path");
  const int nblocks = c.get_int("num.blocks");
  const int niter = c.get_int("num.iters", 10);
  const int reg = c.get_int("regularizer");
  if (reg != 1 && reg != 2) io_error("Only L1 and L2 regularization supported!");
  const bool ignore_value = c.get_bool("binary.feature", false);
  std::vector<float> lambdas = parse_lambdas(c);
  const int L = (int)lambdas.size();
  std::vector<float> rhos;
  if (c.has("rho")) {
    for (auto& t : c.get_list("rho")) rhos.push_back(std::stof(t));
    if ((int)rhos.size() != L) io_error("The number of rho's should be exactly the same as the number of lambda's. OR: don't claim rho!");
  } else for (float l : lambdas) rhos.push_back(l <= 100 ? 1.0f : 10.0f);
  const float boost_rate = c.get_float("initialize.boost.rate", 0);

  Dictionary dict;
  Rows rows;
  read_prepared(c.get("input.paths", out + "/tmp-data"), dict, rows, ignore_value);
  const int D = (int)dict.names.size(), Dt = D + 1;

  // group rows by partition id (AdmmMapper: Integer.parseInt(key), :558; AdmmPartitioner range check :585-588)
  std::vector<std::vector<size_t>> by_part(nblocks);
  for (size_t i = 0; i < rows.n(); i++) {
    const int p = java_parse_int(rows.key[i]);   // Integer.parseInt(key) (AdmmMapper, :558)
    if (p < 0 || p >= nblocks) io_error("Map key is wrong! key has to be in the range of [0,numPartitions-1].");
    by_part[p].push_back(i);
  }
  for (int p = 0; p < nblocks; p++) if (by_part[p].empty()) io_error("Some models failed!");   // an empty reducer emits no model (utils/LinearModelUtils.java:77-83)

  std::vector<float> lambda_map;
  if (!c.get("lambda.map", "").empty()) lambda_map = read_lambda_map(c.get("lambda.map"), dict);
  fprintf(stderr, "[RegressionAdmmTrain] Lambda Map has size = %d\n", (int)std::count_if(lambda_map.begin(), lambda_map.end(), [](float v) { return v > 0; }));

  std::vector<int32_t> devs = gpu_devices(c);
  if ((int)devs.size() > nblocks) devs.resize(nblocks);           // a GPU without a partition has nothing to reduce
  mlease_admm_config cfg; std::memset(&cfg, 0, sizeof(cfg));
  cfg.device = devs[0]; cfg.num_blocks = nblocks; cfg.num_features = D; cfg.num_lambdas = L;
  cfg.lambdas = lambdas.data(); cfg.rhos = rhos.data(); cfg.regularizer = reg;
  cfg.lambda_map = lambda_map.empty() ? nullptr : lambda_map.data();
  cfg.penalize_intercept = c.get_bool("penalize.intercept", false);
  cfg.aggressive_decay = c.get_bool("aggressive.liblinear.epsilon.decay", false);
  cfg.binary_feature = ignore_value;
  cfg.epsilon = c.get_double("epsilon", 0.0001);
  cfg.rho_adapt_coefficient = c.get_float("rho.adapt.coefficient", 0);
  World S;
  ck(mlease_world_create(&cfg, devs.data(), (int32_t)devs.size(), &S.w));
  for (int p = 0; p < nblocks; p++) {
    std::vector<int64_t> rp{0}; std::vector<int32_t> ci; std::vector<float> vv, ww, oo; std::vector<int32_t> rr;
    for (size_t i : by_part[p]) {
      for (int64_t j = rows.rowptr[i]; j < rows.rowptr[i + 1]; j++) { ci.push_back(rows.colidx[j]); vv.push_back(rows.vals[j]); }
      rp.push_back((int64_t)ci.size()); rr.push_back(rows.response[i]); ww.push_back(rows.weight[i]); oo.push_back(rows.offset[i]);
    }
    ck(mlease_world_add_partition_csr(S.w, p, (int64_t)rr.size(), rp.data(), ci.data(), vv.data(), rr.data(), ww.data(), oo.data()));
  }

  // lambda-rho map (:200-201, :721-734)
  {
    AvroWriter w(out + "/lambda-rho/part-r-00000.avro", SCHEMA_LAMBDA_RHO);
    for (int l = 0; l < L; l++) { Value r; r.type = Schema::Record; r.items = {Value::of_float(lambdas[l]), Value::of_float(rhos[l])}; w.append(r); }
    w.close();
  }
  // optional per-iteration test loglik on the first file under test.path (:204-232)
  Rows test; std::vector<int> test2model; bool test_per_iter = false;
  {
    std::string tp = c.get("test.path", "");
    auto tf = tp.empty() ? std::vector<std::string>() : list_avro_files(tp);
    if (!tf.empty()) {
      Dictionary td; read_raw(tf[0], td, test, ignore_value);
      test2model.resize(td.names.size());
      for (size_t k = 0; k < td.names.size(); k++) test2model[k] = dict.find(td.names[k]);
      test_per_iter = test.n() > 0;
      // the reference opens and closes an empty writer here (:217-232): sample-test-loglik/write-test-00000.avro
      AvroWriter w0(out + "/sample-test-loglik/write-test-00000.avro", SCHEMA_SAMPLE_LOGLIK);
      w0.close();
    }
  }
  float best_loglik = -9999999.0f;
  auto models_z = [&](bool as_float) {
    std::vector<std::pair<std::string, std::vector<float>>> m;
    for (int l = 0; l < L; l++) {
      std::vector<double> z(Dt); ck(mlease_world_get_z(S.w, l, z.data()));
      std::vector<float> zf(Dt); for (int k = 0; k < Dt; k++) zf[k] = (float)z[k];
      m.emplace_back(java_float_to_string(lambdas[l]), zf);
    }
    (void)as_float;
    return m;
  };
  const bool initialized = boost_rate > 0 && reg == 2;   // jobs/RegressionAdmmTrain.java:236
  if (initialized) {
    // Mean-model initialization: one RegressionNaiveTrain fit per (lambda, partition) -- prior variance 1/lambda, intercept
    // variance 100000 unless penalize.intercept, prior mean 0, start 0 (jobs/RegressionNaiveTrain.java:333-343,395) -- kept
    // under <out>/initialModel like the reference (:239-260), then averaged as float models (cons/MeanLinearModelConsumer.java:44-70).
    std::vector<double> z0((size_t)L * Dt, 0.0);
    std::vector<std::pair<std::string, std::vector<float>>> init_models;
    // like every NaiveTrain model, an initial model lists the features its partition's rows list (+ the intercept)
    std::vector<std::vector<int32_t>> present(nblocks);
    for (int p = 0; p < nblocks; p++) {
      std::vector<char> seen(D, 0);
      for (size_t i : by_part[p]) for (int64_t j = rows.rowptr[i]; j < rows.rowptr[i + 1]; j++) seen[rows.colidx[j]] = 1;
      for (int k = 0; k < D; k++) if (seen[k]) present[p].push_back(k);
    }
    std::vector<const std::vector<int32_t>*> init_feats;
    for (int l = 0; l < L; l++) {
      std::vector<double> q(Dt, (double)lambdas[l]), zero(Dt, 0.0);
      for (int k = 0; k < D; k++) if (!lambda_map.empty() && lambda_map[k] > 0) q[k] = (double)lambda_map[k];   // propsIni.put(LAMBDA_MAP, ...) (:248)
      if (!cfg.penalize_intercept) q[D] = 1.0 / 100000.0;
      for (int p = 0; p < nblocks; p++) {
        std::vector<double> x(Dt, 0.0);
        int32_t steps = 0;
        ck(mlease_world_fit_partition(S.w, p, x.data(), zero.data(), q.data(), &steps));
        std::vector<float> xf(Dt);
        for (int k = 0; k < Dt; k++) { xf[k] = (float)x[k]; z0[(size_t)l * Dt + k] = 1.0 * z0[(size_t)l * Dt + k] + (1.0 / nblocks) * (double)xf[k]; }
        init_models.emplace_back(java_float_to_string(lambdas[l]) + "#" + std::to_string(p), xf);
        init_feats.push_back(&present[p]);
      }
    }
    write_model_records(out + "/initialModel/part-r-00000.avro", dict, init_models, nullptr, &init_feats);
    if (test_per_iter) {   // updateLogLikBestModel(conf, 0, z, ...) (:272-275): the mean model's sample log-likelihood; no best-model at iteration 0 (:833)
      AvroWriter w(out + "/sample-test-loglik/iteration-0.avro", SCHEMA_SAMPLE_LOGLIK);
      for (int l = 0; l < L; l++) {
        std::vector<double> z(z0.begin() + (size_t)l * Dt, z0.begin() + (size_t)(l + 1) * Dt);
        Value r; r.type = Schema::Record;
        r.items = {Value::of_string(java_float_to_string(lambdas[l])), Value::of_int(0), Value::of_float((float)sample_test_loglik(test, dict, test2model, z))};
        w.append(r);
      }
      w.close();
    }
    ck(mlease_world_begin_initialized(S.w, z0.data(), boost_rate));
  } else {
    ck(mlease_world_begin(S.w));
  }
  // write.iteration.files (not a reference key; default true = the reference's layout): false skips the per-iteration state files
  // iter-<i>/{u,init-value,model} -- with the state resident on the GPUs nothing reads them back, and at 10k features x 24
  // reducers they cost more host time per iteration than the iteration itself; final-model, best-model and sample-test-loglik stay
  const bool iter_files = c.get_bool("write.iteration.files", true);
  int i;
  for (i = 1; i <= niter; i++) {
    const std::string it = out + "/iter-" + std::to_string(i);
    // u of this iteration (empty file at i == 1, :310-313) and z as the reducers see it (:330-331)
    if (iter_files) {
      std::vector<std::pair<std::string, std::vector<float>>> us;
      if (i > 1)
        for (int p = 0; p < nblocks; p++) for (int l = 0; l < L; l++) {
          std::vector<float> u(Dt); ck(mlease_world_get_u(S.w, p, l, u.data()));
          us.emplace_back(java_float_to_string(lambdas[l]) + "#" + std::to_string(p), u);
        }
      write_linear_models(it + "/u/part-r-00000.avro", dict, us);
      if (i > 1 || initialized) write_linear_models(it + "/init-value/part-r-00000.avro", dict, models_z(true));
      else {   // z = {lambda -> new LinearModel()} (:184): one record per lambda holding only the zero intercept
        Dictionary none; std::vector<std::pair<std::string, std::vector<float>>> z0;
        for (int l = 0; l < L; l++) z0.emplace_back(java_float_to_string(lambdas[l]), std::vector<float>(1, 0.f));
        write_linear_models(it + "/init-value/part-r-00000.avro", none, z0);
      }
    }
    double maxdiff = 0; int32_t stop = 0;
    ck(mlease_world_iterate(S.w, &maxdiff, &stop));
    // reducer outputs (:706-711)
    if (iter_files) {
      std::vector<std::pair<std::string, std::vector<float>>> xs;
      std::vector<std::vector<float>> uxs;
      for (int p = 0; p < nblocks; p++) for (int l = 0; l < L; l++) {
        std::vector<double> x(Dt); std::vector<float> xf(Dt), ux(Dt);
        ck(mlease_world_get_x(S.w, p, l, x.data())); ck(mlease_world_get_uplusx(S.w, p, l, ux.data()));
        for (int k = 0; k < Dt; k++) xf[k] = (float)x[k];
        xs.emplace_back(java_float_to_string(lambdas[l]) + "#" + std::to_string(p), std::move(xf));
        uxs.push_back(std::move(ux));
      }
      write_model_records(it + "/model/part-r-00000.avro", dict, xs, &uxs);
    }
    fprintf(stderr, "[RegressionAdmmTrain] iteration %d: max |z - z_prev| = %.6g\n", i, maxdiff);
    if (c.get_bool("remove.tmp.dir", false) && i >= 2) remove_tree(out + "/iter-" + std::to_string(i - 1));
    if (test_per_iter) {   // updateLogLikBestModel (:812-845)
      AvroWriter w(out + "/sample-test-loglik/iteration-" + std::to_string(i) + ".avro", SCHEMA_SAMPLE_LOGLIK);
      for (int l = 0; l < L; l++) {
        std::vector<double> z(Dt); ck(mlease_world_get_z(S.w, l, z.data()));
        double ll = sample_test_loglik(test, dict, test2model, z);
        Value r; r.type = Schema::Record; r.items = {Value::of_string(java_float_to_string(lambdas[l])), Value::of_int(i), Value::of_float((float)ll)};
        w.append(r);
        if (ll > best_loglik) {
          remove_tree(out + "/best-model");
          std::vector<float> zf(Dt); for (int k = 0; k < Dt; k++) zf[k] = (float)z[k];
          write_linear_models(out + "/best-model/best-iteration-" + std::to_string(i) + ".avro", dict, {{java_float_to_string(lambdas[l]), zf}});
          best_loglik = (float)ll;
        }
      }
      w.close();
    }
    if (stop) break;
  }
  write_linear_models(out + "/final-model/part-r-00000.avro", dict, models_z(true));
  if (c.get_bool("remove.tmp.dir", false)) {   // :503-520
    remove_tree(out + "/initialModel");
    for (int j = std::min(i, niter) - 2; j <= std::min(i, niter); j++) remove_tree(out + "/iter-" + std::to_string(j));
    remove_tree(out + "/tmp-data");
  }
}

// ============================================================================================ RegressionTest
void run_test(const JobConfig& c) {
  const std::string in = c.get("input.paths", "");
  if (in.empty()) return;   // "test.input.paths is empty! So no test will be done!"
  const std::string outBase = c.get("output.base.path");
  const bool ignore_value = c.get_bool("binary.feature", false);
  const std::string modelBase = c.get("model.base.path");
  auto test_one = [&](const std::string& modelPath, const std::string& modelKey, const std::string& outPath) {
    auto models = read_linear_models(modelPath);
    const std::unordered_map<std::string, double>* m = nullptr;
    if (!modelKey.empty()) { auto it = models.find(modelKey); if (it == models.end()) io_error("no model for lambda " + modelKey + " under " + modelPath); m = &it->second; }
    else { if (models.empty()) io_error("no best-model"); m = &models.begin()->second; }
    int part = 0;
    for (auto& f : list_avro_files(in)) {
      Dictionary td; Rows rows;
      read_raw(f, td, rows, ignore_value);
      const int D = (int)td.names.size();
      std::vector<double> coef(D + 1, 0.0);
      for (int k = 0; k < D; k++) { auto it = m->find(td.names[k]); if (it != m->end()) coef[k] = it->second; }
      { auto it = m->find(INTERCEPT); coef[D] = it == m->end() ? 0.0 : it->second; }
      std::vector<float> pred(rows.n());
      if (rows.n())
        ck(mlease_score(c.get_int("gpu.device", 0), nullptr, D, (int64_t)rows.n(), rows.rowptr.data(), rows.colidx.data(), rows.vals.data(), 0,
                        rows.offset.data(), coef.data(), 1, ignore_value ? 1 : 0, pred.data()));
      char nm[64]; snprintf(nm, sizeof nm, "/part-r-%05d.avro", part++);
      write_test_output(f, outPath + nm, pred);
    }
  };
  for (auto& lam : c.get_list("lambda"))
    test_one(modelBase + "/final-model", java_float_to_string(std::stof(lam)), outBase + "/lambda-" + lam);
  if (path_exists(modelBase + "/best-model")) test_one(modelBase + "/best-model", "", outBase + "/best-model");
}

// ============================================================================================ RegressionTestLoglik
void run_test_loglik(const JobConfig& c) {
  if (!c.get_bool("get.test.loglik", true)) return;
  const std::string inBase = c.get("input.base.paths"), outBase = c.get("output.base.path");
  auto one = [&](const std::string& inPath, const std::string& outPath) {
    if (!path_exists(inPath)) return;
    std::vector<int32_t> resp; std::vector<float> pred, weight;
    for (auto& f : list_avro_files(inPath)) read_scored(f, resp, pred, weight);
    if (resp.empty()) return;
    float ll; double cnt;
    // one combiner call per map task; local runs have one split per file -> combiner_block = everything
    ck(mlease_test_loglik(c.get_int("gpu.device", 0), nullptr, (int64_t)resp.size(), resp.data(), pred.data(), weight.data(), (int64_t)resp.size(), &ll, &cnt));
    AvroWriter w(outPath + "/part-r-00000.avro", SCHEMA_TEST_LOGLIK);
    Value r; r.type = Schema::Record; r.items = {Value::of_string("averageTestLoglik"), Value::of_float(ll), Value::of_double(cnt)};
    w.append(r); w.close();
  };
  if (c.has("lambda"))
    for (auto& lam : c.get_list("lambda")) one(inBase + "/lambda-" + lam, outBase + "/lambda-" + lam + "/_loglik");
  one(inBase + "/best-model", outBase + "/best-model/_loglik");
}

// ============================================================================================ RegressionNaiveTrain
// deterministic partition ids: sorted Utf8 order of "<lambda>#<key>" (single reducer), jobs/PartitionIdAssigner.java:79-88
std::map<std::string, int> assign_partition_ids(const std::set<std::string>& keys, const std::vector<float>& lambdas) {
  std::map<std::string, int> ids;
  for (float l : lambdas) for (auto& k : keys) ids[java_float_to_string(l) + "#" + k] = 0;
  int n = 0; for (auto& kv : ids) kv.second = n++;
  return ids;
}

void run_naive_train(const JobConfig& c) {
  const std::string out = c.get("output.base.path");
  const bool heavy = c.get_bool("heavy.per.item.train", false);
  const bool mean = c.get_bool("compute.model.mean", true);
  const int nblocks = mean ? c.get_int("num.blocks") : -1;
  const bool ignore_value = c.get_bool("binary.feature", false);
  std::set<float> lambda_set; for (auto& t : c.get_list("lambda")) lambda_set.insert(std::stof(t));
  std::vector<float> lambdas(lambda_set.begin(), lambda_set.end());
  const int L = (int)lambdas.size();
  Dictionary dict; Rows rows;
  read_prepared(c.get("input.paths", out + "/tmp-data"), dict, rows, ignore_value);
  const int D = (int)dict.names.size(), Dt = D + 1;
  std::vector<float> lambda_map;
  if (!c.get("lambda.map", "").empty()) lambda_map = read_lambda_map(c.get("lambda.map"), dict);
  // intercept.key (jobs/RegressionNaiveTrain.java:146,309,340-343): the reducer puts the intercept's prior variance 100000 under THIS
  // name, while the dataset's intercept is always "(INTERCEPT)" (llf/LibLinearDataset.java INTERCEPT_NAME).  With another name the
  // entry lands on a feature of that name, if there is one, and the real intercept keeps the default variance 1/lambda.
  bool penalize_intercept = c.get_bool("penalize.intercept", false);
  {
    const std::string ikey = c.get("intercept.key", INTERCEPT);
    if (!penalize_intercept && ikey != INTERCEPT) {
      penalize_intercept = true;
      const int k = dict.find(ikey);
      if (k >= 0) { if (lambda_map.empty()) lambda_map.assign(D, 0.f); lambda_map[k] = (float)(1.0 / 100000.0); }
    }
  }
  std::map<std::string, std::vector<size_t>> by_key;
  for (size_t i = 0; i < rows.n(); i++) by_key[rows.key[i]].push_back(i);
  if (heavy) {
    std::set<std::string> ks; for (auto& kv : by_key) ks.insert(kv.first);
    AvroWriter w(out + "/partitionIds/part-r-00000.avro", SCHEMA_PARTITION_ID);
    for (auto& kv : assign_partition_ids(ks, lambdas)) { Value r; r.type = Schema::Record; r.items = {Value::of_string(kv.first), Value::of_int(kv.second)}; w.append(r); }
    w.close();
  }
  // per-key sparse datasets (jobs/RegressionNaiveTrain.java:360-378): the rows of one key are contiguous in ONE CSR, uploaded
  // once for all lambdas; a feature no row of the key lists is not part of that key's model
  const int K = (int)by_key.size();
  std::vector<int64_t> krs{0}, rp{0}; std::vector<std::string> knames;
  std::vector<int32_t> ci, rr; std::vector<float> vv, ww, oo;
  for (auto& kv : by_key) {
    knames.push_back(kv.first);
    for (size_t i : kv.second) {
      std::vector<std::pair<int32_t, float>> ent;
      for (int64_t j = rows.rowptr[i]; j < rows.rowptr[i + 1]; j++) ent.emplace_back(rows.colidx[j], rows.vals[j]);
      std::sort(ent.begin(), ent.end(), [](auto& a, auto& b) { return a.first < b.first; });   // rows sorted by index (llf/LibLinearDataset.java:481-482)
      for (auto& e : ent) { ci.push_back(e.first); vv.push_back(e.second); }
      rp.push_back((int64_t)ci.size());
      rr.push_back(rows.response[i]); ww.push_back(rows.weight[i]); oo.push_back(rows.offset[i]);
    }
    krs.push_back((int64_t)rr.size());
  }
  std::vector<std::pair<std::string, std::vector<float>>> models;
  // a key's model lists the features its rows list, plus the intercept (the reducer's dataset holds nothing else:
  // llf/LibLinear.java:343-350, no prior-mean map in NaiveTrain, jobs/RegressionNaiveTrain.java:395): not all D of the job
  std::vector<std::vector<int32_t>> present(K);
  for (int k = 0; k < K; k++) {
    std::vector<int32_t>& pk = present[k];
    pk.assign(ci.begin() + rp[krs[k]], ci.begin() + rp[krs[k + 1]]);
    std::sort(pk.begin(), pk.end());
    pk.erase(std::unique(pk.begin(), pk.end()), pk.end());
  }
  std::vector<const std::vector<int32_t>*> model_feats;
  std::map<std::string, std::pair<int, std::vector<double>>> sums;
  std::vector<double> m((size_t)L * K * Dt); std::vector<int32_t> skipped(K);
  const std::vector<int32_t> devs = gpu_devices(c);
  const float prior_mean = c.get_float("prior.mean", 0.0f);
  const bool has_intercept = c.get_bool("has.intercept", true);
  const int threshold = c.get_int("data.size.threshold", 0);
  if (devs.size() == 1 || K == 0) {
    ck(mlease_naive_train(devs[0], nullptr, K, D, krs.data(), rp.data(), ci.data(), vv.data(), 0, rr.data(), ww.data(), oo.data(), L, lambdas.data(),
                          lambda_map.empty() ? nullptr : lambda_map.data(), prior_mean, penalize_intercept, has_intercept, threshold, ignore_value ? 1 : 0,
                          m.data(), skipped.data()));
  } else {
    // one key range per device (shard_keys); each range's models go to their slice of m
    run_shards(devs, shard_keys(krs, rp, D, (int)devs.size()), [&](int32_t dev, int k0, int k1) {
      const KeySlice s(krs, rp, k0, k1);
      const int Ks = k1 - k0;
      std::vector<double> ms((size_t)L * Ks * Dt);
      ck(mlease_naive_train(dev, nullptr, Ks, D, s.krs.data(), s.rowptr.data(), ci.data() + s.nz0, vv.data() + s.nz0, 0, rr.data() + s.row0,
                            ww.data() + s.row0, oo.data() + s.row0, L, lambdas.data(), lambda_map.empty() ? nullptr : lambda_map.data(), prior_mean,
                            penalize_intercept, has_intercept, threshold, ignore_value ? 1 : 0, ms.data(), skipped.data() + k0));
      for (int l = 0; l < L; l++)
        std::copy(ms.begin() + (size_t)l * Ks * Dt, ms.begin() + (size_t)(l + 1) * Ks * Dt, m.begin() + ((size_t)l * K + k0) * Dt);
    });
  }
  for (int l = 0; l < L; l++) {
    const std::string ls = java_float_to_string(lambdas[l]);
    auto& acc = sums[ls]; acc.second.assign(Dt, 0.0);
    for (int k = 0; k < K; k++) {
      if (skipped[k]) continue;
      std::vector<float> mf(Dt); for (int j = 0; j < Dt; j++) mf[j] = (float)m[((size_t)l * K + k) * Dt + j];
      models.emplace_back(ls + "#" + knames[k], mf);
      model_feats.push_back(&present[k]);
      acc.first++;
      if (mean) for (int j = 0; j < Dt; j++) acc.second[j] = 1.0 * acc.second[j] + (1.0 / nblocks) * (double)mf[j];   // cons/MeanLinearModelConsumer.java:59-63
    }
  }
  write_model_records(out + "/models/part-r-00000.avro", dict, models, nullptr, &model_feats);
  if (mean) {
    int total = 0; for (auto& kv : sums) total += kv.second.first;
    if (total != (int)lambdas.size() * nblocks) throw std::runtime_error("Some models failed!");
    std::vector<std::pair<std::string, std::vector<float>>> fin;
    for (auto& kv : sums) { std::vector<float> f(Dt); for (int j = 0; j < Dt; j++) f[j] = (float)kv.second.second[j]; fin.emplace_back(kv.first, f); }
    write_linear_models(out + "/final-model/part-r-00000.avro", dict, fin);
  }
  if (c.get_bool("remove.tmp.dir", true)) remove_tree(out + "/tmp-data");
}

// ============================================================================================ Regression (chain)
void run_regression(const JobConfig& c) {
  const std::string out = c.get("output.base.path");
  if (c.get_bool("force.output.overwrite", false)) remove_tree(out);
  JobConfig cp = c; cp.kv["output.path"] = out + "/tmp-data";
  run_prepare(cp);
  JobConfig ct = c; ct.kv["input.paths"] = out + "/tmp-data";
  run_admm_train(ct);
  if (c.has("test.path")) {
    JobConfig cte = c; cte.kv["input.paths"] = c.get("test.path"); cte.kv["model.base.path"] = out; cte.kv["output.base.path"] = out + "/test";
    run_test(cte);
    JobConfig cl = c; cl.kv["input.base.paths"] = out + "/test"; cl.kv["output.base.path"] = out + "/test";
    run_test_loglik(cl);
  }
}

// jobs defined in other translation units (register_job)
std::map<std::string, JobFn>& job_registry() { static std::map<std::string, JobFn> r; return r; }
bool register_job(const std::string& job_class, JobFn run) { job_registry()[job_class] = run; return true; }

}  // namespace mlease_jobs

using namespace mlease_jobs;

extern "C" {
const char* mlease_job_last_error(void) { return g_job_err.c_str(); }

// job_class: Regression | RegressionPrepare | RegressionAdmmTrain | RegressionTest | RegressionTestLoglik | RegressionNaiveTrain |
// ItemModelTest | ItemModelTestLoglik | ItemModelTrain | ItemModelGridTest
// (the README's names AdmmPrepare / AdmmTrain / AdmmTest / AdmmTestLoglik / NaiveTrain are accepted as aliases).
int mlease_job_run(const char* job_class, const char* config_path) {
  try {
    JobConfig c = JobConfig::load(config_path);
    std::string j = job_class;
    // host-layer knobs (not reference keys): zlib level of the files written, worker threads of the avro readers / writers
    set_default_deflate_level(c.get_int("avro.deflate.level", 1));
    if (c.has("host.threads")) set_host_threads(c.get_int("host.threads"));
    if (j == "Regression") run_regression(c);
    else if (j == "RegressionPrepare" || j == "AdmmPrepare") run_prepare(c);
    else if (j == "RegressionAdmmTrain" || j == "AdmmTrain") run_admm_train(c);
    else if (j == "RegressionTest" || j == "AdmmTest") run_test(c);
    else if (j == "RegressionTestLoglik" || j == "AdmmTestLoglik") run_test_loglik(c);
    else if (j == "RegressionNaiveTrain" || j == "NaiveTrain") run_naive_train(c);
    else if (auto it = job_registry().find(j); it != job_registry().end()) it->second(c);
    else { g_job_err = "unknown job class " + j; return 1; }
    return 0;
  } catch (const std::exception& e) {
    g_job_err = e.what();
    return 2;
  }
}

// deterministic host logic exposed for bit-exact tests against the oracle -----------------------------------------
// RegressionPrepare key/weight rule for one record stream (jobs/RegressionPrepare.java:154-186); base_key is either the
// map.key value or the externally drawn floor(random*nblocks).
int mlease_prepare_keys(int64_t nrows, const int32_t* base_key, const int32_t* response, const double* weight_in, int32_t nblocks,
                        int32_t num_click_replicates, int32_t random_key_mode, int32_t* out_keys, int32_t* out_nkeys, float* out_weight) {
  for (int64_t i = 0; i < nrows; i++) {
    double w = weight_in ? weight_in[i] : 1.0;
    if (response[i] == 1) w = w / num_click_replicates;
    out_weight[i] = (float)w;
    int32_t* ok = out_keys + i * num_click_replicates;
    if (random_key_mode && response[i] == 1) {
      int pid = base_key[i];
      for (int c = 0; c < num_click_replicates; c++) { if (pid >= nblocks) pid -= nblocks; ok[c] = pid; pid++; }
      out_nkeys[i] = num_click_replicates;
    } else { ok[0] = base_key[i]; out_nkeys[i] = 1; }
  }
  return 0;
}
// PartitionIdAssigner ids + NaivePartitioner partitions (jobs/PartitionIdAssigner.java:79-88; jobs/RegressionNaiveTrain.java:269-283)
int mlease_partition_ids(int32_t nkeys, const char* keys_packed, const float* lambdas, int32_t L, int32_t num_reducers, int32_t* out_ids,
                         int32_t* out_partition, int32_t* out_hash_partition) {
  std::vector<std::string> keys; const char* p = keys_packed;
  for (int i = 0; i < nkeys; i++) { keys.emplace_back(p); p += keys.back().size() + 1; }
  std::set<std::string> ks(keys.begin(), keys.end());
  std::vector<float> ls(lambdas, lambdas + L);
  auto ids = assign_partition_ids(ks, ls);
  for (int l = 0; l < L; l++)
    for (int i = 0; i < nkeys; i++) {
      std::string full = java_float_to_string(lambdas[l]) + "#" + keys[i];
      int id = ids[full];
      out_ids[(size_t)l * nkeys + i] = id;
      if (out_partition) out_partition[(size_t)l * nkeys + i] = id % num_reducers;
      if (out_hash_partition) { int32_t h = java_string_hash(full); int32_t a = h == INT32_MIN ? h : std::abs(h); out_hash_partition[(size_t)l * nkeys + i] = a % num_reducers; }
    }
  return 0;
}
int mlease_java_float_to_string(float f, char* buf, int32_t buflen) {
  std::string s = java_float_to_string(f);
  if ((int)s.size() + 1 > buflen) return 1;
  std::memcpy(buf, s.c_str(), s.size() + 1);
  return 0;
}
// Model files as the jobs write them (test hook for the direct encoder): `names` / `keys` are NUL-separated lists, coefs is
// [nmodels][nfeatures + 1] with the intercept last; uplusx (same shape, may be NULL) selects RegressionTrainOutput records.
int mlease_models_write(const char* path, int32_t nfeatures, const char* names, int32_t nmodels, const char* keys, const float* coefs, const float* uplusx,
                        int32_t generic) {
  try {
    Dictionary dict;
    const char* p = names;
    for (int k = 0; k < nfeatures; k++) { std::string n(p); p += n.size() + 1; dict.add(n); }
    if ((int)dict.names.size() != nfeatures) io_error("duplicate feature names");
    std::vector<std::pair<std::string, std::vector<float>>> models;
    std::vector<std::vector<float>> ux;
    p = keys;
    for (int m = 0; m < nmodels; m++) {
      std::string k(p); p += k.size() + 1;
      models.emplace_back(k, std::vector<float>(coefs + (size_t)m * (nfeatures + 1), coefs + (size_t)(m + 1) * (nfeatures + 1)));
      if (uplusx) ux.emplace_back(uplusx + (size_t)m * (nfeatures + 1), uplusx + (size_t)(m + 1) * (nfeatures + 1));
    }
    g_force_generic = generic != 0;
    try { write_model_records(path, dict, models, uplusx ? &ux : nullptr); } catch (...) { g_force_generic = false; throw; }
    g_force_generic = false;
    return 0;
  } catch (const std::exception& e) { g_job_err = e.what(); return 2; }
}
// RegressionTest's output step as a library call (and test hook): the records of in_path with unions removed and `pred` appended.
int mlease_test_output_write(const char* in_path, const char* out_path, const float* pred, int64_t npred, int32_t generic) {
  try {
    std::vector<float> pv(pred, pred + npred);
    g_force_generic = generic != 0;
    try { write_test_output(in_path, out_path, pv); } catch (...) { g_force_generic = false; throw; }
    g_force_generic = false;
    return 0;
  } catch (const std::exception& e) { g_job_err = e.what(); return 2; }
}
// RegressionTestLoglik's input step (test hook): (response, pred, weight) of the scored records of one file; returns the count or -1.
int64_t mlease_scored_read(const char* path, int64_t cap, int32_t* response, float* pred, float* weight, int32_t generic) {
  try {
    std::vector<int32_t> r; std::vector<float> p, w;
    g_force_generic = generic != 0;
    try { read_scored(path, r, p, w); } catch (...) { g_force_generic = false; throw; }
    g_force_generic = false;
    const size_t n = std::min<size_t>(r.size(), (size_t)std::max<int64_t>(cap, 0));
    if (response) std::memcpy(response, r.data(), n * 4);
    if (pred) std::memcpy(pred, p.data(), n * 4);
    if (weight) std::memcpy(weight, w.data(), n * 4);
    return (int64_t)r.size();
  } catch (const std::exception& e) { g_job_err = e.what(); return -1; }
}
int mlease_host_set_threads(int32_t n) { set_host_threads(n); return host_threads(); }

// The job layer's record ingest as a library call (and the hook the tests use to compare the block-parallel readers with the
// generic one): prepared (raw = 0, a file or a directory) or raw (raw = 1, one file) records -> CSR with first-seen feature ids.
struct mlease_rows { Dictionary dict; Rows rows; };
int mlease_rows_read(const char* path, int32_t raw, int32_t binary_feature, int32_t generic, mlease_rows** out) {
  try {
    auto r = std::make_unique<mlease_rows>();
    g_force_generic = generic != 0;
    try {
      if (raw) read_raw(path, r->dict, r->rows, binary_feature != 0);
      else read_prepared(path, r->dict, r->rows, binary_feature != 0);
    } catch (...) { g_force_generic = false; throw; }
    g_force_generic = false;
    *out = r.release();
    return 0;
  } catch (const std::exception& e) { g_job_err = e.what(); return 2; }
}
int64_t mlease_rows_count(const mlease_rows* r, int64_t* nnz, int32_t* nfeatures) {
  if (nnz) *nnz = (int64_t)r->rows.colidx.size();
  if (nfeatures) *nfeatures = (int32_t)r->dict.names.size();
  return (int64_t)r->rows.n();
}
int mlease_rows_get(const mlease_rows* r, int64_t* rowptr, int32_t* colidx, float* vals, int32_t* response, float* weight, float* offset) {
  const Rows& w = r->rows;
  if (rowptr) std::memcpy(rowptr, w.rowptr.data(), w.rowptr.size() * sizeof(int64_t));
  if (colidx) std::memcpy(colidx, w.colidx.data(), w.colidx.size() * sizeof(int32_t));
  if (vals) std::memcpy(vals, w.vals.data(), w.vals.size() * sizeof(float));
  if (response) std::memcpy(response, w.response.data(), w.response.size() * sizeof(int32_t));
  if (weight) std::memcpy(weight, w.weight.data(), w.weight.size() * sizeof(float));
  if (offset) std::memcpy(offset, w.offset.data(), w.offset.size() * sizeof(float));
  return 0;
}
const char* mlease_rows_feature(const mlease_rows* r, int32_t k) { return (k >= 0 && (size_t)k < r->dict.names.size()) ? r->dict.names[k].c_str() : nullptr; }
const char* mlease_rows_key(const mlease_rows* r, int64_t i) { return (i >= 0 && (size_t)i < r->rows.key.size()) ? r->rows.key[i].c_str() : nullptr; }
void mlease_rows_free(mlease_rows* r) { delete r; }

// avro helpers for tests: decode a container file into CSR arrays is done in Python; here: count + re-encode round trip
int mlease_avro_copy(const char* in_path, const char* out_path, const char* codec, int64_t* nrecords, int64_t* nblocks) {
  try {
    AvroReader rd(in_path);
    AvroWriter w(out_path, rd.schema_json(), codec);
    Value v; int64_t n = 0;
    while (rd.next(v)) { w.append(v); n++; }
    w.close();
    if (nrecords) *nrecords = n;
    if (nblocks) *nblocks = rd.blocks_read();
    return 0;
  } catch (const std::exception& e) { g_job_err = e.what(); return 2; }
}
}  // extern "C"
