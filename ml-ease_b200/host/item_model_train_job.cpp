// item_model_train_job.cpp -- ItemModelTrain (jobs/ItemModelTrain.java:89-321): per key, one LibLinear fit for every (intercept lambda,
// default lambda) pair, written as LinearModelWithVarAvro records under output.model.path/models.  Reached through mlease_job_run
// (register_job); the fits and their posterior variance are one mlease_item_model_train call, or with prior.model.path the fit of
// item_model_prior.cpp.
#include <cmath>

#include "jobs_common.hpp"

namespace mlease_jobs {
namespace {

// intercept.prior.mean.map: Pair records {key, value}, value = Double.parseDouble(value.toString()) (:293-301), so a float value
// is read through its Float.toString digits
std::unordered_map<std::string, double> read_prior_mean_map(const std::string& path) {
  std::unordered_map<std::string, double> out;
  for (auto& f : list_avro_files(path)) {
    AvroReader rd(f);
    const Schema& s = rec_schema(rd.schema());
    Value rec;
    while (rd.next(rec)) {
      const Value* k = field(rec, s, "key");
      const Value* v = field(rec, s, "value");
      if (!k || !v) io_error("intercept.prior.mean.map: a record without key or value");
      double d;
      if (v->type == Schema::String) {
        try { d = std::stod(JobConfig::trim(v->s)); } catch (const std::exception&) { io_error("For input string: \"" + v->s + "\""); }
      } else if (v->type == Schema::Float) d = std::stod(java_float_to_string((float)v->d));
      else if (v->type == Schema::Double) d = v->d;
      else if (v->type == Schema::Int || v->type == Schema::Long) d = (double)v->i;
      else io_error("intercept.prior.mean.map: value of key " + k->s + " is not a number or a string");
      out[k->s] = d;   // HashMap.put: the last record of a key wins
    }
  }
  return out;
}

ItemPriorHooks& prior_hooks() {
  static ItemPriorHooks h{nullptr, nullptr};
  return h;
}

// the fits of every key and grid point into f's dense outputs (mlease_item_model_train), one key range per device
void fit_dense(ItemModelFit& f) {
  const int K = (int)f.knames.size(), D = f.D, Dt = D + 1, IL = (int)f.il.size(), DL = (int)f.dl.size();
  const float* lm = f.lambda_map.empty() ? nullptr : f.lambda_map.data();
  if (f.devs.size() == 1)
    ck(mlease_item_model_train(f.devs[0], nullptr, K, D, f.krs.data(), f.rp.data(), f.ci.data(), f.vv.data(), f.rr.data(), f.ww.data(),
                               f.oo.data(), f.means.data(), IL, f.il.data(), DL, f.dl.data(), lm, f.binary ? 1 : 0, f.compute_var ? 1 : 0,
                               f.m.data(), f.compute_var ? f.var.data() : nullptr));
  else
    // one key range per device (shard_keys); each range's models and variances go to their slices
    run_shards(f.devs, shard_keys(f.krs, f.rp, D, (int)f.devs.size()), [&](int32_t dev, int k0, int k1) {
      const KeySlice s(f.krs, f.rp, k0, k1);
      const int Ks = k1 - k0;
      std::vector<double> ms((size_t)IL * DL * Ks * Dt), vs(f.compute_var ? ms.size() : 0);
      ck(mlease_item_model_train(dev, nullptr, Ks, D, s.krs.data(), s.rowptr.data(), f.ci.data() + s.nz0, f.vv.data() + s.nz0,
                                 f.rr.data() + s.row0, f.ww.data() + s.row0, f.oo.data() + s.row0, f.means.data() + k0, IL, f.il.data(), DL,
                                 f.dl.data(), lm, f.binary ? 1 : 0, f.compute_var ? 1 : 0, ms.data(), f.compute_var ? vs.data() : nullptr));
      for (int g = 0; g < IL * DL; g++) {
        std::copy(ms.begin() + (size_t)g * Ks * Dt, ms.begin() + (size_t)(g + 1) * Ks * Dt, f.m.begin() + ((size_t)g * K + k0) * Dt);
        if (f.compute_var) std::copy(vs.begin() + (size_t)g * Ks * Dt, vs.begin() + (size_t)(g + 1) * Ks * Dt, f.var.begin() + ((size_t)g * K + k0) * Dt);
      }
    });
}

void run_item_model_train(const JobConfig& c) {
  const std::string out = c.get("output.model.path");
  ItemModelFit f;
  f.binary = c.get_bool("binary.feature", false);
  f.compute_var = c.get_bool("compute.var", false);
  f.il = lambda_list(c, "intercept.lambdas"); f.dl = lambda_list(c, "default.lambdas");
  // conf.setFloat / getFloat (:112, :165): the default intercept prior mean is float-rounded
  const double default_mean = (double)(float)c.get_double("intercept.default.prior.mean", 0.0);
  std::unordered_map<std::string, double> mean_map;
  if (!c.get("intercept.prior.mean.map", "").empty()) mean_map = read_prior_mean_map(c.get("intercept.prior.mean.map"));
  // liblinear.epsilon, report.frequency and short.feature.index are accepted; the fit is an exact Newton solve
  Dictionary dict; Rows rows;
  read_prepared(c.get("input.paths"), dict, rows, f.binary);
  // prior.model.path: an earlier run's models as each key's prior; the features they name join the dictionary, no row listing them
  std::shared_ptr<ItemPriors> prior;
  if (!c.get("prior.model.path", "").empty()) {
    if (!prior_hooks().read) io_error("prior.model.path: this build of ItemModelTrain has no per-key priors");
    prior = prior_hooks().read(c, dict);
  }
  const int D = (int)dict.names.size(), Dt = D + 1;
  f.D = D;
  std::vector<std::pair<std::string, float>> lm_entries;
  if (!c.get("lambda.map", "").empty()) {
    lm_entries = read_lambda_map_entries(c.get("lambda.map"));
    f.lambda_map.assign(D, 0.f);
    for (auto& e : lm_entries) if (const int k = dict.find(e.first); k >= 0) f.lambda_map[k] = e.second;
  }
  // one dataset per key (:227-239), keys in Avro string order; a row's features sorted by id (llf/LibLinearDataset.java:481-482)
  std::map<std::string, std::vector<size_t>> by_key;
  for (size_t i = 0; i < rows.n(); i++) by_key[rows.key[i]].push_back(i);
  const int K = (int)by_key.size();
  for (auto& kv : by_key) {
    f.knames.push_back(kv.first);
    auto it = mean_map.find(kv.first);
    f.means.push_back(it != mean_map.end() ? it->second : default_mean);   // :240-248
    for (size_t i : kv.second) {
      std::vector<std::pair<int32_t, float>> ent;
      for (int64_t j = rows.rowptr[i]; j < rows.rowptr[i + 1]; j++) ent.emplace_back(rows.colidx[j], rows.vals[j]);
      std::sort(ent.begin(), ent.end(), [](auto& a, auto& b) { return a.first < b.first; });
      for (auto& e : ent) { f.ci.push_back(e.first); f.vv.push_back(e.second); }
      f.rp.push_back((int64_t)f.ci.size());
      f.rr.push_back(rows.response[i]); f.ww.push_back(rows.weight[i]); f.oo.push_back(rows.offset[i]);
    }
    f.krs.push_back((int64_t)f.rr.size());
  }
  // a key's model lists the intercept and the features its rows list (llf/LibLinear.java:343-350)
  f.cols.resize(K);
  for (int k = 0; k < K; k++) {
    std::vector<int32_t>& pk = f.cols[k];
    pk.assign(f.ci.begin() + f.rp[f.krs[k]], f.ci.begin() + f.rp[f.krs[k + 1]]);
    std::sort(pk.begin(), pk.end());
    pk.erase(std::unique(pk.begin(), pk.end()), pk.end());
  }
  f.var_cols = f.cols;
  const int IL = (int)f.il.size(), DL = (int)f.dl.size();
  f.m.assign((size_t)IL * DL * K * Dt, 0.0);
  f.var.assign(f.compute_var ? f.m.size() : 0, 0.0);
  f.devs = gpu_devices(c);
  if (K > 0 && prior) prior_hooks().fit(*prior, f);
  else if (K > 0) fit_dense(f);
  // posteriorVar also lists every lambda.map feature it does not list yet, at its prior variance 1/lambda (llf/LibLinear.java:384-397),
  // after the dataset's (and the prior's) features, in the map's order; the intercept's entry is always the dataset's
  auto absent_map_entries = [&](int k) {
    std::vector<int32_t> listed(f.var_cols[k]);
    std::sort(listed.begin(), listed.end());
    std::vector<std::pair<std::string, float>> ex;
    for (auto& e : lm_entries) {
      if (e.first == INTERCEPT) continue;
      const int id = dict.find(e.first);
      if (id >= 0 && std::binary_search(listed.begin(), listed.end(), id)) continue;
      ex.emplace_back(e.first, (float)(1.0 / (double)e.second));
    }
    return ex;
  };
  AvroWriter w(out + "/models/part-r-00000.avro", SCHEMA_MODEL_WITH_VAR);
  const bool generic = host_generic_ingest();
  const FeaturePrefix fp(dict);
  std::vector<float> mf(Dt), vf(Dt);
  std::string rec;
  for (int k = 0; k < K; k++) {
    const auto extra = f.compute_var ? absent_map_entries(k) : std::vector<std::pair<std::string, float>>();
    const std::vector<int32_t>& mc = f.cols[k];
    const std::vector<int32_t>& vc = f.var_cols[k];
    for (int a = 0; a < IL; a++)
      for (int b = 0; b < DL; b++) {
        const size_t base = (((size_t)a * DL + b) * K + k) * Dt;
        for (int j = 0; j < Dt; j++) { mf[j] = (float)f.m[base + j]; vf[j] = f.compute_var ? (float)f.var[base + j] : 0.f; }
        const std::string key = java_float_to_string(f.il[a]) + ":" + java_float_to_string(f.dl[b]) + "#" + f.knames[k];   // :265
        if (generic) {   // Value-tree encoder: the reference implementation the tests compare with
          Value r; r.type = Schema::Record; r.items.resize(3);
          r.items[0] = Value::of_string(key);
          Value& ml = r.items[1]; ml.type = Schema::Array;
          ml.items.push_back(feature_value(INTERCEPT, mf[D]));
          for (int32_t j : mc) ml.items.push_back(feature_value(dict.names[j], mf[j]));
          Value& vl = r.items[2]; vl.type = Schema::Array;
          vl.items.push_back(feature_value(INTERCEPT, vf[D]));   // without compute.var: new LinearModel().toAvro, (INTERCEPT) 0 (:271-274)
          if (f.compute_var) {
            for (int32_t j : vc) vl.items.push_back(feature_value(dict.names[j], vf[j]));
            for (auto& e : extra) vl.items.push_back(feature_value(e.first, e.second));
          }
          w.append(r);
        } else {
          rec.clear();
          put_str(rec, key.data(), key.size());
          fp.encode_subset(rec, mf.data(), mc);
          if (f.compute_var) {
            put_long(rec, (int64_t)(1 + vc.size() + extra.size()));
            rec.append(fp.bytes, fp.off[0], fp.off[1] - fp.off[0]); put_float(rec, vf[D]);
            for (int32_t j : vc) { rec.append(fp.bytes, fp.off[(size_t)j + 1], fp.off[(size_t)j + 2] - fp.off[(size_t)j + 1]); put_float(rec, vf[j]); }
            for (auto& e : extra) { put_feature_key(rec, e.first); put_float(rec, e.second); }
            put_long(rec, 0);
          } else {
            put_long(rec, 1); put_feature_key(rec, INTERCEPT); put_float(rec, 0.f); put_long(rec, 0);
          }
          w.append_encoded(rec.data(), rec.size(), 1);
        }
      }
  }
  w.close();
  if (c.get_bool("remove.tmp.dir", true)) remove_tree(out + "/tmp-data");   // :122-127
}

[[maybe_unused]] const bool registered = register_job("ItemModelTrain", run_item_model_train);

}  // namespace

bool register_item_model_prior(const ItemPriorHooks& h) {
  prior_hooks() = h;
  return true;
}
}  // namespace mlease_jobs
