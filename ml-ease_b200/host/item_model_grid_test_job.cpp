// item_model_grid_test_job.cpp -- ItemModelGridTest: scores held-out records with every (intercept lambda, default lambda) model
// ItemModelTrain wrote for their key ("<il>:<dl>#<key>" LinearModelWithVarAvro records), with each record's predictive variance
// under the model's diagonal posterior when compute.var is set, and one test log-likelihood per grid point, so that a user can
// pick the pair that does best on held-out data.  Reached through mlease_job_run (register_job); the scores are one
// mlease_score_keyed(_var) call per device and the log-likelihoods one mlease_test_loglik_keyed call.
#include <cmath>

#include "jobs_common.hpp"

namespace mlease_jobs {
namespace {

// one "<il>:<dl>#<key>" record: its coefficients and, when the file has the field, its posteriorVar list (feature key -> value;
// a repeated feature keeps its last value)
struct GridModel {
  std::unordered_map<std::string, double> coef;
  std::vector<std::pair<std::string, float>> var;
  bool has_var = false;
};

std::string feature_key_of(const Value& fv) { return fv.items[1].s.empty() ? fv.items[0].s : fv.items[0].s + "\x01" + fv.items[1].s; }

// model and posteriorVar of every record under path; a repeated key keeps its last record (HashMap.put)
std::map<std::string, GridModel> read_grid_models(const std::string& path) {
  std::map<std::string, GridModel> out;
  for (auto& f : list_avro_files(path)) {
    AvroReader rd(f);
    const Schema& s = rec_schema(rd.schema());
    const int ki = s.field_index("key"), mi = s.field_index("model"), vi = s.field_index("posteriorVar");
    if (ki < 0 || mi < 0) io_error("model.path: " + f + " holds no {key, model} records");
    Value rec;
    while (rd.next(rec)) {
      GridModel& m = out[rec.items[ki].s];
      m = GridModel();
      for (auto& fv : rec.items[mi].items) m.coef[feature_key_of(fv)] = fv.items[2].d;
      if (vi >= 0 && !rec.items[vi].is_null()) {
        m.has_var = true;
        for (auto& fv : rec.items[vi].items) m.var.emplace_back(feature_key_of(fv), (float)fv.items[2].d);
      }
    }
  }
  return out;
}

std::string display_feature(std::string k) {
  std::replace(k.begin(), k.end(), '\x01', ' ');
  return k;
}

void run_item_model_grid_test(const JobConfig& c) {
  const std::string in = c.get("input.paths"), outBase = c.get("output.base.path"), itemKey = c.get("item.key");
  const bool ignore_value = c.get_bool("binary.feature", false);
  const bool compute_var = c.get_bool("compute.var", false);
  const std::vector<float> il = lambda_list(c, "intercept.lambdas"), dl = lambda_list(c, "default.lambdas");
  const std::vector<std::string> il_typed = c.get_list("intercept.lambdas"), dl_typed = c.get_list("default.lambdas");
  // the grid: the cross product in config order, g = a * DL + b, as ItemModelTrain writes it; a repeated point is refused
  const int IL = (int)il.size(), DL = (int)dl.size(), G = IL * DL;
  std::vector<std::string> gkey(G), gdir(G);
  for (int a = 0; a < IL; a++)
    for (int b = 0; b < DL; b++) {
      const int g = a * DL + b;
      gkey[g] = java_float_to_string(il[a]) + ":" + java_float_to_string(dl[b]);
      gdir[g] = outBase + "/lambda-" + il_typed[a] + "_" + dl_typed[b];
      for (int h = 0; h < g; h++)
        if (gkey[h] == gkey[g]) io_error("intercept.lambdas x default.lambdas: grid point " + gkey[g] + " is repeated");
    }
  const auto files = list_avro_files(in);
  if (files.empty()) io_error("no input files under " + in);
  Dictionary td; Rows rows;
  std::vector<size_t> file_end;   // one combiner group per input file
  for (auto& f : files) { read_raw(f, td, rows, ignore_value, itemKey); file_end.push_back(rows.n()); }
  const size_t n = rows.n();
  KeyedRows kr(rows);
  const int K = (int)kr.knames.size();
  const int Dg = std::max<int>((int)td.names.size(), 1);
  if (compute_var) {
    // a record's entries in dictionary order, each feature once: the device counts every listing as an independent feature
    std::vector<std::pair<int32_t, float>> ent;
    for (int k = 0; k < K; k++)
      for (int64_t i = kr.krs[k]; i < kr.krs[k + 1]; i++) {
        ent.clear();
        for (int64_t j = kr.rp[i]; j < kr.rp[i + 1]; j++) ent.emplace_back(kr.ci[j], kr.vv[j]);
        std::stable_sort(ent.begin(), ent.end(), [](auto& x, auto& y) { return x.first < y.first; });
        for (size_t e = 0; e < ent.size(); e++) {
          if (e > 0 && ent[e].first == ent[e - 1].first)
            io_error("a record of key " + kr.knames[k] + " lists feature " + display_feature(td.names[ent[e].first]) +
                     " more than once; its predictive variance would count the listings as independent features");
          kr.ci[kr.rp[i] + e] = ent[e].first; kr.vv[kr.rp[i] + e] = ent[e].second;
        }
      }
  }
  // models and variance lists over (grid point, key), m = g * K + k, mapped to the test dictionary as ItemModelTest maps them:
  // features the test data never lists are dropped, "(INTERCEPT)" is column Dg.  A key without a model gets the empty model and an
  // empty variance list (predVar NaN).  var_default = 1/dl, the prior variance of a feature outside lambda.map
  // (jobs/ItemModelTrain.java:262); lambda.map features a key's rows never list are already in its posteriorVar.
  const auto models = read_grid_models(c.get("model.path"));
  std::vector<int64_t> mp{0}, vp{0};
  std::vector<int32_t> mc, vc;
  std::vector<float> mv, vv, vdef;
  std::map<int32_t, float> ent;
  auto col_of = [&](const std::string& f) { return f == INTERCEPT ? Dg : td.find(f); };
  for (int g = 0; g < G; g++)
    for (int k = 0; k < K; k++) {
      const std::string mkey = gkey[g] + "#" + kr.knames[k];
      auto it = models.find(mkey);
      if (it != models.end()) {
        ent.clear();
        for (auto& fv : it->second.coef) if (const int id = col_of(fv.first); id >= 0) ent[id] = (float)fv.second;
        for (auto& e : ent) { mc.push_back(e.first); mv.push_back(e.second); }
        if (compute_var) {
          const auto& var = it->second.var;
          if (!it->second.has_var || (var.size() == 1 && var[0].first == INTERCEPT && var[0].second == 0.f))
            io_error("model " + mkey + " has no posterior variance (its posteriorVar is the (INTERCEPT) 0 placeholder): rerun ItemModelTrain "
                     "with compute.var=true");
          ent.clear();
          for (auto& fv : var) if (const int id = col_of(fv.first); id >= 0) ent[id] = fv.second;
          for (auto& e : ent) { vc.push_back(e.first); vv.push_back(e.second); }
        }
      }
      mp.push_back((int64_t)mc.size());
      vp.push_back((int64_t)vc.size());
      vdef.push_back((float)(1.0 / (double)dl[g % DL]));
    }
  std::vector<float> pred((size_t)G * n), pvar(compute_var ? pred.size() : 0);
  auto score = [&](int32_t dev, int Ks, const int64_t* krs, const int64_t* rp, const int32_t* ci, const float* v, const float* o,
                   const int64_t* smp, const int32_t* smc, const float* smv, const int64_t* svp, const int32_t* svc, const float* svv,
                   const float* svd, float* out, float* out_var) {
    if (compute_var)
      ck(mlease_score_keyed_var(dev, nullptr, Dg, Ks, krs, rp, ci, v, o, G, smp, smc, smv, svp, svc, svv, svd, ignore_value ? 1 : 0, out, out_var));
    else
      ck(mlease_score_keyed(dev, nullptr, Dg, Ks, krs, rp, ci, v, o, G, smp, smc, smv, ignore_value ? 1 : 0, out));
  };
  const std::vector<int32_t> devs = gpu_devices(c);
  if (devs.size() == 1 || K == 0) {
    score(devs[0], K, kr.krs.data(), kr.rp.data(), kr.ci.data(), kr.vv.data(), kr.oo.data(), mp.data(), mc.data(), mv.data(), vp.data(),
          vc.data(), vv.data(), vdef.data(), pred.data(), pvar.data());
  } else {
    // one key range per device (shard_keys) with its models and variance lists; each range's results go to their slices
    run_shards(devs, shard_keys(kr.krs, kr.rp, Dg, (int)devs.size()), [&](int32_t dev, int k0, int k1) {
      const KeySlice s(kr.krs, kr.rp, k0, k1);
      const int Ks = k1 - k0;
      const int64_t ns = s.krs[Ks];
      std::vector<int64_t> smp, svp; std::vector<int32_t> smc, svc; std::vector<float> smv, svv, svd;
      slice_model_lists(mp, mc, mv, G, K, k0, k1, smp, smc, smv);
      slice_model_lists(vp, vc, vv, G, K, k0, k1, svp, svc, svv);
      for (int g = 0; g < G; g++) svd.insert(svd.end(), vdef.begin() + (size_t)g * K + k0, vdef.begin() + (size_t)g * K + k1);
      std::vector<float> sp((size_t)G * ns), sv(compute_var ? sp.size() : 0);
      score(dev, Ks, s.krs.data(), s.rowptr.data(), kr.ci.data() + s.nz0, kr.vv.data() + s.nz0, kr.oo.data() + s.row0, smp.data(), smc.data(),
            smv.data(), svp.data(), svc.data(), svv.data(), svd.data(), sp.data(), sv.data());
      for (int g = 0; g < G; g++) {
        std::copy(sp.begin() + (size_t)g * ns, sp.begin() + (size_t)(g + 1) * ns, pred.begin() + (size_t)g * n + s.row0);
        if (compute_var) std::copy(sv.begin() + (size_t)g * ns, sv.begin() + (size_t)(g + 1) * ns, pvar.begin() + (size_t)g * n + s.row0);
      }
    });
  }
  // one log-likelihood per grid point (ItemModelTestLoglik's rounding points): an entry per (record, grid point) with entry key = grid
  // point, records in input order, one combiner group per input file
  std::vector<float> ll(G, std::nanf("")); std::vector<double> cnt(G, 0.0);
  if (n > 0) {
    std::vector<size_t> pos(n);
    for (size_t q = 0; q < n; q++) pos[kr.order[q]] = q;
    std::vector<int32_t> ekey, egroup, eresp;
    std::vector<float> ew, ep;
    size_t i = 0;
    for (size_t f = 0; f < files.size(); f++)
      for (; i < file_end[f]; i++)
        for (int g = 0; g < G; g++) {
          ekey.push_back(g); egroup.push_back((int32_t)f); eresp.push_back(rows.response[i]); ew.push_back(rows.weight[i]);
          ep.push_back(pred[(size_t)g * n + pos[i]]);
        }
    ck(mlease_test_loglik_keyed(devs[0], nullptr, (int64_t)ekey.size(), ekey.data(), egroup.data(), eresp.data(), ew.data(), ep.data(), G,
                                ll.data(), cnt.data()));
  }
  // output per grid point: every input field (unions removed) + pred (+ predVar), grouped by key as ItemModelTest writes them
  AvroReader first(files[0]);
  for (size_t f = 1; f < files.size(); f++)
    if (AvroReader(files[f]).schema_json() != first.schema_json()) io_error("input files of one ItemModelGridTest job must share one schema: " + files[f]);
  const std::string schema = test_output_schema(first.schema(), "ItemModelGridTestOutput", "com.linkedin.lab.regression.avro", compute_var);
  std::vector<std::string> plain;
  bool fast = !host_generic_ingest();
  for (size_t f = 0; fast && f < files.size(); f++) fast = plain_records(files[f], plain);
  std::vector<Value> recs;
  if (!fast) {
    for (auto& f : files) { AvroReader rd(f); Value v; while (rd.next(v)) recs.push_back(v); }
  }
  for (int g = 0; g < G; g++) {
    AvroWriter w(gdir[g] + "/part-r-00000.avro", schema);
    const float* pg = pred.data() + (size_t)g * n;
    const float* vg = compute_var ? pvar.data() + (size_t)g * n : nullptr;
    std::string rec;
    for (size_t q = 0; q < n; q++) {
      const size_t i = kr.order[q];
      if (fast) {
        rec = plain[i]; put_float(rec, pg[q]);
        if (vg) put_float(rec, vg[q]);
        w.append_encoded(rec.data(), rec.size(), 1);
      } else {
        Value r = recs[i]; r.items.push_back(Value::of_float(pg[q]));
        if (vg) r.items.push_back(Value::of_float(vg[q]));
        w.append(r);
      }
    }
    w.close();
  }
  AvroWriter w(outBase + "/_loglik/part-r-00000.avro", SCHEMA_TEST_LOGLIK);
  for (int g = 0; g < G; g++) {
    Value r; r.type = Schema::Record;
    r.items = {Value::of_string(gkey[g]), Value::of_float(ll[g]), Value::of_double(cnt[g])};
    w.append(r);
  }
  w.close();
}

[[maybe_unused]] const bool registered = register_job("ItemModelGridTest", run_item_model_grid_test);

}  // namespace
}  // namespace mlease_jobs
