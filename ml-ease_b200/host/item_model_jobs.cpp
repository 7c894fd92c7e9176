// item_model_jobs.cpp -- ItemModelTest (jobs/ItemModelTest.java:53-248) and ItemModelTestLoglik (jobs/ItemModelTestLoglik.java:40-142):
// per-key scoring of RegressionNaiveTrain's "<lambda>#<key>" models and one test log-likelihood per key.  Reached through
// mlease_job_run (register_job).
#include <cmath>

#include "jobs_common.hpp"

namespace mlease_jobs {
namespace {

// ============================================================================================ ItemModelTest
// jobs/ItemModelTest.java:65-248.  Records are grouped by item key in Avro string order (unsigned bytes); inside a key they keep
// input order (files in listing order, records in file order).  One mlease_score_keyed call scores every lambda.
void run_item_model_test(const JobConfig& c) {
  const std::string in = c.get("input.paths"), outBase = c.get("output.base.path"), itemKey = c.get("item.key");
  const bool ignore_value = c.get_bool("binary.feature", false);
  const std::vector<std::string> lams = c.get_list("lambda");
  const int L = (int)lams.size();
  const auto files = list_avro_files(in);
  if (files.empty()) io_error("no input files under " + in);
  Dictionary td; Rows rows;
  for (auto& f : files) read_raw(f, td, rows, ignore_value, itemKey);
  const size_t n = rows.n();
  const KeyedRows kr(rows);
  const std::vector<size_t>& order = kr.order;
  const std::vector<std::string>& knames = kr.knames;
  const std::vector<int64_t> &krs = kr.krs, &rp = kr.rp;
  const std::vector<int32_t>& ci = kr.ci;
  const std::vector<float> &vv = kr.vv, &oo = kr.oo;
  const int K = (int)knames.size();
  // model "String.valueOf(float lambda)#itemKey" (:187); its features mapped to the test dictionary, the ones the test data never
  // lists dropped (they cannot contribute), "(INTERCEPT)" to column Dg.  A key without a model gets the empty model (:189-197).
  const int Dg = std::max<int>((int)td.names.size(), 1);
  const auto models = read_linear_models(c.get("model.path"), true);
  std::vector<int64_t> mp{0}; std::vector<int32_t> mc; std::vector<float> mv;
  std::vector<std::pair<int32_t, float>> ent;
  for (int l = 0; l < L; l++) {
    const std::string prefix = java_float_to_string(std::stof(lams[l])) + "#";
    for (int k = 0; k < K; k++) {
      auto it = models.find(prefix + knames[k]);
      if (it != models.end()) {
        ent.clear();
        for (auto& fv : it->second) {
          if (fv.first == INTERCEPT) ent.emplace_back(Dg, (float)fv.second);
          else if (const int id = td.find(fv.first); id >= 0) ent.emplace_back(id, (float)fv.second);
        }
        std::sort(ent.begin(), ent.end());
        for (auto& e : ent) { mc.push_back(e.first); mv.push_back(e.second); }
      }
      mp.push_back((int64_t)mc.size());
    }
  }
  std::vector<float> pred((size_t)L * n);
  const std::vector<int32_t> devs = gpu_devices(c);
  if (devs.size() == 1 || K == 0) {
    ck(mlease_score_keyed(devs[0], nullptr, Dg, K, krs.data(), rp.data(), ci.data(), vv.data(), oo.data(), L, mp.data(),
                          mc.data(), mv.data(), ignore_value ? 1 : 0, pred.data()));
  } else {
    // one key range per device (shard_keys) with its models; each range's preds go to their slice of pred
    run_shards(devs, shard_keys(krs, rp, Dg, (int)devs.size()), [&](int32_t dev, int k0, int k1) {
      const KeySlice s(krs, rp, k0, k1);
      const int Ks = k1 - k0;
      const int64_t ns = s.krs[Ks];
      std::vector<int64_t> smp; std::vector<int32_t> smc; std::vector<float> smv;
      slice_model_lists(mp, mc, mv, L, K, k0, k1, smp, smc, smv);
      std::vector<float> sp((size_t)L * ns);
      ck(mlease_score_keyed(dev, nullptr, Dg, Ks, s.krs.data(), s.rowptr.data(), ci.data() + s.nz0, vv.data() + s.nz0, oo.data() + s.row0, L,
                            smp.data(), smc.data(), smv.data(), ignore_value ? 1 : 0, sp.data()));
      for (int l = 0; l < L; l++) std::copy(sp.begin() + (size_t)l * ns, sp.begin() + (size_t)(l + 1) * ns, pred.begin() + (size_t)l * n + s.row0);
    });
  }
  // output: every input field (unions removed) + pred, schema PerItemTestOutput (:214-248)
  AvroReader first(files[0]);
  for (size_t f = 1; f < files.size(); f++)
    if (AvroReader(files[f]).schema_json() != first.schema_json()) io_error("input files of one ItemModelTest job must share one schema: " + files[f]);
  const std::string schema = test_output_schema(first.schema(), "PerItemTestOutput", "com.linkedin.lab.regression.avro");
  std::vector<std::string> plain;
  bool fast = !host_generic_ingest();
  for (size_t f = 0; fast && f < files.size(); f++) fast = plain_records(files[f], plain);
  std::vector<Value> recs;
  if (!fast) {
    for (auto& f : files) { AvroReader rd(f); Value v; while (rd.next(v)) recs.push_back(v); }
  }
  for (int l = 0; l < L; l++) {
    AvroWriter w(outBase + "/lambda-" + lams[l] + "/part-r-00000.avro", schema);
    const float* pl = pred.data() + (size_t)l * n;
    std::string rec;
    for (size_t q = 0; q < n; q++) {
      const size_t i = order[q];
      if (fast) { rec = plain[i]; put_float(rec, pl[q]); w.append_encoded(rec.data(), rec.size(), 1); }
      else { Value r = recs[i]; r.items.push_back(Value::of_float(pl[q])); w.append(r); }
    }
    w.close();
  }
}

// ============================================================================================ ItemModelTestLoglik
// jobs/ItemModelTestLoglik.java:60-142: one loglik per pred-map key.  One map task, hence one combiner group, per input file.
void run_item_model_test_loglik(const JobConfig& c) {
  const std::string in = c.get("input.paths"), out = c.get("output.path");
  std::vector<std::string> ekey;
  std::vector<int32_t> egroup, eresp;
  std::vector<float> ew, ep;
  int g = 0;
  for (auto& f : list_avro_files(in)) {
    AvroReader rd(f);
    const Schema& s = rec_schema(rd.schema());
    Value rec;
    while (rd.next(rec)) {
      const Value* r = field(rec, s, "response");
      const Value* pm = field(rec, s, "pred");
      if (!r || !pm) io_error("response/pred is null");
      const int resp = (int)num_of(*r);
      if (resp != 1 && resp != 0 && resp != -1) io_error("response should be 1,0 or -1!");   // :74-77
      if (pm->type != Schema::Map) io_error("pred is not a map<string, float>");
      const Value* w = field(rec, s, "weight");
      const float wt = w ? (float)num_of(*w) : 1.0f;
      for (auto& e : pm->items) { ekey.push_back(e.map_key); egroup.push_back(g); eresp.push_back(resp); ew.push_back(wt); ep.push_back((float)num_of(e)); }
    }
    g++;
  }
  std::map<std::string, int32_t> ids;   // key order of the reducer's output
  for (auto& k : ekey) ids.emplace(k, 0);
  int32_t K = 0;
  for (auto& kv : ids) kv.second = K++;
  std::vector<int32_t> eid(ekey.size());
  for (size_t e = 0; e < ekey.size(); e++) eid[e] = ids[ekey[e]];
  std::vector<float> ll(K); std::vector<double> cnt(K);
  if (!eid.empty())
    ck(mlease_test_loglik_keyed(c.get_int("gpu.device", 0), nullptr, (int64_t)eid.size(), eid.data(), egroup.data(), eresp.data(), ew.data(), ep.data(), K,
                                ll.data(), cnt.data()));
  AvroWriter w(out + "/part-r-00000.avro", SCHEMA_TEST_LOGLIK);
  for (auto& kv : ids) {
    Value r; r.type = Schema::Record;
    r.items = {Value::of_string(kv.first), Value::of_float(ll[kv.second]), Value::of_double(cnt[kv.second])};
    w.append(r);
  }
  w.close();
}

[[maybe_unused]] const bool registered = register_job("ItemModelTest", run_item_model_test) &&
                                         register_job("ItemModelTestLoglik", run_item_model_test_loglik);

}  // namespace
}  // namespace mlease_jobs
