// regression_posterior_job.cpp -- RegressionPosterior: the posterior variance of the models RegressionAdmmTrain wrote to
// <output.base.path>/final-model, one LinearModelWithVarAvro record per lambda under <output.base.path>/final-model-var.  The Prepare
// output is reloaded into a mlease_world partition by partition as RegressionAdmmTrain loads it, and each lambda's posterior is one
// mlease_world_admm_posterior call at that lambda's final model: 1 / hessianDiagonal, or diag(H^-1) with compute.full.var (the
// computePosteriorVar / computeFullPostVar tail of llf/LibLinear.java:315-334).  Reached through mlease_job_run (register_job); kept
// out of regression_jobs.cpp so that the libraries built from that file do not reference the posterior entry points.
#include <algorithm>
#include <cstring>

#include "jobs_common.hpp"

namespace mlease_jobs {
namespace {

void run_regression_posterior(const JobConfig& c) {
  const std::string out = c.get("output.base.path");
  const int nblocks = c.get_int("num.blocks");
  if (c.get_int("regularizer", 2) == 1) io_error("RegressionPosterior: the L1 penalty has no Hessian (regularizer must be 2)");
  const bool binary = c.get_bool("binary.feature", false);
  const bool full = c.get_bool("compute.full.var", false);
  std::vector<float> lambdas = parse_lambdas(c);
  const int L = (int)lambdas.size();
  if (L == 0) io_error("RegressionPosterior: lambda is empty");

  Dictionary dict;
  Rows rows;
  read_prepared(c.get("input.paths", out + "/tmp-data"), dict, rows, binary);
  const int D = (int)dict.names.size(), Dt = D + 1;
  std::vector<std::vector<size_t>> by_part(nblocks);
  for (size_t i = 0; i < rows.n(); i++) {
    const int p = java_parse_int(rows.key[i]);
    if (p < 0 || p >= nblocks) io_error("Map key is wrong! key has to be in the range of [0,numPartitions-1].");
    by_part[p].push_back(i);
  }
  for (int p = 0; p < nblocks; p++) if (by_part[p].empty()) io_error("Some models failed!");
  std::vector<float> lambda_map;
  if (!c.get("lambda.map", "").empty()) lambda_map = read_lambda_map(c.get("lambda.map"), dict);

  // final-model: one record per lambda, keyed by Float.toString(lambda); its model list is copied to the output as it is
  std::vector<Value> finals;
  std::vector<int> lam_of;
  {
    const auto files = list_avro_files(out + "/final-model");
    if (files.empty()) io_error("RegressionPosterior: no final-model under " + out + " (run RegressionAdmmTrain first)");
    for (auto& f : files) {
      AvroReader rd(f);
      const Schema& s = rec_schema(rd.schema());
      Value rec;
      while (rd.next(rec)) {
        const Value* k = field(rec, s, "key");
        const Value* m = field(rec, s, "model");
        if (!k || !m) io_error("RegressionPosterior: a final-model record without key or model");
        int l = -1;
        for (int j = 0; j < L; j++) if (java_float_to_string(lambdas[j]) == k->s) l = j;
        if (l < 0) io_error("RegressionPosterior: final-model key " + k->s + " is not one of the job's lambdas");
        Value r; r.type = Schema::Record; r.items = {*k, *m};
        finals.push_back(r);
        lam_of.push_back(l);
      }
    }
  }

  std::vector<int32_t> devs = gpu_devices(c);
  if ((int)devs.size() > nblocks) devs.resize(nblocks);
  mlease_admm_config cfg; std::memset(&cfg, 0, sizeof(cfg));
  cfg.device = devs[0]; cfg.num_blocks = nblocks; cfg.num_features = D; cfg.num_lambdas = L;
  cfg.lambdas = lambdas.data(); cfg.regularizer = 2;
  cfg.lambda_map = lambda_map.empty() ? nullptr : lambda_map.data();
  cfg.penalize_intercept = c.get_bool("penalize.intercept", false);
  cfg.binary_feature = binary;
  struct World { mlease_world* w = nullptr; ~World() { if (w) mlease_world_destroy(w); } } S;
  ck(mlease_world_create(&cfg, devs.data(), (int32_t)devs.size(), &S.w));
  for (int p = 0; p < nblocks; p++) {
    std::vector<int64_t> rp{0}; std::vector<int32_t> ci, rr; std::vector<float> vv, ww, oo;
    for (size_t i : by_part[p]) {
      // a row's features sorted by id, as the reference's dataset holds them (llf/LibLinearDataset.java:481-482)
      std::vector<std::pair<int32_t, float>> ent;
      for (int64_t j = rows.rowptr[i]; j < rows.rowptr[i + 1]; j++) ent.emplace_back(rows.colidx[j], rows.vals[j]);
      std::stable_sort(ent.begin(), ent.end(), [](auto& a, auto& b) { return a.first < b.first; });
      for (auto& e : ent) { ci.push_back(e.first); vv.push_back(e.second); }
      rp.push_back((int64_t)ci.size()); rr.push_back(rows.response[i]); ww.push_back(rows.weight[i]); oo.push_back(rows.offset[i]);
    }
    ck(mlease_world_add_partition_csr(S.w, p, (int64_t)rr.size(), rp.data(), ci.data(), vv.data(), rr.data(), ww.data(), oo.data()));
  }

  AvroWriter w(out + "/final-model-var/part-r-00000.avro", SCHEMA_MODEL_WITH_VAR);
  std::vector<double> z(Dt), var(Dt);
  for (size_t r = 0; r < finals.size(); r++) {
    // z: the final model's coefficients over the dictionary (features outside it have no row to weigh them), intercept last
    std::fill(z.begin(), z.end(), 0.0);
    for (auto& fv : finals[r].items[1].items) {
      const std::string key = fv.items[1].s.empty() ? fv.items[0].s : fv.items[0].s + "\x01" + fv.items[1].s;
      if (key == INTERCEPT) z[D] = num_of(fv.items[2]);
      else if (const int k = dict.find(key); k >= 0) z[k] = num_of(fv.items[2]);
    }
    ck(mlease_world_admm_posterior(S.w, lam_of[r], z.data(), full ? 1 : 0, var.data(), nullptr));
    Value rec = finals[r];
    Value vl; vl.type = Schema::Array;
    vl.items.push_back(feature_value(INTERCEPT, (float)var[D]));
    for (int k = 0; k < D; k++) vl.items.push_back(feature_value(dict.names[k], (float)var[k]));
    rec.items.push_back(vl);
    w.append(rec);
  }
  w.close();
}

[[maybe_unused]] const bool registered = register_job("RegressionPosterior", run_regression_posterior);

}  // namespace
}  // namespace mlease_jobs
