// auc_jobs.cpp -- the area under the ROC curve of held-out predictions, the number CTR models are usually ranked by:
//   RegressionTestAuc      the counterpart of RegressionTestLoglik: one AUC per lambda-<l> and best-model directory RegressionTest
//                          wrote
//   ItemModelGridTestAuc   one AUC per (intercept lambda, default lambda) grid point ItemModelGridTest scored, and one per grid
//                          point and item key, so that a user can pick the pair that ranks held-out records best, overall or
//                          within each item
// Reached through mlease_job_run (register_job); each directory or grid is one mlease_test_auc call.  Kept in its own translation
// unit so that the jobs of regression_jobs.cpp and item_model_grid_test_job.cpp link without that symbol.
#include <cmath>
#include <cstring>

#include "jobs_common.hpp"

namespace mlease_jobs {
namespace {

const char* SCHEMA_TEST_AUC =
    "{\"type\":\"record\",\"name\":\"TestAucOutput\",\"namespace\":\"com.linkedin.mlease.regression.avro\",\"fields\":["
    "{\"name\":\"key\",\"type\":\"string\"},{\"name\":\"auc\",\"type\":\"double\"},{\"name\":\"positiveWeight\",\"type\":\"double\"},"
    "{\"name\":\"negativeWeight\",\"type\":\"double\"}]}";
const char* SCHEMA_GRID_TEST_AUC =
    "{\"type\":\"record\",\"name\":\"ItemModelGridTestAucOutput\",\"namespace\":\"com.linkedin.mlease.regression.avro\",\"fields\":["
    "{\"name\":\"key\",\"type\":\"string\"},{\"name\":\"auc\",\"type\":\"double\"},{\"name\":\"keyAuc\",\"type\":\"double\"},"
    "{\"name\":\"positiveWeight\",\"type\":\"double\"},{\"name\":\"negativeWeight\",\"type\":\"double\"}]}";

Value auc_record(const std::string& key, double auc, const double* wt) {
  Value r; r.type = Schema::Record;
  r.items = {Value::of_string(key), Value::of_double(auc), Value::of_double(wt[0]), Value::of_double(wt[1])};
  return r;
}

void run_test_auc(const JobConfig& c) {
  const std::string inBase = c.get("input.base.paths"), outBase = c.get("output.base.path");
  auto one = [&](const std::string& inPath, const std::string& outPath) {
    if (!path_exists(inPath)) return;
    std::vector<int32_t> resp; std::vector<float> pred, weight;
    for (auto& f : list_avro_files(inPath)) read_scored(f, resp, pred, weight);
    if (resp.empty()) return;
    double auc, wt[2];
    ck(mlease_test_auc(c.get_int("gpu.device", 0), nullptr, (int64_t)resp.size(), 1, pred.data(), resp.data(), weight.data(), 0, nullptr,
                       &auc, wt, nullptr, nullptr));
    AvroWriter w(outPath + "/part-r-00000.avro", SCHEMA_TEST_AUC);
    w.append(auc_record("testAuc", auc, wt));
    w.close();
  };
  if (c.has("lambda"))
    for (auto& lam : c.get_list("lambda")) one(inBase + "/lambda-" + lam, outBase + "/lambda-" + lam + "/_auc");
  one(inBase + "/best-model", outBase + "/best-model/_auc");
}

void run_item_model_grid_test_auc(const JobConfig& c) {
  const std::string inBase = c.get("input.base.path"), outBase = c.get("output.base.path"), itemKey = c.get("item.key");
  const std::vector<float> il = lambda_list(c, "intercept.lambdas"), dl = lambda_list(c, "default.lambdas");
  const std::vector<std::string> il_typed = c.get_list("intercept.lambdas"), dl_typed = c.get_list("default.lambdas");
  // the grid as ItemModelGridTest names and orders it: g = a * DL + b; a repeated point is refused
  const int IL = (int)il.size(), DL = (int)dl.size(), G = IL * DL;
  std::vector<std::string> gkey(G), gdir(G);
  for (int a = 0; a < IL; a++)
    for (int b = 0; b < DL; b++) {
      const int g = a * DL + b;
      gkey[g] = java_float_to_string(il[a]) + ":" + java_float_to_string(dl[b]);
      gdir[g] = inBase + "/lambda-" + il_typed[a] + "_" + dl_typed[b];
      for (int h = 0; h < g; h++)
        if (gkey[h] == gkey[g]) io_error("intercept.lambdas x default.lambdas: grid point " + gkey[g] + " is repeated");
    }
  // every grid directory holds the same records in the same order: grid point 0's response, weight and item key are the job's
  std::vector<int32_t> resp; std::vector<float> weight, pred; std::vector<std::string> key;
  size_t n = 0;
  for (int g = 0; g < G; g++) {
    const auto files = list_avro_files(gdir[g]);
    if (files.empty()) io_error("no scored records under " + gdir[g]);
    size_t at = 0;
    for (auto& f : files) {
      std::vector<int32_t> r; std::vector<float> p, w;
      read_scored(f, r, p, w);
      Dictionary td; Rows rows;
      read_raw(f, td, rows, false, itemKey);
      if (g == 0) {
        resp.insert(resp.end(), r.begin(), r.end()); weight.insert(weight.end(), w.begin(), w.end());
        key.insert(key.end(), rows.key.begin(), rows.key.end());
      } else {
        bool same = at + r.size() <= n;
        for (size_t i = 0; same && i < r.size(); i++)
          same = r[i] == resp[at + i] && std::memcmp(&w[i], &weight[at + i], 4) == 0 && rows.key[i] == key[at + i];
        if (!same) io_error("ItemModelGridTestAuc: " + f + " does not hold the records of " + gdir[0] + " in the same order");
      }
      pred.insert(pred.end(), p.begin(), p.end());
      at += r.size();
    }
    if (g == 0) n = at;
    else if (at != n) io_error("ItemModelGridTestAuc: " + gdir[g] + " holds " + std::to_string(at) + " records, " + gdir[0] + " " + std::to_string(n));
  }
  if (n == 0) io_error("no scored records under " + gdir[0]);
  // records grouped by item key in the grid job's key order (Avro string order), input order inside a key
  std::vector<size_t> order(n);
  for (size_t i = 0; i < n; i++) order[i] = i;
  std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return key[a] < key[b]; });
  std::vector<std::string> knames;
  std::vector<int64_t> krs;
  std::vector<int32_t> gresp(n); std::vector<float> gw(n), gpred((size_t)G * n);
  for (size_t q = 0; q < n; q++) {
    const size_t i = order[q];
    if (q == 0 || key[i] != key[order[q - 1]]) { knames.push_back(key[i]); krs.push_back((int64_t)q); }
    gresp[q] = resp[i]; gw[q] = weight[i];
    for (int g = 0; g < G; g++) gpred[(size_t)g * n + q] = pred[(size_t)g * n + i];
  }
  krs.push_back((int64_t)n);
  const int K = (int)knames.size();
  std::vector<double> auc(G), wt(2), kauc((size_t)G * K), kw((size_t)2 * K);
  ck(mlease_test_auc(gpu_devices(c)[0], nullptr, (int64_t)n, G, gpred.data(), gresp.data(), gw.data(), K, krs.data(), auc.data(), wt.data(),
                     kauc.data(), kw.data()));
  AvroWriter w(outBase + "/_auc/part-r-00000.avro", SCHEMA_GRID_TEST_AUC);
  for (int g = 0; g < G; g++) {
    // keyAuc: the keys' AUCs weighted by their weight P_k + N_k, over the keys whose AUC is defined, summed in key order
    double num = 0.0, den = 0.0;
    for (int k = 0; k < K; k++) {
      const double a = kauc[(size_t)g * K + k];
      if (std::isnan(a)) continue;
      const double wk = kw[2 * k] + kw[2 * k + 1];
      num += wk * a; den += wk;
    }
    Value r; r.type = Schema::Record;
    r.items = {Value::of_string(gkey[g]), Value::of_double(auc[g]), Value::of_double(den > 0.0 ? num / den : std::nan("")),
               Value::of_double(wt[0]), Value::of_double(wt[1])};
    w.append(r);
  }
  w.close();
  AvroWriter wk(outBase + "/_key_auc/part-r-00000.avro", SCHEMA_TEST_AUC);
  for (int g = 0; g < G; g++)
    for (int k = 0; k < K; k++) wk.append(auc_record(gkey[g] + "#" + knames[k], kauc[(size_t)g * K + k], kw.data() + 2 * k));
  wk.close();
}

[[maybe_unused]] const bool registered_test_auc = register_job("RegressionTestAuc", run_test_auc);
[[maybe_unused]] const bool registered_grid_test_auc = register_job("ItemModelGridTestAuc", run_item_model_grid_test_auc);

}  // namespace
}  // namespace mlease_jobs
