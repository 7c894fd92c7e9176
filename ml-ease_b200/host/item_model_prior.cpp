// item_model_prior.cpp -- ItemModelTrain with prior.model.path: each item refreshed from an earlier run's posterior instead of refit
// on its whole history.  The earlier run's LinearModelWithVarAvro records of one grid point become each key's prior lists (means from
// "model", variances from "posteriorVar"), fitted by mlease_item_model_train_prior with the semantics of llf/LibLinear.java:221-245
// and initSetup (:476-497).  Kept in its own translation unit, registered with item_model_train_job.cpp, so that the job links
// without that symbol.
#include <cmath>

#include "jobs_common.hpp"

namespace mlease_jobs {

// an item's prior: (dictionary id, or -1 for the intercept; mean; variance, 0 = the column's usual one), ascending ids
struct ItemPriors {
  std::unordered_map<std::string, std::vector<std::tuple<int32_t, double, double>>> by_item;
};

namespace {

std::string feature_name(const Value& fv) { return fv.items[1].s.empty() ? fv.items[0].s : fv.items[0].s + "\x01" + fv.items[1].s; }

// "<intercept lambda>:<default lambda>" as the earlier run wrote it in its keys (Float.toString of each)
std::string grid_point(const std::string& s) {
  const size_t p = s.find(':');
  try {
    if (p != std::string::npos) return java_float_to_string(std::stof(s.substr(0, p))) + ":" + java_float_to_string(std::stof(s.substr(p + 1)));
  } catch (const std::exception&) {
  }
  io_error("prior.model.lambda: expected <intercept lambda>:<default lambda>, got \"" + s + "\"");
}

std::shared_ptr<ItemPriors> read_priors(const JobConfig& c, Dictionary& dict) {
  const std::string path = c.get("prior.model.path");
  const std::string want = c.get("prior.model.lambda", "").empty() ? "" : grid_point(c.get("prior.model.lambda"));
  // the records of every grid point, by item: the last record of an item wins (as read_prior_mean_map's HashMap.put)
  struct Rec { std::vector<std::pair<std::string, double>> model; std::unordered_map<std::string, double> var; };
  std::vector<std::string> found;
  std::map<std::string, std::map<std::string, Rec>> by_point;
  for (auto& f : list_avro_files(path)) {
    AvroReader rd(f);
    const Schema& s = rec_schema(rd.schema());
    const int ki = s.field_index("key"), mi = s.field_index("model"), vi = s.field_index("posteriorVar");
    if (ki < 0 || mi < 0) io_error("prior.model.path: " + f + " does not hold LinearModelWithVarAvro records");
    Value rec;
    while (rd.next(rec)) {
      const std::string& key = rec.items[ki].s;
      const size_t h = key.find('#');
      if (h == std::string::npos) io_error("prior.model.path: record key \"" + key + "\" is not <intercept lambda>:<default lambda>#<item>");
      const std::string gp = key.substr(0, h);
      if (std::find(found.begin(), found.end(), gp) == found.end()) found.push_back(gp);
      if (!want.empty() && gp != want) continue;
      Rec r;
      for (auto& fv : rec.items[mi].items) r.model.emplace_back(feature_name(fv), fv.items[2].d);
      if (vi >= 0)
        for (auto& fv : rec.items[vi].items) r.var[feature_name(fv)] = fv.items[2].d;
      by_point[gp][key.substr(h + 1)] = std::move(r);
    }
  }
  std::string list;
  for (auto& g : found) list += (list.empty() ? "" : ", ") + g;
  if (found.empty()) io_error("prior.model.path: no models under " + path);
  if (want.empty() && found.size() > 1)
    io_error("prior.model.path holds the models of " + std::to_string(found.size()) + " grid points (" + list +
             "): set prior.model.lambda to one of them");
  const std::string gp = want.empty() ? found[0] : want;
  if (!by_point.count(gp)) io_error("prior.model.lambda " + gp + " is not a grid point of prior.model.path (" + list + ")");
  // items in byte order, features in model order: the order in which features new to today's dictionary get their ids
  auto p = std::make_shared<ItemPriors>();
  for (auto& [item, r] : by_point[gp]) {
    std::map<int32_t, std::pair<double, double>> ent;
    for (auto& [name, mean] : r.model) {
      auto it = r.var.find(name);
      // a posteriorVar value <= 0 (the (INTERCEPT) 0 of a run without compute.var) is no variance: the column's usual one
      const double v = it != r.var.end() && it->second > 0.0 ? it->second : 0.0;
      ent[name == INTERCEPT ? -1 : dict.add(name)] = {mean, v};
    }
    auto& out = p->by_item[item];
    for (auto& [id, mv] : ent) out.emplace_back(id, mv.first, mv.second);
  }
  return p;
}

// every key's fits under its item's prior (mlease_item_model_train_prior), one key range per device; a key's model lists its union
// columns, its posteriorVar its data features, then its prior-only features that have a variance (:384-397)
void fit_priors(const ItemPriors& p, ItemModelFit& f) {
  const int K = (int)f.knames.size(), D = f.D, Dt = D + 1, IL = (int)f.il.size(), DL = (int)f.dl.size(), G = IL * DL;
  std::vector<int64_t> pp{0};
  std::vector<int32_t> pc;
  std::vector<double> pm, pv;
  for (int k = 0; k < K; k++) {
    auto it = p.by_item.find(f.knames[k]);
    if (it != p.by_item.end()) {
      const auto& e = it->second;
      for (auto& [id, mean, var] : e)
        if (id >= 0) { pc.push_back(id); pm.push_back(mean); pv.push_back(var); }
      if (!e.empty() && std::get<0>(e.front()) < 0) { pc.push_back(D); pm.push_back(std::get<1>(e.front())); pv.push_back(std::get<2>(e.front())); }
    }
    pp.push_back((int64_t)pc.size());
  }
  const float* lm = f.lambda_map.empty() ? nullptr : f.lambda_map.data();
  const std::vector<int> cuts = f.devs.size() == 1 ? std::vector<int>{0, K} : shard_keys(f.krs, f.rp, D, (int)f.devs.size());
  run_shards(f.devs, cuts, [&](int32_t dev, int k0, int k1) {
    const KeySlice s(f.krs, f.rp, k0, k1);
    const int Ks = k1 - k0;
    std::vector<int64_t> spp;
    int64_t cap = 0;
    for (int k = k0; k <= k1; k++) spp.push_back(pp[k] - pp[k0]);
    for (int k = k0; k < k1; k++) {
      const int64_t non = pp[k + 1] - pp[k] - (pp[k + 1] > pp[k] && pc[pp[k + 1] - 1] == D ? 1 : 0);
      cap += std::min<int64_t>(f.rp[f.krs[k + 1]] - f.rp[f.krs[k]] + non, D) + 1;
    }
    std::vector<int64_t> key_ptr(Ks + 1);
    std::vector<int32_t> col(std::max<int64_t>(cap, 1));
    std::vector<double> mv((size_t)G * std::max<int64_t>(cap, 1)), vv(f.compute_var ? mv.size() : 0);
    const size_t e0 = (size_t)pp[k0];
    ck(mlease_item_model_train_prior(dev, nullptr, Ks, D, s.krs.data(), s.rowptr.data(), f.ci.data() + s.nz0, f.vv.data() + s.nz0,
                                     f.rr.data() + s.row0, f.ww.data() + s.row0, f.oo.data() + s.row0, f.means.data() + k0, IL, f.il.data(),
                                     DL, f.dl.data(), lm, f.binary ? 1 : 0, f.compute_var ? 1 : 0, cap, key_ptr.data(), col.data(), mv.data(),
                                     f.compute_var ? vv.data() : nullptr, spp.data(), pc.data() + e0, pm.data() + e0, pv.data() + e0));
    for (int k = k0; k < k1; k++) {
      const int64_t a = key_ptr[k - k0], b = key_ptr[k - k0 + 1];
      const std::vector<int32_t> data = f.cols[k];
      std::vector<int32_t>& mc = f.cols[k];
      mc.assign(col.begin() + a, col.begin() + b - 1);   // the intercept is last
      for (int32_t j : mc) {
        if (std::binary_search(data.begin(), data.end(), j)) continue;
        const int64_t e = std::lower_bound(pc.begin() + pp[k], pc.begin() + pp[k + 1], j) - pc.begin();
        if (pv[e] > 0.0) f.var_cols[k].push_back(j);
      }
      for (int g = 0; g < G; g++) {
        const size_t base = ((size_t)g * K + k) * Dt;
        for (int64_t e = a; e < b; e++) {
          f.m[base + col[e]] = mv[(size_t)g * cap + e];
          if (f.compute_var) f.var[base + col[e]] = vv[(size_t)g * cap + e];
        }
      }
    }
  });
}

[[maybe_unused]] const bool registered = register_item_model_prior(ItemPriorHooks{read_priors, fit_priors});

}  // namespace
}  // namespace mlease_jobs
