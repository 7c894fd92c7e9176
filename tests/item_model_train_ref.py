"""Sequential restatement of ItemModelTrain's reducer for the tests (paths relative to /root/reference/src/main/java/com/linkedin/mlease/),
built on the oracle's LibLinear fit and Hessian diagonal, and writers of its two side files (lambda.map, intercept.prior.mean.map)."""
import numpy as np

from oracle import oracle as orc

INTERCEPT = "(INTERCEPT)"
PREPARED_SCHEMA = {"type": "record", "name": "RegressionPrepareOutput", "namespace": "com.linkedin.mlease.regression.avro", "fields": [
    {"name": "key", "type": "string"}, {"name": "response", "type": "int"},
    {"name": "features", "type": {"type": "array", "items": {"type": "record", "name": "feature", "fields": [
        {"name": "name", "type": "string"}, {"name": "term", "type": "string"}, {"name": "value", "type": "float"}]}}},
    {"name": "weight", "type": "float"}, {"name": "offset", "type": "float"}]}


def _fkey(f):
    return f["name"] if not f.get("term") else f["name"] + "\x01" + f["term"]


def _split(key):
    n, _, t = key.partition("\x01")
    return n, t


def lambda_map_entries(lambda_map):
    """[(feature key, lambda)] -> the map's keys in order of first appearance, each with its last value as a float
    (HashMap.put, regression/consumers/ReadLambdaMapConsumer.java:33-52)."""
    out = {}
    for k, lam in lambda_map or []:
        out[k] = float(np.float32(lam))
    return list(out.items())


def item_model_train(prepared, intercept_lambdas, default_lambdas, lambda_map=None, prior_mean_map=None, default_prior_mean=0.0,
                     compute_var=False, binary_feature=False):
    """jobs/ItemModelTrain.java:226-276 on RegressionPrepareOutput records (dicts, input order).  Returns the LinearModelWithVarAvro
    records: keys in byte order, then intercept lambda, then default lambda, each list in config order with repeats kept (:313-321)."""
    ids = {}
    for r in prepared:
        for f in r["features"]:
            ids.setdefault(_fkey(f), len(ids))           # the job's dictionary: ids in order of first appearance
    names = list(ids)
    D = len(names)
    lm = lambda_map_entries(lambda_map)
    lmd = dict(lm)
    by_key = {}
    for r in prepared:                                      # mapper: key = data.key (:136-142)
        by_key.setdefault(r["key"], []).append(r)
    il = [np.float32(x) for x in intercept_lambdas]      # Float.parseFloat (:313-321)
    dl = [np.float32(x) for x in default_lambdas]
    dmean = float(np.float32(default_prior_mean))         # conf.setFloat / getFloat (:112, :165)
    out = []
    for key in sorted(by_key, key=lambda s: s.encode()):
        rows = by_key[key]
        rp, ci, v = [0], [], []
        for r in rows:                                      # LibLinearDataset: a row's features sorted by index
            ent = sorted((ids[_fkey(f)], 1.0 if binary_feature else f["value"]) for f in r["features"])
            ci += [c for c, _ in ent]; v += [x for _, x in ent]
            rp.append(len(ci))
        data = orc.Csr(rp, ci, v, [r["response"] for r in rows], [r["weight"] for r in rows], [r["offset"] for r in rows], D)
        present = sorted(set(ci))
        mean = (prior_mean_map or {}).get(key, dmean)        # :240-248
        for ia in il:
            for db in dl:
                # priorVar (:194-216, :254, :262): 1/(double)lambdaMap, 1/interceptLambda, else 1/defaultLambda; prior mean: intercept only
                pv = np.array([1.0 / np.float64(lmd[nm]) if nm in lmd else 1.0 / np.float64(db) for nm in names] + [1.0 / np.float64(ia)])
                pm = np.zeros(D + 1); pm[D] = mean
                beta, _ = orc.liblinear_train(data, np.zeros(D + 1), pm, pv, 1e-14, 100000)
                # LinearModel.toAvro (models/LinearModel.java:697-720): intercept first, then the dataset's features (llf/LibLinear.java:343-350)
                model = [{"name": INTERCEPT, "term": "", "value": float(np.float32(beta[D]))}]
                model += [dict(zip(("name", "term"), _split(names[j])), value=float(np.float32(beta[j]))) for j in present]
                if compute_var:
                    # diagonal only (llf/LibLinear.java:328-333), then every prior-variance key the dataset lacks (:384-397)
                    var = np.zeros(D + 1)                         # the oracle leaves features outside the dataset 0
                    var[present + [D]] = 1.0 / orc.objective("hessian_diag", data, beta, pm, pv)[present + [D]]
                    pvar = [{"name": INTERCEPT, "term": "", "value": float(np.float32(var[D]))}]
                    pvar += [dict(zip(("name", "term"), _split(names[j])), value=float(np.float32(var[j]))) for j in present]
                    pres = {names[j] for j in present} | {INTERCEPT}
                    pvar += [dict(zip(("name", "term"), _split(k)), value=float(np.float32(1.0 / np.float64(lam)))) for k, lam in lm if k not in pres]
                else:
                    pvar = [{"name": INTERCEPT, "term": "", "value": 0.0}]   # new LinearModel().toAvro (:271-274)
                out.append({"key": orc.java_float_to_string(ia) + ":" + orc.java_float_to_string(db) + "#" + key,   # :265
                            "model": model, "posteriorVar": pvar})
    return out


def write_lambda_map(path, entries):
    """lambda.map records {name, term, value} (regression/consumers/ReadLambdaMapConsumer.java:33-52)."""
    import avro_util as au
    schema = {"type": "record", "name": "feature", "fields": [{"name": "name", "type": "string"}, {"name": "term", "type": "string"},
                                                            {"name": "value", "type": "float"}]}
    au.write_avro(path, schema, [dict(zip(("name", "term"), _split(k)), value=float(lam)) for k, lam in entries])


def write_prior_mean_map(path, entries, value_type="string"):
    """intercept.prior.mean.map: Pair records {key, value} (:293-301); value_type "string", "float", "double" or "int"."""
    import avro_util as au
    schema = {"type": "record", "name": "Pair", "namespace": "org.apache.avro.mapred", "fields": [{"name": "key", "type": "string"},
                                                                                               {"name": "value", "type": value_type}]}
    au.write_avro(path, schema, [{"key": k, "value": v} for k, v in entries])
