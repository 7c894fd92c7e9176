"""Sequential restatements of ItemModelTest's reducer and of ItemModelTestLoglik, for the tests (paths relative to
/root/reference/src/main/java/com/linkedin/mlease/).  Plain Python, one record / one entry at a time, so the order of every sum and
every float rounding point is the reference's."""
import math

import numpy as np


def score_keyed(key_rowstart, rowptr, colidx, vals, offset, models, num_features, binary_feature=False):
    """regression/jobs/ItemModelTest.java:181-211.  models[l][k]: dict feature id -> float coefficient of the model
    "<lambda l>#<key k>", the intercept under id num_features; None = no such model, scored with the empty LinearModel
    (:189-197).  LinearModel.evalInstanceAvro(data, false, ignoreValue) (models/LinearModel.java:241-257, 491-554) with
    num_click_replicates = 1: -log(0 + 1 exp(-b)), then coef * value for every record feature the model holds (containsKey),
    in record order, then float(offset + that).  -> pred [L, nrows] float32."""
    L, n = len(models), len(rowptr) - 1
    pred = np.zeros((L, n), np.float32)
    for l in range(L):
        for k in range(len(key_rowstart) - 1):
            m = models[l][k] or {}
            b = float(m.get(num_features, 0.0))
            for i in range(key_rowstart[k], key_rowstart[k + 1]):
                result = -math.log(1 - 1 + 1 * math.exp(-b))
                for j in range(rowptr[i], rowptr[i + 1]):
                    c = int(colidx[j])
                    if c in m and c != num_features:
                        result += float(m[c]) * (1.0 if binary_feature else float(vals[j]))
                o = float(offset[i]) if offset is not None else 0.0
                pred[l, i] = np.float32(o + result)
    return pred


def item_test_loglik(entry_key, entry_group, response, pred, weight=None):
    """regression/jobs/ItemModelTestLoglik.java:60-142.  Mapper: float(-log1p(exp(-/+p)) * weight) per (record, map key) entry,
    count = weight; combiner per (group, key): float(double sum of the float logliks in entry order), double sum of the counts;
    reducer per key: float(double sum of the float partials in group order / sum of counts).  -> {key: (float32, count)}."""
    comb = {}
    for e in range(len(entry_key)):
        r, p = int(response[e]), float(np.float32(pred[e]))
        w = 1.0 if weight is None else float(np.float32(weight[e]))
        if r not in (1, 0, -1):
            raise ValueError("response should be 1,0 or -1!")
        ll = -math.log1p(math.exp(-p)) * w if r == 1 else -math.log1p(math.exp(p)) * w
        s = comb.setdefault((int(entry_group[e]), entry_key[e]), [0.0, 0.0])
        s[0] += float(np.float32(ll))
        s[1] += w
    red = {}
    for (g, k) in sorted(comb, key=lambda gk: gk[0]):
        s = red.setdefault(k, [0.0, 0.0])
        s[0] += float(np.float32(comb[(g, k)][0]))
        s[1] += comb[(g, k)][1]
    return {k: (np.float32(v[0] / v[1]), v[1]) for k, v in red.items()}


item_test_loglik.__test__ = False


def write_avro_with_maps(path, schema, records, codec="null", block=100):
    """avro_util.write_avro for a record schema whose fields may also be map<string, X> (ItemModelTestLoglik's `pred`); every
    other field type is encoded by avro_util."""
    import json
    import os
    import zlib
    import avro_util as au

    table = {}
    au._named(schema, table)

    def enc(out, sch, v):
        if isinstance(sch, dict) and sch.get("type") == "record":
            for f in sch["fields"]:
                enc(out, f["type"], v[f["name"]])
        elif isinstance(sch, dict) and sch.get("type") == "map":
            if v:
                au._wlong(out, len(v))
                for k, e in v.items():
                    b = k.encode()
                    au._wlong(out, len(b))
                    out.extend(b)
                    enc(out, sch["values"], e)
            au._wlong(out, 0)
        else:
            au._encode(out, sch, v, table)

    out = bytearray(b"Obj\x01")
    au._wlong(out, 2)
    for k, v in (("avro.schema", json.dumps(schema).encode()), ("avro.codec", codec.encode())):
        au._wlong(out, len(k)); out.extend(k.encode()); au._wlong(out, len(v)); out.extend(v)
    au._wlong(out, 0)
    sync = bytes(range(16))
    out.extend(sync)
    for s in range(0, len(records), block):
        body = bytearray()
        chunk = records[s:s + block]
        for r in chunk:
            enc(body, schema, r)
        if codec == "deflate":
            co = zlib.compressobj(6, zlib.DEFLATED, -15)
            body = co.compress(bytes(body)) + co.flush()
        au._wlong(out, len(chunk)); au._wlong(out, len(body)); out.extend(body); out.extend(sync)
    os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
    open(path, "wb").write(bytes(out))
