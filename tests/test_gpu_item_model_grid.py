"""GPU tests of scoring ItemModelTrain's grid models with their posterior variance: mlease_score_keyed_var through the Python
binding (pred bitwise mlease_score_keyed's, pred_var against an fp64 numpy reference, streamed against resident, refusals), and the
ItemModelGridTest job end to end after RegressionPrepare -> ItemModelTrain on the fixture, against numpy on the model file, against
ItemModelTest on the same models and against the ItemModelTestLoglik restatement; on two GPUs, gpu.devices=0,1 against one GPU."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import avro_util as au  # noqa: E402
import item_model_ref as ref  # noqa: E402
import item_model_train_ref as tref  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _ndev():
    import torch
    return torch.cuda.device_count()


@pytest.fixture
def budget():
    from mlease_b200 import _hooks
    yield _hooks.set_keyed_budget
    _hooks.set_keyed_budget(0)


def _problem(rng, K, D, G, max_rows=40, density=0.05):
    """K keys (some without rows) of rows with sorted unique columns (~5 % empty); per (grid point, key) a model (~10 % none, some
    without intercept) and a variance list (~10 % empty; a random column subset, the intercept listed or not), var_default > 0."""
    nk = rng.integers(0, max_rows + 1, K)
    nk[rng.random(K) < 0.1] = 0
    krs = np.concatenate([[0], np.cumsum(nk)]).astype(np.int64)
    n = int(krs[-1])
    nnz = np.minimum(rng.poisson(density * D, n), D)
    nnz[rng.random(n) < 0.05] = 0
    rp = np.concatenate([[0], np.cumsum(nnz)]).astype(np.int64)
    ci = np.concatenate([np.sort(rng.choice(D, c, replace=False)) for c in nnz] + [np.zeros(0, np.int64)]).astype(np.int32)
    v = rng.normal(size=len(ci)).astype(np.float32)
    o = rng.normal(size=n).astype(np.float32)
    mp, mc, mv, vp, vc, vv = [0], [], [], [0], [], []
    for m in range(G * K):
        if rng.random() >= 0.1:
            cols = np.sort(rng.choice(D, rng.integers(1, D // 2), replace=False))
            if rng.random() < 0.8:
                cols = np.append(cols, D)
            mc += list(cols); mv += list(rng.normal(size=len(cols)) * 0.3)
        mp.append(len(mc))
        if rng.random() >= 0.1:
            cols = np.sort(rng.choice(D, rng.integers(0, D), replace=False))
            if rng.random() < 0.7:
                cols = np.append(cols, D)
            if len(cols) == 0:
                cols = np.array([D])
            vc += list(cols); vv += list(rng.uniform(0.0, 2.0, len(cols)))
        vp.append(len(vc))
    vdef = rng.uniform(0.01, 3.0, G * K).astype(np.float32)
    return dict(krs=krs, rp=rp, ci=ci, v=v, o=o, mp=np.array(mp, np.int64), mc=np.array(mc, np.int32), mv=np.array(mv, np.float32),
                vp=np.array(vp, np.int64), vc=np.array(vc, np.int32), vv=np.array(vv, np.float32), vdef=vdef, K=K, D=D, G=G)


def _var_ref(pb, binary):
    """pred_var in fp64: sum over a row's entries of v(c) x^2 (listed variance, else var_default) + the listed intercept variance
    (0 if unlisted), NaN for an empty list -> float32 [G, n]"""
    K, D, G, krs, rp = pb["K"], pb["D"], pb["G"], pb["krs"], pb["rp"]
    n = int(krs[-1])
    row_key = np.repeat(np.arange(K), np.diff(krs))
    ent_row = np.repeat(np.arange(n), np.diff(rp))
    x2 = np.ones(len(pb["ci"])) if binary else pb["v"].astype(np.float64) ** 2
    out = np.zeros((G, n), np.float32)
    for g in range(G):
        dense = np.repeat(pb["vdef"][g * K:(g + 1) * K].astype(np.float64)[:, None], D + 1, axis=1)
        dense[:, D] = 0.0
        empty = np.zeros(K, bool)
        for k in range(K):
            m = g * K + k
            a, b = pb["vp"][m], pb["vp"][m + 1]
            empty[k] = a == b
            dense[k, pb["vc"][a:b]] = pb["vv"][a:b]
        s = np.bincount(ent_row, weights=dense[row_key[ent_row], pb["ci"]] * x2, minlength=n) + dense[row_key, D]
        out[g] = np.where(empty[row_key], np.nan, s).astype(np.float32)
    return out


def _call(pb, binary=False, **kw):
    import mlease_b200 as mb
    return mb.score_keyed_var(pb["v"], pb["krs"], pb["rp"], pb["ci"], pb["D"], pb["mp"], pb["mc"], pb["mv"], pb["vp"], pb["vc"], pb["vv"],
                              pb["vdef"], offset=pb["o"], binary_feature=binary, **kw)


def _within_ulps(got, want, k):
    assert np.array_equal(np.isnan(got), np.isnan(want))
    f = ~np.isnan(want)
    assert np.all(np.abs(got[f].astype(np.float64) - want[f]) <= k * np.spacing(np.abs(want[f])).astype(np.float64))


@pytest.mark.parametrize("G", [1, 2, 3, 4, 5, 7])
def test_score_keyed_var_pred_is_score_keyed_and_var_is_fp64(G):
    import mlease_b200 as mb
    rng = np.random.default_rng(300 + G)
    pb = _problem(rng, K=300, D=400, G=G)
    assert (np.diff(pb["krs"]) == 0).any() and (np.diff(pb["rp"]) == 0).any()
    for binary in (False, True):
        pred, pvar = _call(pb, binary)
        want = mb.score_keyed(pb["v"], pb["krs"], pb["rp"], pb["ci"], pb["D"], pb["mp"], pb["mc"], pb["mv"], offset=pb["o"], binary_feature=binary)
        assert np.array_equal(pred.view(np.uint32), want.view(np.uint32)), binary
        _within_ulps(pvar, _var_ref(pb, binary), 2)
        p2, v2 = _call(pb, binary)   # repeatable
        assert np.array_equal(p2.view(np.uint32), pred.view(np.uint32)) and np.array_equal(v2.view(np.uint32), pvar.view(np.uint32))


@pytest.mark.parametrize("G", [1, 3, 5])
def test_streamed_score_keyed_var_is_bitwise_resident(budget, G):
    import torch

    from mlease_b200 import _hooks
    pb = _problem(np.random.default_rng(80 + G), K=40, D=120, G=G, max_rows=300, density=0.1)
    budget(0)
    want_p, want_v = _call(pb)
    assert not _hooks.keyed_last_call()[1]
    budget(256 << 10)
    got_p, got_v = _call(pb)
    bounds, streamed, _, _ = _hooks.keyed_last_call()
    assert streamed and len(bounds) - 1 >= 4, bounds
    assert np.array_equal(got_p.view(np.uint32), want_p.view(np.uint32)) and np.array_equal(got_v.view(np.uint32), want_v.view(np.uint32))
    n = int(pb["krs"][-1])
    dp = torch.zeros((G, n), dtype=torch.float32, device="cuda")
    dv = torch.zeros((G, n), dtype=torch.float32, device="cuda")
    _call(pb, out=dp, out_var=dv)
    assert _hooks.keyed_last_call()[1]
    assert np.array_equal(dp.cpu().numpy().view(np.uint32), want_p.view(np.uint32))
    assert np.array_equal(dv.cpu().numpy().view(np.uint32), want_v.view(np.uint32))


def test_score_keyed_var_refusals_then_keeps_working():
    import mlease_b200 as mb
    D = 4
    base = dict(vals=np.ones(3, np.float32), key_rowstart=[0, 2], rowptr=[0, 2, 3], colidx=np.array([0, 2, 1], np.int32), num_features=D,
                model_ptr=[0, 2], model_col=np.array([1, D], np.int32), model_val=np.array([0.5, 0.25], np.float32),
                var_ptr=[0, 2], var_col=np.array([0, D], np.int32), var_val=np.array([0.5, 0.1], np.float32), var_default=[1.0])
    cases = [
        (dict(rowptr=[0, 2, 3], colidx=np.array([2, 0, 1], np.int32)), "colidx must be strictly ascending within a row"),
        (dict(rowptr=[0, 2, 3], colidx=np.array([1, 1, 1], np.int32)), "colidx must be strictly ascending within a row"),
        (dict(var_col=np.array([0, D + 1], np.int32)), r"var_col out of range \(model 0\)"),
        (dict(var_col=np.array([2, 1], np.int32)), r"var_col must be strictly ascending within a model \(model 0\)"),
        (dict(var_val=np.array([0.5, -0.1], np.float32)), r"var_val must be finite and >= 0 \(model 0\)"),
        (dict(var_val=np.array([np.nan, 0.1], np.float32)), r"var_val must be finite and >= 0 \(model 0\)"),
        (dict(var_val=np.array([0.5, np.inf], np.float32)), r"var_val must be finite and >= 0 \(model 0\)"),
        (dict(var_default=[-1.0]), r"var_default must be finite and >= 0 \(model 0\)"),
        (dict(var_default=[np.inf]), r"var_default must be finite and >= 0 \(model 0\)"),
    ]
    for change, msg in cases:
        a = dict(base, **change)
        with pytest.raises(mb.MleaseError, match=msg):
            mb.score_keyed_var(a.pop("vals"), a.pop("key_rowstart"), a.pop("rowptr"), a.pop("colidx"), a.pop("num_features"), a.pop("model_ptr"),
                               a.pop("model_col"), a.pop("model_val"), a.pop("var_ptr"), a.pop("var_col"), a.pop("var_val"), a.pop("var_default"))
    a = base
    pred, pvar = mb.score_keyed_var(a["vals"], a["key_rowstart"], a["rowptr"], a["colidx"], D, a["model_ptr"], a["model_col"], a["model_val"],
                                    a["var_ptr"], a["var_col"], a["var_val"], a["var_default"])
    # row 0 lists columns 0, 2: 0.5 + 1.0 (default) + intercept 0.1; row 1 lists column 1: 1.0 + 0.1
    assert pvar.tolist() == [[np.float32(1.6), np.float32(1.1)]] and pred.tolist() == [[np.float32(0.25), np.float32(0.75)]]


# ---------------------------------------------------------------------------------------------------------------- the job
@pytest.fixture(scope="module")
def host():
    import mlease_b200
    mlease_b200.lib()
    h = C.CDLL(os.path.join(ROOT, "ml-ease_b200", "lib", "libmlease_host.so"))
    h.mlease_job_last_error.restype = C.c_char_p
    return h


def _run(host, job, path, kv):
    with open(path, "w") as f:
        f.write("".join("%s=%s\n" % (k, v) for k, v in kv.items()))
    rc = host.mlease_job_run(job, str(path).encode())
    return rc, host.mlease_job_last_error().decode() if rc else ""


def _ok(host, job, path, kv):
    rc, err = _run(host, job, path, kv)
    assert rc == 0, err


IL, DL = ["1", "30.0"], ["0.5", "2"]


@pytest.fixture(scope="module")
def trained(host, tmp_path_factory):
    """RegressionPrepare (map.key) -> ItemModelTrain with a 2 x 2 grid and a lambda.map, with and without compute.var; test records:
    the fixture scrambled, plus records of a key without a model, in two files"""
    d = tmp_path_factory.mktemp("grid_job")
    npz = np.load(os.path.join(GOLDEN, "sample_data.npz"))
    names = [str(x) for x in npz["feature_names"]]
    recs = au.fixture_records(npz, with_key=lambda i: (i * 7) % 9)
    au.write_avro(str(d / "in" / "part-0.avro"), au.pig_schema_with_key(), recs, codec="deflate", block=128)
    _ok(host, b"RegressionPrepare", d / "p.job", {"input.paths": d / "in", "output.path": d / "tmp-data", "map.key": "pkey", "num.blocks": 2})
    tref.write_lambda_map(str(d / "lm" / "lm.avro"), [(names[3], 0.2), ("not-in-data", 5.0), (names[10], 2.0)])
    for var in ("true", "false"):
        _ok(host, b"ItemModelTrain", d / ("t" + var + ".job"), {"input.paths": d / "tmp-data", "output.model.path": d / ("m" + var),
            "intercept.lambdas": ",".join(IL), "default.lambdas": ",".join(DL), "lambda.map": d / "lm", "compute.var": var, "remove.tmp.dir": "false"})
    test = recs[::-1][:700] + [dict(r, pkey=99) for r in recs[:31]] + recs[300:]
    au.write_avro(str(d / "test" / "a.avro"), au.pig_schema_with_key(), test[:500], block=100)
    au.write_avro(str(d / "test" / "b.avro"), au.pig_schema_with_key(), test[500:], codec="deflate", block=300)
    return d, test


def _grid(host, d, out, var="true", model="mtrue", **kw):
    kv = {"input.paths": d / "test", "output.base.path": out, "model.path": d / model / "models", "item.key": "pkey",
          "intercept.lambdas": ",".join(IL), "default.lambdas": ",".join(DL), "compute.var": var}
    kv.update(kw)
    return _run(host, b"ItemModelGridTest", str(out) + ".job", kv)


def _f(x):
    return repr(float(np.float32(x)))   # Java Float.toString of these lambdas


def test_item_model_grid_test_job_end_to_end(host, trained, tmp_path):
    d, test = trained
    out = tmp_path / "grid"
    rc, err = _grid(host, d, out)
    assert rc == 0, err
    models = {r["key"]: r for r in au.read_dir(str(d / "mtrue" / "models"))}
    order = sorted(range(len(test)), key=lambda i: str(test[i]["pkey"]))
    names = sorted({f["name"] for r in test for f in r["features"]})
    fid = {nm: i for i, nm in enumerate(names)}
    D = len(names)
    feats = [sorted(((fid[f["name"]], np.float32(f["value"])) for f in test[i]["features"])) for i in order]   # the rows the device gets
    rp = np.cumsum([0] + [len(f) for f in feats]).astype(np.int64)
    ci = np.array([c for f in feats for c, _ in f], np.int32)
    v = np.array([x for f in feats for _, x in f], np.float32)
    off = np.array([test[i]["offset"] for i in order], np.float32)
    keys = [str(test[i]["pkey"]) for i in order]
    kn = sorted(set(keys))
    krs = [keys.index(k) for k in kn] + [len(keys)]
    grid_preds = []
    for a, il in enumerate(IL):
        for b, dl in enumerate(DL):
            sch, got = au.read_avro(str(out / ("lambda-%s_%s" % (il, dl)) / "part-r-00000.avro"))[:2]
            assert sch["name"] == "ItemModelGridTestOutput"
            assert [f["name"] for f in sch["fields"]] == [f["name"] for f in au.pig_schema_with_key()["fields"]] + ["pred", "predVar"]
            assert [r["pkey"] for r in got] == [test[i]["pkey"] for i in order]
            p = np.array([r["pred"] for r in got], np.float32)
            pv = np.array([r["predVar"] for r in got], np.float32)
            ml, want_v = [], np.zeros(len(order), np.float64)
            for k in kn:
                m = models.get("%s:%s#%s" % (_f(il), _f(dl), k))
                ml.append(None if m is None else {(D if f["name"] == "(INTERCEPT)" else fid[f["name"]]): np.float32(f["value"]) for f in m["model"]
                                                  if f["name"] == "(INTERCEPT)" or f["name"] in fid})
            want_p = ref.score_keyed(krs, rp, ci, v, off, [ml], D)[0]
            assert np.all(np.abs(p - want_p) <= np.spacing(np.abs(want_p))), (il, dl)
            for q in range(len(order)):
                m = models.get("%s:%s#%s" % (_f(il), _f(dl), keys[q]))
                if m is None:
                    want_v[q] = np.nan
                    continue
                var = {f["name"]: float(f["value"]) for f in m["posteriorVar"]}
                dflt = float(np.float32(1.0 / float(np.float32(dl))))
                want_v[q] = sum(var.get(names[c], dflt) * float(x) ** 2 for c, x in feats[q]) + var.get("(INTERCEPT)", 0.0)
            _within_ulps(pv, want_v.astype(np.float32), 2)
            assert np.isnan(pv[np.array(keys) == "99"]).all() and not np.isnan(pv[np.array(keys) != "99"]).any()
            grid_preds.append(p)
    # ItemModelTest on the same models relabelled "<g + 1>#<key>": within one ulp (the grid job sorts each record's features for predVar)
    relabel = []
    for g, (il, dl) in enumerate((a, b) for a in IL for b in DL):
        prefix = "%s:%s#" % (_f(il), _f(dl))
        relabel += [{"key": "%d.0#%s" % (g + 1, r["key"][len(prefix):]), "model": r["model"]} for r in models.values() if r["key"].startswith(prefix)]
    lm_schema = {"type": "record", "name": "LinearModelAvro", "fields": [{"name": "key", "type": "string"}, {"name": "model", "type": {"type": "array", "items": {
        "type": "record", "name": "feature", "fields": [{"name": "name", "type": "string"}, {"name": "term", "type": "string"}, {"name": "value", "type": "float"}]}}}]}
    au.write_avro(str(tmp_path / "relabelled" / "part-r-00000.avro"), lm_schema, relabel)
    _ok(host, b"ItemModelTest", tmp_path / "it.job", {"input.paths": d / "test", "output.base.path": tmp_path / "it", "model.path": tmp_path / "relabelled",
                                                      "item.key": "pkey", "lambda": "1,2,3,4"})
    it = [np.array([r["pred"] for r in au.read_avro(str(tmp_path / "it" / ("lambda-%d" % (g + 1)) / "part-r-00000.avro"))[1]], np.float32) for g in range(4)]
    for g in range(4):
        assert np.all(np.abs(grid_preds[g] - it[g]) <= np.spacing(np.abs(it[g]))), g
    rc, err = _grid(host, d, tmp_path / "novar", var="false")
    assert rc == 0, err
    for g, (il, dl) in enumerate((a, b) for a in IL for b in DL):
        sch, got = au.read_avro(str(tmp_path / "novar" / ("lambda-%s_%s" % (il, dl)) / "part-r-00000.avro"))[:2]
        assert [f["name"] for f in sch["fields"]][-1] == "pred"
        assert np.array_equal(np.array([r["pred"] for r in got], np.float32).view(np.uint32), it[g].view(np.uint32)), g
    # _loglik: one record per grid point in grid order; entry per (record, grid point), one combiner group per input file
    ll = au.read_dir(str(out / "_loglik"))
    assert [r["key"] for r in ll] == ["%s:%s" % (_f(a), _f(b)) for a in IL for b in DL]
    pos = {i: q for q, i in enumerate(order)}
    for g, r in enumerate(ll):
        want = ref.item_test_loglik([0] * len(test), [0 if i < 500 else 1 for i in range(len(test))], [t["response"] for t in test],
                                    np.array([grid_preds[g][pos[i]] for i in range(len(test))], np.float32),
                                    np.array([t["weight"] for t in test], np.float32))[0]
        assert abs(r["testLoglik"] - want[0]) <= 1e-6 * abs(want[0]) and r["count"] == want[1], (g, r, want)


def test_item_model_grid_test_refuses_models_trained_without_compute_var(host, trained, tmp_path):
    d, _ = trained
    rc, err = _grid(host, d, tmp_path / "o", model="mfalse")
    assert rc != 0 and err.endswith("has no posterior variance (its posteriorVar is the (INTERCEPT) 0 placeholder): rerun ItemModelTrain "
                                    "with compute.var=true"), err
    rc, err = _grid(host, d, tmp_path / "o2", var="false", model="mfalse")
    assert rc == 0, err


@pytest.mark.skipif("_ndev() < 2")
def test_item_model_grid_test_on_two_gpus_writes_the_one_gpu_tree(host, trained, tmp_path):
    d, _ = trained

    def tree(root):
        out = {}
        for dp, _, fs in os.walk(root):
            for f in fs:
                if f.endswith(".avro"):
                    data = open(os.path.join(dp, f), "rb").read()
                    out[os.path.relpath(os.path.join(dp, f), root)] = data.replace(data[-16:], bytes(16))
        return out
    for devs in ("0", "0,1"):
        rc, err = _grid(host, d, tmp_path / ("d" + devs.replace(",", "")), **{"gpu.devices": devs})
        assert rc == 0, err
    assert tree(str(tmp_path / "d0")) == tree(str(tmp_path / "d01"))
