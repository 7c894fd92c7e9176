"""CPU tests of the ItemModelGridTest job, linked against the test doubles of the device library (tests/fake_device/: fake_item_model.c
for mlease_score_keyed / mlease_test_loglik_keyed, fake_item_model_grid.c for mlease_score_keyed_var).  The doubles' numbers are
per-key hashes of the key's own rows and model, so only layout, key strings, schemas, grid order, fast/generic byte identity,
sharding and error texts are checked here; test_gpu_item_model_grid.py checks the numbers.  Also the binding's no-GPU failure."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import avro_util as au  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
HOST = os.path.join(ROOT, "ml-ease_b200", "host")
FAKE = os.path.join(ROOT, "tests", "fake_device")

FEATURE = {"type": "record", "name": "feature", "fields": [{"name": "name", "type": "string"}, {"name": "term", "type": "string"},
                                                            {"name": "value", "type": "float"}]}
VAR_SCHEMA = {"type": "record", "name": "LinearModelWithVarAvro", "namespace": "com.linkedin.mlease.avro", "fields": [
    {"name": "key", "type": "string"}, {"name": "model", "type": {"type": "array", "items": FEATURE}},
    {"name": "posteriorVar", "type": {"type": "array", "items": dict(FEATURE, name="featureVar")}}]}


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.fixture(scope="module")
def fake_host(tmp_path_factory):
    d = tmp_path_factory.mktemp("fakehost_grid")
    so = str(d / "libmlease_host_fake.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-o", so] +
                          [os.path.join(HOST, f) for f in ("avro_io.cpp", "regression_jobs.cpp", "item_model_grid_test_job.cpp")] +
                          ["-x", "c"] + [os.path.join(FAKE, f) for f in ("fake_mlease_b200.c", "fake_item_model.c", "fake_item_model_grid.c")] +
                          ["-lz", "-pthread", "-lm"])
    h = C.CDLL(so)
    h.mlease_job_last_error.restype = C.c_char_p
    return h


def _cfg(path, kv):
    with open(path, "w") as f:
        f.write("".join("%s=%s\n" % (k, v) for k, v in kv.items()))
    return str(path)


def _run(h, cfg):
    return h.mlease_job_run(b"ItemModelGridTest", cfg.encode())


def _bytes(root):
    """relative path -> raw bytes of every avro file under root, its random 16-byte sync marker (which also ends the file) zeroed."""
    out = {}
    for dp, _, fs in os.walk(root):
        for f in fs:
            if f.endswith(".avro"):
                p = os.path.join(dp, f)
                data = open(p, "rb").read()
                out[os.path.relpath(p, root)] = data.replace(data[-16:], bytes(16))
    return out


GRID = [("1.0", "10.0"), ("1.0", "0.5"), ("100.0", "10.0"), ("100.0", "0.5")]


def _write_models(path, names, keys, placeholder=False):
    """one LinearModelWithVarAvro record per (grid point, key) for every key in keys; placeholder: posteriorVar = (INTERCEPT) 0, as
    ItemModelTrain writes it without compute.var.  Also a feature the test data never lists, and a repeated key (last wins)."""
    recs = []
    for g, (a, b) in enumerate(GRID):
        for k in keys:
            feats = [{"name": "(INTERCEPT)", "term": "", "value": 0.25 * g}] + [{"name": nm, "term": "", "value": 0.1 * (i + 1)} for i, nm in enumerate(names)]
            var = [{"name": "(INTERCEPT)", "term": "", "value": 0.0}] if placeholder else (
                [{"name": "(INTERCEPT)", "term": "", "value": 0.5}] + [{"name": nm, "term": "", "value": 0.01 * (i + 1)} for i, nm in enumerate(names)] +
                [{"name": "not-in-test-data", "term": "", "value": 3.0}])
            recs.append({"key": "%s:%s#%s" % (a, b, k), "model": feats, "posteriorVar": var})
    recs.append(dict(recs[0], model=[{"name": names[0], "term": "", "value": 2.0}]))
    au.write_avro(path, VAR_SCHEMA, recs)


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    d = tmp_path_factory.mktemp("grid_data")
    npz = np.load(os.path.join(GOLDEN, "sample_data.npz"))
    names = [str(n) for n in npz["feature_names"]]
    recs = au.fixture_records(npz, with_key=lambda i: (i * 7) % 13)
    au.write_avro(str(d / "in" / "part-0.avro"), au.pig_schema_with_key(), recs[:600], codec="deflate", block=64)
    au.write_avro(str(d / "in" / "part-1.avro"), au.pig_schema_with_key(), recs[600:], block=500)
    _write_models(str(d / "models" / "part-r-00000.avro"), names[:20], [k for k in range(13) if k != 5])
    _write_models(str(d / "placeholder" / "part-r-00000.avro"), names[:20], range(13), placeholder=True)
    return d, recs, names


def _grid_cfg(d, out, **kw):
    kv = {"input.paths": str(d / "in"), "output.base.path": str(out), "model.path": str(d / "models"), "item.key": "pkey",
          "intercept.lambdas": "1.0, 100", "default.lambdas": "10,0.5", "compute.var": "true"}
    kv.update(kw)
    return _cfg(str(out) + ".job", kv)


@pytest.mark.parametrize("compute_var", [True, False])
def test_grid_layout_schema_loglik_order_and_fast_generic_bytes(fake_host, data, tmp_path, monkeypatch, compute_var):
    d, recs, _ = data
    trees = {}
    for mode in ("fast", "generic"):
        monkeypatch.setenv("MLEASE_HOST_GENERIC_INGEST", "1" if mode == "generic" else "0")
        out = tmp_path / mode
        assert _run(fake_host, _grid_cfg(d, out, **{"compute.var": str(compute_var).lower()})) == 0, fake_host.mlease_job_last_error().decode()
        trees[mode] = _bytes(str(out))
    assert trees["fast"] == trees["generic"]
    out = tmp_path / "fast"
    dirs = ["lambda-1.0_10", "lambda-1.0_0.5", "lambda-100_10", "lambda-100_0.5"]   # the lambdas as typed, grid in config order
    assert sorted(trees["fast"]) == sorted([x + "/part-r-00000.avro" for x in dirs] + ["_loglik/part-r-00000.avro"])
    order = sorted(range(len(recs)), key=lambda i: str(recs[i]["pkey"]))   # grouped by key in string order, input order inside
    extra = ["pred", "predVar"] if compute_var else ["pred"]
    for x in dirs:
        sch, got = au.read_avro(str(out / x / "part-r-00000.avro"))[:2]
        assert sch["name"] == "ItemModelGridTestOutput" and sch["namespace"] == "com.linkedin.lab.regression.avro"
        assert [f["name"] for f in sch["fields"]] == ["features", "offset", "response", "weight", "pkey"] + extra
        assert [{k: r[k] for k in r if k not in extra} for r in got] == [recs[i] for i in order]
        if compute_var:   # key 5 has no model: no posterior, predVar NaN; every other key has one
            pv = np.array([r["predVar"] for r in got])
            k5 = np.array([r["pkey"] == 5 for r in got])
            assert np.isnan(pv[k5]).all() and not np.isnan(pv[~k5]).any()
    sch, ll = au.read_avro(str(out / "_loglik" / "part-r-00000.avro"))[:2]
    assert sch["name"] == "RegressionTestLoglikOutput"
    assert [r["key"] for r in ll] == ["1.0:10.0", "1.0:0.5", "100.0:10.0", "100.0:0.5"]
    assert all(r["count"] == float(sum(x["weight"] for x in recs)) for r in ll)


def test_grid_shards_write_identical_trees(fake_host, data, tmp_path):
    d, _, _ = data
    trees = []
    for devs in ("0", "0,1", "0,1,2"):
        out = tmp_path / ("d" + devs.replace(",", ""))
        assert _run(fake_host, _grid_cfg(d, out, **{"gpu.devices": devs})) == 0, fake_host.mlease_job_last_error().decode()
        trees.append(_bytes(str(out)))
    assert trees[0] == trees[1] == trees[2]


@pytest.mark.parametrize("case,kw,msg", [
    ("repeat", {"intercept.lambdas": "1.0,100,1"}, "intercept.lambdas x default.lambdas: grid point 1.0:10.0 is repeated"),
    ("repeat_typed", {"default.lambdas": "10,0.5,10.0"}, "intercept.lambdas x default.lambdas: grid point 1.0:10.0 is repeated"),
    ("zero", {"default.lambdas": "10,0"}, "default.lambdas: every lambda must be > 0 (got 0)"),
    ("negative", {"intercept.lambdas": "-1"}, "intercept.lambdas: every lambda must be > 0 (got -1)"),
    ("nan", {"intercept.lambdas": "NaN"}, "intercept.lambdas: every lambda must be > 0 (got NaN)"),
    ("placeholder", {"model.path": "placeholder"}, "model 1.0:10.0#0 has no posterior variance (its posteriorVar is the (INTERCEPT) 0 "
                                                   "placeholder): rerun ItemModelTrain with compute.var=true"),
])
def test_grid_refusals(fake_host, data, tmp_path, case, kw, msg):
    d, _, _ = data
    if kw.get("model.path") == "placeholder":
        kw = dict(kw, **{"model.path": str(d / "placeholder")})
    assert _run(fake_host, _grid_cfg(d, tmp_path / case, **kw)) != 0
    assert fake_host.mlease_job_last_error().decode() == msg


def test_grid_placeholder_models_are_fine_without_compute_var(fake_host, data, tmp_path):
    d, _, _ = data
    cfg = _grid_cfg(d, tmp_path / "o", **{"model.path": str(d / "placeholder"), "compute.var": "false"})
    assert _run(fake_host, cfg) == 0, fake_host.mlease_job_last_error().decode()


def test_grid_refuses_a_record_with_a_repeated_feature(fake_host, tmp_path):
    recs = [{"features": [{"name": "a", "term": "", "value": 1.0}, {"name": "b", "term": "t", "value": 2.0}], "offset": 0, "response": 1, "weight": 1, "pkey": 3},
            {"features": [{"name": "b", "term": "t", "value": 1.0}, {"name": "a", "term": "", "value": 1.0}, {"name": "b", "term": "t", "value": 3.0}],
             "offset": 0, "response": 0, "weight": 1, "pkey": 4}]
    au.write_avro(str(tmp_path / "in" / "p.avro"), au.pig_schema_with_key(), recs)
    _write_models(str(tmp_path / "models" / "p.avro"), ["a"], [3, 4])
    kv = {"input.paths": str(tmp_path / "in"), "output.base.path": str(tmp_path / "o"), "model.path": str(tmp_path / "models"), "item.key": "pkey",
          "intercept.lambdas": "1.0", "default.lambdas": "10.0", "compute.var": "true"}
    assert _run(fake_host, _cfg(str(tmp_path / "t.job"), kv)) != 0
    assert fake_host.mlease_job_last_error().decode() == ("a record of key 4 lists feature b t more than once; its predictive variance would count "
                                                          "the listings as independent features")
    kv["compute.var"] = "false"   # without predVar the record is scored as ItemModelTest scores it
    assert _run(fake_host, _cfg(str(tmp_path / "t.job"), kv)) == 0, fake_host.mlease_job_last_error().decode()


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_score_keyed_var_has_no_cpu_fallback():
    import mlease_b200 as mb
    with pytest.raises(mb.MleaseError, match="no CPU fallback"):
        mb.score_keyed_var(np.ones(1, np.float32), [0, 1], [0, 1], [0], 2, [0, 1], [2], [0.5], [0, 1], [2], [0.1], [1.0])
