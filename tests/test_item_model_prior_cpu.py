"""CPU tests of ItemModelTrain with prior.model.path through the test doubles of the device library (tests/fake_device/:
fake_mlease_b200.c, fake_item_model_train.c, and fake_item_model_prior.c, which builds each key's union list as the library does and
fills it with canned numbers naming their source): reading an earlier run's models and choosing its grid point, the features it adds
to the dictionary, the order of the model and posteriorVar lists, and the refusals.  test_gpu_item_model_prior.py checks the numbers."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import avro_util as au  # noqa: E402
import item_model_train_ref as ref  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "ml-ease_b200", "host")
FAKE = os.path.join(ROOT, "tests", "fake_device")
FEATURE = {"type": "record", "name": "feature", "fields": [{"name": "name", "type": "string"}, {"name": "term", "type": "string"},
                                                         {"name": "value", "type": "float"}]}
MODEL_SCHEMA = {"type": "record", "name": "LinearModelWithVarAvro", "namespace": "com.linkedin.mlease.avro", "fields": [
    {"name": "key", "type": "string"}, {"name": "model", "type": {"type": "array", "items": FEATURE}},
    {"name": "posteriorVar", "type": {"type": "array", "items": dict(FEATURE, name="featureVar")}}]}


@pytest.fixture(scope="module")
def fake_host(tmp_path_factory):
    d = tmp_path_factory.mktemp("fakehost_item_prior")
    so = str(d / "libmlease_host_fake.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-o", so] +
                          [os.path.join(HOST, f) for f in ("avro_io.cpp", "regression_jobs.cpp", "item_model_train_job.cpp", "item_model_prior.cpp")] +
                          ["-x", "c"] + [os.path.join(FAKE, f) for f in ("fake_mlease_b200.c", "fake_item_model_train.c", "fake_item_model_prior.c")] +
                          ["-lz", "-pthread", "-lm"])
    h = C.CDLL(so)
    h.mlease_job_last_error.restype = C.c_char_p
    return h


def _run(h, cfg_path, kv):
    with open(cfg_path, "w") as f:
        f.write("".join("%s=%s\n" % e for e in kv.items()))
    rc = h.mlease_job_run(b"ItemModelTrain", str(cfg_path).encode())
    return rc, h.mlease_job_last_error().decode()


def _feat(key, v):
    n, _, t = key.partition("\x01")
    return {"name": n, "term": t, "value": float(v)}


def _model(key, model, var):
    return {"key": key, "model": [_feat(k, v) for k, v in model], "posteriorVar": [_feat(k, v) for k, v in var]}


def _rec(key, feats):
    return {"key": key, "response": 1, "features": [{"name": f, "term": "", "value": 1.5} for f in feats], "weight": 1.0, "offset": 0.0}


def _inputs(tmp_path):
    """today's records: key a lists f0, f1, f2; key b lists f3, f4 (dictionary f0 .. f4).  The earlier run: two grid points, item a
    twice at 1.0:0.5 (the last record wins), an item without rows today (ghost), and features new to today's dictionary."""
    au.write_avro(str(tmp_path / "in" / "p.avro"), ref.PREPARED_SCHEMA,
                  [_rec("a", ["f0", "f1"]), _rec("a", ["f2"]), _rec("b", ["f3", "f4"]), _rec("a", ["f1"])])
    au.write_avro(str(tmp_path / "prior" / "part-r-00000.avro"), MODEL_SCHEMA, [
        _model("1.0:0.5#a", [("(INTERCEPT)", 9.0), ("f2", 9.0)], [("(INTERCEPT)", 9.0)]),
        _model("2.0:0.5#a", [("(INTERCEPT)", 8.0), ("old", 8.0)], [("(INTERCEPT)", 8.0)]),
        _model("1.0:0.5#a", [("(INTERCEPT)", 0.25), ("f1", 2.0), ("newA", 3.0), ("zz\x01t", -1.0)],
               [("(INTERCEPT)", 0.5), ("f1", 0.125), ("newA", 0.0), ("zz\x01t", 4.0), ("onlyvar", 6.0)]),
        _model("1.0:0.5#ghost", [("(INTERCEPT)", 1.0), ("ghostf", 1.0)], [("(INTERCEPT)", 0.0)]),
    ])
    ref.write_lambda_map(str(tmp_path / "lm" / "a.avro"), [("f3", 4.0), ("newA", 2.0), ("f0", 8.0)])
    return {"input.paths": tmp_path / "in", "intercept.lambdas": "3", "default.lambdas": "0.5,2", "prior.model.path": tmp_path / "prior",
            "compute.var": "true", "lambda.map": tmp_path / "lm"}


def _vals(lst):
    return [(f["name"] + ("\x01" + f["term"] if f["term"] else ""), f["value"]) for f in lst]


def test_prior_lists_dictionary_and_order(fake_host, tmp_path, monkeypatch):
    files = {}
    for mode in ("fast", "generic"):
        monkeypatch.setenv("MLEASE_HOST_GENERIC_INGEST", "1" if mode == "generic" else "0")
        kv = _inputs(tmp_path)
        kv.update({"output.model.path": tmp_path / ("out_" + mode), "prior.model.lambda": " 1:0.5"})   # read as Float.toString does
        rc, err = _run(fake_host, tmp_path / (mode + ".job"), kv)
        assert rc == 0, err
        files[mode] = str(tmp_path / ("out_" + mode) / "models" / "part-r-00000.avro")
    assert au.read_avro(files["fast"])[1] == au.read_avro(files["generic"])[1]
    got = au.read_avro(files["fast"])[1]
    assert [r["key"] for r in got] == ["3.0:0.5#a", "3.0:2.0#a", "3.0:0.5#b", "3.0:2.0#b"]   # no output for ghost
    f32 = lambda x: float(np.float32(x))  # noqa: E731
    for r in got:
        b = 0 if r["key"].startswith("3.0:0.5") else 1
        if r["key"].endswith("#a"):
            # dictionary f0 .. f4, then the prior's new features in item and model order: newA, zz|t (and ghost's ghostf); the model
            # lists the intercept, then the union of the rows' columns and the prior-only ones, in dictionary order
            assert _vals(r["model"]) == [("(INTERCEPT)", 0.25), ("f0", f32(0.001 * 0 + b)), ("f1", 2.5), ("f2", f32(0.002 + b)),
                                         ("newA", 3.0), ("zz\x01t", -1.0)]
            # posteriorVar: the intercept, the data features, the prior-only features with a variance, then the lambda.map entries
            # not listed yet, in map order (newA had no variance, so the map's entry lists it)
            assert _vals(r["posteriorVar"]) == [("(INTERCEPT)", 0.5), ("f0", f32(1 / (1 + b))), ("f1", 0.125), ("f2", f32(1 / (3 + b))),
                                                ("zz\x01t", 4.0), ("f3", 0.25), ("newA", 0.5)]
        else:
            assert _vals(r["model"]) == [("(INTERCEPT)", 0.0), ("f3", f32(0.003 + b)), ("f4", f32(0.004 + b))]
            assert _vals(r["posteriorVar"]) == [("(INTERCEPT)", 7.0), ("f3", f32(1 / (4 + b))), ("f4", f32(1 / (5 + b))), ("newA", 0.5),
                                                ("f0", 0.125)]


def test_one_grid_point_needs_no_lambda_and_a_mean_only_prior(fake_host, tmp_path):
    """A run without compute.var wrote (INTERCEPT) 0 as its only posteriorVar entry: every entry is mean-only (variance 0)."""
    kv = _inputs(tmp_path)
    au.write_avro(str(tmp_path / "one" / "m.avro"), MODEL_SCHEMA, [
        _model("1.0:0.5#b", [("(INTERCEPT)", -0.75), ("f4", 1.25), ("f9", 2.0)], [("(INTERCEPT)", 0.0)])])
    kv.update({"prior.model.path": tmp_path / "one", "output.model.path": tmp_path / "o", "default.lambdas": "0.5"})
    rc, err = _run(fake_host, tmp_path / "a.job", kv)
    assert rc == 0, err
    got = au.read_avro(str(tmp_path / "o" / "models" / "part-r-00000.avro"))[1]
    assert [r["key"] for r in got] == ["3.0:0.5#a", "3.0:0.5#b"]
    f32 = lambda x: float(np.float32(x))  # noqa: E731
    assert _vals(got[0]["model"]) == [("(INTERCEPT)", 0.0), ("f0", 0.0), ("f1", f32(0.001)), ("f2", f32(0.002))]
    assert _vals(got[1]["model"]) == [("(INTERCEPT)", -0.75), ("f3", f32(0.003)), ("f4", 1.75), ("f9", 2.0)]
    # variance 0 everywhere: the intercept entry passes its 0 (the library reads it as the usual variance); f9 is prior-only
    # without a variance, so posteriorVar does not list it
    assert _vals(got[1]["posteriorVar"]) == [("(INTERCEPT)", 0.0), ("f3", 0.25), ("f4", f32(0.2)), ("newA", 0.5), ("f0", 0.125)]


@pytest.mark.parametrize("lam,message", [
    (None, "prior.model.path holds the models of 2 grid points (1.0:0.5, 2.0:0.5): set prior.model.lambda to one of them"),
    ("3:0.5", "prior.model.lambda 3.0:0.5 is not a grid point of prior.model.path (1.0:0.5, 2.0:0.5)"),
    ("1.0", 'prior.model.lambda: expected <intercept lambda>:<default lambda>, got "1.0"'),
])
def test_prior_refusals(fake_host, tmp_path, lam, message):
    kv = _inputs(tmp_path)
    kv["output.model.path"] = tmp_path / "o"
    if lam is not None:
        kv["prior.model.lambda"] = lam
    rc, err = _run(fake_host, tmp_path / "e.job", kv)
    assert rc != 0 and err == message
    assert not os.path.exists(tmp_path / "o" / "models")


def test_prior_refusals_of_the_files(fake_host, tmp_path):
    kv = _inputs(tmp_path)
    os.makedirs(tmp_path / "empty")
    kv.update({"output.model.path": tmp_path / "o", "prior.model.path": tmp_path / "empty"})
    rc, err = _run(fake_host, tmp_path / "e.job", kv)
    assert rc != 0 and err == "prior.model.path: no models under %s" % (tmp_path / "empty")
    au.write_avro(str(tmp_path / "bad" / "m.avro"), MODEL_SCHEMA, [_model("nohash", [("(INTERCEPT)", 1.0)], [])])
    kv["prior.model.path"] = tmp_path / "bad"
    rc, err = _run(fake_host, tmp_path / "e.job", kv)
    assert rc != 0 and err == 'prior.model.path: record key "nohash" is not <intercept lambda>:<default lambda>#<item>'


def test_job_without_the_prior_unit_refuses_prior_model_path(tmp_path):
    """item_model_train_job.cpp links without item_model_prior.cpp (as the other jobs' tests link it): prior.model.path is then
    refused, not ignored."""
    so = str(tmp_path / "libnoprior.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-o", so] +
                          [os.path.join(HOST, f) for f in ("avro_io.cpp", "regression_jobs.cpp", "item_model_train_job.cpp")] +
                          ["-x", "c"] + [os.path.join(FAKE, f) for f in ("fake_mlease_b200.c", "fake_item_model_train.c")] + ["-lz", "-pthread", "-lm"])
    h = C.CDLL(so)
    h.mlease_job_last_error.restype = C.c_char_p
    kv = _inputs(tmp_path)
    kv["output.model.path"] = tmp_path / "o"
    rc, err = _run(h, tmp_path / "e.job", kv)
    assert rc != 0 and err == "prior.model.path: this build of ItemModelTrain has no per-key priors"
