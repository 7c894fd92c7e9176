"""CPU tests of ItemModelTrain: the restatement against the oracle's NaiveTrain, and the job through the test doubles of the device
library (tests/fake_device/fake_mlease_b200.c and fake_item_model_train.c: canned numbers, so only layout, order, schema, key strings,
the prior means handed to the device, the lambda.map-only variances and error texts are checked here; test_gpu_item_model_train.py
checks the numbers), and the no-GPU failure of the new entry point."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import avro_util as au  # noqa: E402
import item_model_train_ref as ref  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "ml-ease_b200", "host")


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def _prepared(n=120, keys=("2", "10", "k"), D=12, seed=3):
    rng = np.random.default_rng(seed)
    recs = []
    for i in range(n):
        key = keys[i % len(keys)]
        cols = rng.choice(D - (4 if key == "k" else 0), 3, replace=False)     # key "k" never lists f8..f11
        recs.append({"key": key, "response": int(rng.integers(0, 2)), "features": [{"name": "f%d" % c, "term": "", "value": float(rng.normal())} for c in cols],
                     "weight": float(rng.uniform(0.5, 2)), "offset": float(rng.normal(0, 0.1))})
    return recs


def test_restatement_is_naive_train_when_the_priors_coincide():
    """With iλ = dλ = λ and intercept mean 0 the reducer is NaiveTrain's with penalize.intercept: the restatement's models equal the
    oracle's orc.naive_train on the same per-key datasets."""
    recs = _prepared()
    got = ref.item_model_train(recs, [2.0], [2.0], compute_var=False)
    names = []
    for r in recs:
        for f in r["features"]:
            if f["name"] not in names:
                names.append(f["name"])
    D = len(names)
    for g in got:
        key = g["key"].split("#", 1)[1]
        rows = [r for r in recs if r["key"] == key]
        rp, ci, v = [0], [], []
        for r in rows:
            ent = sorted((names.index(f["name"]), f["value"]) for f in r["features"])
            ci += [c for c, _ in ent]; v += [x for _, x in ent]; rp.append(len(ci))
        data = orc.Csr(rp, ci, v, [r["response"] for r in rows], [r["weight"] for r in rows], [r["offset"] for r in rows], D)
        want, _, _ = orc.naive_train(data, [0, len(rows)], 2.0, penalize_intercept=True, mode="exact")
        m = {f["name"]: f["value"] for f in g["model"]}
        assert g["key"].startswith("2.0:2.0#")
        assert abs(m["(INTERCEPT)"] - np.float32(want[0, D])) <= 1e-5 * max(1.0, abs(want[0, D]))
        for nm in m:
            if nm != "(INTERCEPT)":
                assert abs(m[nm] - np.float32(want[0, names.index(nm)])) <= 1e-5 * max(1.0, np.abs(want).max())
        assert g["posteriorVar"] == [{"name": "(INTERCEPT)", "term": "", "value": 0.0}]


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_item_model_train_has_no_cpu_fallback():
    import mlease_b200 as mb
    with pytest.raises(mb.MleaseError, match="no CPU fallback"):
        mb.item_model_train(np.ones(2, np.float32), [0, 2], [1, 0], [1.0], [1.0], rowptr=[0, 1, 2], colidx=[0, 1], num_features=2)


@pytest.fixture(scope="module")
def fake_host(tmp_path_factory):
    d = tmp_path_factory.mktemp("fakehost_item_train")
    so = str(d / "libmlease_host_fake.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HOST, "avro_io.cpp"), os.path.join(HOST, "regression_jobs.cpp"),
                           os.path.join(HOST, "item_model_train_job.cpp"), "-x", "c", os.path.join(ROOT, "tests", "fake_device", "fake_mlease_b200.c"),
                           os.path.join(ROOT, "tests", "fake_device", "fake_item_model_train.c"), "-lz", "-pthread", "-lm"])
    h = C.CDLL(so)
    h.mlease_job_last_error.restype = C.c_char_p
    return h


def _run(h, cfg_path, kv):
    with open(cfg_path, "w") as f:
        f.write("".join("%s=%s\n" % e for e in kv.items()))
    rc = h.mlease_job_run(b"ItemModelTrain", str(cfg_path).encode())
    return rc, h.mlease_job_last_error().decode()


def _bytes_after_header(path):
    """the file's data blocks (the header ends with the 16-byte sync marker, which the writer draws at random)"""
    b = open(path, "rb").read()
    sync = b[-16:]
    return b[b.index(sync) + 16:].replace(sync, b"")


def test_job_layout_keys_priors_and_avro_paths(fake_host, tmp_path, monkeypatch):
    recs = _prepared()
    au.write_avro(str(tmp_path / "in" / "part-0.avro"), ref.PREPARED_SCHEMA, recs[:50])
    au.write_avro(str(tmp_path / "in" / "part-1.avro"), ref.PREPARED_SCHEMA, recs[50:], codec="deflate", block=30)
    ref.write_lambda_map(str(tmp_path / "lm" / "a.avro"), [("f9", 4.0), ("zz\x01t", 3.0), ("f1", 0.5), ("zz\x01t", 7.0), ("(INTERCEPT)", 9.0)])
    ref.write_prior_mean_map(str(tmp_path / "pm" / "a.avro"), [("2", "0.1"), ("nokey", "5")])
    ref.write_prior_mean_map(str(tmp_path / "pm" / "b.avro"), [("k", 0.3)], value_type="float")
    files = {}
    for mode in ("fast", "generic"):
        monkeypatch.setenv("MLEASE_HOST_GENERIC_INGEST", "1" if mode == "generic" else "0")
        out = tmp_path / ("out_" + mode)
        os.makedirs(out / "tmp-data")
        rc, err = _run(fake_host, tmp_path / (mode + ".job"), {
            "input.paths": tmp_path / "in", "output.model.path": out, "intercept.lambdas": "1e-4, 1", "default.lambdas": "0.1,1e8,0.1",
            "lambda.map": tmp_path / "lm", "intercept.prior.mean.map": tmp_path / "pm", "intercept.default.prior.mean": "0.1",
            "compute.var": "true", "liblinear.epsilon": "0.01", "short.feature.index": "true", "report.frequency": "5"})
        assert rc == 0, err
        assert sorted(os.listdir(out)) == ["models"] and os.listdir(out / "models") == ["part-r-00000.avro"]   # remove.tmp.dir defaults to true
        files[mode] = str(out / "models" / "part-r-00000.avro")
    assert _bytes_after_header(files["fast"]) == _bytes_after_header(files["generic"])
    sch, got = au.read_avro(files["fast"])[:2]
    assert sch["name"] == "LinearModelWithVarAvro" and sch["namespace"] == "com.linkedin.mlease.avro"
    assert [f["name"] for f in sch["fields"]] == ["key", "model", "posteriorVar"]
    grid = ["1.0E-4:0.1", "1.0E-4:1.0E8", "1.0E-4:0.1", "1.0:0.1", "1.0:1.0E8", "1.0:0.1"]    # config order, the repeated 0.1 kept
    assert [r["key"] for r in got] == [g + "#" + k for k in ("10", "2", "k") for g in grid]   # keys in byte order
    names = []
    for r in recs:
        for f in r["features"]:
            if f["name"] not in names:
                names.append(f["name"])
    for i, r in enumerate(got):
        key = r["key"].split("#")[1]
        a, b = (i % 6) // 3, (i % 6) % 3
        listed = sorted({names.index(f["name"]) for x in recs if x["key"] == key for f in x["features"]})
        assert [f["name"] for f in r["model"]] == ["(INTERCEPT)"] + [names[j] for j in listed]
        assert [f["value"] for f in r["model"][1:]] == [np.float32(10 * a + b + 0.001 * j) for j in listed]
        # the intercept's prior mean: the map's double ("0.1" for key 2; float 0.3 read through "0.3" for key k), else the float-rounded default
        mean = {"2": 0.1, "k": 0.3, "10": float(np.float32(0.1))}[key]
        assert r["model"][0]["value"] == np.float32(mean)
        assert r["posteriorVar"][0]["value"] == np.float32(1e9 * (mean - float(np.float32(mean))))
        assert (r["posteriorVar"][0]["value"] != 0) == (key != "10")
        pv = r["posteriorVar"]
        assert [f["value"] for f in pv[1:1 + len(listed)]] == [np.float32(1.0 / (1 + j + a + b)) for j in listed]
        # then the lambda.map features the key's rows do not list, in map order (last value of a repeat), at float(1/lambda)
        extra = [(f["name"], f["term"], f["value"]) for f in pv[1 + len(listed):]]
        want = [("f9", "", np.float32(1 / 4.0))] if key == "k" else []
        want += [("zz", "t", np.float32(1 / 7.0))]
        assert extra == want, (key, extra)
        assert "f1" in [f["name"] for f in r["model"]]


def test_job_without_compute_var_and_keeping_tmp_data(fake_host, tmp_path):
    au.write_avro(str(tmp_path / "out" / "tmp-data" / "part-0.avro"), ref.PREPARED_SCHEMA, _prepared(30))
    rc, err = _run(fake_host, tmp_path / "a.job", {"input.paths": tmp_path / "out" / "tmp-data", "output.model.path": tmp_path / "out",
                                                   "intercept.lambdas": "2", "default.lambdas": "3", "remove.tmp.dir": "false"})
    assert rc == 0, err
    assert sorted(os.listdir(tmp_path / "out")) == ["models", "tmp-data"]
    got = au.read_avro(str(tmp_path / "out" / "models" / "part-r-00000.avro"))[1]
    assert [r["key"] for r in got] == ["2.0:3.0#10", "2.0:3.0#2", "2.0:3.0#k"]
    assert all(r["posteriorVar"] == [{"name": "(INTERCEPT)", "term": "", "value": 0.0}] for r in got)


@pytest.mark.parametrize("kv,message", [
    ({"default.lambdas": "1"}, "Key intercept.lambdas is not in the job config"),
    ({"intercept.lambdas": "1"}, "Key default.lambdas is not in the job config"),
    ({"intercept.lambdas": "1,0", "default.lambdas": "1"}, "intercept.lambdas: every lambda must be > 0 (got 0)"),
    ({"intercept.lambdas": "1", "default.lambdas": "-2"}, "default.lambdas: every lambda must be > 0 (got -2)"),
    ({"intercept.lambdas": "1", "default.lambdas": "NaN"}, "default.lambdas: every lambda must be > 0 (got NaN)"),
])
def test_job_refusals(fake_host, tmp_path, kv, message):
    au.write_avro(str(tmp_path / "in" / "p.avro"), ref.PREPARED_SCHEMA, _prepared(10))
    rc, err = _run(fake_host, tmp_path / "e.job", dict({"input.paths": tmp_path / "in", "output.model.path": tmp_path / "o"}, **kv))
    assert rc != 0 and err == message


def test_job_refuses_a_lambda_map_lambda_of_zero(fake_host, tmp_path):
    au.write_avro(str(tmp_path / "in" / "p.avro"), ref.PREPARED_SCHEMA, _prepared(10))
    ref.write_lambda_map(str(tmp_path / "lm" / "a.avro"), [("f1", 0.0)])
    rc, err = _run(fake_host, tmp_path / "e.job", {"input.paths": tmp_path / "in", "output.model.path": tmp_path / "o", "intercept.lambdas": "1",
                                                   "default.lambdas": "1", "lambda.map": tmp_path / "lm"})
    assert rc != 0 and err == "lambda.map: lambda of feature f1 must be > 0 (it becomes the prior variance 1/lambda)"
