"""CPU tests of the RegressionPosterior job through the test doubles of the device library (tests/fake_device/fake_mlease_b200.c and
fake_admm_posterior.c: canned numbers): the final-model-var layout, keys, schema and record order, its model lists equal to
final-model's, final-model left byte for byte as RegressionAdmmTrain wrote it, and the refusals.  test_gpu_admm_posterior.py checks the
numbers."""
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


@pytest.fixture(scope="module")
def fake_host(tmp_path_factory):
    d = tmp_path_factory.mktemp("fakehost_posterior")
    so = str(d / "libmlease_host_fake.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HOST, "avro_io.cpp"), os.path.join(HOST, "regression_jobs.cpp"),
                           os.path.join(HOST, "regression_posterior_job.cpp"), "-x", "c", os.path.join(ROOT, "tests", "fake_device", "fake_mlease_b200.c"),
                           os.path.join(ROOT, "tests", "fake_device", "fake_admm_posterior.c"), "-lz", "-pthread", "-lm"])
    h = C.CDLL(so)
    h.mlease_job_last_error.restype = C.c_char_p
    return h


def _run(h, job, path, kv, extra=""):
    with open(path, "w") as f:
        f.write("".join("%s=%s\n" % e for e in kv.items()) + extra)
    rc = h.mlease_job_run(job.encode(), str(path).encode())
    return rc, h.mlease_job_last_error().decode()


def _train(h, tmp_path):
    npz = np.load(os.path.join(GOLDEN, "sample_data.npz"))
    recs = au.fixture_records(npz, with_key=lambda i: i // 250)
    au.write_avro(str(tmp_path / "in" / "part-0.avro"), au.pig_schema_with_key(), recs, block=300)
    out = tmp_path / "out"
    rc, err = _run(h, "Regression", tmp_path / "r.job", {"input.paths": tmp_path / "in", "output.base.path": out, "map.key": "pkey",
                                                          "num.blocks": 4, "num.iters": 3, "regularizer": 2}, "lambda=10,1\n")
    assert rc == 0, err
    return out


@pytest.mark.parametrize("full", [False, True])
def test_final_model_var_layout(fake_host, tmp_path, full):
    out = _train(fake_host, tmp_path)
    fm = out / "final-model" / "part-r-00000.avro"
    before = open(fm, "rb").read()
    kv = {"output.base.path": out, "num.blocks": 4, "compute.full.var": "true" if full else "false"}
    rc, err = _run(fake_host, "RegressionPosterior", tmp_path / "p.job", kv, "lambda=10,1\n")
    assert rc == 0, err
    assert open(fm, "rb").read() == before                                   # final-model untouched
    assert os.listdir(out / "final-model-var") == ["part-r-00000.avro"]
    sch, got = au.read_avro(str(out / "final-model-var" / "part-r-00000.avro"))[:2]
    assert sch["name"] == "LinearModelWithVarAvro" and sch["namespace"] == "com.linkedin.mlease.avro"
    assert [f["name"] for f in sch["fields"]] == ["key", "model", "posteriorVar"]
    final = au.read_avro(str(fm))[1]
    assert [r["key"] for r in got] == [r["key"] for r in final] == ["10.0", "1.0"]   # final-model's keys, in its order
    for l, (r, f) in enumerate(zip(got, final)):
        assert r["model"] == f["model"]
        pv = r["posteriorVar"]
        names = [x["name"] for x in f["model"]]
        assert pv[0]["name"] == "(INTERCEPT)" and [x["name"] for x in pv[1:]] == names[1:]   # intercept, then the dictionary's features
        z = {x["name"]: x["value"] for x in f["model"]}
        D = len(pv) - 1
        for k, x in enumerate(pv[1:]):
            assert x["value"] == np.float32(1.0 / (1 + k + 10 * l) + (1000.0 if full else 0.0) + float(z[x["name"]]) / 1024.0)
        assert pv[0]["value"] == np.float32(1.0 / (1 + D + 10 * l) + (1000.0 if full else 0.0) + float(z["(INTERCEPT)"]) / 1024.0)


@pytest.mark.parametrize("kv,extra,message", [
    ({"regularizer": 1}, "lambda=10,1\n", "RegressionPosterior: the L1 penalty has no Hessian (regularizer must be 2)"),
    ({}, "lambda=10,3\n", "RegressionPosterior: final-model key 1.0 is not one of the job's lambdas"),
    ({"num.blocks": 3}, "lambda=10,1\n", "Map key is wrong! key has to be in the range of [0,numPartitions-1]."),
])
def test_refusals(fake_host, tmp_path, kv, extra, message):
    out = _train(fake_host, tmp_path)
    rc, err = _run(fake_host, "RegressionPosterior", tmp_path / "e.job", dict({"output.base.path": out, "num.blocks": 4}, **kv), extra)
    assert rc != 0 and err == message


def test_refuses_without_final_model(fake_host, tmp_path):
    out = _train(fake_host, tmp_path)
    rc, err = _run(fake_host, "RegressionPosterior", tmp_path / "e.job", {"output.base.path": tmp_path / "none", "num.blocks": 4,
                                                                          "input.paths": out / "tmp-data"}, "lambda=1\n")
    assert rc != 0 and err.startswith("RegressionPosterior: no final-model under")
