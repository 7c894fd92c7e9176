"""CPU tests of ItemModelTest / ItemModelTestLoglik: the sequential restatements against the existing oracle and numpy, both jobs
through the test doubles of the device library (tests/fake_device/fake_mlease_b200.c and fake_item_model.c: canned numbers, so
only layout, order, schemas and error texts are checked here; test_gpu_item_model.py checks the numbers), and the no-GPU failure
of the two new entry points."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import avro_util as au  # noqa: E402
import item_model_ref as ref  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
HOST = os.path.join(ROOT, "ml-ease_b200", "host")


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.parametrize("binary", [False, True])
def test_score_keyed_restatement_equals_per_key_score(binary):
    """Per key and lambda, the keyed restatement is orc.score on that key's rows with that key's model (absent features 0),
    bitwise: including keys without a model (pred = float(offset)), repeated features in a record and a record feature with id
    D - 1 standing for a feature named "(INTERCEPT)" that no model can hold."""
    rng = np.random.default_rng(11)
    K, D, L = 40, 30, 2
    nr = rng.integers(0, 6, K)
    krs = np.concatenate([[0], np.cumsum(nr)]).astype(np.int64)
    n = int(krs[-1])
    rp = np.concatenate([[0], np.cumsum(rng.integers(0, 8, n))]).astype(np.int64)
    ci = rng.integers(0, D, int(rp[-1])).astype(np.int32)
    ci[::5] = D - 1
    v = rng.normal(size=len(ci)).astype(np.float32)
    off = rng.normal(size=n).astype(np.float32)
    models = []
    for _ in range(L):
        ml = []
        for k in range(K):
            if k % 7 == 3:
                ml.append(None)
                continue
            cols = rng.choice(D - 1, 10, replace=False).tolist() + ([D] if k % 2 else [])
            ml.append({c: np.float32(rng.normal()) for c in cols})
        models.append(ml)
    got = ref.score_keyed(krs, rp, ci, v, off, models, D, binary)
    for l in range(L):
        for k in range(K):
            a, b = krs[k], krs[k + 1]
            if a == b:
                continue
            m = np.zeros(D + 1)
            for c, x in (models[l][k] or {}).items():
                m[c] = x
            sub = orc.Csr(rp[a:b + 1] - rp[a], ci[rp[a]:rp[b]], v[rp[a]:rp[b]], np.zeros(b - a, np.int32), offset=off[a:b], n_features=D)
            want = orc.score(sub, m, binary_feature=binary)
            assert np.array_equal(got[l, a:b].view(np.uint32), want.view(np.uint32)), (l, k)
            if models[l][k] is None:
                assert np.array_equal(got[l, a:b], off[a:b])


def test_item_test_loglik_restatement_against_numpy():
    rng = np.random.default_rng(5)
    n = 3000
    key = [("k%d" % i) for i in rng.integers(0, 17, n)]
    grp = np.sort(rng.integers(0, 3, n))
    resp = rng.choice([1, 0, -1], n)
    pred = (rng.normal(size=n) * 2).astype(np.float32)
    w = rng.uniform(0.5, 3, n).astype(np.float32)
    got = ref.item_test_loglik(key, grp, resp, pred, w)
    p, wd = pred.astype(np.float64), w.astype(np.float64)
    ll = np.where(resp == 1, -np.log1p(np.exp(-p)) * wd, -np.log1p(np.exp(p)) * wd).astype(np.float32)
    karr = np.array(key)
    for k in set(key):
        s = c = 0.0
        for g in range(3):
            sel = (karr == k) & (grp == g)
            s += float(np.float32(math.fsum(ll[sel].astype(np.float64))))
            c += float(wd[sel].sum())
        assert abs(got[k][0] - np.float32(s / c)) <= 2 * np.spacing(np.float32(abs(s / c))) and abs(got[k][1] - c) < 1e-9 * c
    with pytest.raises(ValueError, match="response should be 1,0 or -1!"):
        ref.item_test_loglik(["a"], [0], [2], [0.5])


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_keyed_entry_points_have_no_cpu_fallback():
    import mlease_b200 as mb
    with pytest.raises(mb.MleaseError, match="no CPU fallback"):
        mb.score_keyed(np.ones(1, np.float32), [0, 1], [0, 1], [0], 2, [0, 1], [2], [0.5])
    with pytest.raises(mb.MleaseError, match="no CPU fallback"):
        mb.test_loglik_keyed([0], [0], [1], [0.5], 1)


@pytest.fixture(scope="module")
def fake_host(tmp_path_factory):
    d = tmp_path_factory.mktemp("fakehost_item")
    so = str(d / "libmlease_host_fake.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HOST, "avro_io.cpp"), os.path.join(HOST, "regression_jobs.cpp"),
                           os.path.join(HOST, "item_model_jobs.cpp"), "-x", "c", os.path.join(ROOT, "tests", "fake_device", "fake_mlease_b200.c"),
                           os.path.join(ROOT, "tests", "fake_device", "fake_item_model.c"), "-lz", "-pthread", "-lm"])
    h = C.CDLL(so)
    h.mlease_job_last_error.restype = C.c_char_p
    return h


def _cfg(path, lines):
    with open(path, "w") as f:
        f.write("".join("%s=%s\n" % kv for kv in lines.items()))
    return path


def _tree(root):
    out = {}
    for dp, _, fs in os.walk(root):
        for f in fs:
            if f.endswith(".avro"):
                p = os.path.join(dp, f)
                out[os.path.relpath(p, root)] = au.read_avro(p)[:2]
    return out


def _models(path, keys, names):
    schema = {"type": "record", "name": "LinearModelAvro", "fields": [{"name": "key", "type": "string"}, {"name": "model", "type": {"type": "array", "items": {
        "type": "record", "name": "feature", "fields": [{"name": "name", "type": "string"}, {"name": "term", "type": "string"}, {"name": "value", "type": "float"}]}}}]}
    recs = [{"key": k, "model": [{"name": "(INTERCEPT)", "term": "", "value": 0.25}] + [{"name": nm, "term": "", "value": 0.1 * (i + 1)} for i, nm in enumerate(names)]}
            for k in keys]
    recs.append({"key": keys[0], "model": [{"name": names[0], "term": "", "value": 2.0}, {"name": "not-in-test-data", "term": "", "value": 9.0}]})   # last wins
    au.write_avro(path, schema, recs)


def test_item_model_jobs_layout_order_and_avro_paths(fake_host, tmp_path, monkeypatch):
    npz = np.load(os.path.join(GOLDEN, "sample_data.npz"))
    names = [str(n) for n in npz["feature_names"]]
    recs = au.fixture_records(npz, with_key=lambda i: (i * 7) % 13)
    au.write_avro(str(tmp_path / "in" / "part-0.avro"), au.pig_schema_with_key(), recs[:600], codec="deflate", block=64)
    au.write_avro(str(tmp_path / "in" / "part-1.avro"), au.pig_schema_with_key(), recs[600:], block=500)
    _models(str(tmp_path / "models" / "part-r-00000.avro"), ["1.0#%d" % k for k in range(0, 13, 2)] + ["10.0#%d" % k for k in range(1, 13, 3)], names[:20])
    trees = {}
    for mode in ("fast", "generic"):
        monkeypatch.setenv("MLEASE_HOST_GENERIC_INGEST", "1" if mode == "generic" else "0")
        out = str(tmp_path / ("out_" + mode))
        cfg = _cfg(str(tmp_path / (mode + ".job")), {"input.paths": str(tmp_path / "in"), "output.base.path": out, "model.path": str(tmp_path / "models"),
                                                     "item.key": "pkey", "lambda": "1,10.0"})
        assert fake_host.mlease_job_run(b"ItemModelTest", cfg.encode()) == 0, fake_host.mlease_job_last_error().decode()
        trees[mode] = _tree(out)
    assert trees["fast"] == trees["generic"]
    t = trees["fast"]
    assert sorted(t) == ["lambda-1/part-r-00000.avro", "lambda-10.0/part-r-00000.avro"]
    sch, got = t["lambda-1/part-r-00000.avro"]
    assert sch["name"] == "PerItemTestOutput" and sch["namespace"] == "com.linkedin.lab.regression.avro"
    assert [f["name"] for f in sch["fields"]] == ["features", "offset", "response", "weight", "pkey", "pred"]
    # grouped by key in string order ("10" < "2"), input order inside a key, every input field copied
    order = sorted(range(len(recs)), key=lambda i: str(recs[i]["pkey"]))
    assert [{k: r[k] for k in r if k != "pred"} for r in got] == [recs[i] for i in order]

    # ItemModelTestLoglik: output sorted by key (bytes), one record per map key
    schema = {"type": "record", "name": "S", "fields": [{"name": "response", "type": "int"}, {"name": "pred", "type": {"type": "map", "values": "float"}}]}
    ref.write_avro_with_maps(str(tmp_path / "ll" / "a.avro"), schema, [{"response": 1, "pred": {"b": 0.5, "B": 0.1}}, {"response": 0, "pred": {"a": -1.0}}])
    ref.write_avro_with_maps(str(tmp_path / "ll" / "b.avro"), schema, [{"response": -1, "pred": {"b": 0.25, "é": 2.0}}])
    cfg = _cfg(str(tmp_path / "l.job"), {"input.paths": str(tmp_path / "ll"), "output.path": str(tmp_path / "llout")})
    assert fake_host.mlease_job_run(b"ItemModelTestLoglik", cfg.encode()) == 0, fake_host.mlease_job_last_error().decode()
    sch, got = au.read_avro(str(tmp_path / "llout" / "part-r-00000.avro"))[:2]
    assert sch["name"] == "RegressionTestLoglikOutput"
    assert [r["key"] for r in got] == ["B", "a", "b", "é"] and [r["count"] for r in got] == [1.0, 1.0, 2.0, 1.0]


def test_item_model_job_errors(fake_host, tmp_path):
    npz = np.load(os.path.join(GOLDEN, "sample_data.npz"))
    recs = au.fixture_records(npz)[:50]
    au.write_avro(str(tmp_path / "in" / "p.avro"), au.PIG_SCHEMA, recs)
    _models(str(tmp_path / "m" / "p.avro"), ["1.0#0"], ["x"])
    for generic in ("0", "1"):
        os.environ["MLEASE_HOST_GENERIC_INGEST"] = generic
        try:
            cfg = _cfg(str(tmp_path / "t.job"), {"input.paths": str(tmp_path / "in"), "output.base.path": str(tmp_path / "o"), "model.path": str(tmp_path / "m"),
                                                 "item.key": "pkey", "lambda": "1"})
            assert fake_host.mlease_job_run(b"ItemModelTest", cfg.encode()) != 0
            assert fake_host.mlease_job_last_error().decode() == "data does not contain the columnpkey"
        finally:
            del os.environ["MLEASE_HOST_GENERIC_INGEST"]
    schema = {"type": "record", "name": "S", "fields": [{"name": "response", "type": "int"}, {"name": "pred", "type": {"type": "map", "values": "float"}}]}
    ref.write_avro_with_maps(str(tmp_path / "ll" / "a.avro"), schema, [{"response": 1, "pred": {"a": 0.5}}, {"response": 2, "pred": {}}])
    cfg = _cfg(str(tmp_path / "l.job"), {"input.paths": str(tmp_path / "ll"), "output.path": str(tmp_path / "llout")})
    assert fake_host.mlease_job_run(b"ItemModelTestLoglik", cfg.encode()) != 0
    assert fake_host.mlease_job_last_error().decode() == "response should be 1,0 or -1!"
