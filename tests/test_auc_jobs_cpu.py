"""CPU tests of the RegressionTestAuc and ItemModelGridTestAuc jobs, linked against test doubles of the device library
(tests/fake_device/: fake_mlease_b200.c, and fake_auc.c for mlease_test_auc, whose "AUC" of a segment is a hash of the segment's own
rows).  Checked here: output layout and schemas, grid and key order, keyAuc recomputed in numpy from what the double returned, and
the refusals; test_gpu_auc.py checks the numbers."""
import ctypes as C
import math
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
GRID = [("1.0", "10"), ("1.0", "0.5"), ("100", "10"), ("100", "0.5")]
GKEYS = ["1.0:10.0", "1.0:0.5", "100.0:10.0", "100.0:0.5"]


@pytest.fixture(scope="module")
def fake_host(tmp_path_factory):
    d = tmp_path_factory.mktemp("fakehost_auc")
    so = str(d / "libmlease_host_fake.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-o", so] +
                          [os.path.join(HOST, f) for f in ("avro_io.cpp", "regression_jobs.cpp", "auc_jobs.cpp")] +
                          ["-x", "c"] + [os.path.join(FAKE, f) for f in ("fake_mlease_b200.c", "fake_auc.c")] + ["-lz", "-pthread", "-lm"])
    h = C.CDLL(so)
    h.mlease_job_last_error.restype = C.c_char_p
    return h


def _run(h, job, path, kv):
    with open(path, "w") as f:
        f.write("".join("%s=%s\n" % (k, v) for k, v in kv.items()))
    return h.mlease_job_run(job.encode(), str(path).encode())


def _scored_schema():
    s = au.pig_schema_with_key()
    s["fields"].append({"name": "pred", "type": "float"})
    return s


def _mix(a, b):
    return math.fmod(a * 1.0000001 + b * 0.6180339887 + 0.1234567, 97.0)


def _hash(resp, weight, pred):
    """fake_auc.c's value of one segment"""
    h, p, n = 0.0, 0.0, 0.0
    for i, (r, w, x) in enumerate(zip(resp, weight, pred)):
        h = _mix(h, float(i) + 0.5 * r + 0.25 * w + float(np.float32(x)))
        p, n = (p + w, n) if r == 1 else (p, n + w)
    return h / 97.0 if p > 0 and n > 0 else float("nan")


@pytest.fixture(scope="module")
def recs():
    npz = np.load(os.path.join(GOLDEN, "sample_data.npz"))
    out = au.fixture_records(npz, with_key=lambda i: (i * 7) % 13)[:400]
    for i, r in enumerate(out):
        r["weight"] = i % 4                         # zero weights too
        if r["pkey"] == 3:
            r["response"] = 1                       # a key with positives only: its AUC is NaN
    return out


def _write_grid(base, recs, order, tamper=None):
    for g, (a, b) in enumerate(GRID):
        rows = [dict(recs[i], pred=float(np.float32(0.01 * ((i * (g + 3)) % 17) - 0.05))) for i in order]
        if tamper and tamper[0] == g:
            tamper[1](rows)
        au.write_avro(os.path.join(base, "lambda-%s_%s" % (a, b), "part-r-00000.avro"), _scored_schema(), rows[:150])
        au.write_avro(os.path.join(base, "lambda-%s_%s" % (a, b), "part-r-00001.avro"), _scored_schema(), rows[150:])


def _grid_kv(base, out, **kw):
    kv = {"input.base.path": str(base), "output.base.path": str(out), "item.key": "pkey", "intercept.lambdas": "1.0,100",
          "default.lambdas": "10,0.5"}
    kv.update(kw)
    return kv


def test_grid_layout_order_and_key_auc(fake_host, recs, tmp_path):
    order = sorted(range(len(recs)), key=lambda i: str(recs[i]["pkey"]))   # as ItemModelGridTest writes them
    _write_grid(str(tmp_path / "in"), recs, order)
    out = tmp_path / "out"
    assert _run(fake_host, "ItemModelGridTestAuc", tmp_path / "g.job", _grid_kv(tmp_path / "in", out)) == 0, \
        fake_host.mlease_job_last_error().decode()
    sch, top = au.read_avro(str(out / "_auc" / "part-r-00000.avro"))[:2]
    assert sch["name"] == "ItemModelGridTestAucOutput"
    assert [(f["name"], f["type"]) for f in sch["fields"]] == [("key", "string"), ("auc", "double"), ("keyAuc", "double"),
                                                               ("positiveWeight", "double"), ("negativeWeight", "double")]
    assert [r["key"] for r in top] == GKEYS
    sch, per = au.read_avro(str(out / "_key_auc" / "part-r-00000.avro"))[:2]
    assert [f["name"] for f in sch["fields"]] == ["key", "auc", "positiveWeight", "negativeWeight"]
    knames = sorted({str(r["pkey"]) for r in recs})
    assert [r["key"] for r in per] == ["%s#%s" % (g, k) for g in GKEYS for k in knames]
    resp = np.array([recs[i]["response"] for i in order])
    w = np.array([recs[i]["weight"] for i in order], np.float64)
    keys = [str(recs[i]["pkey"]) for i in order]
    P, N = w[resp == 1].sum(), w[resp != 1].sum()
    for g, t in enumerate(top):
        assert t["positiveWeight"] == P and t["negativeWeight"] == N
        pred = [0.01 * ((i * (g + 3)) % 17) - 0.05 for i in order]
        assert t["auc"] == _hash(resp, w, pred)
        rows = per[g * len(knames):(g + 1) * len(knames)]
        num = den = 0.0
        for k, r in zip(knames, rows):
            sel = [q for q in range(len(order)) if keys[q] == k]
            assert r["positiveWeight"] == w[sel][resp[sel] == 1].sum() and r["negativeWeight"] == w[sel][resp[sel] != 1].sum()
            a = _hash(resp[sel], w[sel], [pred[q] for q in sel])
            assert (math.isnan(a) and math.isnan(r["auc"])) or a == r["auc"]
            if not math.isnan(r["auc"]):
                num += (r["positiveWeight"] + r["negativeWeight"]) * r["auc"]
                den += r["positiveWeight"] + r["negativeWeight"]
        assert math.isnan(rows[knames.index("3")]["auc"])
        assert t["keyAuc"] == num / den


def test_grid_groups_records_by_key(fake_host, recs, tmp_path):
    """records in input order (not grouped) give the same files as records grouped by key"""
    grouped = sorted(range(len(recs)), key=lambda i: str(recs[i]["pkey"]))
    _write_grid(str(tmp_path / "a"), recs, grouped)
    _write_grid(str(tmp_path / "b"), recs, list(range(len(recs))))
    got = []
    for x in ("a", "b"):
        assert _run(fake_host, "ItemModelGridTestAuc", tmp_path / (x + ".job"), _grid_kv(tmp_path / x, tmp_path / ("o" + x))) == 0
        got.append(au.read_avro(str(tmp_path / ("o" + x) / "_key_auc" / "part-r-00000.avro"))[1])
    assert [r["key"] for r in got[0]] == [r["key"] for r in got[1]]
    assert [(r["positiveWeight"], r["negativeWeight"]) for r in got[0]] == [(r["positiveWeight"], r["negativeWeight"]) for r in got[1]]


def _flip_response(rows):
    rows[7] = dict(rows[7], response=1 - rows[7]["response"])


def _drop_last(rows):
    rows.pop()


def _swap_keys(rows):
    rows[0], rows[1] = dict(rows[0], pkey=rows[1]["pkey"]), dict(rows[1], pkey=rows[0]["pkey"])


@pytest.mark.parametrize("name,tamper,msg", [
    ("response", (2, _flip_response), "ItemModelGridTestAuc: {in}/lambda-100_10/part-r-00000.avro does not hold the records of "
                                      "{in}/lambda-1.0_10 in the same order"),
    ("count", (1, _drop_last), "ItemModelGridTestAuc: {in}/lambda-1.0_0.5 holds 399 records, {in}/lambda-1.0_10 400"),
    ("key", (3, _swap_keys), "ItemModelGridTestAuc: {in}/lambda-100_0.5/part-r-00000.avro does not hold the records of "
                             "{in}/lambda-1.0_10 in the same order"),
])
def test_grid_refuses_mismatched_directories(fake_host, recs, tmp_path, name, tamper, msg):
    grouped = sorted(range(len(recs)), key=lambda i: str(recs[i]["pkey"]))
    if name == "key":   # two records of different keys
        grouped = [grouped[0], grouped[-1]] + grouped[1:-1]
    _write_grid(str(tmp_path / "in"), recs, grouped, tamper)
    assert _run(fake_host, "ItemModelGridTestAuc", tmp_path / "g.job", _grid_kv(tmp_path / "in", tmp_path / "o")) != 0
    assert fake_host.mlease_job_last_error().decode() == msg.format(**{"in": str(tmp_path / "in")})
    assert not os.path.exists(tmp_path / "o" / "_auc")


def test_grid_refuses_a_shorter_directory(fake_host, recs, tmp_path):
    grouped = sorted(range(len(recs)), key=lambda i: str(recs[i]["pkey"]))
    _write_grid(str(tmp_path / "in"), recs, grouped)
    os.remove(tmp_path / "in" / "lambda-100_0.5" / "part-r-00001.avro")
    assert _run(fake_host, "ItemModelGridTestAuc", tmp_path / "g.job", _grid_kv(tmp_path / "in", tmp_path / "o")) != 0
    assert fake_host.mlease_job_last_error().decode() == "ItemModelGridTestAuc: %s holds 150 records, %s 400" % (
        tmp_path / "in" / "lambda-100_0.5", tmp_path / "in" / "lambda-1.0_10")


def test_grid_refuses_a_repeated_point(fake_host, recs, tmp_path):
    _write_grid(str(tmp_path / "in"), recs, list(range(len(recs))))
    kv = _grid_kv(tmp_path / "in", tmp_path / "o", **{"default.lambdas": "10,0.5,10.0"})
    assert _run(fake_host, "ItemModelGridTestAuc", tmp_path / "g.job", kv) != 0
    assert fake_host.mlease_job_last_error().decode() == "intercept.lambdas x default.lambdas: grid point 1.0:10.0 is repeated"


def test_regression_test_auc_layout(fake_host, recs, tmp_path):
    base = tmp_path / "test"
    preds = {"lambda-1.0": [0.1 * (i % 7) for i in range(len(recs))], "best-model": [0.2 * (i % 5) - 0.3 for i in range(len(recs))]}
    for d, p in preds.items():
        au.write_avro(str(base / d / "part-r-00000.avro"), _scored_schema(), [dict(r, pred=float(np.float32(x))) for r, x in zip(recs, p)])
    kv = {"input.base.paths": str(base), "output.base.path": str(tmp_path / "out"), "lambda": "1.0,2.0"}   # lambda-2.0 was not scored
    assert _run(fake_host, "RegressionTestAuc", tmp_path / "t.job", kv) == 0, fake_host.mlease_job_last_error().decode()
    resp = np.array([r["response"] for r in recs])
    w = np.array([r["weight"] for r in recs], np.float64)
    for d, p in preds.items():
        sch, got = au.read_avro(str(tmp_path / "out" / d / "_auc" / "part-r-00000.avro"))[:2]
        assert sch["name"] == "TestAucOutput"
        assert [(f["name"], f["type"]) for f in sch["fields"]] == [("key", "string"), ("auc", "double"), ("positiveWeight", "double"),
                                                                   ("negativeWeight", "double")]
        assert got == [{"key": "testAuc", "auc": _hash(resp, w, p), "positiveWeight": w[resp == 1].sum(), "negativeWeight": w[resp != 1].sum()}]
    assert not os.path.exists(tmp_path / "out" / "lambda-2.0")
