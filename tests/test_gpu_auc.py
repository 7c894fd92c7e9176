"""GPU tests of mlease_test_auc (k7_auc.cu) against tests/auc_ref.py: bit for bit on integer weights, within the fp64 bound on float
weights, independence of every key and set from the others, set chunking under a device budget, the refusals, and the
RegressionTestAuc / ItemModelGridTestAuc jobs on the fixture."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import avro_util as au  # noqa: E402
from auc_ref import test_auc_ref  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture
def budget():
    from mlease_b200 import _hooks
    yield _hooks.set_keyed_budget
    _hooks.set_keyed_budget(0)


def _bits_equal(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


def _tie_case(seed=0, S=5, K=300):
    """integer weights, a handful of prediction values (both zeros, both infinities), keys of 0 .. 60 rows and two of several tiles,
    single-class and all-zero-weight keys"""
    rng = np.random.default_rng(seed)
    sizes = rng.integers(0, 60, K)
    sizes[::17] = 0
    sizes[5] = 5000
    if K > 250:
        sizes[250] = 2100
    krs = np.r_[0, np.cumsum(sizes)].astype(np.int64)
    n = int(krs[-1])
    vals = np.array([-np.inf, -2.0, -0.0, 0.0, 0.5, 1.0, np.inf], np.float32)
    pred = rng.choice(vals, (S, n)).astype(np.float32)
    resp = rng.choice([1, 0, -1], n).astype(np.int32)
    w = rng.integers(0, 4, n).astype(np.float32)
    for k in (7, 8):
        resp[krs[k]:krs[k + 1]] = 1                      # positives only
    resp[krs[9]:krs[10]] = -1                            # negatives only
    w[krs[11]:krs[12]] = 0                               # no weight at all
    return resp, pred, w, krs


def test_bit_for_bit_on_integer_weights():
    import mlease_b200 as mb
    resp, pred, w, krs = _tie_case()
    got = mb.test_auc(resp, pred, w, krs)
    ref = test_auc_ref(resp, pred, w, krs)
    for g, r in zip(got, ref):
        assert _bits_equal(g, r)
    assert np.isnan(got[2][:, [7, 8, 9, 11]]).all() and not np.isnan(got[0]).any()
    # device inputs give the same bits; weight NULL means 1
    import torch
    dev = mb.test_auc(torch.from_numpy(resp).cuda(), torch.from_numpy(pred).cuda(), torch.from_numpy(w).cuda(), krs)
    for g, r in zip(dev, got):
        assert _bits_equal(g, r)
    one = mb.test_auc(resp, pred, None, krs)
    for g, r in zip(one, test_auc_ref(resp, pred, None, krs)):
        assert _bits_equal(g, r)


def _float_case(n, K, S, seed=1):
    rng = np.random.default_rng(seed)
    cuts = np.sort(rng.choice(np.arange(1, n), K - 1, replace=False))
    krs = np.r_[0, cuts, n].astype(np.int64)
    resp = np.where(rng.random(n) < 0.3, 1, rng.choice([0, -1], n)).astype(np.int32)
    pred = (rng.normal(size=(S, n)) + 0.8 * resp).astype(np.float32)
    w = rng.random(n).astype(np.float32) * 3
    return resp, pred, w, krs


def test_float_weights_within_the_fp64_bound_and_repeatable():
    import mlease_b200 as mb
    n = 10 ** 6
    resp, pred, w, krs = _float_case(n, 1000, 2)
    a = mb.test_auc(resp, pred, w, krs)
    b = mb.test_auc(resp, pred, w, krs)
    for x, y in zip(a, b):
        assert _bits_equal(x, y)
    ref = test_auc_ref(resp, pred, w, None)
    tol = 4 * n * 2.0 ** -53
    assert np.all(np.abs(a[0] - ref[0]) <= tol * np.abs(ref[0]))
    assert np.all(np.abs(a[1] - ref[1]) <= tol * np.abs(ref[1]))
    for k in range(0, 1000, 97):
        s, e = krs[k], krs[k + 1]
        rk = test_auc_ref(resp[s:e], pred[:, s:e], w[s:e])
        assert np.all(np.abs(a[2][:, k] - rk[0]) <= tol * np.abs(rk[0]))
        assert np.all(np.abs(a[3][k] - rk[1]) <= tol * np.abs(rk[1]))


@pytest.mark.parametrize("case", ["ties", "float"])
def test_each_key_and_each_set_alone_is_bitwise_the_full_call(case):
    import mlease_b200 as mb
    if case == "ties":
        resp, pred, w, krs = _tie_case(seed=2, S=3, K=60)
        w = w * np.float32(0.37)   # inexact sums: the association is what is compared
    else:
        resp, pred, w, krs = _float_case(300000, 40, 3, seed=3)
    auc, wt, kauc, kw = mb.test_auc(resp, pred, w, krs)
    for k in range(len(krs) - 1):
        s, e = krs[k], krs[k + 1]
        if e == s:
            continue
        a1, w1, ka1, kw1 = mb.test_auc(resp[s:e], pred[:, s:e], w[s:e], [0, e - s])
        assert _bits_equal(ka1[:, 0], kauc[:, k]) and _bits_equal(kw1[0], kw[k])
    for si in range(pred.shape[0]):
        a1, w1, ka1, kw1 = mb.test_auc(resp, pred[si], w, krs)
        assert _bits_equal(a1[0], auc[si]) and _bits_equal(ka1[0], kauc[si]) and _bits_equal(w1, wt) and _bits_equal(kw1, kw)


def test_sets_stream_in_chunks_bitwise(budget):
    import mlease_b200 as mb
    from mlease_b200 import _hooks
    resp, pred, w, krs = _float_case(200000, 300, 5, seed=4)
    full = mb.test_auc(resp, pred, w, krs)
    bounds, streamed, _, _ = _hooks.keyed_last_call()
    assert list(bounds) == [0, 5] and not streamed
    budget(1 << 20)
    with pytest.raises(mb.MleaseError, match=r"one set needs \d+ device bytes") as e:
        mb.test_auc(resp, pred, w, krs)
    need = int(re.search(r"one set needs (\d+) device bytes", str(e.value)).group(1))
    budget(need)
    got = mb.test_auc(resp, pred, w, krs)
    bounds, streamed, _, _ = _hooks.keyed_last_call()
    assert list(bounds) == [0, 1, 2, 3, 4, 5] and streamed
    for g, r in zip(got, full):
        assert _bits_equal(g, r)
    budget(need + 2 * (4 * 200000 + 8 * 301))   # room for two more sets: their predictions and results
    got = mb.test_auc(resp, pred, w, krs)
    assert list(_hooks.keyed_last_call()[0]) == [0, 3, 5]
    for g, r in zip(got, full):
        assert _bits_equal(g, r)
    budget(need - 1)
    with pytest.raises(mb.MleaseError, match="one set needs %d device bytes" % need):
        mb.test_auc(resp, pred, w, krs)


def test_refusals_then_a_valid_call():
    import mlease_b200 as mb
    from mlease_b200._native import lib, ptr
    resp, pred, w, krs = _tie_case(seed=5, S=2, K=40)
    ref = test_auc_ref(resp, pred, w, krs)
    n = len(resp)

    def valid():
        for g, r in zip(mb.test_auc(resp, pred, w, krs), ref):
            assert _bits_equal(g, r)

    bad_pred = pred.copy(); bad_pred[1, n // 2] = np.nan
    bad_resp = resp.copy(); bad_resp[3] = 2
    neg_w = w.copy(); neg_w[4] = -1
    nan_w = w.copy(); nan_w[n - 1] = np.nan
    dec = krs.copy(); dec[3] = dec[4] + 1
    cases = [
        (lambda: mb.test_auc(resp[:0], pred[:, :0], w[:0]), "nrows must be in"),
        (lambda: mb.test_auc(resp, pred[:0], w), "num_sets must be >= 1"),
        (lambda: mb.test_auc(resp, bad_pred, w, krs), "pred holds NaN"),
        (lambda: mb.test_auc(bad_resp, pred, w, krs), "response should be 1,0 or -1!"),
        (lambda: mb.test_auc(resp, pred, neg_w, krs), "weight must be >= 0 and not NaN"),
        (lambda: mb.test_auc(resp, pred, nan_w, krs), "weight must be >= 0 and not NaN"),
        (lambda: mb.test_auc(resp, pred, w, krs + 1), "key_rowstart must start at 0"),
        (lambda: mb.test_auc(resp, pred, w, dec), "key_rowstart decreases at key"),
        (lambda: mb.test_auc(resp, pred, w, np.r_[krs[:-1], n - 1]), "key_rowstart must end at nrows"),
    ]
    for call, msg in cases:
        with pytest.raises(mb.MleaseError, match=re.escape(msg)):
            call()
        valid()
    out_w = np.full(2, -7.0)
    rc = lib().mlease_test_auc(0, None, n, 2, ptr(pred), ptr(resp), ptr(w), len(krs) - 1, ptr(krs), None, ptr(out_w), None, None)
    assert rc != 0 and "both NULL" in lib().mlease_last_error().decode()
    assert (out_w == -7.0).all()   # nothing written
    valid()


# ---------------------------------------------------------------------------------------------------------------- the jobs
@pytest.fixture(scope="module")
def host():
    import mlease_b200
    mlease_b200.lib()
    h = C.CDLL(os.path.join(ROOT, "ml-ease_b200", "lib", "libmlease_host.so"))
    h.mlease_job_last_error.restype = C.c_char_p
    return h


def _ok(host, job, path, kv):
    with open(path, "w") as f:
        f.write("".join("%s=%s\n" % (k, v) for k, v in kv.items()))
    rc = host.mlease_job_run(job, str(path).encode())
    assert rc == 0, host.mlease_job_last_error().decode()


def _scored(path):
    """the scored records of the files directly under path (not those of its _loglik / _auc directories), in file order"""
    recs = []
    for f in sorted(os.listdir(path)):
        if f.endswith(".avro") and not f.startswith(("_", ".")):
            recs += au.read_avro(os.path.join(path, f))[1]
    return (np.array([r["response"] for r in recs], np.int32), np.array([r["pred"] for r in recs], np.float32),
            np.array([1.0 if r.get("weight") is None else r["weight"] for r in recs], np.float32), recs)


def test_regression_test_auc_job(host, tmp_path):
    npz = np.load(os.path.join(GOLDEN, "sample_data.npz"))
    recs = au.fixture_records(npz, with_key=lambda i: i // 250)
    au.write_avro(str(tmp_path / "in" / "part-0.avro"), au.pig_schema_with_key(), recs, codec="deflate", block=128)
    out = tmp_path / "out"
    _ok(host, b"Regression", tmp_path / "r.job", {"input.paths": tmp_path / "in", "output.base.path": out, "test.path": tmp_path / "in",
                                                  "map.key": "pkey", "num.blocks": 4, "num.iters": 10, "regularizer": 2, "lambda": "1,10"})
    _ok(host, b"RegressionTestAuc", tmp_path / "a.job", {"input.base.paths": out / "test", "output.base.path": tmp_path / "auc",
                                                         "lambda": "1,10"})
    for d in ("lambda-1", "lambda-10", "best-model"):
        if not os.path.exists(out / "test" / d):
            continue
        resp, pred, w, _ = _scored(out / "test" / d)
        ref = test_auc_ref(resp, pred, w)
        got = au.read_dir(str(tmp_path / "auc" / d / "_auc"))
        assert got == [{"key": "testAuc", "auc": ref[0][0], "positiveWeight": ref[1][0], "negativeWeight": ref[1][1]}]


def test_item_model_grid_test_auc_job(host, tmp_path):
    npz = np.load(os.path.join(GOLDEN, "sample_data.npz"))
    recs = au.fixture_records(npz, with_key=lambda i: (i * 7) % 9)
    au.write_avro(str(tmp_path / "in" / "part-0.avro"), au.pig_schema_with_key(), recs, codec="deflate", block=128)
    _ok(host, b"RegressionPrepare", tmp_path / "p.job", {"input.paths": tmp_path / "in", "output.path": tmp_path / "tmp-data",
                                                         "map.key": "pkey", "num.blocks": 2})
    il, dl = ["1", "30.0"], ["0.5", "2"]
    _ok(host, b"ItemModelTrain", tmp_path / "t.job", {"input.paths": tmp_path / "tmp-data", "output.model.path": tmp_path / "m",
                                                      "intercept.lambdas": ",".join(il), "default.lambdas": ",".join(dl)})
    test = recs[::-1][:700] + [dict(r, pkey=99) for r in recs[:31]] + recs[300:]
    au.write_avro(str(tmp_path / "test" / "a.avro"), au.pig_schema_with_key(), test[:500], block=100)
    au.write_avro(str(tmp_path / "test" / "b.avro"), au.pig_schema_with_key(), test[500:], block=300)
    grid = tmp_path / "grid"
    _ok(host, b"ItemModelGridTest", tmp_path / "g.job", {"input.paths": tmp_path / "test", "output.base.path": grid,
                                                         "model.path": tmp_path / "m" / "models", "item.key": "pkey",
                                                         "intercept.lambdas": ",".join(il), "default.lambdas": ",".join(dl)})
    _ok(host, b"ItemModelGridTestAuc", tmp_path / "a.job", {"input.base.path": grid, "output.base.path": tmp_path / "auc", "item.key": "pkey",
                                                            "intercept.lambdas": ",".join(il), "default.lambdas": ",".join(dl)})
    top = au.read_dir(str(tmp_path / "auc" / "_auc"))
    per = au.read_dir(str(tmp_path / "auc" / "_key_auc"))
    gkeys = ["%s:%s" % (repr(float(np.float32(a))), repr(float(np.float32(b)))) for a in il for b in dl]
    assert [r["key"] for r in top] == gkeys
    preds = []
    for a in il:
        for b in dl:
            resp, pred, w, rs = _scored(grid / ("lambda-%s_%s" % (a, b)))
            preds.append(pred)
    keys = [str(r["pkey"]) for r in rs]
    knames = sorted(set(keys))
    order = sorted(range(len(keys)), key=lambda i: keys[i])
    krs = np.searchsorted(np.array([keys[i] for i in order]), knames + [chr(0x10FFFF)], side="left")
    krs[-1] = len(keys)
    P = np.stack(preds)[:, order]
    auc, wt, kauc, kw = test_auc_ref(resp[order], P, w[order], krs)
    assert [r["key"] for r in per] == ["%s#%s" % (g, k) for g in gkeys for k in knames]
    for g, t in enumerate(top):
        assert _bits_equal(t["auc"], auc[g]) and t["positiveWeight"] == wt[0] and t["negativeWeight"] == wt[1]
        ok = ~np.isnan(kauc[g])
        W = kw[:, 0] + kw[:, 1]
        assert abs(t["keyAuc"] - (W[ok] * kauc[g][ok]).sum() / W[ok].sum()) <= 1e-12
        for k, r in enumerate(per[g * len(knames):(g + 1) * len(knames)]):
            assert _bits_equal(r["auc"], kauc[g, k]) and r["positiveWeight"] == kw[k, 0] and r["negativeWeight"] == kw[k, 1]
