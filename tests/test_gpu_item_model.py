"""GPU tests of keyed scoring (ItemModelTest) and keyed test log-likelihood (ItemModelTestLoglik): the kernels through the
Python binding, and both jobs end to end after RegressionPrepare -> RegressionNaiveTrain on the fixture."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from oracle import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import avro_util as au  # noqa: E402
import item_model_ref as ref  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _keyed_problem(rng, K, D, max_rows, density, L, entries_per_model):
    """K keys of 0..max_rows rows (some keys empty, ~5 % empty rows), unsorted columns with repeats; per lambda a model per key
    with a random feature subset, some without intercept, ~10 % of (lambda, key) without a model."""
    nrows_k = rng.integers(0, max_rows + 1, K)
    nrows_k[rng.random(K) < 0.05] = 0
    krs = np.concatenate([[0], np.cumsum(nrows_k)]).astype(np.int64)
    n = int(krs[-1])
    nnz_r = rng.poisson(density * D, n)
    nnz_r[rng.random(n) < 0.05] = 0
    rp = np.concatenate([[0], np.cumsum(nnz_r)]).astype(np.int64)
    ci = rng.integers(0, D, int(rp[-1])).astype(np.int32)
    v = rng.normal(size=int(rp[-1])).astype(np.float32)
    off = rng.normal(size=n).astype(np.float32)
    mp, mc, mv, dense = [0], [], [], []
    for _ in range(L):
        dl = []
        for _ in range(K):
            if rng.random() < 0.1:
                dl.append(None)
                mp.append(mp[-1])
                continue
            cols = np.sort(rng.choice(D, min(D, entries_per_model), replace=False))
            if rng.random() < 0.8:
                cols = np.append(cols, D)
            vals = (rng.normal(size=len(cols)) * 0.3).astype(np.float32)
            mc.append(cols.astype(np.int32)); mv.append(vals)
            mp.append(mp[-1] + len(cols))
            dl.append((cols, vals))
        dense.append(dl)
    mc = np.concatenate(mc) if mc else np.zeros(0, np.int32)
    mv = np.concatenate(mv) if mv else np.zeros(0, np.float32)
    return dict(krs=krs, rp=rp, ci=ci, v=v, off=off, mp=np.array(mp, np.int64), mc=mc, mv=mv, models=dense, D=D, K=K, L=L)


def _score(pb, binary=False, lambdas=None):
    import mlease_b200 as mb
    K, L = pb["K"], pb["L"]
    mp, mc, mv = pb["mp"], pb["mc"], pb["mv"]
    if lambdas is not None:   # the models of these lambdas only
        parts_c, parts_v, ptr = [], [], [0]
        for l in lambdas:
            a, b = mp[l * K], mp[(l + 1) * K]
            parts_c.append(mc[a:b]); parts_v.append(mv[a:b])
            ptr += list(ptr[-1] + mp[l * K + 1:(l + 1) * K + 1] - a)
        mp, mc, mv = np.array(ptr, np.int64), np.concatenate(parts_c), np.concatenate(parts_v)
    return mb.score_keyed(pb["v"], pb["krs"], pb["rp"], pb["ci"], pb["D"], mp, mc, mv, offset=pb["off"], binary_feature=binary)


def _dense_model(pb, l, k):
    m = np.zeros(pb["D"] + 1, np.float64)
    if pb["models"][l][k] is not None:
        cols, vals = pb["models"][l][k]
        m[cols] = vals.astype(np.float64)
    return m


@pytest.mark.parametrize("L", [1, 3, 5])
def test_score_keyed_numerics(L):
    import mlease_b200 as mb
    rng = np.random.default_rng(100 + L)
    pb = _keyed_problem(rng, K=3000, D=5000, max_rows=300, density=0.01, L=L, entries_per_model=120)
    krs, rp, D = pb["krs"], pb["rp"], pb["D"]
    for binary in (False, True):
        p = _score(pb, binary)
        assert p.shape == (L, krs[-1])
        # (a) repeatable
        assert np.array_equal(p.view(np.uint32), _score(pb, binary).view(np.uint32))
        # (c) each lambda equals a call with that lambda's models only
        for l in range(L):
            assert np.array_equal(p[l].view(np.uint32), _score(pb, binary, [l])[0].view(np.uint32)), l
        # (d) bitwise mlease_score on a key's rows with its model widened to double; (e) within one float ulp of the sequential
        # scoring (orc.score is LinearModel.evalInstanceAvro restated with absent features as 0); no model -> float(offset)
        sample = set(rng.choice(pb["K"], 150, replace=False).tolist())
        for l in range(L):
            for k in range(pb["K"]):
                a, b = int(krs[k]), int(krs[k + 1])
                if a == b:
                    continue
                sub_rp = rp[a:b + 1] - rp[a]
                sub = orc.Csr(sub_rp, pb["ci"][rp[a]:rp[b]], pb["v"][rp[a]:rp[b]], np.zeros(b - a, np.int32), offset=pb["off"][a:b], n_features=D)
                m = _dense_model(pb, l, k)
                if pb["models"][l][k] is None:
                    assert np.array_equal(p[l, a:b], pb["off"][a:b])
                o = orc.score(sub, m, binary_feature=binary)
                ulp = np.spacing(np.abs(o)).astype(np.float32)
                assert np.all(np.abs(p[l, a:b] - o) <= ulp), (l, k)
                if k in sample:
                    s = mb.score(sub.val, m, rowptr=sub_rp, colidx=sub.colidx, offset=sub.offset, num_features=D, binary_feature=binary)
                    assert np.array_equal(p[l, a:b].view(np.uint32), s.view(np.uint32)), (l, k)


def test_score_keyed_does_not_depend_on_the_table_chunks():
    """1200 keys x 60 001 features at three lambdas: 1.15 GB of coefficient table (four floats per feature and key), more than
    the 1 GiB chunk cap, so the keys are scored in two chunks; a single lambda needs 288 MB and one chunk."""
    rng = np.random.default_rng(7)
    pb = _keyed_problem(rng, K=1200, D=60001, max_rows=12, density=0.01, L=3, entries_per_model=400)
    p = _score(pb)
    for l in range(3):
        assert np.array_equal(p[l].view(np.uint32), _score(pb, lambdas=[l])[0].view(np.uint32)), l


def test_score_keyed_rejects_unsorted_models():
    import mlease_b200 as mb
    with pytest.raises(mb.MleaseError, match="strictly ascending"):
        mb.score_keyed(np.ones(2, np.float32), [0, 1], [0, 2], [0, 1], 3, [0, 2], np.array([1, 0], np.int32), np.ones(2, np.float32))


def test_test_loglik_keyed_matches_the_reference_restatement():
    import mlease_b200 as mb
    rng = np.random.default_rng(3)
    n, K = 200_000, 500
    groups = np.sort(rng.integers(0, 4, n)).astype(np.int32)
    key = rng.integers(0, K, n).astype(np.int32)
    resp = rng.choice([1, 0, -1], n).astype(np.int32)
    pred = (rng.normal(size=n) * 3).astype(np.float32)
    for weight in (None, rng.uniform(0.5, 2.0, n).astype(np.float32)):
        ll, cnt = mb.test_loglik_keyed(key, groups, resp, pred, K, weight=weight)
        ll2, cnt2 = mb.test_loglik_keyed(key, groups, resp, pred, K, weight=weight)
        assert np.array_equal(ll.view(np.uint32), ll2.view(np.uint32)) and np.array_equal(cnt, cnt2)
        want = ref.item_test_loglik(key.tolist(), groups, resp, pred, weight)
        for k in range(K):
            w_ll, w_cnt = want[k]
            assert abs(ll[k] - w_ll) <= 1e-6 * abs(w_ll), (k, ll[k], w_ll)
            if weight is None:
                assert cnt[k] == w_cnt
            else:
                assert abs(cnt[k] - w_cnt) <= 1e-12 * w_cnt
    with pytest.raises(mb.MleaseError, match="response should be 1,0 or -1!"):
        mb.test_loglik_keyed([0, 1], [0, 0], [1, 2], [0.1, 0.2], 2)


@pytest.fixture(scope="module")
def host():
    import mlease_b200
    mlease_b200.lib()
    h = C.CDLL(os.path.join(ROOT, "ml-ease_b200", "lib", "libmlease_host.so"))
    h.mlease_job_last_error.restype = C.c_char_p
    return h


def _cfg(path, **kv):
    with open(path, "w") as f:
        for k, v in kv.items():
            f.write("%s=%s\n" % (k.replace("_", "."), v))
    return path


def test_item_model_jobs_after_naive_train_on_fixture(host, tmp_path):
    npz = np.load(os.path.join(GOLDEN, "sample_data.npz"))
    recs = au.fixture_records(npz, with_key=lambda i: i // 400)
    au.write_avro(str(tmp_path / "in" / "part-0.avro"), au.pig_schema_with_key(), recs, codec="deflate", block=128)
    out = str(tmp_path / "nt")
    def run(job, cfg):
        assert host.mlease_job_run(job, cfg.encode()) == 0, host.mlease_job_last_error().decode()
    run(b"RegressionPrepare", _cfg(str(tmp_path / "p.job"), input_paths=str(tmp_path / "in"), output_path=out + "/tmp-data", map_key="pkey", num_blocks=2))
    cfg = _cfg(str(tmp_path / "n.job"), output_base_path=out, compute_model_mean="false", remove_tmp_dir="false")
    open(cfg, "a").write("lambda=1,10\n")
    run(b"RegressionNaiveTrain", cfg)
    # test records: the fixture in a scrambled key order, plus records of key 999, which has no model
    extra = [dict(r, pkey=999) for r in recs[:37]]
    test = recs[::-1][:1500] + extra + recs[1500:]
    au.write_avro(str(tmp_path / "test" / "a.avro"), au.pig_schema_with_key(), test[:1000], block=100)
    au.write_avro(str(tmp_path / "test" / "b.avro"), au.pig_schema_with_key(), test[1000:], codec="deflate", block=300)
    cfg = _cfg(str(tmp_path / "t.job"), input_paths=str(tmp_path / "test"), output_base_path=str(tmp_path / "it"), model_path=out + "/models", item_key="pkey")
    open(cfg, "a").write("lambda=1,10.0\n")
    run(b"ItemModelTest", cfg)
    models = {r["key"]: r["model"] for r in au.read_dir(out + "/models")}
    # expected: records grouped by key in string order, input order inside a key
    order = sorted(range(len(test)), key=lambda i: str(test[i]["pkey"]))
    names = sorted({f["name"] for r in test for f in r["features"]})
    fid = {nm: i for i, nm in enumerate(names)}
    D = len(names)
    rp = np.cumsum([0] + [len(test[i]["features"]) for i in order]).astype(np.int64)
    ci = np.array([fid[f["name"]] for i in order for f in test[i]["features"]], np.int32)
    v = np.array([f["value"] for i in order for f in test[i]["features"]], np.float32)
    off = np.array([test[i]["offset"] for i in order], np.float32)
    keys = [str(test[i]["pkey"]) for i in order]
    kn = sorted(set(keys))
    krs = [keys.index(k) for k in kn] + [len(keys)]
    preds = {}
    for lam, typed in (("1.0", "1"), ("10.0", "10.0")):
        ml = []
        for k in kn:
            m = models.get(lam + "#" + k)
            ml.append(None if m is None else {(D if f["name"] == "(INTERCEPT)" else fid[f["name"]]): np.float32(f["value"]) for f in m
                                              if f["name"] == "(INTERCEPT)" or f["name"] in fid})
        want = ref.score_keyed(krs, rp, ci, v, off, [ml], D)[0]
        sch, got, _ = au.read_avro(str(tmp_path / "it" / ("lambda-" + typed) / "part-r-00000.avro"))
        assert sch["name"] == "PerItemTestOutput" and sch["namespace"] == "com.linkedin.lab.regression.avro"
        assert [f["name"] for f in sch["fields"]] == [f["name"] for f in au.pig_schema_with_key()["fields"]] + ["pred"]
        assert [r["pkey"] for r in got] == [test[i]["pkey"] for i in order]
        p = np.array([r["pred"] for r in got], np.float32)
        assert np.all(np.abs(p - want) <= np.spacing(np.abs(want))), typed
        mask = np.array(keys) == "999"
        assert mask.sum() == 37 and np.array_equal(p[mask], off[mask])
        preds[typed] = p
    # ItemModelTestLoglik on pred maps built from those preds: two files = two combiner groups
    schema = {"type": "record", "name": "S", "fields": [{"name": "response", "type": "int"}, {"name": "weight", "type": ["null", "float"]},
                                                       {"name": "pred", "type": {"type": "map", "values": "float"}}]}
    resp = [1 if test[i]["response"] == 1 else 0 for i in order]
    rows = [{"response": resp[q], "weight": float(q % 3 + 1), "pred": {"k" + keys[q]: float(preds["1"][q]), "all": float(preds["10.0"][q])}}
            for q in range(len(order))]
    ref.write_avro_with_maps(str(tmp_path / "ll" / "a.avro"), schema, rows[:900])
    ref.write_avro_with_maps(str(tmp_path / "ll" / "b.avro"), schema, rows[900:])
    run(b"ItemModelTestLoglik", _cfg(str(tmp_path / "l.job"), input_paths=str(tmp_path / "ll"), output_path=str(tmp_path / "llout")))
    got = au.read_dir(str(tmp_path / "llout"))
    ek, eg, er, ep, ew = [], [], [], [], []
    for q, r in enumerate(rows):
        for k, pv in r["pred"].items():
            ek.append(k); eg.append(0 if q < 900 else 1); er.append(r["response"]); ep.append(pv); ew.append(r["weight"])
    want = ref.item_test_loglik(ek, eg, er, np.array(ep, np.float32), np.array(ew, np.float32))
    assert [r["key"] for r in got] == sorted(want, key=lambda s: s.encode())
    for r in got:
        w_ll, w_cnt = want[r["key"]]
        assert abs(r["testLoglik"] - w_ll) <= 1e-6 * abs(w_ll) and r["count"] == w_cnt, r
