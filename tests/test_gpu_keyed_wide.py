"""GPU tests of keyed CSR fits over wide dictionaries (mlease_naive_train, mlease_item_model_train): each key narrower than the
dictionary is solved in the columns its rows list.  Against the oracle fitted on each key's rows relabelled into the key's own compact
space (the reference's per-key dataset), bit for bit against the unchanged full-width path on those relabelled rows, independent of
the call a key shares (split calls, streamed ranges), mixed with full-width keys, the row checks before any fit, and the keyed jobs end
to end over a 100 000-name dictionary."""
import numpy as np
import pytest

from oracle import oracle as orc

pytestmark = pytest.mark.gpu


@pytest.fixture
def budget():
    from mlease_b200 import _hooks
    yield _hooks.set_keyed_budget
    _hooks.set_keyed_budget(0)


def _pools(rng, K, D, lo, hi, shared=0.3):
    """K column pools of lo..hi columns spread over [0, D): about `shared` of them overlap an earlier key's pool"""
    pools = []
    for k in range(K):
        size = int(rng.integers(lo, hi + 1))
        if k and rng.random() < shared:
            prev = pools[int(rng.integers(0, k))]
            take = rng.choice(prev, min(len(prev), size // 2), replace=False)
            rest = rng.choice(D, size - len(take), replace=False)
            pools.append(np.unique(np.concatenate([take, rest])))
        else:
            pools.append(np.unique(rng.choice(D, size, replace=False)))
    return pools


def _keyed(rng, rows, pools, D, per_row=12):
    """key k: rows[k] rows, each listing up to per_row sorted unique columns of pools[k]"""
    rp, ci, keys = [0], [], []
    for k, (n, pool) in enumerate(zip(rows, pools)):
        for _ in range(n):
            c = np.sort(rng.choice(pool, min(per_row, len(pool)), replace=False)) if len(pool) else np.zeros(0, np.int64)
            ci.append(c); rp.append(rp[-1] + len(c)); keys.append(k)
    ci = np.concatenate(ci).astype(np.int32) if ci else np.zeros(0, np.int32)
    n = len(keys)
    v = rng.normal(size=len(ci)).astype(np.float32)
    beta = rng.normal(size=D) * 0.4
    rp = np.array(rp, np.int64)
    z = np.array([float((v[rp[i]:rp[i + 1]] * beta[ci[rp[i]:rp[i + 1]]]).sum()) for i in range(n)])
    y = (rng.random(n) < 1 / (1 + np.exp(-(z - 0.3)))).astype(np.int32)
    krs = np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)
    return dict(krs=krs, rp=rp, ci=ci, v=v, y=y, w=rng.uniform(0.5, 2.0, n).astype(np.float32), o=rng.normal(0, 0.1, n).astype(np.float32),
                D=D, K=len(rows))


def _slice(pb, k0, k1):
    a, b = pb["krs"][k0], pb["krs"][k1]
    z0, z1 = pb["rp"][a], pb["rp"][b]
    return dict(krs=pb["krs"][k0:k1 + 1] - a, rp=pb["rp"][a:b + 1] - z0, ci=pb["ci"][z0:z1], v=pb["v"][z0:z1], y=pb["y"][a:b], w=pb["w"][a:b],
                o=pb["o"][a:b], D=pb["D"], K=k1 - k0)


def _compact(pb, k, vals=None):
    """key k's rows relabelled into its own space: (listed global columns, oracle Csr over them)"""
    a, b = pb["krs"][k], pb["krs"][k + 1]
    rp = pb["rp"][a:b + 1]
    ci = pb["ci"][rp[0]:rp[-1]]
    cols = np.unique(ci)
    v = (pb["v"] if vals is None else vals)[rp[0]:rp[-1]]
    return cols, orc.Csr(rp - rp[0], np.searchsorted(cols, ci).astype(np.int32), v, pb["y"][a:b], pb["w"][a:b], pb["o"][a:b], len(cols))


def _close(got, want):
    """the run-to-run spread of a CSR fit: the K1 gradient sums use float atomics"""
    assert np.abs(got - want).max() <= 1e-6 * max(1.0, np.abs(want).max())


def _naive(pb, lams, budget=None, nbytes=0, **kw):
    import mlease_b200 as mb
    if budget is not None:
        budget(nbytes)
    return mb.naive_train(pb["v"], pb["krs"], pb["y"], list(lams), rowptr=pb["rp"], colidx=pb["ci"], num_features=pb["D"], weight=pb["w"],
                          offset=pb["o"], **kw)


@pytest.mark.parametrize("has_intercept,binary", [(True, False), (False, True)])
def test_naive_train_wide_matches_the_per_key_oracle(has_intercept, binary):
    rng = np.random.default_rng(901)
    K, D = 24, 120000
    pools = _pools(rng, K, D, 8, 400)
    rows = rng.integers(1, 600, K); rows[[4, 15]] = [3, 7]          # below data.size.threshold = 10
    pb = _keyed(rng, rows, pools, D)
    lm = np.zeros(D, np.float32)
    hit = np.concatenate([pools[0][:3], pools[9][:2]])
    lm[hit] = rng.uniform(0.1, 8.0, len(hit)).astype(np.float32)
    lams, pmean = (0.7, 6.0), 0.15
    models, skipped = _naive(pb, lams, lambda_map=lm, prior_mean=pmean, has_intercept=has_intercept, binary_feature=binary,
                             data_size_threshold=10)
    assert models.shape == (2, K, D + 1)
    assert list(np.nonzero(skipped)[0]) == [4, 15]
    assert np.all(models[:, [4, 15]] == 0)
    vals = np.ones_like(pb["v"]) if binary else None
    for k in range(K):
        if skipped[k]:
            continue
        cols, data = _compact(pb, k, vals)
        listed = np.zeros(D + 1, bool); listed[cols] = True; listed[D] = has_intercept
        for li, lam in enumerate(lams):
            q = np.where(lm[cols] > 0, lm[cols], np.float32(lam)).astype(np.float64)
            pm = np.full(len(cols), pmean)
            if has_intercept:
                q = np.append(q, 1.0 / 100000.0); pm = np.append(pm, pmean)
            want, _ = orc.liblinear_train(data, np.zeros(len(q)), pm, 1.0 / q, 1e-14, 100000, has_bias=has_intercept)
            got = models[li, k]
            assert np.all(got[~listed] == 0.0), (k, li)
            g = np.append(got[cols], got[D]) if has_intercept else got[cols]
            assert np.abs(g - want).max() <= 1e-5 * np.abs(want).max(), (k, li)


def test_item_model_train_wide_matches_the_oracle_and_hessian_diag():
    import mlease_b200 as mb
    rng = np.random.default_rng(902)
    K, D = 16, 80000
    pools = _pools(rng, K, D, 8, 300)
    pb = _keyed(rng, rng.integers(1, 500, K), pools, D, per_row=10)
    means = rng.normal(0, 1, K)
    lm = np.zeros(D, np.float32); lm[pools[2][:4]] = [0.05, 8.0, 3.0, 0.5]
    il, dl = [0.5, 20.0], [1.0, 0.25]
    models, var = mb.item_model_train(pb["v"], pb["krs"], pb["y"], il, dl, rowptr=pb["rp"], colidx=pb["ci"], num_features=D,
                                      intercept_prior_mean=means, weight=pb["w"], offset=pb["o"], lambda_map=lm, compute_var=True)
    for k in range(K):
        cols, data = _compact(pb, k)
        listed = np.zeros(D + 1, bool); listed[cols] = True; listed[D] = True
        for a, ia in enumerate(il):
            for b, db in enumerate(dl):
                qg = np.where(lm > 0, lm, np.float32(db)).astype(np.float64)
                pv = np.append(1.0 / qg[cols], 1.0 / np.float64(np.float32(ia)))
                pm = np.zeros(len(cols) + 1); pm[-1] = means[k]
                want, _ = orc.liblinear_train(data, np.zeros(len(pv)), pm, pv, 1e-14, 100000)
                got = models[a, b, k]
                g = np.append(got[cols], got[D])
                assert np.abs(g - want).max() <= 1e-5 * np.abs(want).max(), (k, a, b)
                assert np.all(got[~listed] == 0.0)
                hd = orc.objective("hessian_diag", data, g, pm, pv)
                vg = np.append(var[a, b, k][cols], var[a, b, k][D])
                assert np.abs(vg - 1.0 / hd).max() <= 1e-10 * np.abs(1.0 / hd).max(), (k, a, b)
                qfull = np.append(1.0 / (1.0 / qg), 1.0)
                assert np.array_equal(var[a, b, k][~listed], (1.0 / qfull)[~listed])


def test_one_row_keys_are_bitwise_the_compact_full_width_call():
    """Dk + 1 a multiple of 32: a key's own space is exactly the full-width problem of its relabelled rows (Dk = 2111: ldh > 2048,
    the wide Cholesky).  65 keys of each Dk: the compact call's full-width batch is then above the 64 problems that pipeline their
    Newton slots, like every batch of keys in their own spaces."""
    import mlease_b200 as mb
    rng = np.random.default_rng(903)
    D, R = 160000, 65
    dks = [31, 63, 95, 2111]
    cols = rng.choice(D, R * sum(dks), replace=False)   # disjoint pools: each key's local lambda_map is exactly clm
    cuts = np.cumsum([0] + [dk for dk in dks for _ in range(R)])
    pools = [np.sort(cols[a:b]) for a, b in zip(cuts[:-1], cuts[1:])]
    pb = _keyed(rng, np.ones(len(pools), np.int64), pools, D, per_row=3000)
    lmv = rng.uniform(0.2, 4.0, 5).astype(np.float32)   # the 3rd..7th listed column of every key: the same local lambda_map
    lm = np.zeros(D, np.float32)
    for p in pools:
        lm[p[2:7]] = lmv
    lams = (0.5, 3.0)
    wide, _ = _naive(pb, lams, lambda_map=lm, prior_mean=0.1)
    means = rng.normal(size=len(pools))
    wm, wv = mb.item_model_train(pb["v"], pb["krs"], pb["y"], [2.0], [0.8], rowptr=pb["rp"], colidx=pb["ci"], num_features=D,
                                 intercept_prior_mean=means, weight=pb["w"], offset=pb["o"], lambda_map=lm, compute_var=True)
    for g, dk in enumerate(dks):
        ks = list(range(R * g, R * g + R))
        comp = _slice(pb, ks[0], ks[-1] + 1)
        comp["ci"] = comp["ci"].copy()
        for i, k in enumerate(ks):
            a, b = comp["rp"][i], comp["rp"][i + 1]
            comp["ci"][a:b] = np.searchsorted(pools[k], comp["ci"][a:b])
        comp["D"] = dk
        clm = np.zeros(dk, np.float32); clm[2:7] = lmv
        want, _ = _naive(comp, lams, lambda_map=clm, prior_mean=0.1)
        cm, cv = mb.item_model_train(comp["v"], comp["krs"], comp["y"], [2.0], [0.8], rowptr=comp["rp"], colidx=comp["ci"], num_features=dk,
                                     intercept_prior_mean=means[ks], weight=comp["w"], offset=comp["o"], lambda_map=clm, compute_var=True)
        for i, k in enumerate(ks):
            sel = np.append(pools[k], D)
            assert np.array_equal(wide[:, k][:, sel].view(np.uint64), want[:, i].view(np.uint64)), (dk, k)
            assert np.array_equal(wm[0, 0, k][sel].view(np.uint64), cm[0, 0, i].view(np.uint64)), (dk, k)
            assert np.array_equal(wv[0, 0, k][sel].view(np.uint64), cv[0, 0, i].view(np.uint64)), (dk, k)


def test_multi_row_keys_match_the_compact_call_within_the_spread():
    rng = np.random.default_rng(904)
    D = 60000
    pools = _pools(rng, 10, D, 20, 200, shared=0.0)
    pb = _keyed(rng, rng.integers(50, 400, 10), pools, D)
    wide, _ = _naive(pb, (1.0,))
    for k in range(10):
        one = _slice(pb, k, k + 1)
        cols = np.unique(one["ci"])
        comp = dict(one, ci=np.searchsorted(cols, one["ci"]).astype(np.int32), D=len(cols))
        want, _ = _naive(comp, (1.0,))
        _close(np.append(wide[0, k][cols], wide[0, k][D]), want[0, 0])


def test_a_keys_fit_does_not_depend_on_its_call(budget):
    """one call, split across two calls, streamed through at least 4 ranges: one-row keys (every gradient sum one addition) bit for
    bit in all three; multi-row keys within the spread of the float-atomic gradient sums"""
    from mlease_b200 import _hooks
    rng = np.random.default_rng(905)
    D = 150000
    for rows in (np.ones(48, np.int64), rng.integers(20, 300, 20)):
        K = len(rows)
        pb = _keyed(rng, rows, _pools(rng, K, D, 8, 200), D, per_row=200 if rows.max() == 1 else 12)
        lams = (0.5, 2.0)
        one, _ = _naive(pb, lams, budget, 0)
        assert not _hooks.keyed_last_call()[1]
        h0, _ = _naive(_slice(pb, 0, K // 3), lams, budget, 0)
        h1, _ = _naive(_slice(pb, K // 3, K), lams, budget, 0)
        split = np.concatenate([h0, h1], axis=1)
        streamed, _ = _naive(pb, lams, budget, 64 << 10)
        bounds, st, _, _ = _hooks.keyed_last_call()
        assert st and len(bounds) - 1 >= 4, bounds
        for got in (split, streamed):
            if rows.max() == 1:
                assert np.array_equal(got.view(np.uint64), one.view(np.uint64))
            else:
                _close(got, one)


def test_mixed_call_full_width_keys_are_their_own_call():
    rng = np.random.default_rng(906)
    D = 300
    full = [np.sort(rng.choice(D, int(rng.integers(292, 300)), replace=False)) for _ in range(6)]
    narrow = [np.sort(rng.choice(D, 20, replace=False)) for _ in range(8)]
    order = [("f", 0), ("n", 0), ("n", 1), ("f", 1), ("f", 2), ("n", 2), ("n", 3), ("n", 4), ("f", 3), ("n", 5), ("f", 4), ("n", 6), ("n", 7),
             ("f", 5)]
    pools = [full[i] if t == "f" else narrow[i] for t, i in order]
    rows = np.array([1 if t == "f" else int(rng.integers(40, 200)) for t, _ in order])
    pb = _keyed(rng, rows, pools, D, per_row=300)
    lams = (0.5, 4.0)
    models, _ = _naive(pb, lams)
    fk = [k for k, (t, _) in enumerate(order) if t == "f"]
    parts = [_slice(pb, k, k + 1) for k in fk]
    only = dict(krs=np.concatenate([[0], np.cumsum([p["krs"][-1] for p in parts])]).astype(np.int64),
                rp=np.concatenate([[0], np.cumsum([p["rp"][-1] for p in parts])]).astype(np.int64),
                ci=np.concatenate([p["ci"] for p in parts]), v=np.concatenate([p["v"] for p in parts]),
                y=np.concatenate([p["y"] for p in parts]), w=np.concatenate([p["w"] for p in parts]), o=np.concatenate([p["o"] for p in parts]),
                D=D, K=len(fk))
    want, _ = _naive(only, lams)
    assert np.array_equal(models[:, fk].view(np.uint64), want.view(np.uint64))
    for k, (t, _) in enumerate(order):
        if t != "n":
            continue
        cols, data = _compact(pb, k)
        for li, lam in enumerate(lams):
            q = np.append(np.full(len(cols), np.float64(np.float32(lam))), 1.0 / 100000.0)
            want, _ = orc.liblinear_train(data, np.zeros(len(q)), np.zeros(len(q)), 1.0 / q, 1e-14, 100000)
            g = np.append(models[li, k][cols], models[li, k][D])
            assert np.abs(g - want).max() <= 1e-5 * np.abs(want).max(), (k, li)


@pytest.mark.parametrize("nbytes", [0, 1 << 20])
def test_bad_column_in_a_late_key_fails_before_any_fit(budget, nbytes):
    import mlease_b200 as mb
    from mlease_b200 import _hooks
    rng = np.random.default_rng(907)
    D, K = 90000, 30
    pb = _keyed(rng, rng.integers(20, 120, K), _pools(rng, K, D, 8, 100), D)
    pb["ci"] = pb["ci"].copy()
    j = pb["rp"][pb["krs"][27]] + 1
    good = pb["ci"][j]
    pb["ci"][j] = D
    with pytest.raises(mb.MleaseError, match="feature index out of range") as e:
        _naive(pb, (1.0,), budget, nbytes)
    assert e.value.code == 1
    with pytest.raises(mb.MleaseError, match="feature index out of range"):
        mb.item_model_train(pb["v"], pb["krs"], pb["y"], [1.0], [1.0], rowptr=pb["rp"], colidx=pb["ci"], num_features=D)
    pb["ci"][j] = good
    m, _ = _naive(pb, (1.0,), budget, nbytes)   # the process goes on
    assert _hooks.keyed_last_call()[1] == (nbytes > 0)
    assert np.all(np.isfinite(m))


def test_jobs_over_a_wide_dictionary_end_to_end(tmp_path):
    """RegressionPrepare, NaiveTrain and ItemModelTrain (compute.var) on avro records over a 100 000-name dictionary, each key drawing
    from its own pool of 400 names: every key's model lists exactly its features; values against the oracle and the restatement"""
    import ctypes as C
    import os
    import sys

    import mlease_b200
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import avro_util as au
    import item_model_train_ref as ref
    mlease_b200.lib()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    host = C.CDLL(os.path.join(root, "ml-ease_b200", "lib", "libmlease_host.so"))
    host.mlease_job_last_error.restype = C.c_char_p

    def job(name, **kv):
        cfg = tmp_path / (name + ".job")
        cfg.write_text("".join("%s=%s\n" % (k, v) for k, v in kv.items()))
        assert host.mlease_job_run(name.encode(), str(cfg).encode()) == 0, (name, host.mlease_job_last_error().decode())

    rng = np.random.default_rng(908)
    K, P, E, D = 250, 400, 20, 100000
    names = ["f%06d" % i for i in range(D)]
    perm = rng.permutation(D)
    recs, rp, ci, vals, resp = [], [0], [], [], []
    rows = rng.integers(20, 41, K)
    krs = np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)
    for k in range(K):
        pool = perm[k * P:(k + 1) * P]
        for r in range(rows[k]):
            c = np.sort(pool[r * E:(r + 1) * E] if r * E < P else rng.choice(pool, E, replace=False))   # the first rows cover the pool
            v = rng.normal(size=E).astype(np.float32)
            y = int(rng.random() < 1 / (1 + np.exp(-0.5 * float(v[:5].sum()))))
            recs.append({"features": [{"name": names[j], "term": "", "value": float(x)} for j, x in zip(c, v)], "offset": 0, "response": y,
                         "weight": 1, "pkey": k})
            ci += list(c); vals += list(v); resp.append(y); rp.append(len(ci))
    au.write_avro(str(tmp_path / "in" / "p.avro"), au.pig_schema_with_key(), recs, block=500)
    prep = tmp_path / "prep"
    job("RegressionPrepare", **{"input.paths": tmp_path / "in", "output.path": prep, "map.key": "pkey", "num.blocks": 2})
    job("NaiveTrain", **{"input.paths": prep, "output.base.path": tmp_path / "naive", "lambda": "1,10", "compute.model.mean": "false",
                         "remove.tmp.dir": "false"})
    job("ItemModelTrain", **{"input.paths": prep, "output.model.path": tmp_path / "imt", "intercept.lambdas": "0.5", "default.lambdas": "2",
                             "compute.var": "true"})
    data = orc.Csr(np.array(rp, np.int64), np.array(ci, np.int32), np.array(vals, np.float32), np.array(resp, np.int32), n_features=D)
    models = {r["key"]: r["model"] for r in au.read_dir(str(tmp_path / "naive" / "models"))}
    assert len(models) == 2 * K
    for lam, key in ((1.0, "1.0"), (10.0, "10.0")):
        want, _, _ = orc.naive_train(data, krs, lam, mode="exact", nthreads=8)
        for k in range(K):
            m = models["%s#%d" % (key, k)]
            pool = {names[j] for j in perm[k * P:(k + 1) * P]}
            assert {f["name"] for f in m} == pool | {"(INTERCEPT)"} and len(m) == P + 1, (key, k)
            idx = np.array([D if f["name"] == "(INTERCEPT)" else int(f["name"][1:]) for f in m])
            got = np.array([f["value"] for f in m], np.float64)
            w = want[k][idx]
            assert np.abs(got - w).max() <= 1e-5 * np.abs(w).max(), (key, k)
    got = au.read_dir(str(tmp_path / "imt" / "models"))
    want = ref.item_model_train(au.read_dir(str(prep)), [0.5], [2.0], compute_var=True)
    assert [r["key"] for r in got] == [r["key"] for r in want]
    for g, w in zip(got, want):
        assert len(g["model"]) == P + 1
        for field in ("model", "posteriorVar"):
            assert [(f["name"], f["term"]) for f in g[field]] == [(f["name"], f["term"]) for f in w[field]], (g["key"], field)
            a = np.array([f["value"] for f in g[field]], np.float64)
            b = np.array([f["value"] for f in w[field]], np.float64)
            assert np.abs(a - b).max() <= 1e-5 * np.abs(b).max(), (g["key"], field)
