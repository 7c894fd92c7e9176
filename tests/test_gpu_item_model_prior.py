"""GPU tests of ItemModelTrain under per-key priors (mlease_item_model_train_prior): empty lists are the sparse call, priors that
cannot change the fit leave it as it is, random priors on listed, prior-only and intercept columns against the fp64 replica
(item_model_prior_ref.py), streamed against resident, the refusals, and the job end to end refreshing an earlier run, on one and two
devices."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from oracle import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import avro_util as au  # noqa: E402
import item_model_prior_ref as pref  # noqa: E402
import item_model_train_ref as ref  # noqa: E402
from test_gpu_keyed_sparse import SHAPES, _bitwise, _key_cols, _keyed, _same, _shape  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def budget():
    from mlease_b200 import _hooks
    yield _hooks.set_keyed_budget
    _hooks.set_keyed_budget(0)


def _args(pb):
    return dict(rowptr=pb["rp"], colidx=pb["ci"], num_features=pb["D"], weight=pb["w"], offset=pb["o"])


def _empty(K):
    return np.zeros(K + 1, np.int64), np.zeros(0, np.int32), np.zeros(0), np.zeros(0)


def _prior_call(pb, il, dl, prior, **kw):
    import mlease_b200 as mb
    pp, pc, pm, pv = prior
    return mb.item_model_train_prior(pb["v"], pb["krs"], pb["y"], il, dl, prior_ptr=pp, prior_col=pc, prior_mean=pm, prior_var=pv,
                                     **_args(pb), **kw)


def _lists(entries, K):
    """[(key, col, mean, var)] -> prior lists, each key's entries sorted by column"""
    entries = sorted(entries)
    pp = np.zeros(K + 1, np.int64)
    for k, *_ in entries:
        pp[k + 1] += 1
    return (np.cumsum(pp), np.array([e[1] for e in entries], np.int32), np.array([e[2] for e in entries], np.float64),
            np.array([e[3] for e in entries], np.float64))


def _random_prior(rng, pb, rows):
    """per key: about half its listed columns, a quarter as many prior-only columns, the intercept for most keys; a third of the
    variances 0; the key without rows gets a list too (it is not fitted)"""
    D, ent = pb["D"], []
    for k in range(pb["K"]):
        listed = _key_cols(pb, k) if rows[k] else np.zeros(0, np.int64)
        take = listed[rng.random(len(listed)) < 0.5]
        other = np.setdiff1d(rng.choice(D, max(2, len(listed) // 4), replace=False), listed)
        cols = np.union1d(take, other).tolist() + ([D] if rng.random() < 0.7 else [])
        for c in cols:
            ent.append((k, int(c), float(rng.normal(0, 0.6)), 0.0 if rng.random() < 0.33 else float(rng.uniform(0.05, 3.0))))
    return _lists(ent, pb["K"])


@pytest.mark.parametrize("shape", SHAPES)
def test_empty_lists_are_the_sparse_call(shape):
    """Keys at the global width (with and without a column list), keys in their own column space, and a key without rows."""
    import mlease_b200 as mb
    rng = np.random.default_rng(2100 + SHAPES.index(shape))
    pb, rows = _shape(shape, rng)
    lm = np.zeros(pb["D"], np.float32)
    lm[rng.choice(pb["D"], 6, replace=False)] = rng.uniform(0.2, 5.0, 6).astype(np.float32)
    means = rng.normal(0, 0.5, pb["K"])
    kw = dict(intercept_prior_mean=means, lambda_map=lm, compute_var=True)
    want = mb.item_model_train_sparse(pb["v"], pb["krs"], pb["y"], [0.5, 4.0], [1.0], **_args(pb), **kw)
    got = _prior_call(pb, [0.5, 4.0], [1.0], _empty(pb["K"]), **kw)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    assert got[0][6] == got[0][5]                      # key 5 has no rows: an empty list
    for k in range(pb["K"]):
        a, b = want[0][k], want[0][k + 1]
        for i in (2, 3):
            _same(got[i][:, :, a:b], want[i][:, :, a:b], _bitwise(pb, rows, k))


@pytest.mark.parametrize("shape", ["d20", "d120k_local", "mixed"])
def test_priors_that_cannot_change_the_fit(shape):
    """An intercept-only list with variance 0 is the intercept_prior_mean path; a list of prior-only columns leaves the fitted
    values as they are and adds its columns at exactly their prior mean and variance (1/q where the variance is 0)."""
    import mlease_b200 as mb
    rng = np.random.default_rng(2200 + SHAPES.index(shape))
    pb, rows = _shape(shape, rng)
    D, K = pb["D"], pb["K"]
    lm = np.zeros(D, np.float32)
    lm[rng.choice(D, 6, replace=False)] = rng.uniform(0.2, 5.0, 6).astype(np.float32)
    means = rng.normal(0, 0.5, K)
    il, dl = [0.5], [1.0, 3.0]
    want = mb.item_model_train_sparse(pb["v"], pb["krs"], pb["y"], il, dl, **_args(pb), intercept_prior_mean=means, lambda_map=lm,
                                      compute_var=True)
    got = _prior_call(pb, il, dl, _lists([(k, D, means[k], 0.0) for k in range(K)], K), lambda_map=lm, compute_var=True)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    for k in range(K):
        a, b = want[0][k], want[0][k + 1]
        for i in (2, 3):
            _same(got[i][:, :, a:b], want[i][:, :, a:b], _bitwise(pb, rows, k))
    # prior-only columns
    ent = []
    for k in range(K):
        for c in np.setdiff1d(rng.choice(D, 5, replace=False), _key_cols(pb, k)):
            ent.append((k, int(c), float(rng.normal()), 0.0 if c % 2 else float(rng.uniform(0.1, 2.0))))
    prior = _lists(ent, K)
    got = _prior_call(pb, il, dl, prior, intercept_prior_mean=means, lambda_map=lm, compute_var=True)
    for k in range(K):
        a, b = want[0][k], want[0][k + 1]
        c = got[1][got[0][k]:got[0][k + 1]]
        if rows[k] == 0:
            assert len(c) == 0
            continue
        e = np.arange(prior[0][k], prior[0][k + 1])
        assert np.array_equal(c, np.concatenate([np.union1d(want[1][a:b - 1], prior[1][e]), [D]]))
        keep = np.isin(c, want[1][a:b])
        po = ~keep
        at = np.searchsorted(prior[1][e], c[po])
        for i in (2, 3):
            _same(got[i][:, :, got[0][k]:got[0][k + 1]][:, :, keep], want[i][:, :, a:b], _bitwise(pb, rows, k))
        assert np.all(got[2][:, :, got[0][k]:got[0][k + 1]][:, :, po] == prior[2][e][at])
        for ib, lam in enumerate(dl):
            usual = [pref.usual_var(lm[j]) if lm[j] > 0 else pref.usual_var(lam) for j in c[po]]
            pv = np.where(prior[3][e][at] > 0, prior[3][e][at], usual)
            assert np.all(got[3][0, ib, got[0][k]:got[0][k + 1]][po] == pv)


# binary_feature on the mixed shape is left out: its one-row global-width keys list their whole pool as one all-ones row, perfectly
# collinear features whose fits may stop at the noise floor of the float-atomic objective sums (test_gpu_keyed_sparse.py's _shape)
@pytest.mark.parametrize("shape,binary", [("d20", False), ("d20", True), ("mixed", False)])
def test_random_priors_match_the_replica(shape, binary):
    rng = np.random.default_rng(2300 + 2 * SHAPES.index(shape) + binary)
    pb, rows = _shape(shape, rng)
    D, K = pb["D"], pb["K"]
    lm = np.zeros(D, np.float32)
    lm[rng.choice(D, 8, replace=False)] = rng.uniform(0.2, 5.0, 8).astype(np.float32)
    means = rng.normal(0, 0.5, K)
    il, dl = [0.5, 10.0], [0.3, 1.0, 4.0]
    prior = _random_prior(rng, pb, rows)
    key_ptr, cols, models, var = _prior_call(pb, il, dl, prior, intercept_prior_mean=means, lambda_map=lm, binary_feature=binary,
                                             compute_var=True)
    want = pref.key_fits(pb, il, dl, lm, prior, means, binary)
    for k in range(K):
        a, b = key_ptr[k], key_ptr[k + 1]
        if want[k] is None:
            assert a == b
            continue
        w = want[k]
        assert np.array_equal(cols[a:b], w["cols"]), k
        L, P = w["listed"], ~w["listed"]
        for ia in range(len(il)):
            for ib in range(len(dl)):
                g, wm = models[ia, ib, a:b], w["model"][ia, ib]
                assert np.abs(g[L] - wm[L]).max() <= 1e-5 * max(np.abs(wm[L]).max(), 1e-30), (k, ia, ib)
                assert np.array_equal(g[P], wm[P]) and np.array_equal(var[ia, ib, a:b][P], w["povar"][ia, ib][P]), (k, ia, ib)
                full = np.zeros(D + 1)
                full[w["cols"][L]] = g[L]
                hd = orc.objective("hessian_diag", w["data"], full, w["pm"][ia, ib], w["pv"][ia, ib])[w["cols"][L]]
                assert np.abs(var[ia, ib, a:b][L] - 1.0 / hd).max() <= 1e-10 * np.abs(1.0 / hd).max(), (k, ia, ib)


def test_streamed_ranges_carry_their_prior_slices(budget):
    from mlease_b200 import _hooks
    rng = np.random.default_rng(2400)
    D, K = 5000, 6000
    rows = np.ones(K, np.int64)
    rows[rng.choice(K, 30, replace=False)] = rng.integers(20, 120, 30)
    rows[rng.choice(K, 20, replace=False)] = 0
    pools = [np.sort(rng.choice(D, 24, replace=False)) for _ in range(K)]
    pb = _keyed(rng, rows, pools, D, per_row=10)
    prior = _random_prior(rng, pb, rows)
    budget(0)
    res = _prior_call(pb, [2.0], [0.5, 1.5], prior, compute_var=True)
    assert not _hooks.keyed_last_call()[1]
    budget(4 << 20)
    st = _prior_call(pb, [2.0], [0.5, 1.5], prior, compute_var=True)
    bounds, streamed, _, _ = _hooks.keyed_last_call()
    assert streamed and len(bounds) - 1 >= 2, bounds
    assert np.array_equal(st[0], res[0]) and np.array_equal(st[1], res[1])
    for k in range(K):
        a, b = res[0][k], res[0][k + 1]
        for i in (2, 3):
            _same(st[i][:, :, a:b], res[i][:, :, a:b], rows[k] == 1)


def test_refusals_name_the_key_and_leave_the_library_working():
    import mlease_b200 as mb
    rng = np.random.default_rng(2500)
    pb, rows = _shape("d20", rng)
    D, K = pb["D"], pb["K"]
    good = _lists([(3, 2, 0.5, 1.0), (3, D, 0.1, 0.0), (7, 4, -0.2, 0.0)], K)
    cases = []
    pp = good[0].copy(); pp[5] = pp[6] + 1
    cases.append(((pp,) + good[1:], "prior_ptr must never decrease (key 5)"))
    pp = good[0] + 1
    cases.append(((pp,) + good[1:], "prior_ptr[0] must be 0 (key 0)"))
    c = good[1].copy(); c[2] = D + 1
    cases.append(((good[0], c) + good[2:], "key 7: a prior column outside [0, num_features]"))
    c = good[1].copy(); c[1] = 2
    cases.append(((good[0], c) + good[2:], "key 3: prior columns that are not strictly ascending"))
    m = good[2].copy(); m[2] = np.inf
    cases.append((good[:2] + (m, good[3]), "key 7: a prior mean that is not finite"))
    for bad in (-1.0, np.nan, np.inf):
        v = good[3].copy(); v[0] = bad
        cases.append((good[:3] + (v,), "key 3: a prior variance that is negative or not finite"))
    for prior, msg in cases:
        with pytest.raises(mb.MleaseError) as e:
            _prior_call(pb, [1.0], [1.0], prior)
        assert msg in str(e.value), (msg, str(e.value))
    with pytest.raises(mb.MleaseError, match=r"the sum over fitted keys of min\(stored entries \+ non-intercept prior entries"):
        _prior_call(pb, [1.0], [1.0], good, capacity=3)
    key_ptr, cols, models, _ = _prior_call(pb, [1.0], [1.0], good)
    assert D in cols and key_ptr[-1] == len(cols)


# ------------------------------------------------------------------------------------------ the job


@pytest.fixture(scope="module")
def host():
    from mlease_b200 import build as _b
    _b.build()
    h = C.CDLL(os.path.join(ROOT, "ml-ease_b200", "lib", "libmlease_host.so"))
    h.mlease_job_last_error.restype = C.c_char_p
    return h


def _records(rng, n, keys, feats, shift=0.0):
    out = []
    for i in range(n):
        k = keys[int(rng.integers(0, len(keys)))]
        names = rng.choice(feats, int(rng.integers(2, 6)), replace=False)
        z = sum(0.3 * (ord(nm[1]) % 5 - 2) for nm in names) + shift
        out.append({"key": k, "response": int(rng.random() < 1 / (1 + np.exp(-z))),
                    "features": [{"name": str(nm), "term": "t" if nm.endswith("x") else "", "value": float(rng.normal())} for nm in names],
                    "weight": float(rng.uniform(0.5, 2.0)), "offset": float(rng.normal(0, 0.1))})
    return out


def _fkey(f):
    return f["name"] if not f["term"] else f["name"] + "\x01" + f["term"]


def _job_replica(prepared, prior_recs, gp, il, dl, lm_entries):
    """ItemModelTrain with prior.model.path restated: the dictionary (today's features in order of appearance, then the prior's new
    ones by item in byte order and model order), each key's prior lists, the replica's fits and the records' lists"""
    ids = {}
    for r in prepared:
        for f in r["features"]:
            ids.setdefault(_fkey(f), len(ids))
    pri = {}
    for r in prior_recs:
        g, _, item = r["key"].partition("#")
        if g == gp:
            pri[item] = r
    for item in sorted(pri, key=lambda s: s.encode()):
        for f in pri[item]["model"]:
            if _fkey(f) != ref.INTERCEPT:
                ids.setdefault(_fkey(f), len(ids))
    names, D = list(ids), len(ids)
    keys = sorted({r["key"] for r in prepared}, key=lambda s: s.encode())
    rp, ci, v, y, w, o, krs, ent = [0], [], [], [], [], [], [0], []
    for k, key in enumerate(keys):
        for r in prepared:
            if r["key"] == key:
                e = sorted((ids[_fkey(f)], f["value"]) for f in r["features"])
                ci += [c for c, _ in e]; v += [x for _, x in e]; rp.append(len(ci))
                y.append(r["response"]); w.append(r["weight"]); o.append(r["offset"])
        krs.append(len(y))
        if key in pri:
            pvar = {_fkey(f): f["value"] for f in pri[key]["posteriorVar"]}
            for f in pri[key]["model"]:
                nm = _fkey(f)
                ent.append((k, D if nm == ref.INTERCEPT else ids[nm], f["value"], pvar[nm] if pvar.get(nm, 0) > 0 else 0.0))
    pb = dict(krs=np.array(krs, np.int64), rp=np.array(rp, np.int64), ci=np.array(ci, np.int32), v=np.array(v, np.float32),
              y=np.array(y, np.int32), w=np.array(w, np.float32), o=np.array(o, np.float32), D=D, K=len(keys))
    lmd = dict(ref.lambda_map_entries(lm_entries))
    lm = np.array([lmd.get(nm, 0.0) for nm in names], np.float32)
    prior = _lists(ent, len(keys))
    fits = pref.key_fits(pb, il, dl, lm, prior)
    out = []
    for k, key in enumerate(keys):
        fk = fits[k]
        e = np.arange(prior[0][k], prior[0][k + 1])
        for ia, lam_i in enumerate(il):
            for ib, lam_d in enumerate(dl):
                c, L = fk["cols"], fk["listed"]
                full = np.zeros(D + 1)
                full[c[L]] = fk["model"][ia, ib][L]
                with np.errstate(divide="ignore"):   # the oracle leaves features outside the dataset 0
                    var = 1.0 / orc.objective("hessian_diag", fk["data"], full, fk["pm"][ia, ib], fk["pv"][ia, ib])
                val = dict(zip(c.tolist(), fk["model"][ia, ib]))
                model = [(ref.INTERCEPT, val[D])] + [(names[j], val[j]) for j in c[:-1]]
                pvl = [(ref.INTERCEPT, var[D])] + [(names[j], var[j]) for j in c[:-1][L[:-1]]]
                pvl += [(names[j], prior[3][e][np.searchsorted(prior[1][e], j)]) for j in c[:-1][~L[:-1]]
                        if prior[3][e][np.searchsorted(prior[1][e], j)] > 0]
                listed = {nm for nm, _ in pvl}
                pvl += [(nm, 1.0 / np.float64(lam)) for nm, lam in ref.lambda_map_entries(lm_entries) if nm not in listed and nm != ref.INTERCEPT]
                out.append({"key": orc.java_float_to_string(np.float32(lam_i)) + ":" + orc.java_float_to_string(np.float32(lam_d)) + "#" + key,
                            "model": model, "posteriorVar": pvl})
    return out


def _job(host, tmp_path, name, kv):
    cfg = tmp_path / (name + ".job")
    cfg.write_text("".join("%s=%s\n" % e for e in kv.items()))
    assert host.mlease_job_run(b"ItemModelTrain", str(cfg).encode()) == 0, host.mlease_job_last_error().decode()
    return au.read_avro(str(kv["output.model.path"]) + "/models/part-r-00000.avro")[1]


def _refresh(host, tmp_path, devices):
    rng = np.random.default_rng(2600)
    feats = ["f%d" % i for i in range(30)] + ["g1x", "g2x"]
    day1 = _records(rng, 600, ["i%d" % i for i in range(12)], feats[:24] + ["g1x"])
    day2 = _records(rng, 300, ["i%d" % i for i in range(4, 16)], feats[6:], shift=0.4)   # i12 .. i15 are new; f0 .. f5 only in day 1
    au.write_avro(str(tmp_path / "d1" / "p.avro"), ref.PREPARED_SCHEMA, day1)
    au.write_avro(str(tmp_path / "d2" / "p.avro"), ref.PREPARED_SCHEMA, day2)
    lm_entries = [("f7", 3.0), ("nowhere", 5.0), ("f2", 0.5)]
    ref.write_lambda_map(str(tmp_path / "lm" / "a.avro"), lm_entries)
    base = {"intercept.lambdas": "1", "compute.var": "true", "lambda.map": tmp_path / "lm", "gpu.devices": devices}
    prior = _job(host, tmp_path, "day1", dict(base, **{"input.paths": tmp_path / "d1", "output.model.path": tmp_path / "o1",
                                                       "default.lambdas": "0.5,2"}))
    got = _job(host, tmp_path, "day2", dict(base, **{"input.paths": tmp_path / "d2", "output.model.path": tmp_path / "o2",
                                                     "default.lambdas": "0.25,1", "prior.model.path": tmp_path / "o1" / "models",
                                                     "prior.model.lambda": "1:2"}))
    return got, day2, prior, lm_entries


def test_job_refreshes_an_earlier_run(host, tmp_path):
    got, day2, prior, lm_entries = _refresh(host, tmp_path, "0")
    want = _job_replica(day2, prior, "1.0:2.0", [1.0], [0.25, 1.0], lm_entries)
    assert [r["key"] for r in got] == [r["key"] for r in want]
    assert any(f["name"] in ("f0", "f1") for r in got for f in r["model"])     # features only the prior names
    for g, w in zip(got, want):
        for field in ("model", "posteriorVar"):
            assert [_fkey(f) for f in g[field]] == [nm for nm, _ in w[field]], (g["key"], field)
            a = np.array([f["value"] for f in g[field]], np.float64)
            b = np.array([x for _, x in w[field]], np.float64)
            assert np.abs(a - b).max() <= 1e-5 * max(np.abs(b).max(), 1e-30), (g["key"], field)


def test_job_on_two_devices_matches_one(host, tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    one = _refresh(host, tmp_path / "one", "0")[0]
    two = _refresh(host, tmp_path / "two", "0,1")[0]
    assert [r["key"] for r in one] == [r["key"] for r in two]
    for a, b in zip(one, two):
        for field in ("model", "posteriorVar"):
            assert [_fkey(f) for f in a[field]] == [_fkey(f) for f in b[field]]
            x = np.array([f["value"] for f in a[field]]); y = np.array([f["value"] for f in b[field]])
            assert np.abs(x - y).max() <= 1e-5 * max(np.abs(y).max(), 1e-30)
