"""GPU tests of the keyed calls beyond one resident upload: streamed fits (mlease_naive_train CSR and dense, mlease_item_model_train)
against resident calls on each streamed chunk's keys alone and against the resident call on every key, streamed scoring bitwise
against resident scoring, the row checks of a late chunk, and keyed calls on two devices at once.  The test budget hook makes small
inputs stream through many chunks."""
import ctypes as C
import os
import sys
import threading

import numpy as np
import pytest

from oracle import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import avro_util as au  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _ndev():
    import torch
    return torch.cuda.device_count()


@pytest.fixture
def budget():
    from mlease_b200 import _hooks
    yield _hooks.set_keyed_budget
    _hooks.set_keyed_budget(0)


def _keyed(rng, rows, D, nnz, absent=8):
    """keys of rows[k] rows, sorted unique columns; odd keys never list the last `absent` features."""
    K, n = len(rows), int(np.sum(rows))
    krs = np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)
    key = np.repeat(np.arange(K), rows)
    beta = rng.normal(size=D) / np.sqrt(nnz)
    ci = np.stack([np.sort(rng.choice(D - absent * (key[i] % 2), nnz, replace=False)) for i in range(n)]).astype(np.int32)
    v = rng.normal(size=(n, nnz)).astype(np.float32)
    y = (rng.random(n) < 1 / (1 + np.exp(-((v * beta[ci]).sum(1) - 0.3)))).astype(np.int32)
    return dict(krs=krs, rp=np.arange(n + 1, dtype=np.int64) * nnz, ci=ci.reshape(-1), v=v.reshape(-1), y=y,
                w=rng.uniform(0.5, 2.0, n).astype(np.float32), o=rng.normal(0, 0.1, n).astype(np.float32), D=D, K=K)


def _slice(pb, k0, k1):
    a, b = pb["krs"][k0], pb["krs"][k1]
    z0, z1 = pb["rp"][a], pb["rp"][b]
    return dict(krs=pb["krs"][k0:k1 + 1] - a, rp=pb["rp"][a:b + 1] - z0, ci=pb["ci"][z0:z1], v=pb["v"][z0:z1], y=pb["y"][a:b], w=pb["w"][a:b],
                o=pb["o"][a:b], D=pb["D"], K=k1 - k0)


def _close(got, want):
    """the run-to-run spread of a CSR fit: the K1 gradient sums use float atomics (as in test_gpu_item_model_train.py)"""
    assert np.abs(got - want).max() <= 1e-6 * max(1.0, np.abs(want).max())


def _naive(pb, budget_bytes, budget, lams=(0.5, 3.0), thr=40):
    import mlease_b200 as mb
    lm = np.zeros(pb["D"], np.float32); lm[[1, 9]] = [0.2, 5.0]
    budget(budget_bytes)
    kw = dict(rowptr=pb["rp"], colidx=pb["ci"], num_features=pb["D"], weight=pb["w"], offset=pb["o"], lambda_map=lm, data_size_threshold=thr)
    return mb.naive_train(pb["v"], pb["krs"], pb["y"], list(lams), **kw)


def test_streamed_naive_train_csr_matches_resident_per_chunk(budget):
    from mlease_b200 import _hooks
    rng = np.random.default_rng(71)
    rows = rng.integers(400, 1200, 36); rows[[3, 17, 30]] = [5, 0, 20]          # skipped by data.size.threshold = 40, and a key with no rows
    pb = _keyed(rng, rows, 48, 30)
    models, skipped = _naive(pb, 5 << 20, budget)
    bounds, streamed, _, _ = _hooks.keyed_last_call()
    assert streamed and len(bounds) - 1 >= 6 and bounds[0] == 0 and bounds[-1] == pb["K"], bounds
    assert list(np.nonzero(skipped)[0]) == [3, 17, 30] and np.all(models[:, [3, 17, 30]] == 0)
    for k0, k1 in zip(bounds[:-1], bounds[1:]):
        m1, s1 = _naive(_slice(pb, k0, k1), 0, budget)
        assert not _hooks.keyed_last_call()[1]
        _close(models[:, k0:k1], m1)
        assert np.array_equal(skipped[k0:k1], s1)
    full, _ = _naive(pb, 0, budget)
    _close(models, full)
    for k in range(pb["K"]):   # features a key's rows never list are not in its model
        listed = np.zeros(pb["D"] + 1, bool); listed[np.unique(pb["ci"][pb["rp"][pb["krs"][k]]:pb["rp"][pb["krs"][k + 1]]])] = True; listed[-1] = True
        assert np.all(models[:, k][:, ~listed] == 0)


def test_streamed_naive_train_one_row_keys_are_bitwise(budget):
    """keys of one row: every gradient sum is one addition, so a streamed chunk is bitwise its resident call"""
    from mlease_b200 import _hooks
    rng = np.random.default_rng(72)
    pb = _keyed(rng, np.ones(300, np.int64), 30, 6)
    models, _ = _naive(pb, 120 << 10, budget, thr=0)
    bounds, streamed, _, _ = _hooks.keyed_last_call()
    assert streamed and len(bounds) - 1 >= 6, bounds
    for k0, k1 in list(zip(bounds[:-1], bounds[1:]))[::10]:
        m1, _ = _naive(_slice(pb, k0, k1), 0, budget, thr=0)
        assert np.array_equal(models[:, k0:k1].view(np.uint64), m1.view(np.uint64)), (k0, k1)


def test_streamed_naive_train_dense(budget):
    import mlease_b200 as mb
    from mlease_b200 import _hooks
    rng = np.random.default_rng(73)
    K, D = 24, 40
    rows = rng.integers(300, 900, K)
    krs = np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)
    X = rng.normal(size=(krs[-1], D)).astype(np.float32)
    y = (rng.random(krs[-1]) < 1 / (1 + np.exp(-X[:, :5].sum(1)))).astype(np.int32)
    budget(3 << 20)
    got, _ = mb.naive_train(X, krs, y, [1.0, 4.0])
    bounds, streamed, _, _ = _hooks.keyed_last_call()
    assert streamed and len(bounds) - 1 >= 4, bounds
    budget(0)
    for k0, k1 in zip(bounds[:-1], bounds[1:]):
        a, b = krs[k0], krs[k1]
        want, _ = mb.naive_train(X[a:b], krs[k0:k1 + 1] - a, y[a:b], [1.0, 4.0])
        assert np.abs(got[:, k0:k1] - want).max() <= 1e-6 * np.abs(want).max(), (k0, k1)


def test_streamed_item_model_train_matches_resident_per_chunk(budget):
    import mlease_b200 as mb
    from mlease_b200 import _hooks
    rng = np.random.default_rng(74)
    rows = rng.integers(300, 900, 30); rows[11] = 0
    pb = _keyed(rng, rows, 40, 8)
    means = rng.normal(size=pb["K"])
    lm = np.zeros(pb["D"], np.float32); lm[[2, 30]] = [0.05, 3.0]
    il, dl = [0.5, 4.0, 20.0], [1.0, 0.25]

    def fit(p, m, nbytes):
        budget(nbytes)
        return mb.item_model_train(p["v"], p["krs"], p["y"], il, dl, rowptr=p["rp"], colidx=p["ci"], num_features=p["D"], intercept_prior_mean=m,
                                   weight=p["w"], offset=p["o"], lambda_map=lm, compute_var=True)
    models, var = fit(pb, means, 3 << 19)
    bounds, streamed, _, _ = _hooks.keyed_last_call()
    assert streamed and len(bounds) - 1 >= 6, bounds
    for k0, k1 in zip(bounds[:-1], bounds[1:]):
        m1, v1 = fit(_slice(pb, k0, k1), means[k0:k1], 0)
        _close(models[:, :, k0:k1], m1)
        assert np.abs(var[:, :, k0:k1] - v1).max() <= 1e-6 * np.abs(v1).max()
    for k in (0, 7, 12, 25):   # against the oracle, as test_gpu_item_model_train.py checks the resident call
        a0, b0 = pb["krs"][k], pb["krs"][k + 1]
        rp = pb["rp"][a0:b0 + 1]
        data = orc.Csr(rp - rp[0], pb["ci"][rp[0]:rp[-1]], pb["v"][rp[0]:rp[-1]], pb["y"][a0:b0], pb["w"][a0:b0], pb["o"][a0:b0], pb["D"])
        listed = np.zeros(pb["D"] + 1, bool); listed[np.unique(data.colidx)] = True; listed[-1] = True
        for a, ia in enumerate(il):
            for b, db in enumerate(dl):
                pv = np.where(lm > 0, 1.0 / np.where(lm > 0, lm, 1).astype(np.float64), 1.0 / np.float64(np.float32(db)))
                pv = np.append(pv, 1.0 / np.float64(np.float32(ia)))
                pm = np.zeros(pb["D"] + 1); pm[-1] = means[k]
                want, _ = orc.liblinear_train(data, np.zeros(pb["D"] + 1), pm, pv, 1e-14, 100000)
                want[~listed] = 0.0
                assert np.abs(models[a, b, k] - want).max() <= 1e-5 * np.abs(want).max(), (k, a, b)
    m2, v2 = fit(pb, means, 0)
    _close(models, m2)
    assert np.abs(var - v2).max() <= 1e-6 * np.abs(v2).max()
    assert np.array_equal(var[:, :, 11], v2[:, :, 11])   # no rows: the prior variances


def test_late_chunk_with_a_bad_column_fails_before_it_is_solved(budget):
    import mlease_b200 as mb
    rng = np.random.default_rng(75)
    pb = _keyed(rng, rng.integers(300, 600, 20), 30, 6)
    pb["ci"] = pb["ci"].copy(); pb["ci"][pb["rp"][pb["krs"][18]] + 2] = 30    # column == num_features in key 18
    with pytest.raises(mb.MleaseError, match="feature index out of range") as e:
        _naive(pb, 400 << 10, budget)
    assert e.value.code == 1
    pb["ci"][pb["rp"][pb["krs"][18]] + 2] = 29
    m, _ = _naive(pb, 400 << 10, budget)   # the process goes on
    assert np.all(np.isfinite(m))


@pytest.mark.parametrize("where", ["device", "pinned"])
def test_streamed_naive_train_from_device_and_pinned_input(budget, where):
    """device or pinned rows are copied into the ring directly (no pinned staging copy); same fits as pageable input"""
    import torch

    from mlease_b200 import _hooks
    rng = np.random.default_rng(78)
    rows = rng.integers(400, 1200, 24); rows[5] = 10
    pb = _keyed(rng, rows, 48, 30)
    want, ws = _naive(pb, 2 << 20, budget)
    assert _hooks.keyed_last_call()[1]
    conv = (lambda a: torch.from_numpy(a).cuda()) if where == "device" else (lambda a: torch.from_numpy(a).pin_memory())
    pt = dict(pb, rp=conv(pb["rp"]), ci=conv(pb["ci"]), v=conv(pb["v"]), y=conv(pb["y"]), w=conv(pb["w"]), o=conv(pb["o"]))
    got, gs = _naive(pt, 2 << 20, budget)   # below the device input's resident upload (rows, labels) + first state
    bounds, streamed, _, _ = _hooks.keyed_last_call()
    assert streamed and len(bounds) - 1 >= 6, bounds
    assert np.array_equal(gs, ws)
    _close(got, want)


def _scoring_data(rng, K, D, L):
    rows = rng.integers(50, 400, K); rows[[2, 9]] = 0
    krs = np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)
    n = int(krs[-1])
    nnz = rng.integers(0, 20, n)
    rp = np.concatenate([[0], np.cumsum(nnz)]).astype(np.int64)
    ci = np.concatenate([np.sort(rng.choice(D, c, replace=False)) for c in nnz]).astype(np.int32)
    v = rng.normal(size=len(ci)).astype(np.float32)
    o = rng.normal(size=n).astype(np.float32)
    mp, mc, mv = [0], [], []
    for m in range(L * K):
        if m % 7 == 3:
            mp.append(len(mc)); continue                                  # a key without a model
        cols = np.sort(rng.choice(D + 1, rng.integers(1, D // 2), replace=False))
        mc += list(cols); mv += list(rng.normal(size=len(cols))); mp.append(len(mc))
    return krs, rp, ci, v, o, np.array(mp, np.int64), np.array(mc, np.int32), np.array(mv, np.float32)


@pytest.mark.parametrize("L", [1, 3, 5])
@pytest.mark.parametrize("binary", [False, True])
def test_streamed_score_keyed_is_bitwise_resident(budget, L, binary):
    import torch

    import mlease_b200 as mb
    from mlease_b200 import _hooks
    rng = np.random.default_rng(76 + L)
    K, D = 40, 120
    krs, rp, ci, v, o, mp, mc, mv = _scoring_data(rng, K, D, L)
    budget(0)
    want = mb.score_keyed(v, krs, rp, ci, D, mp, mc, mv, offset=o, binary_feature=binary)
    assert not _hooks.keyed_last_call()[1]
    budget(256 << 10)
    got = mb.score_keyed(v, krs, rp, ci, D, mp, mc, mv, offset=o, binary_feature=binary)
    bounds, streamed, _, _ = _hooks.keyed_last_call()
    assert streamed and len(bounds) - 1 >= 4, bounds
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    dev = torch.zeros((L, int(krs[-1])), dtype=torch.float32, device="cuda")
    mb.score_keyed(v, krs, rp, ci, D, mp, mc, mv, offset=o, binary_feature=binary, out=dev)
    assert _hooks.keyed_last_call()[1]
    assert np.array_equal(dev.cpu().numpy().view(np.uint32), want.view(np.uint32))


@pytest.mark.skipif("_ndev() < 2")
def test_keyed_calls_on_two_devices_at_once_match_one_device():
    import mlease_b200 as mb
    rng = np.random.default_rng(77)
    pb = _keyed(rng, rng.integers(200, 500, 16), 40, 8)
    halves = [_slice(pb, 0, 8), _slice(pb, 8, 16)]
    kw = lambda p: dict(rowptr=p["rp"], colidx=p["ci"], num_features=p["D"], weight=p["w"], offset=p["o"])   # noqa: E731
    serial = [mb.naive_train(p["v"], p["krs"], p["y"], [1.0, 2.0], device=0, **kw(p))[0] for p in halves]
    out = [None, None]
    err = []

    def run(i):
        try:
            out[i] = mb.naive_train(halves[i]["v"], halves[i]["krs"], halves[i]["y"], [1.0, 2.0], device=i, **kw(halves[i]))[0]
        except Exception as e:   # reported below
            err.append(e)
    ts = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not err, err
    for a, b in zip(out, serial):
        _close(a, b)
    # mlease_item_model_train and mlease_score_keyed, one device per thread
    krs, rp, ci, v, o, mp, mc, mv = _scoring_data(rng, 16, 40, 2)
    want = mb.score_keyed(v, krs, rp, ci, 40, mp, mc, mv, offset=o)
    imt = [mb.item_model_train(p["v"], p["krs"], p["y"], [1.0], [0.5, 2.0], rowptr=p["rp"], colidx=p["ci"], num_features=p["D"], compute_var=True)
           for p in halves]
    res = {}

    def both(i):
        try:
            if i == 0:
                res[0] = mb.score_keyed(v, krs, rp, ci, 40, mp, mc, mv, offset=o, device=0)
            else:
                p = halves[0]
                res[1] = mb.item_model_train(p["v"], p["krs"], p["y"], [1.0], [0.5, 2.0], rowptr=p["rp"], colidx=p["ci"], num_features=p["D"],
                                             compute_var=True, device=1)
        except Exception as e:   # reported below
            err.append(e)
    ts = [threading.Thread(target=both, args=(i,)) for i in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not err, err
    assert np.array_equal(res[0].view(np.uint32), want.view(np.uint32))
    _close(res[1][0], imt[0][0])


@pytest.fixture(scope="module")
def host():
    import mlease_b200
    mlease_b200.lib()
    h = C.CDLL(os.path.join(ROOT, "ml-ease_b200", "lib", "libmlease_host.so"))
    h.mlease_job_last_error.restype = C.c_char_p
    return h


def _job(h, job, path, kv):
    with open(path, "w") as f:
        f.write("".join("%s=%s\n" % (k, v) for k, v in kv.items()))
    rc = h.mlease_job_run(job.encode(), str(path).encode())
    return rc, (h.mlease_job_last_error() or b"").decode()


def _bytes(root):
    """relative path -> bytes of every avro file under root, its random 16-byte sync marker (which also ends the file) zeroed"""
    out = {}
    for dp, _, fs in os.walk(root):
        for f in fs:
            if f.endswith(".avro"):
                data = open(os.path.join(dp, f), "rb").read()
                out[os.path.relpath(os.path.join(dp, f), root)] = data.replace(data[-16:], bytes(16))
    return out


def _keyed_input(h, tmp_path, key_of):
    """records of the golden sample keyed by key_of(i), prepared once (RegressionPrepare), and NaiveTrain models for ItemModelTest"""
    inp = tmp_path / ("in_" + key_of.__name__)
    if inp.exists():
        return inp
    npz = np.load(os.path.join(GOLDEN, "sample_data.npz"))
    names = [str(n) for n in npz["feature_names"]]
    au.write_avro(str(inp / "raw" / "p.avro"), au.pig_schema_with_key(), au.fixture_records(npz, with_key=key_of), block=300)
    rc, e = _job(h, "RegressionPrepare", tmp_path / "p.job", {"input.paths": inp / "raw", "output.path": inp / "prep", "map.key": "pkey", "num.blocks": 2})
    assert rc == 0, e
    schema = {"type": "record", "name": "LinearModelAvro", "fields": [{"name": "key", "type": "string"}, {"name": "model", "type": {"type": "array",
              "items": {"type": "record", "name": "feature", "fields": [{"name": "name", "type": "string"}, {"name": "term", "type": "string"},
                                                                      {"name": "value", "type": "float"}]}}}]}
    au.write_avro(str(inp / "models" / "m.avro"), schema, [{"key": "1.0#%d" % k, "model": [{"name": "(INTERCEPT)", "term": "", "value": 0.25}] +
                                                            [{"name": nm, "term": "", "value": 0.1 * (i + 1)} for i, nm in enumerate(names[:30])]}
                                                           for k in range(0, 1000, 3)])
    return inp


def _job_configs(inp, out):
    return (("NaiveTrain", {"input.paths": inp / "prep", "output.base.path": out / "naive", "lambda": "1,10", "compute.model.mean": "false",
                            "remove.tmp.dir": "false"}),
            ("ItemModelTrain", {"input.paths": inp / "prep", "output.model.path": out / "imt", "intercept.lambdas": "0.5,20", "default.lambdas": "1",
                                "compute.var": "true"}),
            ("ItemModelTest", {"input.paths": inp / "raw", "output.base.path": out / "imtest", "model.path": inp / "models", "item.key": "pkey", "lambda": "1"}))


def _keyed_jobs(h, tmp_path, key_of, devs, tag):
    """NaiveTrain, ItemModelTrain and ItemModelTest with gpu.devices = devs -> their output directory"""
    inp, out = _keyed_input(h, tmp_path, key_of), tmp_path / tag
    for job, kv in _job_configs(inp, out):
        rc, e = _job(h, job, tmp_path / (tag + job + ".job"), dict(kv, **{"gpu.devices": devs}))
        assert rc == 0, (job, devs, e)
    return out


def _by_ten(i):
    return i // 10


def _one_row(i):
    return i


@pytest.mark.skipif("_ndev() < 2")
def test_keyed_jobs_on_two_gpus_write_the_one_gpu_tree(host, tmp_path):
    """gpu.devices=0,1: the same files, records and key order as gpu.devices=0; ItemModelTest preds byte-identical; models within
    the CSR kernels' run-to-run spread.  With one row per key every fit is order-independent, so the trees are byte-identical
    and each shard's models are bitwise its single-device call's."""
    one = _keyed_jobs(host, tmp_path, _by_ten, "0", "a1")
    two = _keyed_jobs(host, tmp_path, _by_ten, "0,1", "a2")
    b1, b2 = _bytes(one), _bytes(two)
    assert sorted(b1) == sorted(b2)
    for rel in b1:
        if rel.startswith("imtest/"):
            assert b1[rel] == b2[rel], rel
            continue
        r1, r2 = au.read_avro(str(one / rel))[1], au.read_avro(str(two / rel))[1]
        assert [r["key"] for r in r1] == [r["key"] for r in r2], rel
        for x, y in zip(r1, r2):
            for field in ("model", "posteriorVar"):
                if field in x:
                    assert [(f["name"], f["term"]) for f in x[field]] == [(f["name"], f["term"]) for f in y[field]]
                    vx, vy = np.array([f["value"] for f in x[field]]), np.array([f["value"] for f in y[field]])
                    assert np.abs(vx - vy).max() <= 1e-5 * max(1.0, np.abs(vx).max()), (rel, x["key"], field)
    o1 = _bytes(_keyed_jobs(host, tmp_path, _one_row, "0", "b1"))
    o2 = _bytes(_keyed_jobs(host, tmp_path, _one_row, "0,1", "b2"))
    assert o1 == o2


def test_keyed_job_shard_error_is_the_one_device_error(host, tmp_path):
    """gpu.devices=0,99: the shard on device 0 runs, the one on the missing device 99 fails; the job fails with the text a one-device
    job on device 99 reports, after every shard thread is joined"""
    inp = _keyed_input(host, tmp_path, _by_ten)
    for job, kv in _job_configs(inp, tmp_path / "err"):
        rc1, e1 = _job(host, job, tmp_path / "e1.job", dict(kv, **{"gpu.devices": "99"}))
        rc2, e2 = _job(host, job, tmp_path / "e2.job", dict(kv, **{"gpu.devices": "0,99"}))
        assert rc1 != 0 and e1 and (rc2, e2) == (rc1, e1), (job, rc1, e1, rc2, e2)
        rc, e = _job(host, job, tmp_path / "ok.job", dict(kv, **{"gpu.devices": "0"}))   # the process goes on
        assert rc == 0, e
