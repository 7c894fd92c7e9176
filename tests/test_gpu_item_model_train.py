"""GPU tests of ItemModelTrain: mlease_item_model_train against the oracle (fits per (key, intercept lambda, default lambda), the
batched posterior variance against 1 / hessian_diag at the GPU's own fit), the shared keyed driver (bitwise NaiveTrain), the batched
variance against the single-partition one, a call that spans two key chunks, and the job end to end after RegressionPrepare."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from oracle import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import avro_util as au  # noqa: E402
import item_model_train_ref as ref  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _keyed_csr(rng, K, rows, D, nnz, absent=10):
    """K keys of `rows` rows each, sorted unique columns; odd keys never list the last `absent` features."""
    n = K * rows
    beta = rng.normal(size=D) / np.sqrt(nnz)
    ci = np.stack([np.sort(rng.choice(D - absent * (i // rows % 2), nnz, replace=False)) for i in range(n)]).astype(np.int32)
    v = rng.normal(size=(n, nnz)).astype(np.float32)
    y = (rng.random(n) < 1 / (1 + np.exp(-((v * beta[ci]).sum(1) - 0.4)))).astype(np.int32)
    w = rng.uniform(0.5, 2.0, n).astype(np.float32)
    o = rng.normal(0, 0.1, n).astype(np.float32)
    rp = np.arange(n + 1, dtype=np.int64) * nnz
    return dict(rp=rp, ci=ci.reshape(-1), v=v.reshape(-1), y=y, w=w, o=o, krs=np.arange(K + 1, dtype=np.int64) * rows, D=D, K=K)


def _key_data(pb, k, vals=None):
    a, b = pb["krs"][k], pb["krs"][k + 1]
    rp = pb["rp"][a:b + 1]
    v = pb["v"] if vals is None else vals
    return orc.Csr(rp - rp[0], pb["ci"][rp[0]:rp[-1]], v[rp[0]:rp[-1]], pb["y"][a:b], pb["w"][a:b], pb["o"][a:b], pb["D"])


def _prior(D, lm, il, dl, mean):
    pv = np.where(lm > 0, 1.0 / np.where(lm > 0, lm, 1).astype(np.float64), 1.0 / np.float64(np.float32(dl)))
    pv = np.append(pv, 1.0 / np.float64(np.float32(il)))
    pm = np.zeros(D + 1); pm[D] = mean
    return pm, pv


@pytest.mark.parametrize("binary", [False, True])
def test_item_model_train_matches_oracle_and_hessian_diag(binary):
    import mlease_b200 as mb
    rng = np.random.default_rng(31)
    pb = _keyed_csr(rng, 6, 300, 60, 8)
    D, K = pb["D"], pb["K"]
    lm = np.zeros(D, np.float32); lm[[2, 7, 55]] = [0.05, 8.0, 3.0]
    il, dl = [0.5, 20.0], [1.0, 0.25, 1.0]
    means = np.array([0.7, -1.3, 0.0, 2.5, -0.25, 0.1])
    models, var = mb.item_model_train(pb["v"], pb["krs"], pb["y"], il, dl, rowptr=pb["rp"], colidx=pb["ci"], num_features=D,
                                      intercept_prior_mean=means, weight=pb["w"], offset=pb["o"], lambda_map=lm, binary_feature=binary,
                                      compute_var=True)
    assert models.shape == (2, 3, K, D + 1) and var.shape == models.shape
    vals = np.ones_like(pb["v"]) if binary else None
    for k in range(K):
        data = _key_data(pb, k, vals)
        listed = np.zeros(D + 1, bool); listed[np.unique(data.colidx)] = True; listed[D] = True
        for a, ia in enumerate(il):
            for b, db in enumerate(dl):
                pm, pv = _prior(D, lm, ia, db, means[k])
                want, _ = orc.liblinear_train(data, np.zeros(D + 1), pm, pv, 1e-14, 100000)
                want[~listed] = 0.0
                got = models[a, b, k]
                assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max(), (k, a, b)
                assert np.all(got[~listed] == 0.0)
                hd = orc.objective("hessian_diag", data, got, pm, pv)[listed]    # the oracle leaves features outside the dataset 0
                assert np.abs(var[a, b, k][listed] - 1.0 / hd).max() <= 1e-10 * np.abs(1.0 / hd).max(), (k, a, b)
                assert np.array_equal(var[a, b, k][~listed], (1.0 / (1.0 / pv))[~listed])   # absent: 1/q, no data term
    # a repeated default lambda is fitted again: the same fit up to the float-atomic gradient sums of the CSR K1
    assert np.abs(models[:, 0] - models[:, 2]).max() <= 1e-6 * np.abs(models).max()


def test_shared_driver_is_naive_train_bitwise():
    """iλ = dλ = λ with zero intercept means is NaiveTrain with penalize.intercept and prior.mean 0: the same driver, the same bits.
    The CSR K1 sums a key's gradient with float shared-memory atomics, so two CSR calls agree bitwise only where that sum does not
    depend on the order: keys of one row each (every column, the bias included, gets one addition).  Keys of many rows agree to the
    run-to-run spread of those sums."""
    import mlease_b200 as mb
    rng = np.random.default_rng(32)
    for rows, K in ((1, 400), (150, 40)):
        pb = _keyed_csr(rng, K, rows, 90, 12)
        lm = np.zeros(pb["D"], np.float32); lm[[3, 80]] = [0.5, 4.0]
        for lam in (0.3, 2.0):
            got, _ = mb.item_model_train(pb["v"], pb["krs"], pb["y"], [lam], [lam], rowptr=pb["rp"], colidx=pb["ci"], num_features=pb["D"],
                                         weight=pb["w"], offset=pb["o"], lambda_map=lm)
            want, _ = mb.naive_train(pb["v"], pb["krs"], pb["y"], [lam], rowptr=pb["rp"], colidx=pb["ci"], num_features=pb["D"], weight=pb["w"],
                                     offset=pb["o"], lambda_map=lm, prior_mean=0.0, penalize_intercept=True)
            if rows == 1:
                assert np.array_equal(got[0, 0].view(np.uint64), want[0].view(np.uint64)), lam
            else:
                assert np.abs(got[0, 0] - want[0]).max() <= 1e-6 * np.abs(want).max(), lam


def test_batched_variance_of_one_key_equals_single_partition_variance():
    import mlease_b200 as mb
    rng = np.random.default_rng(33)
    pb = _keyed_csr(rng, 1, 2500, 45, 9, absent=0)
    D = pb["D"]
    lm = np.zeros(D, np.float32)
    models, var = mb.item_model_train(pb["v"], pb["krs"], pb["y"], [3.0], [0.7], rowptr=pb["rp"], colidx=pb["ci"], num_features=D,
                                      intercept_prior_mean=[0.4], weight=pb["w"], offset=pb["o"], lambda_map=lm, compute_var=True)
    _, pv = _prior(D, lm, 3.0, 0.7, 0.4)
    with mb.AdmmSession(1, D, [1.0], epsilon=0.0) as s:
        s.add_partition_csr(0, pb["rp"], pb["ci"], pb["v"], pb["y"], pb["w"], pb["o"])
        single = s.posterior_variance(0, models[0, 0, 0], 1.0 / pv)
    assert np.abs(var[0, 0, 0] - single).max() <= 1e-12 * np.abs(single).max()


def test_key_chunks_keep_each_keys_intercept_mean():
    """More than 16 384 keys: the call runs in two key chunks; every key's intercept mean must follow it into its chunk."""
    import mlease_b200 as mb
    rng = np.random.default_rng(34)
    K, rows, D, nnz = 16384 + 700, 12, 20, 3
    n = K * rows
    ci = np.sort(np.stack([rng.choice(D, nnz, replace=False) for _ in range(n)]), axis=1).astype(np.int32).reshape(-1)
    v = rng.normal(size=n * nnz).astype(np.float32)
    y = rng.integers(0, 2, n).astype(np.int32)
    krs = np.arange(K + 1, dtype=np.int64) * rows
    rp = np.arange(n + 1, dtype=np.int64) * nnz
    means = rng.normal(0, 2, K)
    models, var = mb.item_model_train(v, krs, y, [50.0], [1.0], rowptr=rp, colidx=ci, num_features=D, intercept_prior_mean=means,
                                      compute_var=True)
    pb = dict(rp=rp, ci=ci, v=v, y=y, w=np.ones(n, np.float32), o=np.zeros(n, np.float32), krs=krs, D=D)
    for k in list(range(0, 30)) + list(range(16370, 16400)) + list(range(K - 30, K)):
        data = _key_data(pb, k)
        pm, pv = _prior(D, np.zeros(D, np.float32), 50.0, 1.0, means[k])
        want, _ = orc.liblinear_train(data, np.zeros(D + 1), pm, pv, 1e-14, 100000)
        listed = np.zeros(D + 1, bool); listed[np.unique(data.colidx)] = True; listed[D] = True
        want[~listed] = 0.0
        assert np.abs(models[0, 0, k] - want).max() <= 1e-5 * np.abs(want).max(), k
        hd = orc.objective("hessian_diag", data, models[0, 0, k], pm, pv)[listed]
        assert np.abs(var[0, 0, k][listed] - 1.0 / hd).max() <= 1e-10 * np.abs(1.0 / hd).max(), k


@pytest.fixture(scope="module")
def host():
    from mlease_b200 import build as _b
    _b.build()
    h = C.CDLL(os.path.join(ROOT, "ml-ease_b200", "lib", "libmlease_host.so"))
    h.mlease_job_last_error.restype = C.c_char_p
    return h


def test_prepare_then_item_model_train_job_against_restatement(host, tmp_path):
    npz = np.load(os.path.join(GOLDEN, "sample_data.npz"))
    names = [str(x) for x in npz["feature_names"]]
    recs = au.fixture_records(npz)
    au.write_avro(str(tmp_path / "in" / "part-0.avro"), au.PIG_SCHEMA, recs)
    out = str(tmp_path / "out")
    cfg = tmp_path / "prep.job"
    cfg.write_text("input.paths=%s\noutput.path=%s\nnum.blocks=4\n" % (tmp_path / "in", out + "/tmp-data"))
    assert host.mlease_job_run(b"RegressionPrepare", str(cfg).encode()) == 0, host.mlease_job_last_error().decode()
    prepared = au.read_dir(out + "/tmp-data")
    ref.write_lambda_map(str(tmp_path / "lm" / "lm.avro"), [(names[3], 0.2), ("not-in-data", 5.0), (names[10], 2.0)])
    ref.write_prior_mean_map(str(tmp_path / "pm" / "a.avro"), [("1", "0.75")])
    ref.write_prior_mean_map(str(tmp_path / "pm" / "b.avro"), [("2", -1.5)], value_type="double")
    cfg = tmp_path / "t.job"
    cfg.write_text("input.paths=%s\noutput.model.path=%s\nintercept.lambdas=1,30\ndefault.lambdas=0.5,2\nlambda.map=%s\n"
                   "intercept.prior.mean.map=%s\nintercept.default.prior.mean=0.1\ncompute.var=true\nremove.tmp.dir=false\n"
                   % (out + "/tmp-data", out, tmp_path / "lm", tmp_path / "pm"))
    assert host.mlease_job_run(b"ItemModelTrain", str(cfg).encode()) == 0, host.mlease_job_last_error().decode()
    sch, got = au.read_avro(os.path.join(out, "models", "part-r-00000.avro"))[:2]
    assert sch["name"] == "LinearModelWithVarAvro"
    want = ref.item_model_train(prepared, [1.0, 30.0], [0.5, 2.0], lambda_map=[(names[3], 0.2), ("not-in-data", 5.0), (names[10], 2.0)],
                                prior_mean_map={"1": 0.75, "2": -1.5}, default_prior_mean=0.1, compute_var=True)
    assert [r["key"] for r in got] == [r["key"] for r in want]
    for g, w in zip(got, want):
        for field in ("model", "posteriorVar"):
            assert [(f["name"], f["term"]) for f in g[field]] == [(f["name"], f["term"]) for f in w[field]], (g["key"], field)
            a = np.array([f["value"] for f in g[field]], np.float64)
            b = np.array([f["value"] for f in w[field]], np.float64)
            assert np.abs(a - b).max() <= 1e-5 * max(np.abs(b).max(), 1e-30), (g["key"], field)
