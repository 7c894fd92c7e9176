"""The ADMM model's posterior (mlease_admm_posterior) and scoring with its predictive variance (mlease_score_var), on the GPU,
against numpy fp64: the summed Hessian of every partition at z, its inverse, the diagonal mode, its determinism across calls,
upload orders and further ADMM iterations, the refusals; score_var's pred bit for bit against score and pred_var against g^T S g."""
import numpy as np
import pytest

import mlease_b200 as mb

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -53


def _parts(P, n, Dg, density, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(P):
        nnz_row = rng.binomial(Dg, density, size=n).clip(1, Dg)
        rowptr = np.zeros(n + 1, np.int64)
        rowptr[1:] = np.cumsum(nnz_row)
        cols = np.concatenate([np.sort(rng.choice(Dg, k, replace=False)) for k in nnz_row]).astype(np.int32)
        vals = rng.normal(0, 1, len(cols)).astype(np.float32)
        y = np.where(rng.random(n) < 0.4, 1, 0).astype(np.int32)
        w = rng.uniform(0.5, 2.0, n).astype(np.float32)
        o = rng.normal(0, 0.1, n).astype(np.float32)
        out.append((rowptr, cols, vals, y, w, o))
    return out


def _dense(part, Dg):
    rowptr, cols, vals = part[:3]
    X = np.zeros((len(rowptr) - 1, Dg), np.float64)
    for i in range(len(rowptr) - 1):
        X[i, cols[rowptr[i]:rowptr[i + 1]]] = vals[rowptr[i]:rowptr[i + 1]]
    return X


def _hessian(parts, Dg, z, binary=False):
    """sum over partitions of sum_i w_i p_i (1 - p_i) x~ x~^T at z (fp64); binary: every listed feature counts as 1"""
    import scipy.sparse as sp
    H = np.zeros((Dg + 1, Dg + 1))
    for rowptr, cols, vals, y, w, o in parts:
        n = len(rowptr) - 1
        x = np.ones(len(cols)) if binary else vals.astype(np.float64)
        X = sp.hstack([sp.csr_matrix((x, cols, rowptr), shape=(n, Dg)), np.ones((n, 1))]).tocsr()
        s = X @ z + o.astype(np.float64)
        p = 1.0 / (1.0 + np.exp(-np.where(y > 0, 1.0, -1.0) * s))
        d = w.astype(np.float64) * p * (1 - p)
        H += (X.T @ sp.diags(d) @ X).toarray()
    return H


def _q(Dg, lam, lambda_map=None, penalize_intercept=False):
    """the prior precision of the z-update: lambda, lambda_map's own where > 0, the intercept's only with penalize_intercept"""
    lamf = float(np.float32(lam))
    q = np.full(Dg + 1, lamf)
    if lambda_map is not None:
        lm = np.asarray(lambda_map, np.float32)
        q[:Dg] = np.where(lm > 0, lm.astype(np.float64), lamf)
    q[Dg] = lamf if penalize_intercept else 0.0
    return q


def _session(parts, Dg, lambdas, order=None, dense=False, **kw):
    s = mb.AdmmSession(len(parts), Dg, lambdas, **kw)
    for pid in (order if order is not None else range(len(parts))):
        rowptr, cols, vals, y, w, o = parts[pid]
        if dense:
            s.add_partition_dense(pid, _dense(parts[pid], Dg).astype(np.float32), y, w, o)
        else:
            s.add_partition_csr(pid, rowptr, cols, vals, y, w, o)
    return s


def _check_inverse(cov, H, tag):
    """Sigma against numpy.linalg.inv(H) within 8 Dt kappa_2(H) 2^-53 max|Sigma|; returns the ratio error / bound"""
    ref = np.linalg.inv(H)
    ev = np.linalg.eigvalsh(H)
    kappa = ev[-1] / ev[0]
    bound = 8 * H.shape[0] * kappa * EPS * np.abs(ref).max()
    err = np.abs(cov - ref).max()
    assert err <= bound, (tag, err, bound)
    return err / bound


@pytest.mark.parametrize("Dg", [30, 31, 32, 998, 1000, 2046, 2048])
def test_full_posterior_widths(Dg):
    P, n = 3, 400
    parts = _parts(P, n, Dg, min(0.05, 20.0 / Dg), seed=Dg)
    s = _session(parts, Dg, [1.0])
    s.begin()
    s.iterate()
    z = s.z(0)
    var, cov = s.admm_posterior(0, full=True, want_cov=True)
    H = _hessian(parts, Dg, z) + np.diag(_q(Dg, 1.0))
    r = _check_inverse(cov, H, Dg)
    print("Dt", Dg + 1, "worst ratio", r)
    assert np.array_equal(var, np.diag(cov))


@pytest.mark.parametrize("penalize_intercept", [False, True])
@pytest.mark.parametrize("lambdas", [[1.0], [0.1, 1.0, 10.0]])
def test_lambdas_map_and_intercept(lambdas, penalize_intercept):
    Dg, P = 60, 4
    parts = _parts(P, 300, Dg, 0.1, seed=7)
    lm = np.zeros(Dg, np.float32)
    lm[::7] = 3.5
    s = _session(parts, Dg, lambdas, lambda_map=lm, penalize_intercept=penalize_intercept)
    s.begin()
    s.iterate()
    s.iterate()
    for l, lam in enumerate(lambdas):
        z = s.z(l)
        Hd = _hessian(parts, Dg, z)
        q = _q(Dg, lam, lm, penalize_intercept)
        var, cov = s.admm_posterior(l, full=True, want_cov=True)
        _check_inverse(cov, Hd + np.diag(q), (l, lam))
        # diagonal mode: 1 / (q + diag(H)) within 4 ulps of fp64
        vd = s.admm_posterior(l, full=False)
        ref = 1.0 / (q + np.diag(Hd))
        assert np.all(np.abs(vd - ref) <= 4 * np.spacing(ref)), np.abs(vd - ref).max()


@pytest.mark.parametrize("binary", [False, True])
@pytest.mark.parametrize("dense", [False, True])
def test_deterministic_and_iteration_independent(dense, binary):
    if dense and binary:
        pytest.skip("binary.feature needs CSR input")
    Dg, P = 100, 4
    parts = _parts(P, 500, Dg, 0.08, seed=11)   # non-unit values: with binary_feature the posterior must take x = 1
    a = _session(parts, Dg, [0.5], dense=dense, binary_feature=binary)
    b = _session(parts, Dg, [0.5], order=[2, 0, 3, 1], dense=dense, binary_feature=binary)
    c = _session(parts, Dg, [0.5], dense=dense, binary_feature=binary)
    for s in (a, b, c):
        s.begin()
        s.iterate()
    z = a.z(0)
    assert np.array_equal(z, b.z(0))
    v1, c1 = a.admm_posterior(0, full=True, want_cov=True)
    v2, c2 = a.admm_posterior(0, full=True, want_cov=True)
    v3, c3 = b.admm_posterior(0, full=True, want_cov=True)
    assert np.array_equal(c1, c2) and np.array_equal(c1, c3)
    assert np.array_equal(a.admm_posterior(0), b.admm_posterior(0))
    _check_inverse(c1, _hessian(parts, Dg, z, binary) + np.diag(_q(Dg, 0.5)), "det")
    # the call leaves the ADMM state alone: a iterates bitwise as c, which made no posterior call
    a.iterate()
    c.iterate()
    assert np.array_equal(a.z(0), c.z(0))
    assert np.array_equal(a.x(1, 0), c.x(1, 0))
    # the same explicit z after further iterations gives the same bits
    v4, c4 = a.admm_posterior(0, z=z, full=True, want_cov=True)
    assert np.array_equal(c4, c1)


def test_matrix_free_session_matches_gram_session():
    Dg, P = 80, 3
    parts = _parts(P, 400, Dg, 0.1, seed=5)
    z = np.random.default_rng(1).normal(0, 0.2, Dg + 1)
    a = _session(parts, Dg, [1.0])
    b = _session(parts, Dg, [1.0], hessian_policy=2)
    for s in (a, b):
        s.begin()
    va, ca = a.admm_posterior(0, z=z, full=True, want_cov=True)
    vb, cb = b.admm_posterior(0, z=z, full=True, want_cov=True)
    assert np.array_equal(ca, cb)
    assert np.array_equal(a.admm_posterior(0, z=z), b.admm_posterior(0, z=z))


def test_one_partition_agrees_with_posterior_variance():
    Dg = 50
    parts = _parts(1, 600, Dg, 0.1, seed=3)
    s = _session(parts, Dg, [2.0], penalize_intercept=True)
    s.begin()
    z = np.random.default_rng(2).normal(0, 0.3, Dg + 1)
    q = _q(Dg, 2.0, None, True)
    var, cov = s.admm_posterior(0, z=z, full=True, want_cov=True)
    var2, cov2 = s.posterior_variance(0, z, q, full=True, want_cov=True)
    H = _hessian(parts, Dg, z) + np.diag(q)
    _check_inverse(cov, H, "admm")
    ev = np.linalg.eigvalsh(H)
    bound = 8 * H.shape[0] * ev[-1] / ev[0] * EPS * np.abs(cov2).max()
    assert np.abs(cov - cov2).max() <= bound


def test_wide_shape_4x20000x10001():
    Dg, P = 10000, 4
    parts = _parts(P, 20000, Dg, 0.01, seed=21)
    s = _session(parts, Dg, [1.0])
    s.begin()
    s.iterate()
    z = s.z(0)
    var, cov = s.admm_posterior(0, full=True, want_cov=True)
    H = _hessian(parts, Dg, z) + np.diag(_q(Dg, 1.0))
    print("Dt 10001 worst ratio", _check_inverse(cov, H, "wide"))


def test_refusals():
    Dg = 20
    parts = _parts(2, 50, Dg, 0.2, seed=9)
    s = _session(parts, Dg, [1.0], regularizer=1)
    s.begin()
    with pytest.raises(mb.MleaseError, match="L1 penalty has no Hessian"):
        s.admm_posterior(0, full=True)
    s = _session(parts, Dg, [1.0])
    s.begin()
    with pytest.raises(mb.MleaseError, match="lambda index 1 out of range"):
        s.admm_posterior(1)
    rowptr, cols, vals, y, w, o = parts[0]
    r = int(np.argmax(np.diff(rowptr) >= 2))   # a row of two entries or more: swap its first two
    bad = cols.copy()
    bad[rowptr[r]], bad[rowptr[r] + 1] = cols[rowptr[r] + 1], cols[rowptr[r]]
    u = mb.AdmmSession(1, Dg, [1.0])
    u.add_partition_csr(0, rowptr, bad, vals, y, w, o)
    u.begin()
    with pytest.raises(mb.MleaseError, match="strictly increasing column ids"):
        u.admm_posterior(0, full=True)
    wide = mb.AdmmSession(1, 59999, [1.0], hessian_policy=2)
    wide.add_partition_csr(0, np.array([0, 2], np.int64), np.array([3, 59000], np.int32), np.ones(2, np.float32), np.array([1], np.int32))
    wide.begin()
    with pytest.raises(mb.MleaseError, match="bytes of device memory"):
        wide.admm_posterior(0, full=True)
    assert np.all(np.isfinite(wide.admm_posterior(0, full=False)))


def _score_ref(parts, Dg, model, S, n_rep, binary, diag):
    rowptr, cols, vals = parts[0][:3]
    o = parts[0][5].astype(np.float64)
    b = model[Dg]
    gI = n_rep * np.exp(-b) / (n_rep - 1 + n_rep * np.exp(-b))
    out = []
    for i in range(len(rowptr) - 1):
        c = cols[rowptr[i]:rowptr[i + 1]]
        x = np.ones(len(c)) if binary else vals[rowptr[i]:rowptr[i + 1]].astype(np.float64)
        g = np.append(x, gI)
        idx = np.append(c, Dg)
        out.append(np.sum(S[idx] * g * g) if diag else g @ S[np.ix_(idx, idx)] @ g)
    return np.array(out)


@pytest.mark.parametrize("binary", [False, True])
@pytest.mark.parametrize("n_rep", [1, 5])
def test_score_var(n_rep, binary):
    Dg = 300
    parts = _parts(1, 2000, Dg, 0.05, seed=31)
    rng = np.random.default_rng(4)
    model = rng.normal(0, 0.3, Dg + 1)
    A = rng.normal(0, 1, (Dg + 1, Dg + 1))
    cov = A @ A.T / Dg + np.eye(Dg + 1)
    rowptr, cols, vals, _, _, o = parts[0]
    pred_ref = mb.score(vals, model, rowptr=rowptr, colidx=cols, offset=o, num_features=Dg, num_click_replicates=n_rep,
                        binary_feature=binary)
    pred, pv = mb.score_var(rowptr, cols, vals, model, cov=cov, offset=o, num_click_replicates=n_rep, binary_feature=binary)
    assert np.array_equal(pred, pred_ref)
    ref = _score_ref(parts, Dg, model, cov, n_rep, binary, False)
    assert np.all(np.abs(pv - ref) <= 2 * np.spacing(np.float32(ref)).astype(np.float64))
    v = np.diag(cov).copy()
    pred2, pvd = mb.score_var(rowptr, cols, vals, model, var=v, offset=o, num_click_replicates=n_rep, binary_feature=binary)
    assert np.array_equal(pred2, pred_ref)
    refd = _score_ref(parts, Dg, model, v, n_rep, binary, True)
    assert np.all(np.abs(pvd - refd) <= 2 * np.spacing(np.float32(refd)).astype(np.float64))
    # the diagonal form equals the dense form of a diagonal Sigma within 1 ulp
    _, pvD = mb.score_var(rowptr, cols, vals, model, cov=np.diag(v), offset=o, num_click_replicates=n_rep, binary_feature=binary)
    assert np.all(np.abs(pvD.astype(np.float64) - pvd) <= np.spacing(pvd).astype(np.float64))


def test_score_var_refusals():
    Dg = 10
    model = np.zeros(Dg + 1)
    v = np.ones(Dg + 1)
    rowptr = np.array([0, 2], np.int64)
    with pytest.raises(mb.MleaseError, match="strictly ascending"):
        mb.score_var(rowptr, np.array([4, 2], np.int32), np.ones(2, np.float32), model, var=v)
    for bad in ([2, Dg], [-1, 4]):
        for kw in (dict(var=v), dict(cov=np.eye(Dg + 1))):
            with pytest.raises(mb.MleaseError, match="colidx out of range"):
                mb.score_var(rowptr, np.array(bad, np.int32), np.ones(2, np.float32), model, **kw)
    with pytest.raises(mb.MleaseError, match="exactly one of var and cov"):
        mb.score_var(rowptr, np.array([2, 4], np.int32), np.ones(2, np.float32), model, var=v, cov=np.eye(Dg + 1))
    with pytest.raises(mb.MleaseError, match="exactly one of var and cov"):
        mb.score_var(rowptr, np.array([2, 4], np.int32), np.ones(2, np.float32), model)
    from mlease_b200._native import check
    with pytest.raises(mb.MleaseError, match="CSR rows only"):
        check(mb.lib().mlease_score_var(0, None, Dg, 1, None, None, np.ones(Dg, np.float32).ctypes.data, None, model.ctypes.data, 1, 0,
                                  v.ctypes.data, None, np.zeros(1, np.float32).ctypes.data, np.zeros(1, np.float32).ctypes.data))


def _ngpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.skipif(_ngpus() < 2, reason="needs 2 GPUs")
def test_world_two_gpus_against_one():
    """random partitions at D' = 121, then posterior_cases' window case at D' = 12 289 (the packed all-reduce past one column
    window), against fp64 and one GPU against two"""
    import posterior_cases as pc
    Dg, P = 120, 4
    wc = pc.window_case(12289)
    for parts, Dg, z, lm in [(_parts(P, 300, Dg, 0.08, seed=41), Dg, np.random.default_rng(3).normal(0, 0.2, Dg + 1), None),
                             (wc["parts"], wc["Dg"], wc["z"], wc["lambda_map"])]:
        res = []
        for devs in ([0], [0, 1]):
            w = mb.World(devs, len(parts), Dg, [1.0], lambda_map=lm)
            for pid, (rowptr, cols, vals, y, wt, o) in enumerate(parts):
                w.add_partition_csr(pid, rowptr, cols, vals, y, wt, o)
            w.begin()
            res.append(w.admm_posterior(0, z=z, full=True, want_cov=True))
            w.close()
        if lm is None:
            H = _hessian(parts, Dg, z) + np.diag(_q(Dg, 1.0))
            _check_inverse(res[0][1], H, "1 gpu")
            _check_inverse(res[1][1], H, "2 gpus")
            ev = np.linalg.eigvalsh(H)
            bound = 8 * H.shape[0] * ev[-1] / ev[0] * EPS * np.abs(res[0][1]).max()
        else:
            ref = pc.reference(wc)
            bound = pc.sigma_bound(wc, ref)
            for (_, cov), tag in zip(res, ("1 gpu", "2 gpus")):
                for r0 in range(0, Dg + 1, 2048):
                    r1 = min(Dg + 1, r0 + 2048)
                    assert np.abs(cov[r0:r1] - pc.sigma_rows(ref, Dg + 1, r0, r1)).max() <= bound, (tag, r0)
        assert np.abs(res[0][1] - res[1][1]).max() <= bound


def test_job_chain_on_the_fixture(tmp_path):
    """RegressionPrepare -> RegressionAdmmTrain -> RegressionPosterior on tests/golden/sample_data.npz (4 blocks), against numpy at
    the final model the job wrote"""
    import ctypes as C
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import avro_util as au
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    h = C.CDLL(os.path.join(root, "ml-ease_b200", "lib", "libmlease_host.so"))
    h.mlease_job_last_error.restype = C.c_char_p
    npz = np.load(os.path.join(root, "tests", "golden", "sample_data.npz"))
    recs = au.fixture_records(npz, with_key=lambda i: i // 250)
    au.write_avro(str(tmp_path / "in" / "part-0.avro"), au.pig_schema_with_key(), recs, block=300)
    out = tmp_path / "out"

    def run(job, kv, extra=""):
        p = tmp_path / (job + ".job")
        p.write_text("".join("%s=%s\n" % e for e in kv.items()) + extra)
        assert h.mlease_job_run(job.encode(), str(p).encode()) == 0, h.mlease_job_last_error().decode()

    run("Regression", {"input.paths": tmp_path / "in", "output.base.path": out, "map.key": "pkey", "num.blocks": 4, "num.iters": 5,
                       "regularizer": 2}, "lambda=1,10\n")
    sch, prep = au.read_avro(str(out / "tmp-data" / "part-00000.avro"))[:2]
    names = sorted({f["name"] + ("\x01" + f["term"] if f["term"] else "") for r in prep for f in r["features"]})
    for full in (False, True):
        run("RegressionPosterior", {"output.base.path": out, "num.blocks": 4, "compute.full.var": str(full).lower()}, "lambda=1,10\n")
        got = au.read_avro(str(out / "final-model-var" / "part-r-00000.avro"))[1]
        final = au.read_avro(str(out / "final-model" / "part-r-00000.avro"))[1]
        assert [r["key"] for r in got] == [r["key"] for r in final] and all(a["model"] == b["model"] for a, b in zip(got, final))
        for r in got:
            lam = float(r["key"])
            key = lambda f: f["name"] + ("\x01" + f["term"] if f["term"] else "")
            order = [key(f) for f in r["posteriorVar"][1:]]
            col = {k: j for j, k in enumerate(order)}
            Dg = len(order)
            zm = {key(f): f["value"] for f in r["model"]}
            z = np.array([float(zm.get(k, 0.0)) for k in order] + [float(zm["(INTERCEPT)"])])
            parts = []
            for p in range(4):
                rows = [x for x in prep if int(x["key"]) == p]
                rp, ci, vv = [0], [], []
                for x in rows:
                    ent = sorted((col[key(f)], f["value"]) for f in x["features"])
                    ci += [c for c, _ in ent]; vv += [v for _, v in ent]; rp.append(len(ci))
                parts.append((np.array(rp, np.int64), np.array(ci, np.int32), np.array(vv, np.float32),
                              np.array([x["response"] for x in rows]), np.array([x["weight"] for x in rows], np.float32),
                              np.array([x["offset"] for x in rows], np.float32)))
            H = _hessian(parts, Dg, z) + np.diag(_q(Dg, lam))
            ref = np.diag(np.linalg.inv(H)) if full else 1.0 / np.diag(H)
            v = np.array([f["value"] for f in r["posteriorVar"][1:]] + [r["posteriorVar"][0]["value"]], np.float64)
            assert np.allclose(v, ref.astype(np.float32), rtol=1e-5, atol=0), (full, lam, np.abs(v - ref).max())
