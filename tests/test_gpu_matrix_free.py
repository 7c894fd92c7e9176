"""Matrix-free Newton-CG x-update (-m gpu): the Hv mode of the CSR K1 kernels against the oracle's LogisticRegressionL2.Hv, ADMM
runs with hessian_policy = 2 against oracle-exact, the automatic selection for a model whose Hessian cannot be held, and the
error paths.  Tolerances: Hv 1e-5 relative (the K1 gradient's: fp32 products, fp64 reductions); z 1e-5 relative (north star)."""
import numpy as np
import pytest

from oracle import oracle as orc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mb():
    import mlease_b200
    return mlease_b200


def _sparse_parts(P, n, D, nnz, seed, binary=False):
    """P CSR partitions of n rows with nnz sorted unique columns each (one column per stride of D // nnz), and the pooled Csr.  With
    n >= D // nnz every column below nnz * (D // nnz) occurs in every partition: the reducers of the reference drop the features a
    partition lacks (llf/LibLinear.java:491-493), which the oracle restates."""
    rng = np.random.default_rng(seed)
    beta = rng.normal(size=D) / np.sqrt(nnz)
    stride = D // nnz
    parts, ci_all, v_all, y_all, w_all, o_all = [], [], [], [], [], []
    for p in range(P):
        r = np.random.default_rng(seed + 1 + p)
        ci = np.stack([k * stride + r.permutation(n) % stride for k in range(nnz)], axis=1).astype(np.int32)
        v = r.normal(size=(n, nnz)).astype(np.float32)
        sc = ((1.0 if binary else v) * beta[ci]).sum(1) - 0.5
        y = (r.random(n) < 1 / (1 + np.exp(-sc))).astype(np.int32)
        w = r.uniform(0.5, 2.0, n).astype(np.float32)
        o = r.normal(0, 0.1, n).astype(np.float32)
        parts.append((np.arange(n + 1, dtype=np.int64) * nnz, ci.reshape(-1), v.reshape(-1), y, w, o))
        ci_all.append(ci.reshape(-1)); v_all.append(v.reshape(-1)); y_all.append(y); w_all.append(w); o_all.append(o)
    data = orc.Csr(np.arange(P * n + 1, dtype=np.int64) * nnz, np.concatenate(ci_all), np.concatenate(v_all), np.concatenate(y_all),
                   np.concatenate(w_all), np.concatenate(o_all), n_features=D)
    return parts, data, [p * n for p in range(P + 1)]


# (rows, features, stored values per row, lambdas of the session, hessian_policy, no segment lists): mlease_hessian_vector runs on
# the session's one-problem scratch batch -- the fused kernel (default policy: a Gram-path scratch problem), the column windows
# (two lambdas at 30 001 columns: the 2-wide interleaved beta of the fused kernel does not fit a CTA's shared memory, so the upload
# builds no segment lists), and a width no Gram fits.  The multi-lambda and per-problem variants of the main batch:
# test_batch_hv_and_diagonal_match_oracle
@pytest.mark.parametrize("n,D,nnz,lambdas,policy,no_fused", [(4000, 300, 12, (0.1, 1.0, 10.0), 0, False),
                                                             (3000, 30001, 60, (1.0, 2.0), 2, True),
                                                             (3000, 200001, 100, (1.0,), 2, False)])
def test_hessian_vector_matches_oracle(mb, n, D, nnz, lambdas, policy, no_fused):
    parts, data, _ = _sparse_parts(1, n, D, nnz, seed=D)
    rng = np.random.default_rng(3)
    w = rng.normal(0, 0.3, D + 1); q = rng.uniform(0.5, 2.0, D + 1); v = rng.normal(size=D + 1)
    ref = orc.objective("Hv", data, w, np.zeros(D + 1), 1.0 / q, vec=v)
    outs = []
    for upload in range(2):
        with mb.AdmmSession(1, D, list(lambdas), hessian_policy=policy) as s:
            s.add_partition_csr(0, *parts[0])
            outs.append(s.hessian_vector(0, w, q, v))
            outs.append(s.hessian_vector(0, w, q, v))
            if no_fused:   # a policy-2 batch is cheap to allocate: it shows the partition has no segment lists
                s.begin()
                assert s.stats()["k1_fused"] == 0
    # the oracle leaves the entries of features no row lists at 0 (it drops them from the dataset): there Hv = q v exactly
    present = np.zeros(D + 1, bool); present[parts[0][1]] = True; present[D] = True
    err = np.abs(outs[0] - ref)[present].max() / np.abs(ref).max()
    assert err <= 1e-5, err
    np.testing.assert_array_equal(outs[0][~present], q[~present] * v[~present])
    for o in outs[1:]:
        np.testing.assert_array_equal(o, outs[0])   # call to call and upload to upload


def _part_csr(part, D):
    rp, ci, v, y, w, o = part
    return orc.Csr(rp, ci, v, y, w, o, D)


# (partitions, rows, features, stored values per row, lambdas, no segment lists): the ADMM batch of a policy-2 session through the
# kernels its CG runs -- fused multi-lambda with 4- and 2-wide interleaved vectors, the per-problem fixed-point kernel with its
# accumulators and v in shared memory (5 lambdas: no fused kernel) under the dynamic CTA mapping, the same kernel reading v from
# global memory (3 lambdas at 20 003 columns: the 4-wide interleaved vectors of the fused kernel do not fit), and the column windows
# (2 lambdas at 30 001 columns: no segment lists, see test_hessian_vector_matches_oracle)
@pytest.mark.parametrize("P,n,D,nnz,L,no_fused", [(2, 3000, 300, 12, 3, False), (2, 3000, 300, 12, 2, False), (2, 3000, 300, 12, 5, False),
                                                  (1, 2000, 20003, 40, 3, True), (2, 2000, 30001, 60, 2, True)])
def test_batch_hv_and_diagonal_match_oracle(mb, P, n, D, nnz, L, no_fused):
    """Every (partition, lambda) problem at its own point w and vector v: a wrong lambda's v or d, or a wrong diagonal, fails here (the
    ADMM parity cases could not see it: any SPD model leads the line search to the same minimiser).  Each column is also held to the
    bound of tests/k1_reference.py, with the pass's chunking as the gradient hook reports it for the same batch."""
    import k1_reference as kr
    from mlease_b200._native import ptr, check
    from mlease_b200 import _hooks
    parts, _, _ = _sparse_parts(P, n, D, nnz, seed=D + L)
    rng = np.random.default_rng(L)
    nprob = P * L
    w = rng.normal(0, 0.3, (nprob, D + 1)); v = rng.normal(size=(nprob, D + 1))
    big = np.full(D + 1, 1e30)   # prior variance: the oracle's prior term vanishes, the hook returns the data term
    fn = _hooks.bound().mlease_internal_batch_hv
    with mb.AdmmSession(P, D, [0.5 * (l + 1) for l in range(L)], hessian_policy=2) as s:
        for p, part in enumerate(parts):
            s.add_partition_csr(p, *part)
        s.begin()
        assert s.stats()["k1_fused"] == (0 if no_fused or L > 4 else 1)
        info = _hooks.batch_grad(s, w)   # all problems, as in the Hv / diagonal passes: the same CTA mapping
        assert info["kind"] == ("fused" if s.stats()["k1_fused"] else "fx_window" if D > 28000 else "fx")
        for mode, name in ((1, "Hv"), (2, "hessian_diag")):
            outs = []
            for rep in range(2):
                out = np.zeros((nprob, D + 1))
                check(fn(s._h, mode, ptr(w), ptr(v), ptr(out)))
                outs.append(out)
            np.testing.assert_array_equal(outs[0], outs[1])
            for b in range(nprob):
                data = _part_csr(parts[b // L], D)
                ref = orc.objective(name, data, w[b], np.zeros(D + 1), big, vec=v[b] if mode == 1 else None)
                err = np.abs(outs[0][b] - ref).max() / np.abs(ref).max()
                assert err <= 1e-5, (name, b, err)
                rp, ci, vv, yy, ww, oo = parts[b // L]
                part = kr.Part.from_csr(rp, ci, vv, yy, ww, oo, D)
                rowl1 = np.float32(np.bincount(part.rows, np.abs(vv.astype(np.float64)), part.n).max() * (1 + 1e-5))
                vinf = np.abs(v[b].astype(np.float32)).max()
                ref64, bnd = kr.hv_reference_and_bound(part, w[b], v[b], mode, kr.plan_from_info(info, b, part.n), rowl1, vinf)
                r = kr.ratio(outs[0][b] - ref64, bnd)
                assert np.all(r <= 1.0), (name, b, int(np.argmax(r)), float(r.max()))
                print("Hv bound %s %s L=%d D=%d: worst error/bound %.3e" % (name, info["kind"], L, D, r.max()))


def test_policy2_session_builds_no_gram_list(mb):
    """A matrix-free session builds no block-major Gram list at upload (n D'/512 offsets + 6 B per stored value): the same partition
    holds that much less device memory under hessian_policy = 2 than under the default policy."""
    import torch
    n, D, nnz = 200000, 200000, 50
    parts, _, _ = _sparse_parts(1, n, D, nnz, seed=5)
    torch.cuda.init(); torch.cuda.synchronize()
    used = {}
    z = np.zeros(D + 1)
    for policy in (0, 2):
        with mb.AdmmSession(1, D, [1.0], hessian_policy=policy) as s:
            s.add_partition_csr(0, *parts[0])
            s.hessian_vector(0, z, np.ones(D + 1), np.ones(D + 1))   # finishes the upload, same matrix-free scratch problem for both
            used[policy] = torch.cuda.mem_get_info(0)[1] - torch.cuda.mem_get_info(0)[0]
    list_bytes = 6 * (n * nnz + n) + 8 * (((D + 1 + 3) // 4 * 4 + 127) // 128 * ((n + 31) // 32))
    assert used[0] - used[2] >= 0.9 * list_bytes, (used, list_bytes)


def _fixture_parts(d, prs):
    parts = []
    for p in range(len(prs) - 1):
        r0, r1 = prs[p], prs[p + 1]
        rp = d.rowptr[r0:r1 + 1] - d.rowptr[r0]
        sl = slice(d.rowptr[r0], d.rowptr[r1])
        parts.append((rp, d.colidx[sl], d.val[sl], d.response[r0:r1], d.weight[r0:r1], d.offset[r0:r1]))
    return parts


# case -> (data builder, lambdas, iterations, session / oracle options)
CASES = {
    "fixture": ("fixture", [1.0, 10.0, 100.0], 6, {}),
    "cfg3_equal_rho": ((2, 6000, 1500, 15, 77), [0.1, 1.0, 10.0], 6, {}),
    "cfg3_distinct_rho": ((2, 6000, 1500, 15, 77), [0.1, 1.0, 10.0], 6, dict(rhos=[1.0, 3.0, 0.5])),
    "l1": ((3, 2000, 300, 10, 71), [0.3, 3.0], 8, dict(regularizer=1)),
    "lambda_map": ((2, 3000, 300, 12, 300), [2.0, 30.0], 6, dict(lambda_map="every7")),
    "binary_feature": ((2, 4000, 500, 10, 400), [0.5, 5.0], 6, dict(binary_feature=True)),
    "rho_adapt": ((2, 3000, 400, 10, 500), [1.0, 10.0], 6, dict(rho_adapt_coefficient=0.3)),
    "boost": ("fixture", [1.0, 10.0], 6, dict(boost=2.5)),
    "penalize_intercept": ((2, 3000, 400, 10, 600), [1.0, 10.0], 6, dict(penalize_intercept=True)),
    "stop_rule": ((2, 1500, 60, 6, 700), [10.0], 300, dict(epsilon=1e-3)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_admm_matrix_free_matches_oracle_exact(mb, fixture_data, frozen, case):
    """hessian_policy = 2 pins the matrix-free x-update at sizes where the Gram path also runs: a different solver reaching the same
    minimisers, so the ADMM iterates match oracle-exact at the same iteration count (and the stop rule fires at the same one)."""
    src, lambdas, niters, opts = CASES[case]
    opts = dict(opts)
    if src == "fixture":
        data, prs = fixture_data, frozen["part_rowstart"]
        parts, D = _fixture_parts(data, prs), data.n_features
    else:
        P, n, D, nnz, seed = src
        parts, data, prs = _sparse_parts(P, n, D, nnz, seed, binary=opts.get("binary_feature", False))
    if opts.get("lambda_map") == "every7":
        lm = np.zeros(D, np.float32); lm[::7] = 0.2
        opts["lambda_map"] = lm
    boost = opts.pop("boost", 0.0)
    eps = opts.pop("epsilon", 0.0)
    ref = orc.admm_run(data, prs, lambdas, niters=niters, mode="exact", nthreads=8, epsilon=eps, initialize_boost_rate=boost, **opts)
    with mb.AdmmSession(len(parts), D, lambdas, epsilon=eps, hessian_policy=2, **opts) as s:
        for p, part in enumerate(parts):
            s.add_partition_csr(p, *part)
        if boost:
            s.begin(s.mean_naive_model(range(len(parts))), boost)
            done = 0
            for _ in range(niters):
                s.iterate()
                done += 1
        else:
            done = s.run(niters)
        z = np.stack([s.z(l) for l in range(len(lambdas))])
        st = s.stats()
    assert done == ref["iters_done"], (done, ref["iters_done"])
    zr = ref["z_hist"][-1]
    for l in range(len(lambdas)):
        err = np.abs(z[l] - zr[l]).max() / np.abs(zr[l]).max()
        assert err <= 1e-5, (case, l, err, st)
    assert st["not_converged"] == 0 and st["gram_builds"] == 0, st


def test_wide_model_selects_matrix_free_automatically(mb):
    """2 partitions x 3000 rows x 200 000 features (100 per row), lambda in {0.1, 1, 10}: the Gram path would need ~1 TB per problem,
    so the session builds the batch matrix-free on its own (no Gram build, Hessian-category launches) and lands on oracle-exact,
    bitwise equal to the same run with hessian_policy = 2."""
    D, lambdas, niters = 200000, [0.1, 1.0, 10.0], 4
    parts, data, prs = _sparse_parts(2, 3000, D, 100, seed=900)
    zs = []
    for policy in (0, 2):
        with mb.AdmmSession(2, D, lambdas, epsilon=0.0, hessian_policy=policy) as s:
            for p, part in enumerate(parts):
                s.add_partition_csr(p, *part)
            s.profile(2)
            assert s.run(niters) == niters
            prof = s.profile(-1)
            st = s.stats()
            zs.append(np.stack([s.z(l) for l in range(3)]))
        assert st["gram_builds"] == 0 and st["not_converged"] == 0, st
        assert prof["launches"]["gram"] > 0 and prof["gram_flops"] == 0, prof
    np.testing.assert_array_equal(zs[0], zs[1])
    ref = orc.admm_run(data, prs, lambdas, niters=niters, mode="exact", nthreads=8, epsilon=0.0)
    for l in range(3):
        zr = ref["z_hist"][-1, l]
        err = np.abs(zs[0][l] - zr).max() / np.abs(zr).max()
        assert err <= 1e-5, (l, err)


def test_matrix_free_errors(mb):
    """A Newton step cap that cannot be met is "Model fitting error!" (MLEASE_ERR_NUMERIC), as on the Gram path; dense partitions
    have no Hv pass, so policy 2 rejects them (MLEASE_ERR_INVALID)."""
    parts, _, _ = _sparse_parts(1, 4000, 50, 8, seed=13)
    rp, ci, v, y, w, o = parts[0]
    with mb.AdmmSession(1, 50, [1e-3], rhos=[1e-3], epsilon=0.0, max_newton=1, hessian_policy=2) as s:
        s.add_partition_csr(0, rp, ci, v * 3.0, y, w, o)
        with pytest.raises(mb.MleaseError, match="Model fitting error") as e:
            s.run(3)
        assert e.value.code == 3
    X = np.random.default_rng(1).normal(size=(200, 6)).astype(np.float32)
    with mb.AdmmSession(1, 6, [1.0], hessian_policy=2) as s:
        s.add_partition_dense(0, X, (X[:, 0] > 0).astype(np.int32))
        with pytest.raises(mb.MleaseError, match="hessian_policy 2") as e:
            s.run(1)
        assert e.value.code == 1
