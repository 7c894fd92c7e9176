"""GPU parity tests (-m gpu): the CUDA path, called through the C ABI, against the CPU oracle on the same
seeded inputs.  Tolerances: objective/gradient 1e-5 relative (fp32 data path, fp64 reductions); Gram (bf16
tensor-core operands) 2e-2 vs the fp64 Hessian and 1e-3 vs the fp32 SIMT kernel on the same bf16 operand;
coefficients / z: 1e-5 relative (north star)."""
import os
import sys

import numpy as np
import pytest

from oracle import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gram_reference import e4m3_round  # noqa: E402

pytestmark = pytest.mark.gpu


def _mk(n, d, seed, sparse=False, density=0.3):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)).astype(np.float32)
    if sparse:
        X *= rng.random((n, d)) < density
    beta = rng.normal(size=d) / np.sqrt(d)
    y = (rng.random(n) < 1 / (1 + np.exp(-(X @ beta - 0.5)))).astype(np.int32)
    w = rng.uniform(0.5, 2.0, n).astype(np.float32)
    o = rng.normal(0, 0.1, n).astype(np.float32)
    return X, y, w, o


def _csr_of(X):
    rp, ci, v = [0], [], []
    for i in range(X.shape[0]):
        nz = np.nonzero(X[i])[0]
        ci += list(nz); v += list(X[i, nz]); rp.append(len(ci))
    return np.array(rp, np.int64), np.array(ci, np.int32), np.array(v, np.float32)


def _session(mb, D, lambdas=(1.0,), P=1, **kw):
    return mb.AdmmSession(P, D, list(lambdas), **kw)


@pytest.fixture(scope="module")
def mb():
    import mlease_b200
    return mlease_b200


@pytest.mark.parametrize("n,d,sparse", [(1000, 37, False), (777, 100, False), (300, 1100, False), (500, 2500, False), (1000, 50, True),
                                        (4000, 3000, True), (50, 20, True), (20000, 700, True)])
def test_k1_objective_and_gradient(mb, n, d, sparse):
    """One K1 pass (loss + gradient) against the oracle's fun/grad.  CSR partitions with sorted unique rows take the fused
    segment-list kernel (column sums in registers in row order, no atomics); the pass must be bitwise reproducible from
    call to call AND from upload to upload (the layout is rebuilt), whatever order the warps retire in."""
    X, y, w, o = _mk(n, d, seed=n + d, sparse=sparse)
    rng = np.random.default_rng(1)
    wv = rng.normal(0, 0.3, d + 1); pm = rng.normal(0, 0.3, d + 1); pv = rng.uniform(0.2, 2.0, d + 1)
    if sparse:
        with _session(mb, d) as s0:
            s0.add_partition_csr(0, *_csr_of(X), y, w, o)
            f0, g0, _ = s0.objective(0, wv, pm, 1.0 / pv)
    with _session(mb, d) as s:
        if sparse:
            rp, ci, v = _csr_of(X)
            s.add_partition_csr(0, rp, ci, v, y, w, o)
            data = orc.Csr(rp, ci, v, y, w, o, d)
        else:
            s.add_partition_dense(0, X, y, w, o)
            data = orc.Csr.from_dense(X, y, w, o)
        f, g, _ = s.objective(0, wv, pm, 1.0 / pv)
        f2, g2, _ = s.objective(0, wv, pm, 1.0 / pv)
    f_ref, g_ref = orc.objective("grad", data, wv, pm, pv)
    assert abs(f - f_ref) <= 1e-5 * abs(f_ref), (f, f_ref)
    assert np.abs(g - g_ref).max() <= 1e-5 * np.abs(g_ref).max(), np.abs(g - g_ref).max() / np.abs(g_ref).max()
    assert f == f2 and np.array_equal(g, g2)
    if sparse:
        assert f == f0 and np.array_equal(g, g0)


@pytest.mark.parametrize("n,d", [(1000, 50), (4000, 3000)])
def test_k1_per_problem_csr_kernels_without_segment_lists(mb, n, d):
    """The pre-fusion CSR K1 (two-word fixed-point accumulation with native integer shared-memory atomics) stays the path for
    partitions without segment lists (more than 4 lambdas, feature spaces too wide for the builder): same parity gate.  A session
    of 5 lambdas uploads its partitions without them."""
    X, y, w, o = _mk(n, d, seed=n + d, sparse=True)
    rng = np.random.default_rng(1)
    wv = rng.normal(0, 0.3, d + 1); pm = rng.normal(0, 0.3, d + 1); pv = rng.uniform(0.2, 2.0, d + 1)
    rp, ci, v = _csr_of(X)
    with _session(mb, d, lambdas=(0.1, 0.3, 1.0, 3.0, 10.0)) as s:
        s.add_partition_csr(0, rp, ci, v, y, w, o)
        f, g, _ = s.objective(0, wv, pm, 1.0 / pv)
        f2, g2, _ = s.objective(0, wv, pm, 1.0 / pv)
        x, _ = s.fit_partition(0, np.zeros(d + 1), pm, 1.0 / pv)
        s.begin()
        assert s.stats()["k1_fused"] == 0
    data = orc.Csr(rp, ci, v, y, w, o, d)
    f_ref, g_ref = orc.objective("grad", data, wv, pm, pv)
    assert abs(f - f_ref) <= 1e-5 * abs(f_ref) and np.abs(g - g_ref).max() <= 1e-5 * np.abs(g_ref).max()
    assert f == f2 and np.array_equal(g, g2)
    x_ref, _ = orc.liblinear_train(data, np.zeros(d + 1), pm, pv, 1e-14, 100000)
    assert np.abs(x - x_ref).max() <= 1e-5 * np.abs(x_ref).max()


def test_csr_rows_with_repeated_and_unsorted_columns(mb):
    """Rows may list a column twice or out of order (TRON's fun/grad/Hv accept that: llf/LogisticRegressionL2.java:115-150;
    only the reference's hessian() insists on sorted rows, :277).  Such partitions take the general CSR kernels (float
    gradient accumulation, dense bf16 Gram operand): same objective, gradient, Hessian and fit as the merged rows."""
    n, d = 1500, 60
    X, y, w, o = _mk(n, d, seed=91, sparse=True)
    rng = np.random.default_rng(4)
    rp, ci, v = [0], [], []
    for i in range(n):
        cols = np.nonzero(X[i])[0]
        vals = X[i, cols].astype(np.float32)
        if len(cols):   # split the first entry in two, then shuffle the row
            cols = np.concatenate([cols, cols[:1]]); vals = np.concatenate([vals, vals[:1] * np.float32(0.25)]); vals[0] *= np.float32(0.75)
            perm = rng.permutation(len(cols)); cols, vals = cols[perm], vals[perm]
        ci += list(cols); v += list(vals); rp.append(len(ci))
    rp = np.array(rp, np.int64); ci = np.array(ci, np.int32); v = np.array(v, np.float32)
    Xm = np.zeros((n, d), np.float32)
    for i in range(n):
        np.add.at(Xm[i], ci[rp[i]:rp[i + 1]], v[rp[i]:rp[i + 1]])
    data = orc.Csr.from_dense(Xm, y, w, o)
    wv = rng.normal(0, 0.3, d + 1); pm = rng.normal(0, 0.2, d + 1); pv = np.full(d + 1, 0.7)
    with _session(mb, d) as s:
        s.add_partition_csr(0, rp, ci, v, y, w, o)
        f, g, H = s.objective(0, wv, pm, 1.0 / pv, want_hessian=True, tensor=True)
        _, _, H_simt = s.objective(0, wv, pm, 1.0 / pv, want_hessian=True, tensor=False)   # the dense operand exists on this path
        x, _ = s.fit_partition(0, np.zeros(d + 1), pm, 1.0 / pv)
    f_ref, g_ref = orc.objective("grad", data, wv, pm, pv)
    H_ref = orc.objective("hessian", data, wv, pm, pv)
    assert abs(f - f_ref) <= 1e-5 * abs(f_ref)
    assert np.abs(g - g_ref).max() <= 1e-5 * np.abs(g_ref).max()
    assert np.abs(H - H_ref).max() <= 2e-2 * np.abs(H_ref).max() and np.abs(H - H_simt).max() <= 1e-3 * np.abs(H_ref).max()
    x_ref, _ = orc.liblinear_train(data, np.zeros(d + 1), pm, pv, 1e-14, 100000)
    assert np.abs(x - x_ref).max() <= 1e-5 * np.abs(x_ref).max()


@pytest.mark.parametrize("fused", [False, True])
def test_csr_feature_space_wider_than_one_gradient_window(mb, fused):
    """30 001 columns: the per-CTA fixed-point gradient (8 bytes per column) no longer fits shared memory in one piece, so
    K1 runs one launch for the margins + the first 28 128 columns and one more per further column window; the Gram tile
    list, the DMMA factorisation and the fp32 inverse copy are exercised at ldh = 30 016 as well.  With one lambda the
    partition gets segment lists and the fused kernel takes the 30k columns in one launch; with two, the 2-wide interleaved
    beta (240 032 B) does not fit a CTA's shared memory, so there are no lists and the column-window kernels run."""
    lambdas = (1.0,) if fused else (1.0, 2.0)
    n, D, nnz = 3000, 30000, 8
    r = np.random.default_rng(12)
    ci = np.stack([np.sort(r.choice(D, nnz, replace=False)) for _ in range(n)]).astype(np.int32)
    ci[:, -1] = D - 1 - (np.arange(n) % 5)            # make sure the last window and the columns next to the intercept are hit
    ci.sort(axis=1)
    for i in range(n):                                 # keep rows strictly increasing after the overwrite
        while len(np.unique(ci[i])) < nnz:
            ci[i] = np.sort(r.choice(D, nnz, replace=False))
    v = r.normal(size=(n, nnz)).astype(np.float32)
    beta = r.normal(size=D) / np.sqrt(nnz)
    y = (r.random(n) < 1 / (1 + np.exp(-((v * beta[ci]).sum(1) - 0.3)))).astype(np.int32)
    w = r.uniform(0.5, 2.0, n).astype(np.float32); o = r.normal(0, 0.1, n).astype(np.float32)
    rp = np.arange(n + 1, dtype=np.int64) * nnz
    data = orc.Csr(rp, ci.reshape(-1), v.reshape(-1), y, w, o, D)
    wv = r.normal(0, 0.3, D + 1); pm = r.normal(0, 0.3, D + 1); pv = r.uniform(0.5, 2.0, D + 1)
    # columns that never occur in the partition are not part of the reference's local problem (llf/LibLinear.java:491-493;
    # their coefficient is the prior mean, :374-383): evaluate at a point that agrees with that, so that fun/grad compare
    absent = np.ones(D + 1, bool); absent[ci.reshape(-1)] = False; absent[D] = False
    wv[absent] = pm[absent]
    with _session(mb, D, lambdas) as s:
        s.add_partition_csr(0, rp, ci.reshape(-1), v.reshape(-1), y, w, o)
        f, g, _ = s.objective(0, wv, pm, 1.0 / pv)
        l0 = s.stats()["kernel_launches"]
        f2, g2, _ = s.objective(0, wv, pm, 1.0 / pv)
        launches = s.stats()["kernel_launches"] - l0
        x, steps = s.fit_partition(0, np.zeros(D + 1), pm, 1.0 / pv)
    if not fused:   # the same upload with one lambda: the column windows are one launch more than the fused kernel's one
        with _session(mb, D) as s1:
            s1.add_partition_csr(0, rp, ci.reshape(-1), v.reshape(-1), y, w, o)
            s1.objective(0, wv, pm, 1.0 / pv)
            l0 = s1.stats()["kernel_launches"]
            s1.objective(0, wv, pm, 1.0 / pv)
            assert launches == s1.stats()["kernel_launches"] - l0 + 1, launches
    f_ref, g_ref = orc.objective("grad", data, wv, pm, pv)
    assert abs(f - f_ref) <= 1e-5 * abs(f_ref), (f, f_ref)
    assert np.abs(g - g_ref).max() <= 1e-5 * np.abs(g_ref).max(), np.abs(g - g_ref).max() / np.abs(g_ref).max()
    assert f == f2 and np.array_equal(g, g2)
    x_ref, _ = orc.liblinear_train(data, np.zeros(D + 1), pm, pv, 1e-14, 100000)
    assert np.abs(x - x_ref).max() <= 1e-5 * np.abs(x_ref).max(), (np.abs(x - x_ref).max() / np.abs(x_ref).max(), steps)


@pytest.mark.parametrize("n,d,sparse", [(1000, 37, False), (2000, 100, False), (700, 300, False), (1000, 50, True), (3000, 700, True),
                                        (333, 255, True)])
def test_gram_tcgen05_vs_oracle_hessian(mb, n, d, sparse):
    """Dense partitions: the wgmma Gram against the fp64 Hessian and against the fp32 SIMT kernel on the same bf16 operand.
    CSR partitions assemble their operand tiles from the CSR rows inside the Gram kernel (no dense copy exists, so no SIMT
    run) as e4m3 with a power-of-two scale (wgmma .e4m3, twice the bf16 MMA rate; H only preconditions): the check is against
    a numpy emulation of the e4m3-rounded scaled rows."""
    X, y, w, o = _mk(n, d, seed=3 * n + d, sparse=sparse)
    rng = np.random.default_rng(2)
    wv = rng.normal(0, 0.3, d + 1); pm = np.zeros(d + 1); pv = np.full(d + 1, 0.5)
    with _session(mb, d) as s:
        if sparse:
            rp, ci, v = _csr_of(X)
            s.add_partition_csr(0, rp, ci, v, y, w, o)
            data = orc.Csr(rp, ci, v, y, w, o, d)
        else:
            s.add_partition_dense(0, X, y, w, o)
            data = orc.Csr.from_dense(X, y, w, o)
        _, _, H_tc = s.objective(0, wv, pm, 1.0 / pv, want_hessian=True, tensor=True)
        if sparse:
            with pytest.raises(mb.MleaseError):
                s.objective(0, wv, pm, 1.0 / pv, want_hessian=True, tensor=False)
        else:
            _, _, H_simt = s.objective(0, wv, pm, 1.0 / pv, want_hessian=True, tensor=False)
    H_ref = orc.objective("hessian", data, wv, pm, pv)
    scale = np.abs(H_ref).max()
    if sparse:
        Xb = np.hstack([X.astype(np.float64), np.ones((n, 1))])
        p = 1.0 / (1.0 + np.exp(-(Xb @ wv + o)))
        dd = w * p * (1 - p)
        prior = H_ref - (Xb * dd[:, None]).T @ Xb
        sd = np.sqrt(dd).astype(np.float32)
        amax = 0.5 * np.sqrt(np.float32(w.max())) * max(float(np.abs(v).max()), 1.0)
        g = 2.0 ** (np.frexp(np.float32(224.0) / np.float32(amax))[1] - 1)           # the library's power-of-two operand scale
        Xt = e4m3_round((Xb.astype(np.float32) * (sd * np.float32(g))[:, None]).astype(np.float32)) / g
        H_simt = Xt.T @ Xt + prior
    e_simt = np.abs(H_simt - H_ref).max() / scale
    e_tc = np.abs(H_tc - H_ref).max() / scale
    e_x = np.abs(H_tc - H_simt).max() / scale
    assert e_simt < 2e-2, ("simt vs oracle", e_simt)
    assert e_tc < 2e-2, ("wgmma vs oracle", e_tc, e_simt, e_x)
    assert e_x < 1e-3, ("wgmma vs simt", e_x)


@pytest.mark.parametrize("n,d,sparse", [(1500, 100, False), (3000, 700, False), (2500, 1100, False), (4000, 2303, False), (5000, 2600, True)])
def test_inverse_times_hessian_is_identity(mb, n, d, sparse):
    """The explicit inverse behind every Newton direction, for both factorisation paths: ldh <= 1000 (NB=32 right-looking
    Cholesky, substitution inverse, SIMT product) and ldh > 1000 (outer panels + DMMA trailing updates, recursive inverse
    with DMMA merges, DMMA Y^T Y), including a width that is not a multiple of the leaf / panel size."""
    X, y, w, o = _mk(n, d, seed=7 * n + d, sparse=sparse, density=0.05 if sparse else 0.3)
    rng = np.random.default_rng(5)
    wv = rng.normal(0, 0.3 / np.sqrt(d), d + 1); pm = np.zeros(d + 1); pv = np.full(d + 1, 0.5)
    with _session(mb, d) as s:
        if sparse:
            rp, ci, v = _csr_of(X)
            s.add_partition_csr(0, rp, ci, v, y, w, o)
        else:
            s.add_partition_dense(0, X, y, w, o)
        _, _, H = s.objective(0, wv, pm, 1.0 / pv, want_hessian=True, tensor=True)
        _, _, Hinv = s.objective(0, wv, pm, 1.0 / pv, want_hessian=True, tensor=2)
    assert np.abs(Hinv - Hinv.T).max() == 0.0
    err = np.abs(Hinv @ H - np.eye(d + 1)).max()
    assert err < 1e-9, err


@pytest.mark.parametrize("n,d", [(1500, 20), (3000, 100), (800, 300)])
def test_fit_partition_matches_exact_tron(mb, n, d):
    X, y, w, o = _mk(n, d, seed=11 * n + d)
    rng = np.random.default_rng(3)
    pm = rng.normal(0, 0.2, d + 1); pv = np.full(d + 1, 1.0); init = rng.normal(0, 0.1, d + 1)
    with _session(mb, d) as s:
        s.add_partition_dense(0, X, y, w, o)
        x, steps = s.fit_partition(0, init, pm, 1.0 / pv)
        st = s.stats()
    x_ref, _ = orc.liblinear_train(orc.Csr.from_dense(X, y, w, o), init, pm, pv, 1e-14, 100000)
    err = np.abs(x - x_ref).max() / np.abs(x_ref).max()
    assert err < 1e-6, (err, steps, st)
    assert 1 <= steps <= 30 and st["not_converged"] == 0


def _run_gpu_admm(mb, parts, D, lambdas, niters, csr, **kw):
    P = len(parts)
    with mb.AdmmSession(P, D, lambdas, **kw) as s:
        for p, part in enumerate(parts):
            (s.add_partition_csr if csr else s.add_partition_dense)(p, *part)
        done = s.run(niters)
        z = np.stack([s.z(l) for l in range(len(lambdas))])
        xs = np.stack([[s.x(p, l) for l in range(len(lambdas))] for p in range(P)])
        us = np.stack([[s.u(p, l) for l in range(len(lambdas))] for p in range(P)])
        st = s.stats()
    return done, z, xs, us, st


def test_admm_fixture_csr_matches_oracle_exact(mb, fixture_data, frozen):
    d = fixture_data
    prs = frozen["part_rowstart"]
    parts = []
    for p in range(len(prs) - 1):
        r0, r1 = prs[p], prs[p + 1]
        rp = d.rowptr[r0:r1 + 1] - d.rowptr[r0]
        sl = slice(d.rowptr[r0], d.rowptr[r1])
        parts.append((rp, d.colidx[sl], d.val[sl], d.response[r0:r1], d.weight[r0:r1], d.offset[r0:r1]))
    lambdas = [1.0, 10.0, 100.0]
    for niters in (1, 2, 20):
        done, z, xs, us, st = _run_gpu_admm(mb, parts, d.n_features, lambdas, niters, csr=True, epsilon=0.0)
        ref = frozen["exact_z_hist"][niters - 1]
        for l in range(3):
            err = np.abs(z[l] - ref[l]).max() / np.abs(ref[l]).max()
            assert err < 1e-5, (niters, l, err, st)
    # last-iteration reducer outputs (x double, u float) vs the oracle
    assert np.abs(xs - frozen["exact_x_last"]).max() / np.abs(frozen["exact_x_last"]).max() < 1e-5
    # u after consensus of iteration 20 = what computeU writes for iteration 21: float(uplusx_20 - z_20)
    oracle_run = orc.admm_run(d, prs, lambdas, niters=20, mode="exact", nthreads=4, epsilon=0.0)
    u_next = (oracle_run["uplusx_last"].astype(np.float64) - oracle_run["z_hist"][-1][None]).astype(np.float32)
    assert np.abs(us - u_next).max() / np.abs(u_next).max() < 2e-5
    assert st["not_converged"] == 0


def test_admm_dense_config1_shape_matches_oracle_exact(mb):
    # BASELINE config 0: 2 partitions x 10k x 100 dense, lambda = 1
    P, n, D = 2, 10000, 100
    parts, Xs, ys = [], [], []
    rng = np.random.default_rng(1000)
    beta = rng.normal(size=D) / np.sqrt(D)
    for p in range(P):
        r = np.random.default_rng(1000 + p)
        X = r.normal(size=(n, D)).astype(np.float32)
        y = (r.random(n) < 1 / (1 + np.exp(-(X @ beta - 1.0)))).astype(np.int32)
        parts.append((X, y)); Xs.append(X); ys.append(y)
    data = orc.Csr.from_dense(np.vstack(Xs), np.concatenate(ys))
    ref = orc.admm_run(data, [0, n, 2 * n], [1.0], niters=10, mode="exact", nthreads=4, epsilon=0.0)
    done, z, xs, us, st = _run_gpu_admm(mb, parts, D, [1.0], 10, csr=False, epsilon=0.0)
    err = np.abs(z[0] - ref["z_hist"][-1, 0]).max() / np.abs(ref["z_hist"][-1, 0]).max()
    assert done == 10 and err < 1e-5, (err, st)
    fa = orc.admm_run(data, [0, n, 2 * n], [1.0], niters=10, mode="faithful", nthreads=4, epsilon=0.0)
    gap = np.abs(z[0] - fa["z_hist"][-1, 0]).max() / np.abs(z[0]).max()
    assert gap < 5e-2   # informational bound vs the loose-tolerance reference schedule (SURVEY 8c iii)


def test_admm_sparse_config3_shape_multi_lambda(mb):
    # BASELINE config 2 shape in small: sparse rows (1% nnz), multi-lambda {0.1,1,10} in one run, 2 partitions
    P, n, D, nnz = 2, 6000, 1500, 15
    rng = np.random.default_rng(77)
    beta = rng.normal(size=D) / np.sqrt(nnz)
    parts, rp_all, ci_all, v_all, y_all = [], [0], [], [], []
    for p in range(P):
        r = np.random.default_rng(1000 + p)
        ci = np.stack([np.sort(r.choice(D, nnz, replace=False)) for _ in range(n)]).astype(np.int32)
        v = r.normal(size=(n, nnz)).astype(np.float32)
        s = (v * beta[ci]).sum(1) - 0.5
        y = (r.random(n) < 1 / (1 + np.exp(-s))).astype(np.int32)
        rp = np.arange(n + 1, dtype=np.int64) * nnz
        parts.append((rp, ci.reshape(-1), v.reshape(-1), y))
        ci_all.append(ci.reshape(-1)); v_all.append(v.reshape(-1)); y_all.append(y)
    data = orc.Csr(np.arange(P * n + 1, dtype=np.int64) * nnz, np.concatenate(ci_all), np.concatenate(v_all), np.concatenate(y_all), n_features=D)
    lambdas = [0.1, 1.0, 10.0]
    ref = orc.admm_run(data, [0, n, 2 * n], lambdas, niters=6, mode="exact", nthreads=8, epsilon=0.0)
    done, z, xs, us, st = _run_gpu_admm(mb, parts, D, lambdas, 6, csr=True, epsilon=0.0)
    for l in range(3):
        err = np.abs(z[l] - ref["z_hist"][-1, l]).max() / np.abs(ref["z_hist"][-1, l]).max()
        assert err < 1e-5, (l, err, st)
    assert st["not_converged"] == 0
    # equal rho (the default) lets the cold start share one Gram AND one factorisation per partition across the lambdas;
    # distinct rho shares only the Gram: both must land on the oracle
    rhos = [1.0, 3.0, 0.5]
    ref = orc.admm_run(data, [0, n, 2 * n], lambdas, rhos=rhos, niters=6, mode="exact", nthreads=8, epsilon=0.0)
    done, z, xs, us, st = _run_gpu_admm(mb, parts, D, lambdas, 6, csr=True, epsilon=0.0, rhos=rhos)
    for l in range(3):
        err = np.abs(z[l] - ref["z_hist"][-1, l]).max() / np.abs(ref["z_hist"][-1, l]).max()
        assert err < 1e-5, (l, err, st)
    assert st["not_converged"] == 0


def test_admm_wide_systems_keep_the_cold_start_factor(mb):
    """D' > 2048: the cost model marks a refactorisation as too expensive to repeat mid-run, so every x-update after the
    first runs on the factor of the cold start (shared across the lambdas), corrected by L-BFGS pairs and the self-scaling
    of the stale inverse; the wide (DMMA) Cholesky / inverse path is the one in use.  Same gate: oracle-exact z to 1e-5."""
    P, n, D, nnz = 2, 8000, 2300, 20
    rng = np.random.default_rng(5)
    beta = rng.normal(size=D) / np.sqrt(nnz)
    parts, ci_all, v_all, y_all = [], [], [], []
    for p in range(P):
        r = np.random.default_rng(2000 + p)
        ci = np.stack([np.sort(r.choice(D, nnz, replace=False)) for _ in range(n)]).astype(np.int32)
        v = r.normal(size=(n, nnz)).astype(np.float32)
        s = (v * beta[ci]).sum(1) - 0.5
        y = (r.random(n) < 1 / (1 + np.exp(-s))).astype(np.int32)
        parts.append((np.arange(n + 1, dtype=np.int64) * nnz, ci.reshape(-1), v.reshape(-1), y))
        ci_all.append(ci.reshape(-1)); v_all.append(v.reshape(-1)); y_all.append(y)
    data = orc.Csr(np.arange(P * n + 1, dtype=np.int64) * nnz, np.concatenate(ci_all), np.concatenate(v_all), np.concatenate(y_all), n_features=D)
    lambdas = [1.0, 10.0]
    ref = orc.admm_run(data, [0, n, 2 * n], lambdas, niters=5, mode="exact", nthreads=8, epsilon=0.0)
    done, z, xs, us, st = _run_gpu_admm(mb, parts, D, lambdas, 5, csr=True, epsilon=0.0)
    for l in range(2):
        err = np.abs(z[l] - ref["z_hist"][-1, l]).max() / np.abs(ref["z_hist"][-1, l]).max()
        assert err < 1e-5, (l, err, st)
    # one factorisation per (partition, lambda) at the cold start; at most one more each if the cold x-update spent a dozen steps
    # on that factor without contracting by 2x (the "stuck" rule of k1_reduce_decide_kernel) -- never one per iteration
    assert st["not_converged"] == 0 and 4 <= st["gram_builds"] <= 8, st
    # distinct rho: the lambdas share the cold-start Gram but factorise separately, so each streams its own Y in the direction
    # kernels (with equal rho, above, the group reads the leader's Y once for all its lambdas)
    rhos = [1.0, 2.5]
    ref = orc.admm_run(data, [0, n, 2 * n], lambdas, rhos=rhos, niters=3, mode="exact", nthreads=8, epsilon=0.0)
    done, z, xs, us, st = _run_gpu_admm(mb, parts, D, lambdas, 3, csr=True, epsilon=0.0, rhos=rhos)
    for l in range(2):
        err = np.abs(z[l] - ref["z_hist"][-1, l]).max() / np.abs(ref["z_hist"][-1, l]).max()
        assert err < 1e-5, (l, err, st)
    assert st["not_converged"] == 0


def test_admm_initialize_boost_rate(mb, fixture_data, frozen):
    """initialize.boost.rate (jobs/RegressionAdmmTrain.java:236-266, 313-316): start from the mean NaiveTrain model, the reducers of
    iteration 1 on rho * boost (the per-iteration JobConf is rebuilt, so the rate is back to 1 afterwards; with
    rho.adapt.coefficient > 0 the usual schedule applies from iteration 2)."""
    d = fixture_data
    prs = frozen["part_rowstart"]
    parts = []
    for p in range(len(prs) - 1):
        r0, r1 = prs[p], prs[p + 1]
        rp = d.rowptr[r0:r1 + 1] - d.rowptr[r0]
        sl = slice(d.rowptr[r0], d.rowptr[r1])
        parts.append((rp, d.colidx[sl], d.val[sl], d.response[r0:r1], d.weight[r0:r1], d.offset[r0:r1]))
    lambdas = [1.0, 10.0]
    for coef in (0.0, 0.05):
        ref = orc.admm_run(d, prs, lambdas, niters=6, mode="exact", nthreads=8, epsilon=0.0, initialize_boost_rate=2.5, rho_adapt_coefficient=coef)
        with mb.AdmmSession(len(parts), d.n_features, lambdas, epsilon=0.0, rho_adapt_coefficient=coef) as s:
            for p, part in enumerate(parts):
                s.add_partition_csr(p, *part)
            z0 = s.mean_naive_model(range(len(parts)))
            s.begin(z0, 2.5)
            for it in range(6):
                s.iterate()
                for l in range(2):
                    zr = ref["z_hist"][it, l]
                    assert np.abs(s.z(l) - zr).max() / np.abs(zr).max() < 1e-5, (coef, it, l)
            assert s.stats()["not_converged"] == 0


def test_naive_train_many_keys(mb):
    # BASELINE config 4 shape in small: many independent per-key fits in lock-step batches
    K, n, D = 300, 120, 24
    X, y, w, o = _mk(K * n, D, seed=31)
    krs = np.arange(K + 1) * n
    ref, _, _ = orc.naive_train(orc.Csr.from_dense(X, y, w, o), krs, 1.0, mode="exact", nthreads=8)
    got, skipped = mb.naive_train_dense(X, krs, y, 1.0, weight=w, offset=o)
    assert not skipped.any()
    assert np.abs(got - ref).max() / np.abs(ref).max() < 1e-5


def test_admm_fixed_point_is_pooled_sklearn_fit_and_invariants(mb):
    """Parity protocol (ii), SURVEY 8c: after enough iterations the GPU ADMM reaches the minimiser of the POOLED problem
    sum_i logloss + (lambda/2)|beta|^2 (intercept unpenalised) computed by scikit-learn -- independent of the oracle --
    and size-independent invariants hold: the unpenalised intercept makes mean_p u_p[intercept] = 0 after every consensus."""
    from sklearn.linear_model import LogisticRegression
    P, n, D, lam = 4, 30000, 120, 10.0
    rng = np.random.default_rng(5)
    beta = rng.normal(size=D) / np.sqrt(D)
    Xs, ys = [], []
    for p in range(P):
        X = rng.normal(size=(n, D)).astype(np.float32) * (1.0 + 0.3 * p)    # heterogeneous partitions -> real consensus work
        y = (rng.random(n) < 1 / (1 + np.exp(-(X @ beta - 0.7 + 0.2 * p)))).astype(np.int32)
        Xs.append(X); ys.append(y)
    # rho is a free ADMM parameter (the fixed point does not depend on it); matched to the data curvature it converges fast
    with mb.AdmmSession(P, D, [lam], rhos=[5000.0], epsilon=0.0) as s:
        for p in range(P):
            s.add_partition_dense(p, Xs[p], ys[p])
        s.begin()
        for it in range(400):
            md, stop = s.iterate()
            if it in (0, 5, 50):
                usum = sum(s.u(p, 0)[-1].astype(np.float64) for p in range(P))
                assert abs(usum) <= 1e-6 * P, (it, usum)
        z = s.z(0)
        st = s.stats()
    clf = LogisticRegression(C=1.0 / lam, fit_intercept=True, solver="newton-cholesky", tol=1e-12, max_iter=200)
    clf.fit(np.vstack(Xs).astype(np.float64), np.concatenate(ys))
    ref = np.concatenate([clf.coef_.ravel(), clf.intercept_])
    err = np.abs(z - ref).max() / np.abs(ref).max()
    assert err < 2e-5, (err, md, st)
    assert st["not_converged"] == 0 and md < 1e-6


def test_admm_stop_rule_and_options(mb):
    X, y, w, o = _mk(600, 8, seed=5)
    parts = [(X[:300], y[:300], w[:300], o[:300]), (X[300:], y[300:], w[300:], o[300:])]
    data = orc.Csr.from_dense(X, y, w, o)
    for kw, okw in ((dict(penalize_intercept=True), dict(penalize_intercept=True)),
                    (dict(rho_adapt_coefficient=0.3), dict(rho_adapt_coefficient=0.3)),
                    (dict(rhos=[2.0]), dict(rhos=[2.0]))):
        rhos = kw.pop("rhos", None)
        ref = orc.admm_run(data, [0, 300, 600], [10.0], rhos=okw.pop("rhos", None), niters=6, mode="exact", epsilon=0.0, **okw)
        done, z, _, _, st = _run_gpu_admm(mb, parts, 8, [10.0], 6, csr=False, epsilon=0.0, rhos=rhos, **kw)
        err = np.abs(z[0] - ref["z_hist"][-1, 0]).max() / np.abs(ref["z_hist"][-1, 0]).max()
        assert err < 1e-5, (kw, err)
    # Stop rule (:493-496): maxdiff < epsilon && liblinearEpsilon <= 1e-5, with the schedule of :338-346.  The oracle in exact
    # mode runs the SAME schedule and rule on exact x-updates (what the GPU computes), so the iteration counts must be equal;
    # the faithful run (TRON stopped at the reference's loose tolerances) may differ by an iteration or two (informational).
    for eps, aggressive in ((1e-3, False), (1e-4, False), (1e-3, True)):
        ref = orc.admm_run(data, [0, 300, 600], [10.0], niters=300, mode="exact", epsilon=eps, aggressive_decay=aggressive)
        done, z, _, _, st = _run_gpu_admm(mb, parts, 8, [10.0], 300, csr=False, epsilon=eps, aggressive_liblinear_epsilon_decay=aggressive)
        assert done == ref["iters_done"] and done < 300, (eps, aggressive, done, ref["iters_done"])
        err = np.abs(z[0] - ref["z_hist"][-1, 0]).max() / np.abs(ref["z_hist"][-1, 0]).max()
        assert err < 1e-5, (eps, aggressive, err)


def _sparse_parts(P, n, D, nnz, seed, binary=False):
    rng = np.random.default_rng(seed)
    beta = rng.normal(size=D) / np.sqrt(nnz)
    parts, ci_all, v_all, y_all, w_all, o_all = [], [], [], [], [], []
    for p in range(P):
        r = np.random.default_rng(seed + 1 + p)
        ci = np.stack([np.sort(r.choice(D, nnz, replace=False)) for _ in range(n)]).astype(np.int32)
        v = r.normal(size=(n, nnz)).astype(np.float32)
        sc = ((1.0 if binary else v) * beta[ci]).sum(1) - 0.5
        y = (r.random(n) < 1 / (1 + np.exp(-sc))).astype(np.int32)
        w = r.uniform(0.5, 2.0, n).astype(np.float32); o = r.normal(0, 0.1, n).astype(np.float32)
        parts.append((np.arange(n + 1, dtype=np.int64) * nnz, ci.reshape(-1), v.reshape(-1), y, w, o))
        ci_all.append(ci.reshape(-1)); v_all.append(v.reshape(-1)); y_all.append(y); w_all.append(w); o_all.append(o)
    data = orc.Csr(np.arange(P * n + 1, dtype=np.int64) * nnz, np.concatenate(ci_all), np.concatenate(v_all), np.concatenate(y_all),
                   np.concatenate(w_all), np.concatenate(o_all), n_features=D)
    return parts, data, [p * n for p in range(P + 1)]


def test_admm_lambda_map_overrides_per_feature_weights(mb):
    """lambda.map (jobs/RegressionAdmmTrain.java:186-196, 382-386): listed features get z-weight P rho / (lambdaMap[k] + P rho)
    instead of P rho / (lambda + P rho); the reducers are untouched.  Dense and CSR, two lambdas, against oracle-exact."""
    P, n, D = 3, 1500, 40
    X, y, w, o = _mk(P * n, D, seed=61)
    lm = np.zeros(D, np.float32)
    lm[[0, 3, 7, 20, 39]] = [0.01, 5.0, 100.0, 1.0, 0.5]
    data = orc.Csr.from_dense(X, y, w, o)
    prs = [p * n for p in range(P + 1)]
    parts = [(X[prs[p]:prs[p + 1]], y[prs[p]:prs[p + 1]], w[prs[p]:prs[p + 1]], o[prs[p]:prs[p + 1]]) for p in range(P)]
    lambdas = [1.0, 30.0]
    ref = orc.admm_run(data, prs, lambdas, niters=8, mode="exact", nthreads=6, epsilon=0.0, lambda_map=lm)
    plain = orc.admm_run(data, prs, lambdas, niters=8, mode="exact", nthreads=6, epsilon=0.0)
    assert np.abs(ref["z_hist"][-1] - plain["z_hist"][-1]).max() > 1e-3          # the map really changes the answer
    done, z, xs, us, st = _run_gpu_admm(mb, parts, D, lambdas, 8, csr=False, epsilon=0.0, lambda_map=lm)
    for l in range(2):
        err = np.abs(z[l] - ref["z_hist"][-1, l]).max() / np.abs(ref["z_hist"][-1, l]).max()
        assert err < 1e-5, (l, err)
    sparts, sdata, sprs = _sparse_parts(2, 3000, 300, 12, seed=300)
    lm2 = np.zeros(300, np.float32); lm2[::7] = 0.2
    ref = orc.admm_run(sdata, sprs, [2.0], niters=6, mode="exact", nthreads=4, epsilon=0.0, lambda_map=lm2)
    done, z, xs, us, st = _run_gpu_admm(mb, sparts, 300, [2.0], 6, csr=True, epsilon=0.0, lambda_map=lm2)
    assert np.abs(z[0] - ref["z_hist"][-1, 0]).max() / np.abs(ref["z_hist"][-1, 0]).max() < 1e-5


def test_admm_binary_feature_ignores_values(mb):
    """binary.feature (llf/LibLinearBinaryDataset.java:426-515): every listed feature counts as 1, the stored value is ignored.
    The CSR upload rewrites the values; the result must equal the oracle's binary run AND a GPU run on explicit 1.0 values."""
    parts, data, prs = _sparse_parts(2, 4000, 500, 10, seed=400, binary=True)
    lambdas = [0.5, 5.0]
    ref = orc.admm_run(data, prs, lambdas, niters=6, mode="exact", nthreads=4, epsilon=0.0, binary_feature=True)
    nonbin = orc.admm_run(data, prs, lambdas, niters=6, mode="exact", nthreads=4, epsilon=0.0)
    assert np.abs(ref["z_hist"][-1] - nonbin["z_hist"][-1]).max() > 1e-2
    done, z, xs, us, st = _run_gpu_admm(mb, parts, 500, lambdas, 6, csr=True, epsilon=0.0, binary_feature=True)
    ones = [(rp, ci, np.ones_like(v), y, w, o) for rp, ci, v, y, w, o in parts]
    done1, z1, _, _, _ = _run_gpu_admm(mb, ones, 500, lambdas, 6, csr=True, epsilon=0.0)
    for l in range(2):
        err = np.abs(z[l] - ref["z_hist"][-1, l]).max() / np.abs(ref["z_hist"][-1, l]).max()
        assert err < 1e-5, (l, err)
    np.testing.assert_array_equal(z, z1)
    # scoring with binary.feature (models/LinearModel.java:491-554 with ignoreValue)
    pred = mb.score(data.val, z[0], rowptr=data.rowptr, colidx=data.colidx, offset=data.offset, binary_feature=True)
    pref = orc.score(data, z[0], binary_feature=True)
    assert np.abs(pred - pref).max() <= 2e-6 * np.abs(pref).max()


def test_admm_l1_regularizer_thresholded_z_update(mb):
    """regularizer = 1 (jobs/RegressionAdmmTrain.java:406-451): same reducers, z = thresholded mean of x + u with threshold
    lambda / (rho P); as the reference is written, values inside the threshold band are left untouched.  Oracle-exact parity."""
    P, n, D = 3, 2000, 30
    X, y, w, o = _mk(P * n, D, seed=71)
    X[:, 20:] *= 0.02                                                    # weak features: their coefficients sit inside the band
    data = orc.Csr.from_dense(X, y, w, o)
    prs = [p * n for p in range(P + 1)]
    parts = [(X[prs[p]:prs[p + 1]], y[prs[p]:prs[p + 1]], w[prs[p]:prs[p + 1]], o[prs[p]:prs[p + 1]]) for p in range(P)]
    lambdas = [0.3, 3.0]
    for pen in (False, True):
        ref = orc.admm_run(data, prs, lambdas, niters=10, mode="exact", nthreads=6, epsilon=0.0, regularizer=1, penalize_intercept=pen)
        l2 = orc.admm_run(data, prs, lambdas, niters=10, mode="exact", nthreads=6, epsilon=0.0)
        assert np.abs(ref["z_hist"][-1] - l2["z_hist"][-1]).max() > 1e-2
        done, z, xs, us, st = _run_gpu_admm(mb, parts, D, lambdas, 10, csr=False, epsilon=0.0, regularizer=1, penalize_intercept=pen)
        for l in range(2):
            err = np.abs(z[l] - ref["z_hist"][-1, l]).max() / np.abs(ref["z_hist"][-1, l]).max()
            assert err < 1e-5, (pen, l, err)
        assert np.abs(xs - ref["x_last"]).max() / np.abs(ref["x_last"]).max() < 1e-5


def test_admm_config2_shape_eight_dense_partitions(mb):
    """BASELINE configs[1] at reduced rows: 8 partitions x 12k x 1000 dense features, lambda = 1 (the bench's config-2 shape:
    same D' = 1001 kernels, tile plans, Cholesky path and 8-problem batch), against oracle-exact."""
    P, n, D = 8, 12000, 1000
    beta = (np.random.default_rng(999).normal(size=D) / np.sqrt(D)).astype(np.float32)
    parts, Xs, ys = [], [], []
    for p in range(P):
        r = np.random.default_rng(1000 + p)
        X = r.normal(size=(n, D)).astype(np.float32)
        y = (r.random(n) < 1 / (1 + np.exp(-(X @ beta - 1.0)))).astype(np.int32)
        parts.append((X, y)); Xs.append(X); ys.append(y)
    data = orc.Csr.from_dense(np.vstack(Xs), np.concatenate(ys))
    prs = [p * n for p in range(P + 1)]
    ref = orc.admm_run(data, prs, [1.0], niters=5, mode="exact", nthreads=8, epsilon=0.0)
    done, z, xs, us, st = _run_gpu_admm(mb, parts, D, [1.0], 5, csr=False, epsilon=0.0)
    err = np.abs(z[0] - ref["z_hist"][-1, 0]).max() / np.abs(ref["z_hist"][-1, 0]).max()
    assert done == 5 and err < 1e-5 and st["not_converged"] == 0, (err, st)
    assert np.abs(xs - ref["x_last"]).max() / np.abs(ref["x_last"]).max() < 1e-5


def test_unconverged_x_update_is_a_fit_error(mb):
    """A reducer whose fit fails kills the job with IOException("Model fitting error!") (jobs/RegressionAdmmTrain.java:713-716):
    an x-update that runs out of Newton steps must not be averaged into z silently."""
    X, y, w, o = _mk(4000, 50, seed=13)
    with mb.AdmmSession(1, 50, [1e-3], rhos=[1e-3], epsilon=0.0, max_newton=1) as s:
        s.add_partition_dense(0, X * 3.0, y, w, o)
        with pytest.raises(mb.MleaseError, match="Model fitting error"):
            s.run(3)
        assert s.stats()["not_converged"] >= 1


def test_score_and_loglik_match_oracle(mb, fixture_data, frozen):
    d = fixture_data
    model = frozen["exact_z_hist"][-1, 0]
    pred = mb.score(d.val, model, rowptr=d.rowptr, colidx=d.colidx, offset=d.offset)
    ref = frozen["score_pred"]
    assert np.abs(pred - ref).max() <= 2e-6 * np.abs(ref).max()
    ll, cnt = mb.test_loglik(d.response, ref, d.weight, combiner_block=128)
    assert abs(float(ll) - float(frozen["loglik"])) <= 1e-6 * abs(float(frozen["loglik"])) and cnt == 1000
    X, y, w, o = _mk(500, 33, seed=9)
    m = np.random.default_rng(0).normal(size=34)
    p2 = mb.score(X, m, offset=o, num_click_replicates=3)
    r2 = orc.score(orc.Csr.from_dense(X, y, w, o), m, num_click_replicates=3)
    assert np.abs(p2 - r2).max() <= 2e-6 * np.abs(r2).max()
    with pytest.raises(mb.MleaseError):
        mb.test_loglik([5], [0.0])


def test_naive_train_matches_oracle(mb):
    X, y, w, o = _mk(1200, 16, seed=21)
    krs = [0, 400, 800, 1200]
    ref, _, _ = orc.naive_train(orc.Csr.from_dense(X, y, w, o), krs, 2.0, mode="exact")
    got, skipped = mb.naive_train_dense(X, krs, y, 2.0, weight=w, offset=o)
    assert not skipped.any()
    assert np.abs(got - ref).max() / np.abs(ref).max() < 1e-5
    got2, sk2 = mb.naive_train_dense(X, krs, y, 2.0, weight=w, offset=o, data_size_threshold=500)
    assert sk2.all() and not got2.any()
    ref3, _, _ = orc.naive_train(orc.Csr.from_dense(X, y, w, o), krs, 2.0, has_intercept=False, penalize_intercept=True, mode="exact")
    got3, _ = mb.naive_train_dense(X, krs, y, 2.0, weight=w, offset=o, has_intercept=False, penalize_intercept=True)
    assert np.abs(got3 - ref3).max() / np.abs(ref3).max() < 1e-5


def test_errors_follow_reference_conventions(mb):
    X, y, w, o = _mk(50, 4, seed=1)
    with pytest.raises(mb.MleaseError, match="Only L1 and L2"):
        mb.AdmmSession(1, 4, [1.0], regularizer=3)
    with _session(mb, 4) as s:
        with pytest.raises(mb.MleaseError, match="response"):
            s.add_partition_dense(0, X, np.full(50, 2, np.int32))
        with pytest.raises(mb.MleaseError, match="weight"):
            s.add_partition_dense(0, X, y, -w)
        with pytest.raises(mb.MleaseError, match="Map key is wrong"):
            s.add_partition_dense(3, X, y)
    with mb.AdmmSession(2, 4, [1.0]) as s:
        s.add_partition_dense(0, X, y)
        with pytest.raises(mb.MleaseError, match="Some models failed"):
            s.run(2)
    # CSR: label errors are immediate; the colidx range check of a partition runs while the NEXT partition is copied, so it is
    # reported by the next call on the session, naming the partition
    rp, ci, v = _csr_of(X)
    with mb.AdmmSession(2, 4, [1.0]) as s:
        with pytest.raises(mb.MleaseError, match="response"):
            s.add_partition_csr(0, rp, ci, v, np.full(50, 2, np.int32))
        bad = ci.copy(); bad[3] = 4
        s.add_partition_csr(0, rp, bad, v, y)
        with pytest.raises(mb.MleaseError, match="partition 0: feature index out of range"):
            s.add_partition_csr(1, rp, ci, v, y)
    with mb.AdmmSession(1, 4, [1.0]) as s:
        bad = ci.copy(); bad[0] = -1
        s.add_partition_csr(0, rp, bad, v, y)
        with pytest.raises(mb.MleaseError, match="partition 0: feature index out of range"):
            s.run(1)


@pytest.mark.parametrize("d", [45, 1100])
@pytest.mark.parametrize("sparse", [False, True])
def test_posterior_variance_diag_and_full(mb, sparse, d):
    """ItemModelTrain's "posteriorVar" (jobs/ItemModelTrain.java:257-266): LibLinear.train's computePosteriorVar tail
    (llf/LibLinear.java:315-334).  Diagonal mode = 1 / hessianDiagonal (llf/LogisticRegressionL2.java:304-327); full mode =
    diag of the inverse of hessian() (:258-297).  The GPU accumulates the Hessian in fp64 from the fp32 data, so the
    tolerance is 1e-9 / 1e-8 relative, not the bf16 Gram's.  d = 1100 (ldh 1120) runs the inverse of systems wider than 1000:
    256-wide leaves, the fp64 DMMA merges and Y^T Y."""
    n = 2500
    X, y, w, o = _mk(n, d, seed=17, sparse=sparse, density=0.25)
    rng = np.random.default_rng(2)
    pm = rng.normal(0, 0.2, d + 1); pv = rng.uniform(0.3, 3.0, d + 1)
    with _session(mb, d) as s:
        if sparse:
            rp, ci, v = _csr_of(X)
            s.add_partition_csr(0, rp, ci, v, y, w, o)
            data = orc.Csr(rp, ci, v, y, w, o, d)
        else:
            s.add_partition_dense(0, X, y, w, o)
            data = orc.Csr.from_dense(X, y, w, o)
        x, _ = s.fit_partition(0, np.zeros(d + 1), pm, 1.0 / pv)
        var_d = s.posterior_variance(0, x, 1.0 / pv)
        var_f, cov = s.posterior_variance(0, x, 1.0 / pv, full=True, want_cov=True)
        x2, _ = s.fit_partition(0, np.zeros(d + 1), pm, 1.0 / pv)        # the scratch factor was overwritten: the next fit rebuilds
    hd = orc.objective("hessian_diag", data, x, pm, pv)
    assert np.abs(var_d - 1.0 / hd).max() <= 1e-9 * np.abs(1.0 / hd).max()
    H = orc.objective("hessian", data, x, pm, pv)
    ref = np.linalg.inv(H)
    assert np.abs(cov - ref).max() <= 1e-8 * np.abs(ref).max()
    assert np.array_equal(var_f, np.diag(cov)) and np.abs(cov - cov.T).max() == 0.0
    assert np.all(var_f >= var_d * (1 - 1e-12))                           # diag(H^-1) >= 1 / diag(H) for SPD H
    assert np.abs(x2 - x).max() <= 1e-9 * np.abs(x).max()
    with _session(mb, d) as s:
        s.add_partition_dense(0, X, y, w, o)
        with pytest.raises(mb.MleaseError, match="full = 1"):
            import ctypes as C
            from mlease_b200._native import check, lib, ptr
            cov = np.zeros((d + 1, d + 1)); var = np.zeros(d + 1)
            check(lib().mlease_posterior_variance(s._h, 0, ptr(x), ptr(1.0 / pv), 0, ptr(var), ptr(cov)))


def test_naive_train_csr_multi_lambda_lambda_map_and_absent_features(mb):
    """RegressionNaiveTrain on per-key SPARSE datasets (jobs/RegressionNaiveTrain.java:360-398): one CSR upload, keys = row ranges,
    all lambdas in one call.  A feature no row of a key lists is not in that key's model (coefficient 0 even with prior.mean != 0);
    lambda.map gives listed features their own prior variance; binary.feature counts every listed feature as 1."""
    K, n, D, nnz = 6, 400, 80, 9
    r = np.random.default_rng(8)
    beta = r.normal(size=D) / np.sqrt(nnz)
    ci = np.stack([np.sort(r.choice(D - 10 * (i // n % 2), nnz, replace=False)) for i in range(K * n)]).astype(np.int32)   # odd keys never see the last 10 features
    v = r.normal(size=(K * n, nnz)).astype(np.float32)
    y = (r.random(K * n) < 1 / (1 + np.exp(-((v * beta[ci]).sum(1) - 0.4)))).astype(np.int32)
    w = r.uniform(0.5, 2.0, K * n).astype(np.float32); o = r.normal(0, 0.1, K * n).astype(np.float32)
    rp = np.arange(K * n + 1, dtype=np.int64) * nnz
    krs = np.arange(K + 1) * n
    data = orc.Csr(rp, ci.reshape(-1), v.reshape(-1), y, w, o, D)
    lm = np.zeros(D, np.float32); lm[[1, 5, 40]] = [0.02, 9.0, 2.0]
    lambdas = [0.5, 4.0]
    got, skipped = mb.naive_train(v.reshape(-1), krs, y, lambdas, rowptr=rp, colidx=ci.reshape(-1), num_features=D, weight=w, offset=o,
                                  lambda_map=lm, prior_mean=0.3)
    assert got.shape == (2, K, D + 1) and not skipped.any()
    for li, lam in enumerate(lambdas):
        ref, _, _ = orc.naive_train(data, krs, lam, lambda_map=lm, prior_mean=0.3, mode="exact", nthreads=6)
        assert np.abs(got[li] - ref).max() / np.abs(ref).max() < 1e-5, li
        assert np.all(got[li][1::2, D - 10:D] == 0.0) and np.all(ref[1::2, D - 10:D] == 0.0)     # absent features: not in the model
    # binary.feature == the same call on explicit ones; has.intercept = false; data.size.threshold
    gb, _ = mb.naive_train(v.reshape(-1), krs, y, [1.0], rowptr=rp, colidx=ci.reshape(-1), num_features=D, weight=w, offset=o, binary_feature=True)
    ones = orc.Csr(rp, ci.reshape(-1), np.ones(K * n * nnz, np.float32), y, w, o, D)
    rb, _, _ = orc.naive_train(ones, krs, 1.0, mode="exact", nthreads=6)
    assert np.abs(gb[0] - rb).max() / np.abs(rb).max() < 1e-5
    gn, sk = mb.naive_train(v.reshape(-1), krs, y, [1.0], rowptr=rp, colidx=ci.reshape(-1), num_features=D, has_intercept=False, data_size_threshold=401)
    assert sk.all() and not gn.any()
    gn, sk = mb.naive_train(v.reshape(-1), krs, y, [1.0], rowptr=rp, colidx=ci.reshape(-1), num_features=D, weight=w, has_intercept=False, penalize_intercept=True)
    rn, _, _ = orc.naive_train(orc.Csr(rp, ci.reshape(-1), v.reshape(-1), y, w, None, D), krs, 1.0, has_intercept=False, penalize_intercept=True, mode="exact", nthreads=6)
    assert np.abs(gn[0] - rn).max() / np.abs(rn).max() < 1e-5 and np.all(gn[0][:, -1] == 0)
    # the dense entry point is the same code on dense rows
    Xd = np.zeros((K * n, D), np.float32)
    np.put_along_axis(Xd, ci.astype(np.int64), v, axis=1)
    gd, _ = mb.naive_train(Xd, krs, y, lambdas, weight=w, offset=o)
    g1, _ = mb.naive_train_dense(Xd, krs, y, lambdas[1], weight=w, offset=o)
    assert np.array_equal(gd[1], g1)
    rd, _, _ = orc.naive_train(orc.Csr.from_dense(Xd, y, w, o), krs, lambdas[1], mode="exact", nthreads=6)
    assert np.abs(g1 - rd).max() / np.abs(rd).max() < 1e-5


def test_world_of_one_gpu_is_a_session(mb, fixture_data, frozen):
    """mlease_world with a single device = the session calls (no NCCL involved): same z, x, u as the frozen oracle run."""
    d = fixture_data
    prs = frozen["part_rowstart"]
    with mb.World([0], len(prs) - 1, d.n_features, [1.0, 10.0, 100.0], epsilon=0.0) as w:
        for p in range(len(prs) - 1):
            r0, r1 = prs[p], prs[p + 1]
            sl = slice(d.rowptr[r0], d.rowptr[r1])
            w.add_partition_csr(p, d.rowptr[r0:r1 + 1] - d.rowptr[r0], d.colidx[sl], d.val[sl], d.response[r0:r1], d.weight[r0:r1], d.offset[r0:r1])
        assert w.run(20) == 20
        for l in range(3):
            ref = frozen["exact_z_hist"][19, l]
            assert np.abs(w.z(l) - ref).max() / np.abs(ref).max() < 1e-5
        xs = np.stack([[w.x(p, l) for l in range(3)] for p in range(len(prs) - 1)])
        assert np.abs(xs - frozen["exact_x_last"]).max() / np.abs(frozen["exact_x_last"]).max() < 1e-5
        assert w.stats()["not_converged"] == 0


def _ngpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.skipif(_ngpus() < 2, reason="needs 2 GPUs")
def test_two_gpus_world_and_process_per_gpu_match_the_oracle(mb, fixture_data, frozen, tmp_path):
    """N = 2, both ways the boundary offers it: (b) one process, mlease_world over GPUs 0 and 1; (a) one process per GPU with the
    library's NCCL communicator (tests/dist_worker.py under torch.distributed.run).  Same z as the oracle's exact run."""
    import subprocess
    import sys
    d = fixture_data
    prs = frozen["part_rowstart"]
    with mb.World([0, 1], len(prs) - 1, d.n_features, [1.0, 10.0, 100.0], epsilon=0.0) as w:
        for p in range(len(prs) - 1):
            r0, r1 = prs[p], prs[p + 1]
            sl = slice(d.rowptr[r0], d.rowptr[r1])
            w.add_partition_csr(p, d.rowptr[r0:r1 + 1] - d.rowptr[r0], d.colidx[sl], d.val[sl], d.response[r0:r1], d.weight[r0:r1], d.offset[r0:r1])
        w.begin()
        for it in range(20):
            md, stop = w.iterate()
        zw = np.stack([w.z(l) for l in range(3)])
        us = np.stack([w.u(p, 0) for p in range(len(prs) - 1)])
    for l in range(3):
        ref = frozen["exact_z_hist"][19, l]
        assert np.abs(zw[l] - ref).max() / np.abs(ref).max() < 1e-5
    assert abs(us[:, -1].astype(np.float64).sum()) < 1e-5
    out = str(tmp_path / "z.npy")
    root = __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29531", __import__("os").path.join(root, "tests", "dist_worker.py"), out], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    zp = np.load(out)
    for l in range(3):
        ref = frozen["exact_z_hist"][19, l]
        assert np.abs(zp[l] - ref).max() / np.abs(ref).max() < 1e-5
    assert np.abs(zp - zw).max() <= 1e-6 * np.abs(zw).max()


def test_admm_csr_long_run_warm_starts_reach_the_pooled_fixed_point(mb):
    """CSR partitions take the fused K1, and from the second iteration on every x-update starts from the ANALYTIC gradient at the
    previous x_p (no pass for the start point, k4_consensus.cu).  Near the ADMM fixed point the x-updates are tiny and that
    estimate is all noise: the run must still follow the oracle (exact mode, iteration 40) and end at scikit-learn's pooled fit."""
    from sklearn.linear_model import LogisticRegression
    from scipy.sparse import csr_matrix
    parts, data, prs = _sparse_parts(3, 4000, 150, 12, seed=900)
    parts = [(rp, ci, v, y) for rp, ci, v, y, w, o in parts]                     # unit weights, no offsets (sklearn has none)
    data = orc.Csr(data.rowptr, data.colidx, data.val, data.response, n_features=150)
    lambdas, rhos = [0.5, 5.0], [40.0, 40.0]
    ref = orc.admm_run(data, prs, lambdas, rhos=rhos, niters=40, mode="exact", nthreads=6, epsilon=0.0)
    with mb.AdmmSession(3, 150, lambdas, rhos=rhos, epsilon=0.0) as s:
        for p, part in enumerate(parts):
            s.add_partition_csr(p, *part)
        s.begin()
        for it in range(300):
            md, stop = s.iterate()
            if it == 39:
                for l in range(2):
                    zr = ref["z_hist"][39, l]
                    assert np.abs(s.z(l) - zr).max() / np.abs(zr).max() < 1e-5, l
        z = np.stack([s.z(l) for l in range(2)])
        st = s.stats()
    assert st["not_converged"] == 0 and st["k1_fused"] == 1 and md < 1e-6, (st, md)
    assert st["k1_passes"] < 2.2 * 2 * 3 * 300, st          # ~1-2 passes per warm x-update, not 3
    X = csr_matrix((data.val.astype(np.float64), data.colidx, data.rowptr), shape=(12000, 150))
    for l, lam in enumerate(lambdas):
        clf = LogisticRegression(C=1.0 / lam, fit_intercept=True, solver="newton-cholesky", tol=1e-12, max_iter=300)
        clf.fit(X.toarray(), data.response)
        fp = np.concatenate([clf.coef_.ravel(), clf.intercept_])
        assert np.abs(z[l] - fp).max() / np.abs(fp).max() < 3e-5, (l, np.abs(z[l] - fp).max() / np.abs(fp).max())
