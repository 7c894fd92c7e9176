"""GPU tests of ItemModelTrain with the full posterior (mlease_item_model_train_cov): each key's Sigma = H^-1 at its fit against an fp64
assembly and Cholesky inverse of H in numpy, within a bound derived from fp64 Cholesky arithmetic; the variances as Sigma's
diagonal and against a session's mlease_posterior_variance(full = 1); fits equal to the sparse call's, and Sigma independent of the
chunking and the streaming; the refusals; and a 50 000-key fit over 2 000 000 features."""
import ctypes as C
import resource

import numpy as np
import pytest

import item_model_cov_ref as ref
from test_gpu_keyed_sparse import _bitwise, _close, _key_cols, _keyed, _pools, _same, _wide

pytestmark = pytest.mark.gpu

IL, DL = [0.5, 20.0], [1.0, 0.25, 4.0]


@pytest.fixture
def budget():
    from mlease_b200 import _hooks
    yield _hooks.set_keyed_budget
    _hooks.set_keyed_budget(0)


def _cov(pb, il=IL, dl=DL, **kw):
    import mlease_b200 as mb
    return mb.item_model_train_cov(pb["v"], pb["krs"], pb["y"], il, dl, rowptr=pb["rp"], colidx=pb["ci"], num_features=pb["D"],
                                   weight=pb["w"], offset=pb["o"], **kw)


def _sparse(pb, il=IL, dl=DL, **kw):
    import mlease_b200 as mb
    return mb.item_model_train_sparse(pb["v"], pb["krs"], pb["y"], il, dl, rowptr=pb["rp"], colidx=pb["ci"], num_features=pb["D"],
                                      weight=pb["w"], offset=pb["o"], compute_var=True, **kw)


def _shape(name, rng):
    """D = 20: every key at the global width without a column list; 60 000 features: keys in their own spaces; D = 40: keys that list
    all 40 columns run at the global width through their lists, the others in their own 32-column spaces; widths on both sides of
    32 (30 / 31 and 33 / 34 columns) and of 1000 (K3's DMMA path: 960 and 1100 columns)."""
    D, per_row, full = 60000, 12, False
    if name == "d20":
        D, K = 20, 24
        pools = _pools(rng, K, D, 8, 20, shared=0.0)
        rows = rng.integers(1, 60, K)
        per_row = 6
    elif name == "own60k":
        K = 24
        pools = _pools(rng, K, D, 8, 200)
        rows = rng.integers(1, 150, K)
        rows[::4] = 1
    elif name == "global_list":
        D, K = 40, 16
        pools = [np.arange(D) if k % 2 == 0 else np.sort(rng.choice(D, 20, replace=False)) for k in range(K)]
        rows = rng.integers(2, 80, K)
        full = True
    elif name == "w32":
        K = 8
        pools = [np.sort(rng.choice(D, s, replace=False)) for s in (30, 31, 33, 34, 30, 31, 33, 34)]
        rows = np.array([1, 40, 1, 40, 25, 60, 25, 60])
        full = True
    else:   # "w1000"
        K = 2
        pools = [np.sort(rng.choice(D, s, replace=False)) for s in (960, 1100)]
        rows = np.array([150, 160])
        per_row, full = 30, True
    return _keyed(rng, rows, pools, D, per_row=per_row, full_first=full), rows


def _fits_agree(got, want, one_row, binary):
    """the cov call's models against the sparse call's: bit for bit for one-row keys in their own spaces; otherwise within the
    run-to-run spread, which under binary_feature reaches past the sparse tests' 1e-6 relative on multi-row keys at the global
    width (on an H100, two sparse calls on the d20 shape below differed by 1.05e-6, two cov calls by 2.5e-6, relative to max |beta|
    ~ 2.7).  It is not the reset between priors: the cov and sparse calls differed by 1.5e-6 at the first prior, which both fit from
    the same freshly allocated state before any posterior is formed.  1e-5 there"""
    if one_row or not binary:
        _same(got, want, one_row)
    elif want.size:
        assert np.abs(got - want).max() <= 1e-5 * max(1.0, np.abs(want).max())


def _check_sigma(pb, k, cols, beta, var, block, lm, il, dl, binary):
    """Sigma of key k at one prior against fp64; returns the worst error over the bound's c = 1 scale"""
    D = pb["D"]
    n = len(cols)
    q = ref.prior_precision(cols, D, lm, il, dl)
    H = ref.hessian(pb, k, cols, beta, q, binary)
    want, _ = ref.inverse(H)
    got = ref.unpack(block, n)
    assert np.array_equal(var.view(np.uint64), np.diag(got).copy().view(np.uint64)), k
    assert np.all(var >= (1.0 / np.diag(H)) * (1 - 1e-12)), k
    bound = ref.sigma_bound(H, want)
    err = np.abs(got - want).max()
    assert err <= bound, (k, err, bound)
    return err / (bound / 8.0)


@pytest.mark.parametrize("shape", ["d20", "own60k", "global_list", "w32", "w1000"])
@pytest.mark.parametrize("binary", [False, True])
def test_sigma_against_fp64(shape, binary):
    rng = np.random.default_rng(2100 + ["d20", "own60k", "global_list", "w32", "w1000"].index(shape))
    pb, rows = _shape(shape, rng)
    D, K = pb["D"], pb["K"]
    lm = np.zeros(D, np.float32)
    lm[rng.choice(D, min(D, 8), replace=False)] = rng.uniform(0.1, 8.0, min(D, 8)).astype(np.float32)
    means = rng.normal(0, 1, K)
    kw = dict(intercept_prior_mean=means, lambda_map=lm, binary_feature=binary)
    key_ptr, cols, models, var, cov_ptr, cov = _cov(pb, **kw)
    skp, scols, smodels, _ = _sparse(pb, **kw)
    assert np.array_equal(key_ptr, skp) and np.array_equal(cols, scols)
    n_k = np.diff(key_ptr)
    assert np.array_equal(np.diff(cov_ptr), n_k * (n_k + 1) // 2)
    worst = 0.0
    for k in range(K):
        a, b = key_ptr[k], key_ptr[k + 1]
        c = cols[a:b]
        assert np.array_equal(c, np.append(_key_cols(pb, k), D))
        for ia in range(len(IL)):
            for ib in range(len(DL)):
                _fits_agree(models[ia, ib, a:b], smodels[ia, ib, a:b], _bitwise(pb, rows, k), binary)
                worst = max(worst, _check_sigma(pb, k, c, models[ia, ib, a:b], var[ia, ib, a:b],
                                                cov[ia, ib, cov_ptr[k]:cov_ptr[k + 1]], lm, IL[ia], DL[ib], binary))
    print("%s binary=%d: worst |Sigma - fp64| = %.3g x Dt kappa 2^-53 max|Sigma|" % (shape, binary, worst))


def test_widths_at_the_explicit_inverse_limit():
    """a key of 2047 columns (a 2048-column system) is fitted and checked against fp64; one of 2048 columns (2080) is refused before
    its chunk is solved, the message naming the key and its width"""
    import mlease_b200 as mb
    rng = np.random.default_rng(2200)
    D = 60000

    def key_of(ncols):
        cols = np.sort(rng.choice(D, ncols, replace=False))
        pools = [cols]
        pb = _keyed(rng, [1], pools, D, per_row=ncols)   # one row listing every column, then rows of ~40 of them
        extra = [np.sort(rng.choice(cols, 40, replace=False)) for _ in range(120)]
        ci = np.concatenate([pb["ci"]] + extra).astype(np.int32)
        rp = np.concatenate([[0], np.cumsum([ncols] + [40] * 120)]).astype(np.int64)
        n = 121
        return dict(krs=np.array([0, n], np.int64), rp=rp, ci=ci, v=rng.normal(size=len(ci)).astype(np.float32),
                    y=(rng.random(n) < 0.4).astype(np.int32), w=rng.uniform(0.5, 2.0, n).astype(np.float32),
                    o=rng.normal(0, 0.1, n).astype(np.float32), D=D, K=1)
    pb = key_of(2047)
    key_ptr, cols, models, var, cov_ptr, cov = _cov(pb, il=[2.0], dl=[0.5])
    assert key_ptr[-1] == 2048 and cov_ptr[-1] == 2048 * 2049 // 2
    r = _check_sigma(pb, 0, cols, models[0, 0], var[0, 0], cov[0, 0], None, 2.0, 0.5, False)
    print("2047 columns: worst |Sigma - fp64| = %.3g x Dt kappa 2^-53 max|Sigma|" % r)
    wide = key_of(2048)
    with pytest.raises(mb.MleaseError, match=r"key 0: .*2080-column system \(its own column space\).*2048") as e:
        _cov(wide, il=[2.0], dl=[0.5])
    assert e.value.code == 1


def test_variances_match_the_session_posterior_variance():
    """for a few keys, mlease_posterior_variance(full = 1) on a session holding the key's rows at the same beta and q: diag(Sigma)
    and Sigma restricted to the key's list within 1e-10 relative"""
    import mlease_b200 as mb
    rng = np.random.default_rng(2300)
    pb, rows = _shape("d20", rng)
    D = pb["D"]
    lm = np.zeros(D, np.float32)
    lm[[2, 7, 11]] = [0.5, 3.0, 7.0]
    key_ptr, cols, models, var, cov_ptr, cov = _cov(pb, lambda_map=lm, intercept_prior_mean=rng.normal(0, 1, pb["K"]))
    for k in [0, 1, 2, 3, 9]:
        a, b = key_ptr[k], key_ptr[k + 1]
        c = cols[a:b]
        rp, ci, v, y, w, o = ref.key_rows(pb, k)
        for ia, ib in [(0, 0), (1, 2)]:
            beta = np.zeros(D + 1); beta[c] = models[ia, ib, a:b]
            q = ref.prior_precision(np.arange(D + 1), D, lm, IL[ia], DL[ib])
            with mb.AdmmSession(1, D, [1.0]) as s:
                s.add_partition_csr(0, rp, ci, v, y, w, o)
                sv, sc = s.posterior_variance(0, beta, q, full=True, want_cov=True)
            got = ref.unpack(cov[ia, ib, cov_ptr[k]:cov_ptr[k + 1]], len(c))
            want = sc[np.ix_(c, c)]
            assert np.abs(var[ia, ib, a:b] - sv[c]).max() <= 1e-10 * np.abs(sv[c]).max(), k
            assert np.abs(got - want).max() <= 1e-10 * np.abs(want).max(), k


def test_fits_unchanged_and_sigma_independent_of_chunks_and_streaming(budget):
    """one-row keys in their own spaces: models bit for bit the sparse call's, and Sigma bit for bit the same from a resident call in
    one chunk, a resident call in several chunks and a streamed call; multi-row keys within the run-to-run spread"""
    from mlease_b200 import _hooks
    rng = np.random.default_rng(2400)
    D, K = 60000, 400
    rows = np.ones(K, np.int64)
    multi = rng.choice(K, 12, replace=False)
    rows[multi] = rng.integers(5, 60, 12)
    pb = _keyed(rng, rows, _pools(rng, K, D, 8, 60), D, per_row=20)
    one = rows == 1
    kw = dict(il=[2.0, 0.5], dl=[1.0])
    budget(0)
    res = _cov(pb, **kw)
    bounds, streamed, _, _ = _hooks.keyed_last_call()
    assert not streamed and len(bounds) == 2, bounds
    sp = _sparse(pb, **kw)
    assert np.array_equal(sp[0], res[0]) and np.array_equal(sp[1], res[1])
    chunked = streamed_run = None
    nbytes = 256 << 20
    while nbytes >= (64 << 10) and streamed_run is None:
        budget(nbytes)
        out = _cov(pb, **kw)
        bounds, streamed, _, _ = _hooks.keyed_last_call()
        if streamed:
            streamed_run = out
        elif len(bounds) > 2 and chunked is None:
            chunked = out
        nbytes //= 2
    assert chunked is not None and streamed_run is not None
    kp, cp = res[0], res[4]
    for other in (chunked, streamed_run):
        assert np.array_equal(other[0], kp) and np.array_equal(other[1], res[1]) and np.array_equal(other[4], cp)
    for k in range(K):
        a, b = kp[k], kp[k + 1]
        for p in range(2):
            _same(res[2][p, 0, a:b], sp[2][p, 0, a:b], one[k])
            for other in (chunked, streamed_run):
                _same(other[2][p, 0, a:b], res[2][p, 0, a:b], one[k])
                _same(other[3][p, 0, a:b], res[3][p, 0, a:b], one[k])
                got, want = other[5][p, 0, cp[k]:cp[k + 1]], res[5][p, 0, cp[k]:cp[k + 1]]
                if one[k]:
                    assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), k
                else:
                    _close(got, want)


def _raw(pb, cap, ccap, key_ptr, cols, models, var, cov_ptr, cov):
    import mlease_b200 as mb
    from mlease_b200._native import ptr
    il, dl = np.array([1.0], np.float32), np.array([1.0], np.float32)
    im = np.zeros(pb["K"])
    return mb.lib().mlease_item_model_train_cov(0, None, pb["K"], pb["D"], ptr(pb["krs"]), ptr(pb["rp"]), ptr(pb["ci"]), ptr(pb["v"]),
                                                ptr(pb["y"]), None, None, ptr(im), 1, ptr(il), 1, ptr(dl), None, 0, int(cap), ptr(key_ptr),
                                                ptr(cols), ptr(models), ptr(var), int(ccap), ptr(cov_ptr), ptr(cov))


def test_refusals_and_variances_without_blocks():
    import mlease_b200 as mb
    rng = np.random.default_rng(2500)
    D, K = 60000, 20
    rows = rng.integers(1, 40, K); rows[::3] = 1
    pb = _keyed(rng, rows, _pools(rng, K, D, 8, 80), D)
    nnz = np.diff(pb["rp"][pb["krs"]])
    cap = int((np.minimum(nnz, D) + 1).sum())
    n_k = np.array([len(_key_cols(pb, k)) + 1 for k in range(K)])
    need = int((n_k * (n_k + 1) // 2).sum())
    # a short cov_capacity: refused, the message giving the size, nothing written
    kp, cols, models, var = np.full(K + 1, -7, np.int64), np.full(cap, -7, np.int32), np.full(cap, -7.0), np.full(cap, -7.0)
    cp, cov = np.full(K + 1, -7, np.int64), np.full(need, -7.0)
    assert _raw(pb, cap, need - 1, kp, cols, models, var, cp, cov) == 1
    msg = mb.lib().mlease_last_error().decode()
    assert "cov_capacity" in msg and str(need) in msg, msg
    assert np.all(cov == -7.0) and np.all(models == -7.0)
    with pytest.raises(mb.MleaseError, match=str(need)):
        _cov(pb, il=[1.0], dl=[1.0], cov_capacity=need - 1)
    assert _raw(pb, cap, need, kp, cols, models, var, cp, cov) == 0 and cp[-1] == need
    # null pointers: out_var is required; out_cov_ptr with out_cov
    for args in ([kp, cols, models, None, cp, cov], [kp, cols, models, var, None, cov], [None, cols, models, var, cp, cov],
                 [kp, None, models, var, cp, cov], [kp, cols, None, var, cp, cov]):
        assert _raw(pb, cap, need, *args) == 1
        assert "bad argument" in mb.lib().mlease_last_error().decode()
    # out_cov = NULL: diag(Sigma) only, cov_capacity and out_cov_ptr ignored
    var2 = np.full(cap, -7.0)
    assert _raw(pb, cap, 0, kp, cols, models, var2, None, None) == 0
    one = np.repeat(rows == 1, np.diff(kp))
    assert np.array_equal(var2[:kp[-1]][one].view(np.uint64), var[:kp[-1]][one].view(np.uint64))
    _close(var2[:kp[-1]], var[:kp[-1]])
    out = _cov(pb, il=[1.0], dl=[1.0], want_cov=False)
    assert out[4] is None and out[5] is None and out[3].shape == (1, 1, kp[-1])
    # rows with a repeated or descending column: refused with the session's text
    bad = dict(pb, ci=pb["ci"].copy())
    r0 = bad["rp"][bad["krs"][4]]
    bad["ci"][r0], bad["ci"][r0 + 1] = bad["ci"][r0 + 1], bad["ci"][r0]
    with pytest.raises(mb.MleaseError, match="strictly increasing column ids") as e:
        _cov(bad, il=[1.0], dl=[1.0])
    assert e.value.code == 1
    kp2, c2, m2, v2, cp2, cv2 = _cov(pb, il=[1.0], dl=[1.0])   # the process goes on
    assert np.all(np.isfinite(cv2)) and cp2[-1] == need


def test_a_dictionary_of_two_million_features():
    """50 000 keys of 1 - 8 rows over 2 000 000 features: the call completes with the process's peak RSS less than 2 GB above what it
    was, and the blocks of sampled keys match fp64 at their fits"""
    rng = np.random.default_rng(2600)
    K, D = 50000, 2000000
    pb = _wide(rng, K, D, 1, 8, 40, 20)
    small = dict(pb, krs=pb["krs"][:9], K=8)
    _cov(small, il=[1.0], dl=[1.0])   # modules and allocator
    rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024
    key_ptr, cols, models, var, cov_ptr, cov = _cov(pb, il=[1.0], dl=[1.0])
    grown = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024 - rss0
    assert grown < 2 << 30, grown
    n_k = np.diff(key_ptr)
    assert np.all(n_k > 0) and np.array_equal(np.diff(cov_ptr), n_k * (n_k + 1) // 2)
    worst = 0.0
    for k in rng.choice(K, 40, replace=False):
        a, b = key_ptr[k], key_ptr[k + 1]
        assert np.array_equal(cols[a:b], np.append(_key_cols(pb, k), D))
        worst = max(worst, _check_sigma(pb, k, cols[a:b], models[0, 0, a:b], var[0, 0, a:b], cov[0, 0, cov_ptr[k]:cov_ptr[k + 1]], None,
                                        1.0, 1.0, False))
    print("2M features: worst |Sigma - fp64| = %.3g x Dt kappa 2^-53 max|Sigma|" % worst)
