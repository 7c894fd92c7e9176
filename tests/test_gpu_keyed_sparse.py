"""GPU tests of the keyed CSR fits with sparse outputs (mlease_naive_train_sparse, mlease_item_model_train_sparse): each key's list is
exactly the distinct columns its rows list (then the intercept), its values those the dense call writes at those columns (bit for bit
for one-row keys in their own column spaces, within the run-to-run spread of the float-atomic gradient sums otherwise), across the three ways a key's list is
gathered on the device (a key in its own column space, a global-width key with a column list, a key without one compacted by its
presence mask), streamed and chunked calls, the refusals before any fit, a shape whose dense output no host could hold, fit then
score without a dense model, and two devices."""
import ctypes as C
import resource
import threading

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


def _keyed(rng, rows, pools, D, per_row=12, full_first=False):
    """key k: rows[k] rows, each listing up to per_row sorted unique columns of pools[k]; full_first: a key's first row lists its
    whole pool, so the key lists every column of it while its other rows differ from one another"""
    rp, ci, keys = [0], [], []
    for k, (n, pool) in enumerate(zip(rows, pools)):
        for i in range(n):
            take = len(pool) if (full_first and i == 0) else min(per_row, len(pool))
            c = np.sort(rng.choice(pool, take, replace=False)) if len(pool) else np.zeros(0, np.int64)
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


def _key_cols(pb, k):
    a, b = pb["krs"][k], pb["krs"][k + 1]
    return np.unique(pb["ci"][pb["rp"][a]:pb["rp"][b]])


def _close(got, want):
    """the run-to-run spread of a CSR fit: the K1 gradient sums use float atomics"""
    if want.size:
        assert np.abs(got - want).max() <= 1e-6 * max(1.0, np.abs(want).max())


def _same(got, want, one_row):
    if one_row:
        assert np.array_equal(np.asarray(got).view(np.uint64), np.asarray(want).view(np.uint64))
    else:
        _close(got, want)


def _naive(pb, lams, sparse, **kw):
    import mlease_b200 as mb
    fn = mb.naive_train_sparse if sparse else mb.naive_train
    return fn(pb["v"], pb["krs"], pb["y"], list(lams), rowptr=pb["rp"], colidx=pb["ci"], num_features=pb["D"], weight=pb["w"],
              offset=pb["o"], **kw)


def _item(pb, il, dl, sparse, **kw):
    import mlease_b200 as mb
    fn = mb.item_model_train_sparse if sparse else mb.item_model_train
    return fn(pb["v"], pb["krs"], pb["y"], il, dl, rowptr=pb["rp"], colidx=pb["ci"], num_features=pb["D"], weight=pb["w"], offset=pb["o"], **kw)


def _shape(name, rng):
    """the four kinds of call: D = 20 (no column lists: every key compacted by its mask), D = 256 with every key at the global width
    (gathered through its list), D = 120 000 (keys in their own spaces), and a call mixing global-width and local keys.  Every shape
    has one-row keys (key 1 among them), a two-row key (key 2) and a key without rows (key 5)."""
    if name == "d20":
        D, K = 20, 40
        pools = _pools(rng, K, D, 8, 20, shared=0.0)
        rows = rng.integers(1, 60, K)
    elif name == "d256_global":
        D, K = 256, 24
        pools = [np.arange(D)] * K
        rows = rng.integers(1, 30, K)
    elif name == "d120k_local":
        D, K = 120000, 30
        pools = _pools(rng, K, D, 8, 400)
        rows = rng.integers(1, 300, K)
        rows[::4] = 1
    else:
        D, K = 300, 28
        pools = [np.arange(D) if k % 3 == 0 else np.sort(rng.choice(D, 20, replace=False)) for k in range(K)]
        rows = np.array([1 if k % 3 == 0 else int(rng.integers(1, 200)) for k in range(K)])
        rows[[4, 10, 17, 22]] = 1
    rows[1], rows[2], rows[5] = 1, 2, 0          # one row, two rows, no rows
    # rows list fewer columns than their key's pool (global-width keys list all of it through their first row), so that no key's
    # rows are all the same vector under binary_feature: such a key's features are perfectly collinear, and its fit's line search may
    # fail at the noise floor of the float-atomic objective sums, in the dense call as in the sparse one
    wide = name in ("d256_global", "mixed")
    per_row = {"d20": 6, "d256_global": 96}.get(name, 12)
    return _keyed(rng, rows, pools, D, per_row=per_row, full_first=wide), rows


def _check_lists(pb, key_ptr, cols, fitted, intercept):
    D = pb["D"]
    assert key_ptr[0] == 0 and np.all(np.diff(key_ptr) >= 0)
    for k in range(pb["K"]):
        got = cols[key_ptr[k]:key_ptr[k + 1]]
        if not fitted[k]:
            assert len(got) == 0, k
            continue
        want = _key_cols(pb, k)
        if intercept:
            want = np.append(want, D)
        assert np.array_equal(got, want), k


SHAPES = ["d20", "d256_global", "d120k_local", "mixed"]


def _bitwise(pb, rows, k):
    """one-row keys solved in their own column space (round_up(Dk + 1, 32) < round_up(D + 1, 32)) compare bit for bit: their batches
    run in lockstep, so a key's bits depend on its own rows alone.  Global-width keys share batches of up to 64 problems whose slot
    pipeline couples the problems' rebuilds, so there a one-row key follows the float-atomic spread of the multi-row keys beside it,
    in the dense call as in the sparse one: within the spread"""
    def up(x):
        return (x + 31) // 32 * 32
    return rows[k] == 1 and up(len(_key_cols(pb, k)) + 1) < up(pb["D"] + 1)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("has_intercept,binary", [(True, False), (False, True)])
def test_naive_train_lists_and_values_match_the_dense_call(shape, has_intercept, binary):
    rng = np.random.default_rng(1100 + SHAPES.index(shape))
    pb, rows = _shape(shape, rng)
    D = pb["D"]
    lm = np.zeros(D, np.float32)
    lm[rng.choice(D, min(D, 12), replace=False)] = rng.uniform(0.1, 8.0, min(D, 12)).astype(np.float32)
    thr = 0 if has_intercept else 2   # with 2, the one-row keys are skipped
    kw = dict(lambda_map=lm, prior_mean=0.1, has_intercept=has_intercept, binary_feature=binary, data_size_threshold=thr)
    lams = (0.7, 6.0)
    dense, dskip = _naive(pb, lams, False, **kw)
    key_ptr, cols, models, skipped = _naive(pb, lams, True, **kw)
    fitted = (rows >= thr) & (rows > 0)
    assert np.array_equal(skipped, dskip) and np.array_equal(~skipped, fitted)
    assert skipped[5] and skipped[1] == (thr == 2) and not skipped[2]
    _check_lists(pb, key_ptr, cols, fitted, has_intercept)
    assert models.shape == (2, key_ptr[-1])
    for k in range(pb["K"]):
        c = cols[key_ptr[k]:key_ptr[k + 1]]
        unlisted = np.ones(D + 1, bool); unlisted[c] = False
        for li in range(2):
            _same(models[li, key_ptr[k]:key_ptr[k + 1]], dense[li, k, c], _bitwise(pb, rows, k))
            assert np.all(dense[li, k, unlisted] == 0.0), (k, li)


@pytest.mark.parametrize("shape", ["d20", "d120k_local", "mixed"])
def test_item_model_train_values_and_variance_match_the_dense_call(shape):
    rng = np.random.default_rng(1200 + SHAPES.index(shape))
    pb, rows = _shape(shape, rng)
    D, K = pb["D"], pb["K"]
    means = rng.normal(0, 1, K)
    lm = np.zeros(D, np.float32)
    lm[rng.choice(D, min(D, 6), replace=False)] = rng.uniform(0.1, 8.0, min(D, 6)).astype(np.float32)
    il, dl = [0.5, 20.0], [1.0, 0.25, 4.0]
    kw = dict(intercept_prior_mean=means, lambda_map=lm, compute_var=True)
    dm, dv = _item(pb, il, dl, False, **kw)
    key_ptr, cols, models, var = _item(pb, il, dl, True, **kw)
    fitted = rows > 0
    _check_lists(pb, key_ptr, cols, fitted, True)
    assert models.shape == var.shape == (2, 3, key_ptr[-1])
    for k in range(K):
        c = cols[key_ptr[k]:key_ptr[k + 1]]
        unlisted = np.ones(D + 1, bool); unlisted[c] = False
        for a in range(2):
            for b in range(3):
                _same(models[a, b, key_ptr[k]:key_ptr[k + 1]], dm[a, b, k, c], _bitwise(pb, rows, k))
                _same(var[a, b, key_ptr[k]:key_ptr[k + 1]], dv[a, b, k, c], _bitwise(pb, rows, k))
                q = np.append(np.where(lm > 0, lm, np.float32(dl[b])).astype(np.float64), np.float64(np.float32(il[a])))
                q = 1.0 / (1.0 / q)
                assert np.all(dm[a, b, k, unlisted] == 0.0)
                assert np.array_equal(dv[a, b, k, unlisted], (1.0 / q)[unlisted]), (k, a, b)


def test_streamed_and_chunked_calls_match_the_resident_call(budget):
    """more than 16 384 fitted keys: the resident call runs several chunks; under a small budget the call streams several ranges.
    The lists are contiguous in key order across chunks and ranges; one-row keys bit for bit, multi-row keys within the spread."""
    from mlease_b200 import _hooks
    rng = np.random.default_rng(1300)
    D, K = 5000, 17000
    rows = np.ones(K, np.int64)
    multi = rng.choice(K, 40, replace=False)
    rows[multi] = rng.integers(20, 120, 40)
    rows[rng.choice(K, 30, replace=False)] = 0
    pools = [np.sort(rng.choice(D, 24, replace=False)) for _ in range(K)]
    pb = _keyed(rng, rows, pools, D, per_row=10)
    one = rows == 1
    budget(0)
    res = _naive(pb, (1.0,), True)
    bounds, streamed, _, _ = _hooks.keyed_last_call()
    assert not streamed and len(bounds) - 1 >= 2, bounds
    _check_lists(pb, res[0], res[1], rows > 0, True)
    budget(4 << 20)
    st = _naive(pb, (1.0,), True)
    bounds, streamed, _, _ = _hooks.keyed_last_call()
    assert streamed and len(bounds) - 1 >= 4, bounds
    assert np.array_equal(st[0], res[0]) and np.array_equal(st[1], res[1])
    for k in range(K):
        a, b = res[0][k], res[0][k + 1]
        _same(st[2][0, a:b], res[2][0, a:b], one[k])
    # ItemModelTrain with its variance, streamed against resident
    budget(0)
    r2 = _item(pb, [2.0], [0.5], True, compute_var=True)
    budget(4 << 20)
    s2 = _item(pb, [2.0], [0.5], True, compute_var=True)
    assert _hooks.keyed_last_call()[1]
    assert np.array_equal(s2[0], r2[0]) and np.array_equal(s2[1], r2[1])
    for k in range(K):
        a, b = r2[0][k], r2[0][k + 1]
        _same(s2[2][0, 0, a:b], r2[2][0, 0, a:b], one[k])
        _same(s2[3][0, 0, a:b], r2[3][0, 0, a:b], one[k])


def _raw_naive(pb, cap, key_ptr, cols, models, skipped, lam=1.0):
    import mlease_b200 as mb
    from mlease_b200._native import ptr
    lams = np.array([lam], np.float32)
    return mb.lib().mlease_naive_train_sparse(0, None, pb["K"], pb["D"], ptr(pb["krs"]), ptr(pb["rp"]), ptr(pb["ci"]), ptr(pb["v"]),
                                              ptr(pb["y"]), None, None, 1, ptr(lams), None, C.c_float(0.0), 0, 1, 0, 0, int(cap),
                                              ptr(key_ptr), ptr(cols), ptr(models), ptr(skipped))


def test_refusals_before_any_fit(budget):
    import mlease_b200 as mb
    rng = np.random.default_rng(1400)
    D, K = 90000, 30
    rows = rng.integers(20, 120, K)
    pb = _keyed(rng, rows, _pools(rng, K, D, 8, 100), D)
    nnz = np.diff(pb["rp"][pb["krs"]])
    need = int((np.minimum(nnz, D) + 1).sum())
    # capacity one short: refused, naming the bound, and nothing written
    kp = np.full(K + 1, -7, np.int64); cols = np.full(need, -7, np.int32); models = np.full(need, -7.0); skipped = np.full(K, -7, np.int32)
    rc = _raw_naive(pb, need - 1, kp, cols, models, skipped)
    assert rc == 1
    msg = mb.lib().mlease_last_error().decode()
    assert str(need) in msg, msg
    assert np.all(kp == -7) and np.all(cols == -7) and np.all(models == -7.0) and np.all(skipped == -7)
    with pytest.raises(mb.MleaseError, match=str(need)):
        _naive(pb, (1.0,), True, capacity=need - 1)
    # the bound itself is enough
    assert _raw_naive(pb, need, kp, cols, models, skipped) == 0
    assert kp[-1] <= need
    # null outputs
    for i in range(4):
        args = [kp, cols, models, skipped]
        args[i] = None
        if i == 3:   # skipped may be NULL, as in the dense call
            assert _raw_naive(pb, need, *args) == 0
            continue
        assert _raw_naive(pb, need, *args) == 1
        assert "bad argument" in mb.lib().mlease_last_error().decode()
    # a bad column in a late key: the dense call's text, resident and streamed, before the outputs are touched
    bad = dict(pb, ci=pb["ci"].copy())
    bad["ci"][bad["rp"][bad["krs"][27]] + 1] = D
    for nbytes in (0, 1 << 20):
        budget(nbytes)
        kp[:] = -7
        with pytest.raises(mb.MleaseError, match="feature index out of range") as e:
            _naive(bad, (1.0,), True)
        assert e.value.code == 1
        with pytest.raises(mb.MleaseError, match="feature index out of range"):
            _item(bad, [1.0], [1.0], True)
        if nbytes == 0:
            assert _raw_naive(bad, need, kp, cols, models, skipped) == 1 and np.all(kp == -7)
    budget(0)
    kp2, c2, m2, _ = _naive(pb, (1.0,), True)   # the process goes on
    assert np.all(np.isfinite(m2)) and kp2[-1] == len(c2)


def _wide(rng, K, D, lo_rows, hi_rows, pool, per_row):
    """K keys of lo..hi rows, each row per_row sorted unique columns of the key's pool of `pool` random columns of [0, D)"""
    nk = rng.integers(lo_rows, hi_rows + 1, K)
    pools = np.sort(rng.integers(0, D, (K, pool)), axis=1)
    ci, rl = [], []
    for k in range(K):
        p = np.unique(pools[k])
        pick = np.sort(np.argsort(rng.random((nk[k], len(p))), axis=1)[:, :per_row], axis=1)
        ci.append(p[pick].reshape(-1)); rl.append(np.full(nk[k], pick.shape[1]))
    ci = np.concatenate(ci).astype(np.int32)
    rp = np.concatenate([[0], np.cumsum(np.concatenate(rl))]).astype(np.int64)
    n = int(nk.sum())
    v = rng.normal(size=len(ci)).astype(np.float32)
    y = (rng.random(n) < 0.4).astype(np.int32)
    krs = np.concatenate([[0], np.cumsum(nk)]).astype(np.int64)
    return dict(krs=krs, rp=rp, ci=ci, v=v, y=y, w=rng.uniform(0.5, 2.0, n).astype(np.float32), o=rng.normal(0, 0.1, n).astype(np.float32),
                D=D, K=K)


def test_a_dictionary_the_dense_output_cannot_hold():
    """50 000 keys of 1 - 8 rows over 2 000 000 features: the dense output would be 800 GB.  The sparse call completes with the
    process's peak RSS less than 2 GB above what it was, and sampled keys match the oracle fitted on their relabelled rows."""
    rng = np.random.default_rng(1500)
    K, D = 50000, 2000000
    pb = _wide(rng, K, D, 1, 8, 40, 20)
    lam = 1.0
    _naive(_slice(pb, 0, 8), (lam,), True)   # modules and allocator
    rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024
    key_ptr, cols, models, skipped = _naive(pb, (lam,), True)
    grown = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024 - rss0
    assert grown < 2 << 30, grown
    assert not skipped.any() and key_ptr[-1] == len(cols)
    for k in rng.choice(K, 50, replace=False):
        c = _key_cols(pb, k)
        assert np.array_equal(cols[key_ptr[k]:key_ptr[k + 1]], np.append(c, D))
        a, b = pb["krs"][k], pb["krs"][k + 1]
        rp = pb["rp"][a:b + 1]
        ci = pb["ci"][rp[0]:rp[-1]]
        data = orc.Csr(rp - rp[0], np.searchsorted(c, ci).astype(np.int32), pb["v"][rp[0]:rp[-1]], pb["y"][a:b], pb["w"][a:b], pb["o"][a:b],
                       len(c))
        q = np.append(np.full(len(c), np.float64(np.float32(lam))), 1.0 / 100000.0)
        want, _ = orc.liblinear_train(data, np.zeros(len(q)), np.zeros(len(q)), 1.0 / q, 1e-14, 100000)
        got = models[0, key_ptr[k]:key_ptr[k + 1]]
        assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max(), k


def test_fit_then_score_without_a_dense_model():
    import mlease_b200 as mb
    rng = np.random.default_rng(1600)
    D, K = 40000, 60
    rows = rng.integers(1, 150, K); rows[::4] = 1
    pools = _pools(rng, K, D, 10, 120)
    tr = _keyed(rng, rows, pools, D)
    # held-out rows of the same keys: half their columns from the key's pool, half never listed by its training rows
    te_pools = [np.unique(np.concatenate([p, rng.choice(D, 30, replace=False)])) for p in pools]
    te = _keyed(rng, rng.integers(1, 20, K), te_pools, D, per_row=16)
    lams = (0.5, 3.0)
    key_ptr, cols, models, _ = _naive(tr, lams, True)
    dense, _ = _naive(tr, lams, False)
    mp, mc, mv = mb.keyed_models_for_scoring(key_ptr, cols, models)
    pred = mb.score_keyed(te["v"], te["krs"], te["rp"], te["ci"], D, mp, mc, mv, offset=te["o"])
    # the dense call's model restricted to the same lists
    dv = np.concatenate([dense[l, k, cols[key_ptr[k]:key_ptr[k + 1]]] for l in range(2) for k in range(K)]).astype(np.float32)
    want = mb.score_keyed(te["v"], te["krs"], te["rp"], te["ci"], D, mp, mc, dv, offset=te["o"])
    key_of_row = np.repeat(np.arange(K), np.diff(te["krs"]))
    one = rows[key_of_row] == 1
    assert np.array_equal(pred[:, one].view(np.uint32), want[:, one].view(np.uint32))
    # an fp64 evaluation of the sparse models (their float32 values widened): ref = offset + sum over listed columns of beta * x,
    # the intercept's x = 1; S = the same sum of magnitudes, X = sum of |x| over the listed columns
    n = len(key_of_row)
    ref, S, X, m = np.zeros((2, n)), np.zeros((2, n)), np.zeros(n), np.zeros(n)
    for i, k in enumerate(key_of_row):
        c = cols[key_ptr[k]:key_ptr[k + 1]]
        x = np.zeros(D + 1); x[D] = 1.0
        a, b = te["rp"][i], te["rp"][i + 1]
        x[te["ci"][a:b]] = te["v"][a:b]
        X[i], m[i] = np.abs(x[c]).sum(), b - a
        for l in range(2):
            terms = mv[mp[l * K + k]:mp[l * K + k + 1]].astype(np.float64) * x[c]
            ref[l, i] = np.float64(te["o"][i]) + terms.sum()
            S[l, i] = abs(np.float64(te["o"][i])) + np.abs(terms).sum()
    eps = np.float64(np.finfo(np.float32).eps)
    # multi-row keys: each coefficient differs from the dense call's by the spread, and each side rounds its fp32 copy and its score
    spread = 1e-6 * max(1.0, np.abs(dense).max())
    bound = X * spread + 4 * eps * S
    assert np.all(np.abs(pred.astype(np.float64) - want.astype(np.float64)) <= bound)
    assert np.all(np.abs(pred.astype(np.float64) - ref) <= (m + 4) * eps * S)


def test_two_devices_shard_the_keys():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    rng = np.random.default_rng(1700)
    D, K = 60000, 400
    pb = _keyed(rng, np.ones(K, np.int64), _pools(rng, K, D, 8, 200), D, per_row=200)
    one = _naive(pb, (0.5, 2.0), True)
    halves, out = [(0, K // 2 + 7), (K // 2 + 7, K)], [None, None]

    def run(i):
        out[i] = _naive(_slice(pb, *halves[i]), (0.5, 2.0), True, device=i)
    ts = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    kp = np.concatenate([out[0][0], out[1][0][1:] + out[0][0][-1]])
    assert np.array_equal(kp, one[0])
    assert np.array_equal(np.concatenate([out[0][1], out[1][1]]), one[1])
    assert np.array_equal(np.concatenate([out[0][2], out[1][2]], axis=1).view(np.uint64), one[2].view(np.uint64))
