"""GPU tests of keyed scoring under the full posterior (mlease_score_keyed_cov): pred bit for bit mlease_score_keyed's for 1 - 7 models
per key and for rows of up to 1 100 entries; pred_var within 2 float ulps of numpy's fp64 x_L^T Sigma x_L + unlisted terms, with
lambda_map and binary_feature; a diagonal Sigma within 1 ulp of mlease_score_keyed_var; NaN for an empty block; streamed equal to
resident bit for bit, two devices equal to one; the refusals; and fit then score of 50 000 keys over 2 000 000 features."""
import resource
import threading

import numpy as np
import pytest

from test_gpu_keyed_sparse import _key_cols, _wide

pytestmark = pytest.mark.gpu


@pytest.fixture
def budget():
    from mlease_b200 import _hooks
    yield _hooks.set_keyed_budget
    _hooks.set_keyed_budget(0)


def _data(rng, K, G, D=5000, empty=(), row_lens=None):
    """K keys; model g*K + k lists a sorted pool of the key's columns then the intercept, with a random SPD Sigma; test rows list half
    their columns from the key's pool and half outside it (unlisted); models in `empty` have no block.  row_lens: pools of 600 - 700
    columns and 1 - 3 rows per key whose lengths cycle through row_lens (ceil(len / 2) listed, the last among them, the rest
    unlisted), so that a row's pairs span several 256-entry tiles of score_keyed_cov_kernel"""
    lo, hi = (600, 700) if row_lens else (4, 60)
    pools = [np.sort(rng.choice(D, int(rng.integers(lo, hi)), replace=False)) for _ in range(K)]
    nk = rng.integers(1, 4 if row_lens else 40, K)
    nk[3] = 0
    rp, ci = [0], []
    for k in range(K):
        for _ in range(nk[k]):
            if row_lens:
                L = row_lens[(len(rp) - 1) % len(row_lens)]
                a = rng.choice(pools[k], (L + 1) // 2, replace=False)
                out = np.setdiff1d(np.arange(D), pools[k])
                b = rng.choice(out[out < a.max()], L // 2, replace=False)   # the row's last entry is listed: it pairs across tiles
            else:
                a = rng.choice(pools[k], min(len(pools[k]), int(rng.integers(1, 12))), replace=False)
                b = rng.choice(D, int(rng.integers(0, 8)), replace=False)
            c = np.unique(np.concatenate([a, b]))
            ci.append(c); rp.append(rp[-1] + len(c))
    ci = np.concatenate(ci).astype(np.int32)
    pb = dict(krs=np.concatenate([[0], np.cumsum(nk)]).astype(np.int64), rp=np.array(rp, np.int64), ci=ci,
              v=rng.normal(size=len(ci)).astype(np.float32), o=rng.normal(0, 0.1, int(nk.sum())).astype(np.float32), D=D, K=K)
    mp, mc, mv, cp, cv = [0], [], [], [0], []
    for g in range(G):
        for k in range(K):
            cols = np.append(pools[k], D)
            n = len(cols)
            mc.append(cols); mv.append(rng.normal(size=n).astype(np.float32)); mp.append(mp[-1] + n)
            if g * K + k in empty:
                cp.append(cp[-1]); continue
            A = rng.normal(size=(n, n)) * 0.05
            S = A @ A.T + np.diag(rng.uniform(0.5, 2.0, n))
            cv.append(S[np.tril_indices(n)]); cp.append(cp[-1] + n * (n + 1) // 2)
    models = dict(mp=np.array(mp, np.int64), mc=np.concatenate(mc).astype(np.int32), mv=np.concatenate(mv),
                  cp=np.array(cp, np.int64), cv=np.concatenate(cv) if cv else np.zeros(0), vd=rng.uniform(0.1, 3.0, G * K).astype(np.float32))
    return pb, models


def _score(pb, md, **kw):
    import mlease_b200 as mb
    return mb.score_keyed_cov(pb["v"], pb["krs"], pb["rp"], pb["ci"], pb["D"], md["mp"], md["mc"], md["mv"], md["cp"], md["cv"], md["vd"],
                              offset=pb["o"], **kw)


def _ref(pb, md, G, lm=None, binary=False):
    """fp64 x_L^T Sigma x_L + sum over unlisted columns of v_c x_c^2 for every (model, record); NaN for an empty block"""
    K, D = pb["K"], pb["D"]
    out = np.zeros((G, pb["krs"][-1]))
    for g in range(G):
        for k in range(K):
            m = g * K + k
            cols = md["mc"][md["mp"][m]:md["mp"][m + 1]]
            n = len(cols)
            blk = md["cv"][md["cp"][m]:md["cp"][m + 1]]
            S = None
            if len(blk):
                S = np.zeros((n, n)); S[np.tril_indices(n)] = blk; S = S + np.tril(S, -1).T
            for i in range(pb["krs"][k], pb["krs"][k + 1]):
                if S is None:
                    out[g, i] = np.nan; continue
                c = pb["ci"][pb["rp"][i]:pb["rp"][i + 1]]
                x = np.ones(len(c)) if binary else pb["v"][pb["rp"][i]:pb["rp"][i + 1]].astype(np.float64)
                p = np.searchsorted(cols, c)
                listed = (p < n) & (cols[np.minimum(p, n - 1)] == c)
                xl = np.zeros(n); xl[p[listed]] = x[listed]
                if cols[-1] == D:
                    xl[-1] = 1.0
                vu = np.full(len(c), np.float64(md["vd"][m]))
                if lm is not None:
                    vu = np.where(lm[c] > 0, 1.0 / lm[c].astype(np.float64), vu)
                out[g, i] = xl @ S @ xl + (vu[~listed] * x[~listed] ** 2).sum()
    return out


def _ulps(got, want, n):
    ok = np.isnan(want)
    assert np.array_equal(np.isnan(got), ok)
    w = want[~ok]
    assert np.all(np.abs(got[~ok].astype(np.float64) - w) <= n * np.spacing(np.abs(w).astype(np.float32)).astype(np.float64))


LONG_ROWS = (1, 255, 256, 257, 512, 513, 1100)   # entries per row: one tile, a full tile, one past it, two, two and one, four


@pytest.mark.parametrize("G,row_lens", [pytest.param(G, None, id=str(G)) for G in (1, 2, 3, 4, 5, 7)] +
                         [pytest.param(G, LONG_ROWS, id="long-%d" % G) for G in (1, 3)])
def test_pred_and_pred_var(G, row_lens):
    import mlease_b200 as mb
    rng = np.random.default_rng(3100 + G + (100 if row_lens else 0))
    K = 12
    pb, md = _data(rng, K, G, empty={1, G * K - 1}, row_lens=row_lens)
    lm = np.zeros(pb["D"], np.float32)
    lm[rng.choice(pb["D"], 800, replace=False)] = rng.uniform(0.2, 5.0, 800).astype(np.float32)
    for binary, lmap in [(False, None), (True, lm), (False, lm)]:
        pred, pv = _score(pb, md, lambda_map=lmap, binary_feature=binary)
        want = mb.score_keyed(pb["v"], pb["krs"], pb["rp"], pb["ci"], pb["D"], md["mp"], md["mc"], md["mv"], offset=pb["o"],
                              binary_feature=binary)
        assert np.array_equal(pred.view(np.uint32), want.view(np.uint32))
        _ulps(pv, _ref(pb, md, G, lmap, binary), 2)
        for m in (1, G * K - 1):   # the empty blocks
            g, k = divmod(m, K)
            assert np.all(np.isnan(pv[g, pb["krs"][k]:pb["krs"][k + 1]]))


def test_diagonal_sigma_matches_score_keyed_var():
    import mlease_b200 as mb
    rng = np.random.default_rng(3200)
    K, G = 16, 3
    pb, md = _data(rng, K, G)
    vp, vc, vv, cv = [0], [], [], []
    for m in range(G * K):
        cols = md["mc"][md["mp"][m]:md["mp"][m + 1]]
        d = rng.uniform(0.1, 2.0, len(cols)).astype(np.float32)
        vc.append(cols); vv.append(d); vp.append(vp[-1] + len(cols))
        S = np.diag(d.astype(np.float64))
        cv.append(S[np.tril_indices(len(cols))])
    dmd = dict(md, cv=np.concatenate(cv))
    pred, pv = _score(pb, dmd)
    p2, pv2 = mb.score_keyed_var(pb["v"], pb["krs"], pb["rp"], pb["ci"], pb["D"], md["mp"], md["mc"], md["mv"], np.array(vp, np.int64),
                                 np.concatenate(vc), np.concatenate(vv), md["vd"], offset=pb["o"])
    assert np.array_equal(pred.view(np.uint32), p2.view(np.uint32))
    _ulps(pv, pv2.astype(np.float64), 1)


def test_streamed_equals_resident(budget):
    from mlease_b200 import _hooks
    rng = np.random.default_rng(3300)
    pb, md = _data(rng, 300, 2)
    budget(0)
    r = _score(pb, md)
    assert not _hooks.keyed_last_call()[1]
    budget(256 << 10)
    s = _score(pb, md)
    bounds, streamed, _, _ = _hooks.keyed_last_call()
    assert streamed and len(bounds) > 2
    assert np.array_equal(r[0].view(np.uint32), s[0].view(np.uint32)) and np.array_equal(r[1].view(np.uint32), s[1].view(np.uint32))


def test_two_devices_equal_one():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    rng = np.random.default_rng(3400)
    K = 40
    pb, md = _data(rng, K, 1)
    one = _score(pb, md)
    h = 17
    out = [None, None]

    def part(i, k0, k1):
        a, b = pb["krs"][k0], pb["krs"][k1]
        z0, z1 = pb["rp"][a], pb["rp"][b]
        sp = dict(krs=pb["krs"][k0:k1 + 1] - a, rp=pb["rp"][a:b + 1] - z0, ci=pb["ci"][z0:z1], v=pb["v"][z0:z1], o=pb["o"][a:b], D=pb["D"])
        m0, m1 = md["mp"][k0], md["mp"][k1]
        c0, c1 = md["cp"][k0], md["cp"][k1]
        sm = dict(mp=md["mp"][k0:k1 + 1] - m0, mc=md["mc"][m0:m1], mv=md["mv"][m0:m1], cp=md["cp"][k0:k1 + 1] - c0, cv=md["cv"][c0:c1],
                  vd=md["vd"][k0:k1])
        out[i] = _score(sp, sm, device=i)
    ts = [threading.Thread(target=part, args=(0, 0, h)), threading.Thread(target=part, args=(1, h, K))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert np.array_equal(np.concatenate([out[0][1], out[1][1]], axis=1).view(np.uint32), one[1].view(np.uint32))


def test_refusals():
    import mlease_b200 as mb
    rng = np.random.default_rng(3500)
    pb, md = _data(rng, 8, 1)
    short = dict(md, cp=md["cp"].copy())
    short["cp"][3:] -= 1
    with pytest.raises(mb.MleaseError, match="covariance block of .* entries") as e:
        _score(pb, dict(short, cv=md["cv"][:-1]))
    assert e.value.code == 1
    bad = dict(md, cv=md["cv"].copy())
    bad["cv"][5] = np.inf
    with pytest.raises(mb.MleaseError, match="cov_val must be finite"):
        _score(pb, bad)
    rows = dict(pb, ci=pb["ci"].copy())
    i = int(np.argmax(np.diff(pb["rp"]) >= 2))
    r0 = pb["rp"][i]
    rows["ci"][r0], rows["ci"][r0 + 1] = rows["ci"][r0 + 1], rows["ci"][r0]
    with pytest.raises(mb.MleaseError, match="strictly ascending"):
        _score(rows, md)
    assert np.all(np.isfinite(_score(pb, md)[1]))   # the process goes on


def test_fit_then_score_at_two_million_features():
    """50 000 keys of 1 - 8 rows over 2 000 000 features: fit with the full posterior, then score the rows under it, with the process's
    peak RSS less than 2 GB above what it was; sampled records against numpy's fp64 quadratic form"""
    import mlease_b200 as mb
    rng = np.random.default_rng(3600)
    K, D = 50000, 2000000
    pb = _wide(rng, K, D, 1, 8, 40, 20)
    rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024
    key_ptr, cols, models, var, cov_ptr, cov = mb.item_model_train_cov(pb["v"], pb["krs"], pb["y"], [1.0], [1.0], rowptr=pb["rp"],
                                                                       colidx=pb["ci"], num_features=D, weight=pb["w"], offset=pb["o"])
    mp, mc, mv = mb.keyed_models_for_scoring(key_ptr, cols, models)
    cp, cv = mb.keyed_cov_for_scoring(key_ptr, cov_ptr, cov)
    vd = np.ones(K, np.float32)
    pred, pv = mb.score_keyed_cov(pb["v"], pb["krs"], pb["rp"], pb["ci"], D, mp, mc, mv, cp, cv, vd, offset=pb["o"])
    grown = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024 - rss0
    assert grown < 2 << 30, grown
    want = mb.score_keyed(pb["v"], pb["krs"], pb["rp"], pb["ci"], D, mp, mc, mv, offset=pb["o"])
    assert np.array_equal(pred.view(np.uint32), want.view(np.uint32))
    for k in rng.choice(K, 60, replace=False):
        c = np.append(_key_cols(pb, k), D)
        n = len(c)
        S = np.zeros((n, n)); S[np.tril_indices(n)] = cv[cp[k]:cp[k + 1]]; S = S + np.tril(S, -1).T
        for i in range(pb["krs"][k], pb["krs"][k + 1]):
            x = np.zeros(n); x[-1] = 1.0
            x[np.searchsorted(c, pb["ci"][pb["rp"][i]:pb["rp"][i + 1]])] = pb["v"][pb["rp"][i]:pb["rp"][i + 1]]
            r = x @ S @ x
            assert abs(float(pv[0, i]) - r) <= 2 * float(np.spacing(np.float32(r))), (k, i)
