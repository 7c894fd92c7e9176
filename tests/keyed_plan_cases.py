"""Seeded keyed calls whose plans are pinned by tests/golden/keyed_plans.npz (tests/test_gpu_keyed_plans.py, written by
tests/golden/make_keyed_plans.py).

Every case is one keyed C ABI call on small seeded data: NaiveTrain over CSR (pageable, pinned and device input, and one-row keys),
NaiveTrain over dense rows (host and device input), ItemModelTrain with the posterior variance, NaiveTrain over a 90 000-feature
dictionary (the column lists are built), and score_keyed / score_keyed_var at L = 1, 3, 5 with pred on the host and on the device.
Each runs under the budgets of the keyed-budget hook its plans name (by default the first three): 0 (resident, one chunk), a cap under
which the call is still resident but solves or scores in several chunks (chunked), a cap under which it streams in exactly one key
range (one_range), and a cap that streams it through several key ranges (streamed).  Three more cases reach a one-range streamed
plan (dense host rows, scoring many models over few rows) and streamed scoring ranges of several keys.  run() returns what the call recorded
(key bounds, streamed) and its outputs."""
import numpy as np

DENSE_HOST_D = 1000   # a resident dense call from host rows counts 256 MB of staging: its keys need states that large to chunk


def _csr_keys(rng, rows, D, nnz):
    K, n = len(rows), int(np.sum(rows))
    krs = np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)
    ci = np.stack([np.sort(rng.choice(D, nnz, replace=False)) for _ in range(n)]).astype(np.int32).reshape(-1)
    v = rng.normal(size=n * nnz).astype(np.float32)
    beta = rng.normal(size=D) / np.sqrt(nnz)
    z = (v.reshape(n, nnz) * beta[ci.reshape(n, nnz)]).sum(1)
    y = (rng.random(n) < 1 / (1 + np.exp(-(z - 0.3)))).astype(np.int32)
    return dict(krs=krs, rp=np.arange(n + 1, dtype=np.int64) * nnz, ci=ci, v=v, y=y, w=rng.uniform(0.5, 2.0, n).astype(np.float32),
                o=rng.normal(0, 0.1, n).astype(np.float32), D=D, K=K)


def _wide_keys(rng, K, D, per_row=10):
    """K keys of 5 .. 20 rows, each listing columns of its own pool of 20 .. 200 of D features: few entries per key, so that the width
    bound of the first key (its stored entries) lets the call stay resident under a budget its keys' states exceed"""
    pools = [np.unique(rng.choice(D, int(rng.integers(20, 201)), replace=False)) for _ in range(K)]
    rows = rng.integers(5, 21, K)
    rp, ci = [0], []
    for n, pool in zip(rows, pools):
        for _ in range(n):
            c = np.sort(rng.choice(pool, per_row, replace=False))
            ci.append(c); rp.append(rp[-1] + len(c))
    ci = np.concatenate(ci).astype(np.int32)
    n = int(rows.sum())
    y = (rng.random(n) < 0.4).astype(np.int32)
    return dict(krs=np.concatenate([[0], np.cumsum(rows)]).astype(np.int64), rp=np.array(rp, np.int64), ci=ci,
                v=rng.normal(size=len(ci)).astype(np.float32), y=y, w=rng.uniform(0.5, 2.0, n).astype(np.float32),
                o=rng.normal(0, 0.1, n).astype(np.float32), D=D, K=K)


def _dense_keys(rng, K, D, lo, hi):
    rows = rng.integers(lo, hi, K)
    krs = np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)
    X = rng.normal(size=(int(krs[-1]), D)).astype(np.float32)
    y = (rng.random(int(krs[-1])) < 1 / (1 + np.exp(-X[:, :5].sum(1)))).astype(np.int32)
    return dict(krs=krs, X=X, y=y)


def _model_lists(rng, M, D, var):
    """M sparse lists over columns [0, D] (D = the intercept); every 7th from the 4th on is empty"""
    ptr, col, val = [0], [], []
    for m in range(M):
        if m % 7 != 3:
            cols = np.sort(rng.choice(D + 1, int(rng.integers(1, min(60, D + 1))), replace=False))
            col += list(cols)
            val += list(rng.uniform(0.01, 1.0, len(cols)) if var else rng.normal(size=len(cols)))
        ptr.append(len(col))
    return np.array(ptr, np.int64), np.array(col, np.int32), np.array(val, np.float32)


def _scoring(rng, L, var, D=20000):
    """30 keys; at 20 000 features the model table, not the rows, decides the resident chunks, and a streamed range holds one key"""
    K = 30
    rows = rng.integers(5, 40, K); rows[[2, 9]] = 0
    krs = np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)
    n = int(krs[-1])
    nnz = rng.integers(0, 20, n)
    rp = np.concatenate([[0], np.cumsum(nnz)]).astype(np.int64)
    ci = np.concatenate([np.sort(rng.choice(D, c, replace=False)) for c in nnz]).astype(np.int32)
    d = dict(krs=krs, rp=rp, ci=ci, v=rng.normal(size=len(ci)).astype(np.float32), o=rng.normal(size=n).astype(np.float32), D=D, K=K, L=L)
    d["mp"], d["mc"], d["mv"] = _model_lists(rng, L * K, D, False)
    if var:
        d["vp"], d["vc"], d["vv"] = _model_lists(rng, L * K, D, True)
        d["vd"] = rng.uniform(0.5, 2.0, L * K).astype(np.float32)
    return d


def _scoring_few_rows(rng, L=8, K=10, D=20):
    """many models over few rows: the models alone can exceed three quarters of a budget whose quarter holds every row, so the call
    streams in one range"""
    krs = np.arange(K + 1, dtype=np.int64) * 2
    n = int(krs[-1])
    ci = np.concatenate([np.sort(rng.choice(D, 3, replace=False)) for _ in range(n)]).astype(np.int32)
    d = dict(krs=krs, rp=np.arange(n + 1, dtype=np.int64) * 3, ci=ci, v=rng.normal(size=len(ci)).astype(np.float32),
             o=rng.normal(size=n).astype(np.float32), D=D, K=K, L=L)
    d["mp"] = np.arange(L * K + 1, dtype=np.int64) * (D + 1)
    d["mc"] = np.tile(np.arange(D + 1, dtype=np.int32), L * K)
    d["mv"] = rng.normal(size=L * K * (D + 1)).astype(np.float32)
    return d


def _naive_csr(seed, where, one_row=False):
    def make():
        rng = np.random.default_rng(seed)
        if one_row:
            return _csr_keys(rng, np.ones(200, np.int64), 30, 6)
        rows = rng.integers(200, 600, 16); rows[[3, 11]] = [5, 0]      # below data.size.threshold = 40, and a key without rows
        return _csr_keys(rng, rows, 48, 12)
    return dict(kind="naive_csr", where=where, make=make, bitwise=one_row)


CASES = {
    "naive_csr_pageable": _naive_csr(501, "pageable"),
    "naive_csr_pinned": _naive_csr(501, "pinned"),
    "naive_csr_device": _naive_csr(501, "device"),
    "naive_csr_one_row": _naive_csr(502, "pageable", one_row=True),
    "naive_dense_host": dict(kind="naive_dense", where="pageable", make=lambda: _dense_keys(np.random.default_rng(503), 8, DENSE_HOST_D, 100, 200)),
    "naive_dense_device": dict(kind="naive_dense", where="device", make=lambda: _dense_keys(np.random.default_rng(504), 16, 40, 200, 500)),
    "item_model_var": dict(kind="item_model", where="pageable", make=lambda: _csr_keys(np.random.default_rng(505), np.arange(20) * 23 % 400 + 200, 40, 8)),
    "naive_wide": dict(kind="naive_csr", where="pageable", wide=True, make=lambda: _wide_keys(np.random.default_rng(506), 24, 90000)),
    # host rows count 256 MB of staging against a resident call: far below that, the call streams, in one range while its rows and
    # states fit a quarter of the budget
    "naive_dense_host_one_range": dict(kind="naive_dense", where="pageable", plans=("resident", "one_range", "streamed"),
                                       make=lambda: _dense_keys(np.random.default_rng(507), 16, 40, 300, 301)),
    # 50 features: a streamed range is cut by its rows' bytes and holds several keys
    "score_L3_host_multi_key": dict(kind="score", var=False, pred="host", bitwise=True, plans=("resident", "streamed"),
                                    make=lambda: _scoring(np.random.default_rng(508), 3, False, D=50)),
    "score_L8_host_one_range": dict(kind="score", var=False, pred="host", bitwise=True, plans=("resident", "one_range", "streamed"),
                                    make=lambda: _scoring_few_rows(np.random.default_rng(509))),
}
for _var in (False, True):
    for _L in (1, 3, 5):
        for _pred in ("host", "device"):
            CASES["score%s_L%d_%s" % ("_var" if _var else "", _L, _pred)] = dict(
                kind="score", var=_var, pred=_pred, bitwise=True, make=(lambda L=_L, v=_var: _scoring(np.random.default_rng(600 + 10 * L + v), L, v)))


def _placed(a, where):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a))
    return t.pin_memory() if where == "pinned" else t.cuda() if where == "device" else a


def run(mb, name, budget, data=None):
    """case `name` under keyed budget `budget` -> (bounds, streamed, {output name: array}); data: the case's make(), if made"""
    from mlease_b200 import _hooks
    c = CASES[name]
    d = c["make"]() if data is None else data
    _hooks.set_keyed_budget(budget)
    try:
        if c["kind"] == "naive_csr":
            p = {k: _placed(d[k], c["where"]) for k in ("rp", "ci", "v", "y", "w", "o")}
            lm = np.zeros(d["D"], np.float32); lm[[1, 9]] = [0.2, 5.0]
            thr = 0 if c.get("bitwise") else 10 if c.get("wide") else 40
            lams = [1.0] if c.get("wide") else [0.5, 3.0]
            m, s = mb.naive_train(p["v"], d["krs"], p["y"], lams, rowptr=p["rp"], colidx=p["ci"], num_features=d["D"], weight=p["w"],
                                  offset=p["o"], lambda_map=lm, data_size_threshold=thr)
            out = dict(model=m, skipped=s)
        elif c["kind"] == "naive_dense":
            m, s = mb.naive_train(_placed(d["X"], c["where"]), d["krs"], _placed(d["y"], c["where"]), [1.0, 4.0][:1 if c["where"] == "pageable" else 2])
            out = dict(model=m, skipped=s)
        elif c["kind"] == "item_model":
            means = np.linspace(-1.0, 1.0, d["K"])
            m, v = mb.item_model_train(d["v"], d["krs"], d["y"], [0.5, 4.0], [1.0], rowptr=d["rp"], colidx=d["ci"], num_features=d["D"],
                                       intercept_prior_mean=means, weight=d["w"], offset=d["o"], compute_var=True)
            out = dict(model=m, var=v)
        else:
            import torch
            n = len(d["rp"]) - 1
            dev = c["pred"] == "device"
            pred = torch.zeros((d["L"], n), dtype=torch.float32, device="cuda") if dev else None
            args = (d["v"], d["krs"], d["rp"], d["ci"], d["D"], d["mp"], d["mc"], d["mv"])
            if c["var"]:
                pv = torch.zeros((d["L"], n), dtype=torch.float32, device="cuda") if dev else None
                p, q = mb.score_keyed_var(*args, d["vp"], d["vc"], d["vv"], d["vd"], offset=d["o"], out=pred, out_var=pv)
                out = dict(pred=p, pred_var=q)
            else:
                out = dict(pred=mb.score_keyed(*args, offset=d["o"], out=pred))
            out = {k: (a.cpu().numpy() if hasattr(a, "cpu") else a) for k, a in out.items()}
        bounds, streamed, _, _ = _hooks.keyed_last_call()
    finally:
        _hooks.set_keyed_budget(0)
    return np.array(bounds, np.int64), bool(streamed), out
