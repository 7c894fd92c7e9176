"""The K1 gradient pass of multi-problem ADMM batches (-m gpu), problem by problem and column by column, against the fp64 reference of
tests/k1_reference.py within the per-column bound derived from each kernel's arithmetic: every variant batch_k1 picks (dense
G = 1 with 16 .. 1 row slices, G = 2, G = 4; CSR fixed point with beta in shared / global memory and with column windows; general
CSR with float atomics; fused multi-lambda with LP = 1, 2, 4), both CTA mappings, active subsets and repeats.  The loss and the
emitted sqrt(d) (sdvec) or bf16 Xt operand are checked the same way."""
import numpy as np
import pytest

import k1_reference as kr

pytestmark = pytest.mark.gpu

WORST = {}   # variant -> worst ratio of |error| to bound seen (gradient columns)


@pytest.fixture(scope="module")
def mb():
    import mlease_b200
    return mlease_b200


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    for k in sorted(WORST):
        print("K1 worst error/bound %-28s %.3e" % (k, WORST[k]))


def _grad(s, W, active=None, rows=None, sd=False, xt=False):
    from mlease_b200 import _hooks
    return _hooks.batch_grad(s, W, active=active, rows=rows, want_sd=sd, want_xt=xt)


def _session(mb, D, L, cases, policy=0, binary=False):
    s = mb.AdmmSession(len(cases), D, [0.5 * (l + 1) for l in range(L)], hessian_policy=policy, binary_feature=binary)
    for p, c in enumerate(cases):
        if "X" in c:
            s.add_partition_dense(p, c["X"], c["response"], c["weight"], c["offset"])
        else:
            s.add_partition_csr(p, c["rowptr"], c["colidx"], c["vals"], c["response"], c["weight"], c["offset"])
    s.begin()
    return s


def _variant(res):
    k = res["kind"]
    if k == "dense":
        return "dense G=%d nsl=%d" % (res["G"], res["nsl"])
    if k == "fused":
        return "fused LP=%d" % res["G"]
    if k == "fx":
        return "fx beta in %s" % ("smem" if res["G"] else "global")
    return k


def _check(res, parts, betas, L, active, sd=False, xt=False):
    """Every active problem within its bounds (gradient per column, loss, sqrt(d) / Xt); inactive problems NaN."""
    tag = _variant(res) + (" dyn" if res["dyn"] else " static")
    for b in range(len(betas)):
        if not active[b]:
            assert np.all(np.isnan(res["g"][b])) and np.isnan(res["f"][b]) and res["chunks"][b] == 0
            continue
        part = parts[b // L]
        ref = kr.reference(part, betas[b])
        plan = kr.plan_from_info(res, b, part.n)
        err = kr.row_errors(part, ref, plan)
        assert plan.chunks >= 1
        bnd, terms = kr.grad_bound(part, ref, plan, err)
        r = kr.ratio(res["g"][b] - ref.g, bnd)
        if plan.kind.startswith("fx"):   # the documented fixed-point resolution against the fp32 rounding it sits beside
            on = terms["fp32"] > 0
            key = "fixed-point/fp32 term " + tag
            WORST[key] = max(WORST.get(key, 0.0), float((terms["fx"][on] / terms["fp32"][on]).max()))
        assert np.all(r <= 1.0), (tag, b, int(np.argmax(r)), float(r.max()), res["g"][b][np.argmax(r)], ref.g[np.argmax(r)])
        WORST[tag] = max(WORST.get(tag, 0.0), float(r.max()))
        assert abs(res["f"][b] - ref.f) <= kr.loss_bound(part, ref, plan, err), (tag, b, res["f"][b], ref.f)
        if sd:
            rs = kr.ratio(res["sd"][b].astype(np.float64) - ref.sd, kr.sd_bound(ref, err))
            assert np.all(rs <= 1.0), ("sd", tag, b, float(rs.max()))
            WORST["sqrt(d) " + tag] = max(WORST.get("sqrt(d) " + tag, 0.0), float(rs.max()))
        if xt:
            rx = kr.xt_check(part, ref, err, res["xt"][b])
            WORST["Xt " + tag] = max(WORST.get("Xt " + tag, 0.0), rx)


def _dense_plan(D):
    ncg = (D + 1 + 3) // 4
    G = -(-ncg // 256)
    G = 4 if G == 3 else G
    RT = 4 if G == 4 else 8
    nsl = min(16, max(1, 256 // ncg)) if G == 1 else 1
    return G, RT, nsl


def _betas(parts_seeds, Dg, L, seed, edge):
    out = []
    for p, ps in enumerate(parts_seeds):
        out += kr.make_betas(Dg, L, seed + p, edge_seed=ps if edge else None)
    return out


def _run_subsets(s, parts, betas, L, rows, sd, xt, fixed_chunking):
    """All problems, then a strict subset, then one: the bound holds for each; problems whose chunking does not depend on the others
    (static mapping, fused) are bitwise their all-active values, under the dynamic mapping k1_chunks changes.  Then a repeat of the
    all-active pass, bitwise (every variant here is deterministic)."""
    nprob = len(betas)
    W = np.array(betas)
    full = np.ones(nprob, np.int32)
    r0 = _grad(s, W, full, rows, sd, xt)
    _check(r0, parts, betas, L, full, sd, xt)
    subsets = [np.array([b % 2 for b in range(nprob)], np.int32), np.eye(nprob, dtype=np.int32)[nprob - 1]] if nprob > 1 else []
    for act in subsets:
        r = _grad(s, W, act, rows, sd, xt)
        _check(r, parts, betas, L, act, sd, xt)
        on = act.astype(bool)
        if fixed_chunking:
            np.testing.assert_array_equal(r["g"][on], r0["g"][on])
            np.testing.assert_array_equal(r["f"][on], r0["f"][on])
            np.testing.assert_array_equal(r["chunks"][on], r0["chunks"][on])
        else:
            assert np.all(r["chunks"][on] != r0["chunks"][on]), (r["chunks"], r0["chunks"])
    r1 = _grad(s, W, full, rows, sd, xt)
    np.testing.assert_array_equal(r1["g"], r0["g"])
    np.testing.assert_array_equal(r1["f"], r0["f"])
    if sd:
        for a, b in zip(r0["sd"], r1["sd"]):
            np.testing.assert_array_equal(a, b)
    return r0


DENSE_D = [1, 3, 29, 61, 125, 253, 509, 1021, 2045, 4095]


# (features, partitions, lambdas): G = 1 with nsl 16 (D = 1 .. 61), 8, 4, 2, 1, then G = 2 and G = 4.  P x L = 1 x 3 (dynamic
# mapping) for every width, on many tiles with a partial last one; 3 x 1, 3 x 2 (dynamic) and 9 x 4 = 36 problems (static) with the
# partitions' rows cycling through below one tile, exactly one tile, and many tiles with a partial last one.
@pytest.mark.parametrize("D,P,L", [(d, 1, 3) for d in DENSE_D] + [(509, 3, 1), (4095, 3, 1), (125, 3, 2), (2045, 3, 2), (61, 9, 4),
                                                                   (1021, 9, 4)])
def test_dense_batches(mb, D, P, L):
    G, RT, nsl = _dense_plan(D)
    R = RT * nsl
    sizes = [R * max(3, 3000 // R) + max(1, R // 2 - 1), max(1, R // 2), R]
    edge = D >= 3 and (D + P) % 2 == 0
    seeds = [100 + D + p for p in range(P)]
    built = [kr.synth(sd_, sizes[p % 3], D, dense=True, edge=edge) for p, sd_ in enumerate(seeds)]
    cases, parts = [c for c, _ in built], [p for _, p in built]
    betas = _betas(seeds, D, L, 7 + D, edge)
    with _session(mb, D, L, cases) as s:
        r = _run_subsets(s, parts, betas, L, [p.n for p in parts], False, True, fixed_chunking=P * L > 32)
    assert r["kind"] == "dense" and r["G"] == G and r["nsl"] == nsl and r["RT"] == RT
    assert (r["dyn"] > 0) == (P * L <= 32)


# fused multi-lambda kernel: two partitions of 4097 rows (nine segments of 456 rows, the last one shorter), empty rows, a column of the first
# rows only (one segment), columns no row lists, edge data; L = 3 runs LP = 4 with an idle lane.  The last case reads
# binary_feature (every stored value 1).
@pytest.mark.parametrize("L,edge,binary", [(1, True, False), (2, True, False), (3, True, False), (4, True, False), (2, False, True)])
def test_fused_batches(mb, L, edge, binary):
    D = 301
    seeds = [500 + L, 600 + L]
    built = [kr.synth(sd_, 4097, D, nnz=10, edge=edge, empty_rows=True, binary=binary) for p, sd_ in enumerate(seeds)]
    cases, parts = [c for c, _ in built], [p for _, p in built]
    betas = _betas(seeds, D, L, 11 + L, edge)
    with _session(mb, D, L, cases, binary=binary) as s:
        r = _run_subsets(s, parts, betas, L, [p.n for p in parts], True, False, fixed_chunking=True)
    assert r["kind"] == "fused" and r["G"] == {1: 1, 2: 2, 3: 4, 4: 4}[L] and r["dyn"] == 0
    assert np.all(r["chunks"] >= 9)


# CSR fixed point (no fused kernel): L = 5 with beta in shared memory, L = 3 at ~20 000 features (beta read from global memory; the
# 4-wide interleaved vectors of the fused kernel do not fit), L = 2 at 30 001 features (column windows).  Matrix-free sessions:
# the pass is the same, and no Gram is allocated for the wide ones.
@pytest.mark.parametrize("P,L,D,n,kind,bsm", [(2, 5, 1001, 3000, "fx", 1), (1, 3, 20003, 3000, "fx", 0), (1, 2, 30001, 2500, "fx_window", 0)])
def test_fixed_point_batches(mb, P, L, D, n, kind, bsm):
    seeds = [700 + D + p for p in range(P)]
    built = [kr.synth(sd_, n - 111 * p, D, nnz=40, edge=True, empty_rows=True) for p, sd_ in enumerate(seeds)]
    cases, parts = [c for c, _ in built], [p for _, p in built]
    betas = _betas(seeds, D, L, 13 + L, True)
    with _session(mb, D, L, cases, policy=2) as s:
        r = _run_subsets(s, parts, betas, L, [p.n for p in parts], True, False, fixed_chunking=False)
    assert r["kind"] == kind and r["G"] == bsm and r["dyn"] == P * L


# general CSR (repeated and unsorted columns: float atomics, serial bf16 emit of the repeated columns): bound and Xt; no bitwise
# repeat (the float atomics commute only up to rounding)
@pytest.mark.parametrize("P,L", [(2, 2), (1, 1)])
def test_general_csr_batches(mb, P, L):
    D = 257
    seeds = [800 + P + p for p in range(P)]
    built = [kr.synth(sd_, 3000 + 77 * p, D, nnz=12, edge=True, dup=True, empty_rows=True) for p, sd_ in enumerate(seeds)]
    cases, parts = [c for c, _ in built], [p for _, p in built]
    assert any(len(set(c["colidx"][c["rowptr"][i]:c["rowptr"][i + 1]])) < c["rowptr"][i + 1] - c["rowptr"][i] for c in cases for i in range(100))
    betas = _betas(seeds, D, L, 17, True)
    nprob = P * L
    with _session(mb, D, L, cases) as s:
        full = np.ones(nprob, np.int32)
        r = _grad(s, np.array(betas), full, [p.n for p in parts], False, True)
        _check(r, parts, betas, L, full, xt=True)
        if nprob > 1:
            act = np.eye(nprob, dtype=np.int32)[0]
            _check(_grad(s, np.array(betas), act, [p.n for p in parts], False, True), parts, betas, L, act, xt=True)
    assert r["kind"] == "csr" and r["G"] == 1 and (r["dyn"] > 0) == (nprob > 1)


def test_hook_refusals(mb):
    from mlease_b200._native import MleaseError
    case, part = kr.synth(5, 200, 30, dense=True)
    s = mb.AdmmSession(1, 30, [1.0])
    s.add_partition_dense(0, case["X"], case["response"], case["weight"], case["offset"])
    W = np.zeros((1, 31))
    with pytest.raises(MleaseError):
        _grad(s, W)   # no batch before begin()
    s.begin()
    with pytest.raises(MleaseError):
        _grad(s, W, rows=[200], sd=True)   # a dense batch has no sdvec
    r = _grad(s, W, rows=[200], xt=True)
    assert r["kind"] == "dense" and r["dyn"] == 0 and r["chunks"][0] >= 1
    s.close()
