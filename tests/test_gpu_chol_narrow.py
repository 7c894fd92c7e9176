"""GPU tests (-m gpu) of the explicit-inverse Cholesky (ldh <= 2048) on the ADMM batch, through the test hook
mlease_internal_batch_factor (not part of the C ABI), which runs the solver's rebuild code (batch_factor):

- exactly representable systems H = (I + E)(I + E)^T factorised bit for bit (Lc, Ldinv, Yinv, Hinv, padding included) at widths
  that end mid-tile, on both code paths (narrow: ldh <= 992; mid: 1024 <= ldh <= 2048), with the pairs of E placed by
  chol_reference.chol_pairs and their coverage asserted in each case;
- batch composition: every problem's bits equal its batch-of-one bits, in batch order and over a reversed subset of a batch of
  more than 64 problems (the grids over compacted Problem copies); problems marked done keep the sentinel and their Ctrl;
- the cold starts of a multi-lambda run (equal rho: followers share the leader's outcome and H^-1; distinct rho: followers
  factorise the leader's Gram partials plus their own q) and non-positive pivots;
- real Hessians within the fp64 bounds of chol_reference, and run-to-run bit equality;
- the L-BFGS direction on the explicit inverse (mlease_internal_direction) against chol_reference.two_loop."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import chol_reference as cr  # noqa: E402
from factored_reference import VALUES, ldh_of  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mb():
    import mlease_b200
    return mlease_b200


def _part(D, n, nnz, seed):
    r = np.random.default_rng(seed)
    nnz = min(nnz, D)
    ci = np.stack([np.sort(r.choice(D, nnz, replace=False)) for _ in range(n)]).astype(np.int32)
    v = r.normal(size=(n, nnz)).astype(np.float32)
    y = (r.random(n) < 0.5).astype(np.int32)
    return np.arange(n + 1, dtype=np.int64) * nnz, ci.reshape(-1), v.reshape(-1), y


class _Sess:
    """An ADMM session of P CSR partitions x L lambdas, begun, with the factor hook."""

    def __init__(self, mb, P, D, L, n=64, rhos=None):
        lam = [1.0 + l for l in range(L)]
        self.s = mb.AdmmSession(P, D, lam, rhos)
        self.s.__enter__()
        for p in range(P):
            self.s.add_partition_csr(p, *_part(D, n, 6, 1000 * p + D))
        self.s.begin()
        self.nprob, self.Dt, self.ldh = P * L, D + 1, ldh_of(D + 1)

    def factor(self, mode, **kw):
        from mlease_b200 import _hooks
        self.s.begin()
        return _hooks.batch_factor(self.s, mode, **kw)

    def close(self):
        self.s.__exit__(None, None, None)


def _pairs(Dt, b):
    """chol_pairs with problem b's own values (the same positions, the values rotated and signed per problem)."""
    p = cr.chol_pairs(Dt)
    sgn = -1.0 if b % 2 else 1.0
    return {k: sgn * VALUES[(n + b) % len(VALUES)] for n, k in enumerate(p)}


def _spd(Dt, seed, m=96):
    r = np.random.default_rng(seed)
    X = r.normal(size=(Dt, m)) * r.uniform(0.5, 2.0, (Dt, 1))
    H = X @ X.T / m
    H[np.diag_indices(Dt)] += r.uniform(0.1, 2.0, Dt)
    return H


def _gram(Dt, seed):
    """(fp32 Gram, q): an SPD G + diag(q) with G exactly fp32."""
    G = _spd(Dt, seed).astype(np.float32)
    G = (G + G.T) / 2
    return G, np.random.default_rng(seed + 1).uniform(0.5, 1.5, Dt)


def _same(a, b):
    return cr.same_bits(a, b)


def _check_exact(out, b, E, upper_sentinel=False):
    ex = cr.exact_outputs(E)
    L = out["L"][b]
    assert _same(np.tril(L), ex["L"]), "Lc"
    up = np.triu(np.ones(L.shape, bool), 1)
    if upper_sentinel:   # chol_prep writes the lower triangle only
        assert cr.is_sentinel(L[up])
    else:
        assert _same(L[up], 0.0 * L[up])
    assert _same(out["Ldinv"][b], ex["Ldinv"]), "Ldinv"
    assert _same(out["Y"][b], ex["Y"]), "Yinv"
    assert _same(out["Hinv"][b], ex["Hinv"]), "Hinv"
    Hi = out["Hinv"][b]
    assert np.array_equal(Hi.view(np.uint64), Hi.T.view(np.uint64)), "Hinv symmetric"
    assert (out["fail"][b], out["done"][b], out["hess_valid"][b], out["tot_hess"][b]) == (0, 0, 1, 1)


def _check_untouched(out, b, done=1, H=None):
    """No kernel wrote problem b's buffers (H: the Lc the hook put in for a mode-1 problem)."""
    assert cr.is_sentinel(out["L"][b]) if H is None else np.array_equal(out["L"][b], np.tril(H)), "L"
    for k in ("Ldinv", "Hinv"):
        assert cr.is_sentinel(out[k][b]), k
    Y = out["Y"][b]
    lo = np.tri(Y.shape[0], dtype=bool)
    assert cr.is_sentinel(Y[lo]) and not Y[~lo].any(), "Yinv"
    assert (out["fail"][b], out["done"][b], out["hess_valid"][b], out["tot_hess"][b]) == (0, done, 0, 0)


WIDTHS = [1, 30, 31, 32, 63, 64, 200, 991, 992, 1023, 1024, 1300, 2047]


@pytest.mark.parametrize("D", WIDTHS)
def test_exact_factors_bit_for_bit(mb, D):
    """Problem 0 comes through chol_prep (mode 2: G = H - I in fp32, q = 1), the others as H (mode 1); each has its own E."""
    Dt = D + 1
    cr.assert_coverage(Dt, cr.chol_pairs(Dt))
    P, L = (1, 3) if Dt > 1500 else (2, 2)
    t = _Sess(mb, P, D, L)
    try:
        nprob = t.nprob
        Es, H, G = [], np.zeros((nprob, Dt, Dt)), np.zeros((nprob, Dt, Dt), np.float32)
        for b in range(nprob):
            E, Hb = cr.exact_system(Dt, _pairs(Dt, b))
            Es.append(E)
            H[b] = Hb
            G[b] = (Hb - np.eye(Dt)).astype(np.float32)
        mode = np.array([2] + [1] * (nprob - 1), np.int32)
        out = t.factor(mode, H=H, G=G, q=np.ones((nprob, Dt)))
        for b in range(nprob):
            _check_exact(out, b, Es[b], upper_sentinel=(b == 0))
    finally:
        t.close()


def _one(mb, D, inputs):
    """Batch-of-one results of [(mode, H or (G, q))] in a one-problem session."""
    t = _Sess(mb, 1, D, 1)
    try:
        res = []
        for md, x in inputs:
            if md == 1:
                res.append(t.factor(np.array([1], np.int32), H=x[None]))
            else:
                res.append(t.factor(np.array([2], np.int32), G=x[0][None], q=x[1][None]))
        return res
    finally:
        t.close()


_KEYS = ("L", "Y", "Hinv", "Ldinv")


def _assert_as_one(out, b, one):
    for k in _KEYS:
        assert np.array_equal(out[k][b].view(np.uint64), one[k][0].view(np.uint64)), (b, k)
    for k in ("fail", "done", "hess_valid", "tot_hess"):
        assert out[k][b] == one[k][0], (b, k)


@pytest.mark.parametrize("D,P,L", [(200, 17, 4), (1024, 2, 2)])
def test_batch_composition_changes_no_bit(mb, D, P, L):
    """A batch of modes 0, 1 and 2 in batch order, then over a reversed subset (grids over compacted Problem copies; at 68
    problems the solver's own route): each factorised problem bitwise equal to its batch of one, the others untouched."""
    Dt = D + 1
    nprob = P * L
    mode = np.array([(0, 1, 2)[b % 3] for b in range(nprob)], np.int32)
    H = np.zeros((nprob, Dt, Dt))
    G = np.zeros((nprob, Dt, Dt), np.float32)
    q = np.ones((nprob, Dt))
    for b in range(nprob):
        if mode[b] == 1:
            H[b] = _spd(Dt, b)
        elif mode[b] == 2:
            G[b], q[b] = _gram(Dt, b)
    act = [b for b in range(nprob) if mode[b]]
    ones = dict(zip(act, _one(mb, D, [(mode[b], H[b] if mode[b] == 1 else (G[b], q[b])) for b in act])))
    t = _Sess(mb, P, D, L)
    try:
        out = t.factor(mode, H=H, G=G, q=q)
        for b in range(nprob):
            if mode[b]:
                _assert_as_one(out, b, ones[b])
            else:
                _check_untouched(out, b)
        # reversed subset: two of every three active problems (modes 1 and 2 both), mode-0 problems listed too (the kernels
        # must skip them)
        order = np.array([b for b in range(nprob)[::-1] if not mode[b] or act.index(b) % 3 != 2], np.int32)
        assert {1, 2} <= set(mode[order].tolist())
        out = t.factor(mode, H=H, G=G, q=q, order=order)
        for b in range(nprob):
            if mode[b] and b in order:
                _assert_as_one(out, b, ones[b])
            else:
                _check_untouched(out, b, done=0 if mode[b] else 1, H=H[b] if mode[b] == 1 else None)
    finally:
        t.close()


@pytest.mark.parametrize("D", [200, 1024])
def test_cold_start_equal_rho(mb, D):
    """share = L with share_factor: the leaders factorise, every follower gets the leader's Hinv bit for bit and the Ctrl
    chol_share_end_kernel sets; no kernel writes the followers' own Lc / Yinv / Ldinv.  A leader whose H is not positive definite
    fails its whole group and no one else."""
    Dt, P, L = D + 1, 2, 3
    nprob = P * L
    H = np.stack([_spd(Dt, 10 + b) for b in range(nprob)])
    ones = _one(mb, D, [(1, H[g * L]) for g in range(P)])
    t = _Sess(mb, P, D, L)
    try:
        out = t.factor(np.ones(nprob, np.int32), H=H, share=L, share_factor=True)
        for g in range(P):
            _assert_as_one(out, g * L, ones[g])
            for b in range(g * L + 1, g * L + L):
                assert np.array_equal(out["Hinv"][b].view(np.uint64), out["Hinv"][g * L].view(np.uint64))
                assert (out["fail"][b], out["done"][b], out["hess_valid"][b], out["tot_hess"][b]) == (0, 0, 1, 1)
                assert np.array_equal(out["L"][b], np.tril(H[b]))   # as the hook put it: no kernel factorised it
                assert cr.is_sentinel(out["Ldinv"][b])
                assert cr.is_sentinel(out["Y"][b][np.tri(t.ldh, dtype=bool)])
        Hbad = H.copy()
        Hbad[L, 5, 5] = -1.0   # the leader of group 1
        out = t.factor(np.ones(nprob, np.int32), H=Hbad, share=L, share_factor=True)
        for b in range(nprob):
            want = (1, 1, 0) if b >= L else (0, 0, 1)
            assert (out["fail"][b], out["done"][b], out["hess_valid"][b]) == want, b
        _assert_as_one(out, 0, ones[0])
    finally:
        t.close()


@pytest.mark.parametrize("D", [200, 1024])
def test_cold_start_distinct_rho(mb, D):
    """share = L alone: chol_prep_kernel of every follower reads the leader's Gram partials (its own hold NaN) and its own q."""
    Dt, P, L = D + 1, 2, 3
    nprob = P * L
    G = np.full((nprob, Dt, Dt), np.nan, np.float32)
    q = np.zeros((nprob, Dt))
    for b in range(nprob):
        if b % L == 0:
            G[b] = _gram(Dt, 20 + b)[0]
        q[b] = np.random.default_rng(b).uniform(0.5, 1.5, Dt)
    ones = _one(mb, D, [(2, (G[b - b % L], q[b])) for b in range(nprob)])
    t = _Sess(mb, P, D, L)
    try:
        out = t.factor(np.full(nprob, 2, np.int32), G=G, q=q, share=L)
        for b in range(nprob):
            _assert_as_one(out, b, ones[b])
    finally:
        t.close()


@pytest.mark.parametrize("D", [200, 1024])
def test_non_positive_pivots(mb, D):
    """The pivot at column p made exactly 0, negative or NaN (H = (I + E)(I + E)^T, so every other pivot is 1): fail = 1, done = 1,
    hess_valid = 0 on that problem only; its neighbours keep their exact bits."""
    Dt = D + 1
    ps = [0, 31, 32, Dt - 1] + ([255, 256, 511] if cr.is_mid(ldh_of(Dt)) else [])
    nprob = 3
    Es, H = [], np.zeros((nprob, Dt, Dt))
    for b in range(nprob):
        E, H[b] = cr.exact_system(Dt, _pairs(Dt, b))
        Es.append(E)
    t = _Sess(mb, 1, D, nprob)
    try:
        for p in ps:
            for kind in (0.0, -0.5, np.nan):
                Hb = H.copy()
                Hb[1, p, p] = Hb[1, p, p] - 1.0 + kind   # the pivot is H[p][p] - 1 + 1 = kind
                out = t.factor(np.ones(nprob, np.int32), H=Hb)
                assert (out["fail"][1], out["done"][1], out["hess_valid"][1]) == (1, 1, 0), (p, kind)
                for b in (0, 2):
                    _check_exact(out, b, Es[b])
    finally:
        t.close()


@pytest.mark.parametrize("D", [200, 991, 1024, 2047])
@pytest.mark.parametrize("dense", [False, True])
def test_real_hessians_within_fp64_bounds(mb, D, dense):
    """objective(want_hessian=True) at a point where the IRLS weights vary: Lc, Yinv and Hinv inside chol_reference's bounds,
    and the same H twice gives the same bits.  Measured worst error / bound over the eight cases on an H100 80GB (power limit
    not recorded): factor 0.016, inverse 0.0067, Hinv 0.016."""
    Dt = D + 1
    r = np.random.default_rng(D)
    n = 3 * Dt
    with mb.AdmmSession(1, D, [1.0, 2.0]) as s:
        if dense:
            X = (r.normal(size=(n, D)) * (r.random((n, D)) < 0.05)).astype(np.float32)
            y = (r.random(n) < 0.5).astype(np.int32)
            s.add_partition_dense(0, X, y)
        else:
            s.add_partition_csr(0, *_part(D, n, 12, D))
        w = r.normal(0, 0.5, Dt)
        _, _, Hr = s.objective(0, w, np.zeros(Dt), np.full(Dt, 0.3), want_grad=False, want_hessian=True, tensor=True)
        Hr = (np.tril(Hr) + np.tril(Hr, -1).T)
        from mlease_b200 import _hooks
        s.begin()
        out = _hooks.batch_factor(s, np.array([1, 1], np.int32), H=np.stack([Hr, Hr]))
    assert (out["fail"] == 0).all()
    for k in _KEYS:
        assert np.array_equal(out[k][0].view(np.uint64), out[k][1].view(np.uint64)), k
    ef = cr.factor_excess(Hr, out["L"][0])
    ey = cr.inverse_excess(out["L"][0], out["Y"][0], out["Ldinv"][0])
    eh = cr.hinv_excess(out["Y"][0], out["Hinv"][0])
    print("D", D, "dense", dense, "error / bound: factor %.3g inverse %.3g Hinv %.3g" % (ef, ey, eh))
    assert ef <= 1 and ey <= 1 and eh <= 1, (ef, ey, eh)


def test_hook_refusals(mb):
    """Every bad argument is refused before any launch, each with its own text, and the session still works after."""
    from mlease_b200 import _hooks
    D, Dt = 40, 41
    H = np.stack([np.eye(Dt)] * 4)
    with mb.AdmmSession(2, D, [1.0, 2.0]) as s:
        for p in range(2):
            s.add_partition_csr(p, *_part(D, 64, 6, p))
        one = np.ones(4, np.int32)
        with pytest.raises(mb.MleaseError, match="mlease_admm_begin was not called"):
            _hooks.batch_factor(s, one, H=H)
        s.begin()
        cases = [
            (dict(mode=np.array([1, 3, 1, 1], np.int32), H=H), "mode must be 0, 1 or 2"),
            (dict(mode=one), "mode 1 needs H"),
            (dict(mode=np.full(4, 2, np.int32), H=H), "mode 2 needs G and q"),
            (dict(mode=one, H=H, order=[0, 1, 2, 3, 0]), "launch order longer than the batch"),
            (dict(mode=one, H=H, order=[0, 4]), "launch order leaves the batch"),
            (dict(mode=one, H=H, order=[-1]), "launch order leaves the batch"),
            (dict(mode=one, H=H, order=[2, 1, 2]), "launch order repeats a problem"),
            (dict(mode=one, H=H, share=3), "share must be 0 or the batch's group_L"),
            (dict(mode=one, H=H, share=2, order=[0, 1]), "a shared cold start runs over the batch order"),
            (dict(mode=one, H=H, share_factor=True), "share_factor needs share"),
            (dict(mode=np.array([1, 1, 0, 0], np.int32), H=H, share=2, share_factor=True), "share_factor needs every problem in one mode"),
            (dict(mode=np.array([1, 0, 1, 1], np.int32), H=H, share=2), "every problem of a group has its leader's mode"),
        ]
        for kw, text in cases:
            mode = kw.pop("mode")
            with pytest.raises(mb.MleaseError, match=text.replace("(", r"\(")):
                _hooks.batch_factor(s, mode, **kw)
        with pytest.raises(mb.MleaseError, match="launch order leaves the batch"):   # refused before q or Ctrl are touched
            _hooks.batch_factor(s, np.array([1, 2, 1, 2], np.int32), H=H, G=H.astype(np.float32), q=np.ones((4, Dt)), order=[9])
        with pytest.raises(mb.MleaseError, match=r"bfgs_count must be >= 0"):
            args = _dir_args(4, Dt)
            args[5][2] = -1
            _hooks.direction(s, *args)
        # an empty launch order on a batch mixing modes 1 and 2: nothing runs, nothing is written
        out = _hooks.batch_factor(s, np.array([1, 2, 1, 2], np.int32), H=H, G=H.astype(np.float32), q=np.ones((4, Dt)),
                                     order=np.zeros(0, np.int32))
        assert all(cr.is_sentinel(out["Hinv"][b]) for b in range(4)) and (out["tot_hess"] == 0).all()
        out = _hooks.batch_factor(s, one, H=H)
        assert (out["hess_valid"] == 1).all() and np.array_equal(out["Hinv"][:, :Dt, :Dt], H)
        s.begin()
        s.run(2)   # the solver still runs on the batch the hook used
    with mb.AdmmSession(1, D, [1.0], hessian_policy=2) as s:   # matrix-free: no factor at all
        s.add_partition_csr(0, *_part(D, 64, 6, 0))
        s.begin()
        with pytest.raises(mb.MleaseError, match="a matrix-free session forms no factor"):
            _hooks.batch_factor(s, np.ones(1, np.int32), H=H[:1])
        with pytest.raises(mb.MleaseError, match="a matrix-free session forms no factor"):
            _hooks.direction(s, *_dir_args(1, Dt))
    with mb.AdmmSession(1, 3000, [1.0]) as s:   # ldh 3008: the factored direction, no explicit inverse
        s.add_partition_csr(0, *_part(3000, 64, 6, 0))
        s.begin()
        with pytest.raises(mb.MleaseError, match="only systems up to 2048"):
            _hooks.batch_factor(s, np.ones(1, np.int32), H=np.eye(3001)[None])
        with pytest.raises(mb.MleaseError, match="only systems up to 2048"):
            _hooks.direction(s, *_dir_args(1, 3001))


def _dir_args(nprob, Dt):
    M = 6
    return [np.ones(nprob, np.int32), np.ones((nprob, Dt)), np.zeros((nprob, M, Dt)), np.zeros((nprob, M, Dt)),
            np.ones((nprob, M)), np.zeros(nprob, np.int32), np.ones(nprob), np.zeros((nprob, Dt))]


@pytest.mark.parametrize("D", [200, 1024])
@pytest.mark.parametrize("L", [1, 2, 3, 4, 5])
def test_direction_on_the_explicit_inverse(mb, D, L):
    """The L-BFGS direction of a chord slot on the GPU's own Hinv (first loop fused into k1_reduce_decide_kernel,
    newton_gemv_kernel, second loop and h0_scale in newton_solve_kernel) against chol_reference.two_loop in long double:
    bfgs_count in {0, 1, 6, 7, 13} (13: the ring has wrapped twice) and h0_scale in {1, 2.5}, every combination on every problem
    position of an L-lambda batch.  dir, phi0 = dir . g and dirnorm = max |dir| within the running-error bounds; beta_t is
    float(beta + dir) bit for bit."""
    from mlease_b200 import _hooks
    Dt, M = D + 1, cr.BFGS_M
    combos = [(c, h) for c in (0, 1, 6, 7, 13) for h in (1.0, 2.5)]
    Hs = np.stack([_spd(Dt, 50 + b) for b in range(L)])
    r = np.random.default_rng(D + L)
    with mb.AdmmSession(1, D, [1.0 + l for l in range(L)]) as s:
        s.add_partition_csr(0, *_part(D, 64, 6, D))
        s.begin()
        Hinv = _hooks.batch_factor(s, np.ones(L, np.int32), H=Hs)["Hinv"]
        worst = np.zeros(3)
        for i in range(len(combos)):
            cnt = np.array([combos[(i + b) % len(combos)][0] for b in range(L)], np.int32)
            h0 = np.array([combos[(i + b) % len(combos)][1] for b in range(L)])
            g = r.normal(size=(L, Dt))
            S = r.normal(size=(L, M, Dt)) * 0.1
            Y = np.einsum("bjk,bkl->bjl", S, Hs) + 1e-3 * r.normal(size=(L, M, Dt))
            rho = 1.0 / np.einsum("bjk,bjk->bj", S, Y)
            beta = r.normal(0, 0.5, (L, Dt))
            out = _hooks.direction(s, np.ones(L, np.int32), g, S, Y, rho, cnt, h0, beta)
            for b in range(L):
                ref, bound = cr.two_loop(Hinv[b], g[b], S[b], Y[b], rho[b], cnt[b], h0[b])
                e = cr.direction_excess(out["dir"][b], out["phi0"][b], out["dirnorm"][b], g[b], ref, bound)
                worst = np.maximum(worst, e)
                assert max(e) <= 1, (b, cnt[b], h0[b], e)
                want = (beta[b] + out["dir"][b]).astype(np.float32).astype(np.float64)
                assert np.array_equal(out["beta_t"][b].view(np.uint64), want.view(np.uint64)), (b, cnt[b], h0[b])
        print("D", D, "L", L, "error / bound: dir %.3g phi0 %.3g dirnorm %.3g" % tuple(worst))
