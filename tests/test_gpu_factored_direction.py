"""GPU tests (-m gpu) of the factored Newton direction of wide systems (ldh > 2048), against the fp64 reference of
tests/factored_reference.py: the TF32-merged inverse and its bf16 symmetric packing (bitwise on exactly representable factors,
within bounds on a real Hessian), the two triangular GEMVs on the bytes each problem reads (entrywise bounds; shared passes bitwise
equal to single ones), and the rule that a follower of a shared cold-start factor keeps that factor when its leader refactorises.
The hooks are test entry points of the library, not part of its C ABI."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import factored_reference as fr  # noqa: E402

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = 1, 4


@pytest.fixture(scope="module")
def mb():
    import mlease_b200
    return mlease_b200


@pytest.fixture(scope="module")
def hooks(mb):
    from mlease_b200 import _hooks
    return _hooks.bound()


def _check(rc):
    from mlease_b200._native import check
    check(rc)


def _ptr(a):
    return None if a is None else a.ctypes.data


def _part(D, n, nnz, seed):
    r = np.random.default_rng(seed)
    beta = r.normal(size=D) / np.sqrt(nnz)
    ci = np.stack([np.sort(r.choice(D, nnz, replace=False)) for _ in range(n)]).astype(np.int32)
    v = r.normal(size=(n, nnz)).astype(np.float32)
    y = (r.random(n) < 1 / (1 + np.exp(-((v * beta[ci]).sum(1) - 0.5)))).astype(np.int32)
    return np.arange(n + 1, dtype=np.int64) * nnz, ci.reshape(-1), v.reshape(-1), y


def _factor(hooks, s, H, Dt, full):
    ldh = fr.ldh_of(Dt)
    L = np.empty((Dt, Dt)) if full else None
    Y = np.empty((ldh, ldh)) if full else None
    bits = np.empty((ldh, ldh), np.uint16)
    _check(hooks.mlease_internal_factor(s._h, 0, _ptr(np.ascontiguousarray(H)), _ptr(L), _ptr(Y), _ptr(bits)))
    return L, Y, bits


def _ysym(hooks, s, b):
    ldh = s._ldh
    bits = np.empty((ldh, ldh), np.uint16)
    own, th = C.c_int32(-7), C.c_int32(-7)
    _check(hooks.mlease_internal_ysym(s._h, b, _ptr(bits), C.byref(own), C.byref(th)))
    return bits, own.value, th.value


def _direction(hooks, s, active, q):
    nprob, Dt = q.shape
    t = np.full((nprob, Dt), -1.0, np.float32)
    d = np.empty((nprob, Dt))
    _check(hooks.mlease_internal_factored_direction(s._h, _ptr(np.asarray(active, np.int32)), _ptr(q), _ptr(t), _ptr(d)))
    return t, d


@pytest.mark.parametrize("D", [2048, 2079, 2302, 10000])
def test_exact_factor_is_bitwise(mb, hooks, D):
    """H = (I+E)(I+E)^T with E^2 = 0: Lc = I+E, Yinv = I-E (strict upper triangle 0: the TF32 tiles read it), Ysym = bf16(I-E)
    mirrored, identity on the padding -- bit for bit, at every merge level and tile edge the pairs reach."""
    Dt = D + 1
    ldh = fr.ldh_of(Dt)
    pairs = fr.exact_pairs(Dt)
    E, H = fr.exact_system(Dt, pairs)
    full = D < 10000
    with mb.AdmmSession(1, D, [1.0]) as s:
        s.add_partition_csr(0, *_part(D, 300, 8, D))
        L, Y, bits = _factor(hooks, s, H, Dt, full)
    del H
    if full:
        Ed = E.toarray()
        assert np.array_equal(np.tril(L), np.eye(Dt) + Ed)
        Yx = np.eye(ldh)
        Yx[:Dt, :Dt] -= Ed
        bad = np.argwhere(Y != Yx)
        assert bad.size == 0, (len(bad), bad[:5])
    ref = fr.exact_ysym_bits(ldh, pairs)
    # the merges store -(T Y22) as sgn * acc: an exact zero there is -0.0 (bf16 0x8000), numerically the same operand
    bits = np.where(bits == 0x8000, np.uint16(0), bits)
    bad = np.argwhere(bits != ref)
    assert bad.size == 0, (len(bad), bad[:5])


# Measured on an H100 80GB (power limit not recorded): spread ratios 1.000054 (D = 2048) and 1.000162 (D = 2302).
SPREAD_FACTOR = 1.01


@pytest.mark.parametrize("D", [2048, 2302])
def test_generic_factor_against_fp64(mb, hooks, D):
    """A Hessian of CSR data at a point where the IRLS weights vary: Lc is the fp64 Cholesky factor; Ysym is bitwise
    bf16(float(Yinv)) mirrored; every block each TF32 merge writes is within the entrywise bound of factored_reference.merge_excess
    of the fp64 merge of the GPU's own operands; and the preconditioned spread is within SPREAD_FACTOR of that of the rounded fp64
    inverse of Lc."""
    Dt = D + 1
    ldh = fr.ldh_of(Dt)
    rng = np.random.default_rng(D)
    wv = rng.normal(0, 1.0, Dt)
    pm = np.zeros(Dt)
    with mb.AdmmSession(1, D, [1.0]) as s:
        s.add_partition_csr(0, *_part(D, 6000, 20, D + 1))
        _, _, H = s.objective(0, wv, pm, np.full(Dt, 1.0), want_hessian=True, tensor=True)
        L, Y, bits = _factor(hooks, s, H, Dt, True)
    Lref = np.linalg.cholesky(H)
    assert np.abs(np.tril(L) - Lref).max() <= 1e-10 * np.abs(Lref).max()
    assert np.array_equal(bits, fr.ysym_bits(np.tril(Y), ldh))   # Yinv of the padded system, -0.0 included
    assert not np.triu(Y, 1).any()
    Lp = np.eye(ldh)
    Lp[:Dt, :Dt] = np.tril(L)
    x_merge = fr.merge_excess(Lp, Y)
    assert x_merge <= 1.0, x_merge
    Yref = np.linalg.inv(np.tril(L))
    e_merge = np.abs(Y[:Dt, :Dt] - Yref).max() / np.abs(Yref).max()
    Yb = np.tril(fr.bits_to_float(bits)[:Dt, :Dt])
    Yb64 = fr.bits_to_float((fr.bf16_round(Yref.astype(np.float32)).view(np.uint32) >> 16).astype(np.uint16))
    s_gpu, s_ref = fr.spread(Yb, H), fr.spread(Yb64, H)
    print("D=%d merges at %.3f of their bound, |Y - inv(Lc)| %.3e of max|Y|, spread %.6f vs %.6f (ratio %.6f), cond(H) %.3e"
          % (D, x_merge, e_merge, s_gpu, s_ref, s_gpu / s_ref, np.linalg.cond(H)))
    assert s_gpu <= SPREAD_FACTOR * s_ref


def _admm(mb, D, lambdas, rhos, n, nnz, seed, P=1):
    s = mb.AdmmSession(P, D, lambdas, rhos=rhos, epsilon=0.0)
    for p in range(P):
        s.add_partition_csr(p, *_part(D, n, nnz, seed + p))
    s._ldh = fr.ldh_of(D + 1)
    return s


def _masks(L):
    m = [list(range(L))]
    if L >= 4:
        m.append([1, 3])   # leader inactive: member 1 carries member 3's vector
    m.append([L - 1])
    return m


def _check_directions(hooks, s, L, D, distinct, seed):
    Dt = D + 1
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(L, Dt)).astype(np.float32)
    emu = {}
    for b in range(L):
        bits, own, _ = _ysym(hooks, s, b)
        if distinct:
            assert own == b
        else:
            assert own in (0, b)
        if own not in emu:
            emu[own] = fr.halves(bits, Dt)
        emu[b] = emu[own]
    if not distinct and L > 1:   # the shared path is exercised: some follower streams the leader's Y
        assert any(_ysym(hooks, s, b)[1] == 0 for b in range(1, L))
    for mask in _masks(L):
        act = np.zeros(L, np.int32)
        act[mask] = 1
        t, d = _direction(hooks, s, act, q)
        t2, d2 = _direction(hooks, s, act, q)
        assert np.array_equal(t, t2, equal_nan=True) and np.array_equal(d, d2, equal_nan=True)   # bitwise repeatable
        for b in range(L):
            if not act[b]:
                assert np.isnan(d[b]).all(), (mask, b)
                continue
            lo, up = emu[b]
            t_ex, b0 = fr.phase0(lo, q[b])
            assert fr.excess(t[b], t_ex, b0) <= 1.0, (mask, b, fr.excess(t[b], t_ex, b0))
            d_ex, b1 = fr.phase1(up, t[b])
            assert fr.excess(d[b], d_ex, b1) <= 1.0, (mask, b, fr.excess(d[b], d_ex, b1))
            if len(mask) > 1:   # the same vector computed alone: bitwise the same
                one = np.zeros(L, np.int32)
                one[b] = 1
                t1, d1 = _direction(hooks, s, one, q)
                assert np.array_equal(t1[b], t[b]) and np.array_equal(d1[b], d[b]), (mask, b)


@pytest.mark.parametrize("distinct", [False, True])
@pytest.mark.parametrize("L", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("D", [2048, 2079, 2302])
def test_direction_against_fp64_emulation(mb, hooks, D, L, distinct):
    """Both GEMV phases on the bytes each problem reads, for all / leader-inactive / single-member active sets, with equal rho
    (followers read the leader's Y, up to 4 vectors per pass; L = 5 falls back to single-vector passes) and distinct rho."""
    if distinct and L == 1:
        pytest.skip("one lambda: nothing to distinguish")
    # rho = 10: the cold x-update converges on the shared factor (no "stuck" rebuild), so with equal rho the followers still
    # stream the leader's Y afterwards
    rhos = [10.0 + 5.0 * l for l in range(L)] if distinct else [10.0] * L
    with _admm(mb, D, [0.5 * (l + 1) for l in range(L)], rhos, 8000, 20, D + L) as s:
        s.begin()
        s.iterate()
        _check_directions(hooks, s, L, D, distinct, D * L)


@pytest.mark.parametrize("distinct", [False, True])
def test_direction_at_benchmark_width(mb, hooks, distinct):
    D, L = 10000, 3
    # 40000 rows: this shape faulted on a misaligned float4 load of qf before every problem's vector block was padded to 32 bytes
    with _admm(mb, D, [0.1, 1.0, 10.0], [10.0, 20.0, 5.0] if distinct else [10.0] * 3, 40000, 20, 77) as s:
        s.begin()
        s.iterate()
        _check_directions(hooks, s, L, D, distinct, 5)


def test_follower_keeps_the_cold_start_factor(mb, hooks):
    """Equal rho: after the shared cold-start factorisation every follower streams its leader's Y.  When the leader later
    refactorises on its own (here through refresh_next, which a slow x-update sets; the "stuck" rule acts per problem too), a
    follower that did not refactorise must go on reading the factor its secant pairs and h0_scale were built around -- the bytes
    it read after iteration 1 -- not the leader's new Y, another lambda's Hessian at another point.  And a follower that reads
    another problem's factor must have been factorised as often as that problem."""
    P, D, L = 2, 2300, 2   # the shape of test_admm_wide_systems_keep_the_cold_start_factor
    with _admm(mb, D, [1.0, 10.0], None, 8000, 20, 2000, P=P) as s:
        s.begin()
        s.iterate()
        nprob = P * L
        rec = [_ysym(hooks, s, b) for b in range(nprob)]
        for b in range(nprob):
            assert rec[b][1] == b - b % L and rec[b][2] == rec[b - b % L][2], (b, rec[b][1:])   # the shared cold-start factor
        _check(hooks.mlease_internal_request_refresh(s._h, 0))   # the leader of partition 0 refactorises alone
        solo = 0
        for it in range(3):
            s.iterate()
            cur = [_ysym(hooks, s, b) for b in range(nprob)]
            for b in range(nprob):
                bits, own, th = cur[b]
                if own != b:
                    assert cur[own][2] == th, (it, b, own, th, cur[own][2])
                lead = b - b % L
                if b == lead:
                    continue
                solo += cur[lead][2] > th
                if th == rec[b][2]:   # still on the shared cold-start factor
                    assert np.array_equal(bits, rec[b][0]), (it, b, own, th, cur[lead][2])
        print("follower-iterations behind a leader that refactorised alone:", solo, [c[1:] for c in cur])
        assert solo > 0, "no leader refactorised alone: the test did not reach its case"
        assert s.stats()["not_converged"] == 0


def test_hooks_refuse_before_launching(mb, hooks):
    """Every refusal returns before a launch: no Ysym (ldh <= 2048), matrix-free, no ADMM batch, b out of range, partition not
    resident."""
    one = np.ones(1, np.int32)
    q = np.zeros((1, 2301), np.float32)
    with mb.AdmmSession(2, 2300, [1.0]) as s:
        s.add_partition_csr(0, *_part(2300, 300, 8, 1))
        assert hooks.mlease_internal_ysym(s._h, 0, None, None, None) == ERR_STATE                  # no ADMM batch
        assert hooks.mlease_internal_factored_direction(s._h, _ptr(one), _ptr(q), None, None) == ERR_STATE
        assert hooks.mlease_internal_request_refresh(s._h, 0) == ERR_STATE
        H = np.eye(2301)
        assert hooks.mlease_internal_factor(s._h, 1, _ptr(H), None, None, None) == ERR_INVALID    # partition not resident
    with mb.AdmmSession(1, 2300, [1.0, 2.0]) as s:
        s.add_partition_csr(0, *_part(2300, 300, 8, 2))
        s.begin()
        assert hooks.mlease_internal_factored_direction(s._h, _ptr(one), _ptr(q), None, None) == ERR_STATE   # no iteration yet
        assert hooks.mlease_internal_ysym(s._h, 2, None, None, None) == ERR_INVALID               # b out of range
        assert hooks.mlease_internal_ysym(s._h, -1, None, None, None) == ERR_INVALID
        assert hooks.mlease_internal_request_refresh(s._h, 2) == ERR_INVALID
    with mb.AdmmSession(1, 300, [1.0]) as s:   # ldh = 320: no Ysym
        s.add_partition_csr(0, *_part(300, 500, 8, 3))
        H = np.eye(301)
        assert hooks.mlease_internal_factor(s._h, 0, _ptr(H), None, None, None) == ERR_INVALID
        s.run(1)
        assert hooks.mlease_internal_factored_direction(s._h, _ptr(one), _ptr(np.zeros((1, 301), np.float32)), None, None) == ERR_INVALID
        assert hooks.mlease_internal_ysym(s._h, 0, None, None, None) == ERR_INVALID
    with mb.AdmmSession(1, 2300, [1.0], hessian_policy=2) as s:   # matrix-free
        s.add_partition_csr(0, *_part(2300, 500, 8, 4))
        H = np.eye(2301)
        assert hooks.mlease_internal_factor(s._h, 0, _ptr(H), None, None, None) == ERR_INVALID
        s.run(1)
        assert hooks.mlease_internal_factored_direction(s._h, _ptr(one), _ptr(q), None, None) == ERR_INVALID
        assert hooks.mlease_internal_ysym(s._h, 0, None, None, None) == ERR_INVALID
