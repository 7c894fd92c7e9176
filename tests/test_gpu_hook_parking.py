"""GPU tests (-m gpu) of what the test hooks leave in the ADMM batch (mlease_internal.h): every hook that runs kernels on it parks
every problem's control block in the one documented state, and the library refuses to iterate the batch until begin() runs
again; after that begin() the session computes what a fresh one computes."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ERR_STATE = 4
# Ctrl of csrc/common.cuh, field by field with C alignment (checked against sizeof(Ctrl) below)
_I, _D, _L = np.int32, np.float64, np.int64
CTRL = np.dtype([("done", _I), ("have_dir", _I), ("need_solve", _I), ("need_hess", _I), ("emit", _I), ("hess_valid", _I), ("fail", _I),
                 ("newton_steps", _I), ("evals", _I), ("rejects", _I), ("hess_builds", _I), ("stall", _I), ("bfgs_count", _I),
                 ("h0_scale", _D), ("k1_chunks", _I), ("refresh_next", _I), ("skip_eval", _I), ("warm_used", _I), ("build_step", _I),
                 ("worst_ratio", _D), ("alpha", _D), ("phi0", _D), ("f_acc", _D), ("f_t", _D), ("gnorm", _D), ("gnorm_prev", _D),
                 ("dirnorm", _D), ("dirnorm_prev", _D), ("xtol", _D), ("max_newton", _I), ("hess_policy", _I), ("rebuild_is_expensive", _I),
                 ("tot_evals", _L), ("tot_newton", _L), ("tot_rejects", _L), ("tot_hess", _L), ("ysym_use", np.uint64), ("cg_active", _I),
                 ("cg_iter", _I), ("cg_rz", _D), ("cg_g2", _D), ("hv_vinf", np.float32)], align=True)
PARKED = dict(done=1, hess_valid=0, need_solve=0, need_hess=0, have_dir=0, bfgs_count=0, skip_eval=0, refresh_next=0, cg_active=0,
              k1_chunks=0, fail=0, h0_scale=1.0)


@pytest.fixture(scope="module")
def mb():
    import mlease_b200
    return mlease_b200


def _session(mb, D, L, P=2, n=2000, nnz=8, policy=0, seed=0):
    r = np.random.default_rng(seed + D)
    s = mb.AdmmSession(P, D, [1.0 + l for l in range(L)], hessian_policy=policy, epsilon=0.0)
    for p in range(P):
        ci = np.stack([np.sort(r.choice(D, nnz, replace=False)) for _ in range(n)]).astype(np.int32)
        v = r.normal(size=n * nnz).astype(np.float32)
        y = (r.random(n) < 0.5).astype(np.int32)
        s.add_partition_csr(p, np.arange(n + 1, dtype=np.int64) * nnz, ci.reshape(-1), v, y)
    return s


def _ctrl(s):
    """Every problem's control block, through a read of the consensus hook (stages = 0: it runs nothing and parks nothing)."""
    from mlease_b200 import _hooks
    S = _hooks.consensus(s)
    assert S["info"]["ctrl_bytes"] == CTRL.itemsize
    c = S["ctrl_raw"][0].copy().view(CTRL).reshape(-1)
    for i, k in enumerate(_hooks.CONSENSUS_CTRL):
        c[k] = S["ctrl"][:, i]
    return c


def test_iterate_after_a_consuming_hook_needs_begin(mb):
    """After batch_grad, iterate() is refused before any launch; after begin() three iterations give a fresh session's z bits."""
    from mlease_b200 import _hooks
    D, L = 36, 2
    with _session(mb, D, L) as s:
        s.begin()
        s.iterate()
        _hooks.batch_grad(s, np.full((2 * L, D + 1), 0.1))
        launches = s.stats()["kernel_launches"]
        with pytest.raises(mb.MleaseError, match="call mlease_admm_begin again") as e:
            s.iterate()
        assert e.value.code == ERR_STATE
        assert s.stats()["kernel_launches"] == launches
        s.begin()
        for _ in range(3):
            s.iterate()
        z = [s.z(l) for l in range(L)]
    with _session(mb, D, L) as fresh:
        fresh.begin()
        for _ in range(3):
            fresh.iterate()
        for l in range(L):
            assert fresh.z(l).tobytes() == z[l].tobytes(), l


def _run_batch_hv(s, nprob, Dt):
    from mlease_b200 import _hooks
    from mlease_b200._native import check
    w, v, out = np.full((nprob, Dt), 0.1), np.ones((nprob, Dt)), np.zeros((nprob, Dt))
    check(_hooks.bound().mlease_internal_batch_hv(s._h, 1, w.ctypes.data, v.ctypes.data, out.ctypes.data))


def _run_batch_grad(s, nprob, Dt):
    from mlease_b200 import _hooks
    _hooks.batch_grad(s, np.full((nprob, Dt), 0.1), active=np.arange(nprob) % 2)


def _run_batch_factor(s, nprob, Dt):
    from mlease_b200 import _hooks
    _hooks.batch_factor(s, np.ones(nprob, np.int32), H=np.stack([np.eye(Dt) * 2.0] * nprob))


def _run_direction(s, nprob, Dt):
    from mlease_b200 import _hooks
    M = _hooks.BFGS_M
    _hooks.direction(s, np.ones(nprob, np.int32), np.ones((nprob, Dt)), np.zeros((nprob, M, Dt)), np.zeros((nprob, M, Dt)),
                     np.ones((nprob, M)), np.zeros(nprob, np.int32), np.ones(nprob), np.zeros((nprob, Dt)))


def _run_newton_stage(s, nprob, Dt):
    from mlease_b200 import _hooks
    info = _hooks.newton_stage(s)["info"]
    ldx, M = info["ldx"], _hooks.BFGS_M
    _hooks.newton_stage(s, ["begin"], np.zeros(nprob, _hooks.STAGE_CTRL), np.zeros((nprob, 12, ldx)),
                        np.zeros((nprob, 2 * M * ldx + 2 * M)), np.zeros((nprob, 3, ldx), np.float32), begin_args=[1e-8, 10, 0, 0, 0])


def _run_factored_direction(s, nprob, Dt):
    from mlease_b200 import _hooks
    from mlease_b200._native import check
    q = np.ones((nprob, Dt), np.float32)
    act = (np.arange(nprob) % 2).astype(np.int32)
    check(_hooks.bound().mlease_internal_factored_direction(s._h, act.ctypes.data, q.ctypes.data, None, None))


# hook, (D, lambdas, hessian_policy) of a session it accepts
CASES = [(_run_batch_hv, (200, 2, 2)), (_run_batch_grad, (200, 2, 0)), (_run_batch_factor, (200, 2, 0)),
         (_run_direction, (200, 2, 0)), (_run_newton_stage, (200, 2, 0)), (_run_factored_direction, (2300, 2, 0))]


@pytest.mark.parametrize("hook,shape", CASES, ids=[c[0].__name__[5:] for c in CASES])
def test_consuming_hooks_park_one_state(mb, hook, shape):
    """After begin() and one iteration (control blocks holding a factor, secant pairs and h0_scale), each consuming hook leaves
    the parked fields at the documented state and every other field of every problem as it was before the hook."""
    D, L, policy = shape
    with _session(mb, D, L, policy=policy) as s:
        s.begin()
        s.iterate()
        nprob = 2 * L
        pre = _ctrl(s)
        hook(s, nprob, D + 1)
        post = _ctrl(s)
        for k in CTRL.names:
            want = np.full(nprob, PARKED[k], CTRL[k]) if k in PARKED else pre[k]
            assert np.asarray(post[k]).tobytes() == np.asarray(want).tobytes(), (hook.__name__, k, post[k], want)
