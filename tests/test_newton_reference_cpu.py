"""The fp64 replica of the Newton state machine (newton_reference.py) driven, without a GPU, by an exact numpy loss / gradient /
Hessian of a small logistic problem: it must behave as the solver it restates is meant to."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import chol_reference as cr  # noqa: E402
import newton_reference as nr  # noqa: E402


class Logistic:
    def __init__(self, n=300, D=8, seed=0, rho=1.0):
        r = np.random.default_rng(seed)
        self.X = r.normal(size=(n, D)).astype(np.float32).astype(np.float64)
        self.X[:, -1] = 1.0
        self.y = np.where(r.random(n) < 1 / (1 + np.exp(-self.X @ r.normal(size=D))), 1.0, -1.0)
        self.q = np.full(D, rho)
        self.m = r.normal(size=D) * 0.1
        self.D = D

    def data(self, b):
        z = self.y * (self.X @ b)
        f = np.logaddexp(0.0, -z).sum()
        p = 1 / (1 + np.exp(z))
        return f, -(self.X.T @ (self.y * p)), (self.X * (p * (1 - p))[:, None]).T @ self.X

    def minimiser(self):
        b = self.m.copy()
        for _ in range(60):
            _, g, H = self.data(b)
            b = b - np.linalg.solve(H + np.diag(self.q), g + self.q * (b - self.m))
        return b


def run(pb, policy, expensive=0, Hinv=None, valid=0, start=None, xtol=1e-9, max_newton=50, slots=200, spec=lambda s: 0):
    """One x-update through the replica: K1 = pb.data at float(beta_t), a rebuild = the exact inverse at the accepted point."""
    st = nr.new_state(pb.D, matrix_free=(policy == 2))
    st.update(q=pb.q.copy(), m=pb.m.copy(), beta=np.zeros(pb.D) if start is None else start.copy(), hess_valid=valid)
    st = nr.begin(st, xtol, max_newton, policy, 0, expensive)
    trace, cg_log = [], []
    for slot in range(slots):
        f, g, H = pb.data(st["beta_tf"].astype(np.float64))
        st["g_t"], st["k1_chunks"] = g, 1
        st = nr.decide(st, [f], spec(slot))
        if st["need_hess"] and not st["done"]:
            Hinv = np.linalg.inv(H + np.diag(pb.q))
            st = nr.rebuilt(st)
        if st["need_solve"] and not st["done"]:
            if policy == 2:
                st = nr.cg_begin(st)
                st["cg_diag"] = np.diag(H).copy()
                st = nr.cg_init(st)
                rrs = []
                while st["cg_active"]:
                    st["cg_Hp"] = H @ st["hv_vf"].astype(np.float64)
                    st = nr.cg_step(st)
                    rrs.append(st["cg_margin"])
                cg_log.append((rrs, st["cg_iter"]))
                st = nr.solve(st, st["dir"])
            else:
                st = nr.solve(st, Hinv @ st["g_t"])
        trace.append(st)
        if st["done"]:
            break
    return st, trace, cg_log


@pytest.mark.parametrize("policy", [0, 1, 2])
def test_reaches_the_minimiser(policy):
    pb = Logistic()
    st, trace, _ = run(pb, policy)
    assert st["done"] and st["fail"] == 0
    ref = pb.minimiser()
    assert np.abs(st["beta"] - ref).max() <= 1e-6 * np.abs(ref).max()   # trial points are fp32: the last step is taken in double
    if policy == 1:
        assert st["hess_builds"] == st["newton_steps"] + 1
    if policy == 2:
        assert st["hess_builds"] == 0 and st["bfgs_count"] == 0


def test_stale_factor_needs_the_secant_pairs():
    pb = Logistic(rho=0.05)
    _, _, H0 = pb.data(np.zeros(pb.D))
    Hinv = np.linalg.inv(H0 * 3.0 + np.diag(pb.q))   # a factor from far away; expensive: never rebuilt mid-update
    st, trace, _ = run(pb, 0, expensive=1, Hinv=Hinv, valid=1, xtol=1e-6)   # (above the floor of gradients taken at fp32 points)
    assert st["done"] and st["fail"] == 0 and st["hess_builds"] == 0 and st["bfgs_count"] > 0
    # the plain chord iteration on the same factor from the same start
    b, chord = np.zeros(pb.D), 0
    while chord < 500:
        _, g, _ = pb.data(b)
        d = Hinv @ (g + pb.q * (b - pb.m))
        if np.abs(d).max() <= 1e-6 * max(np.abs(b).max(), 1e-2):
            break
        b, chord = b - d, chord + 1
    assert st["newton_steps"] <= 14 and chord > 2 * st["newton_steps"]


def test_too_long_direction_is_shrunk_within_the_clamps():
    pb = Logistic()
    _, _, H0 = pb.data(np.zeros(pb.D))
    Hinv = 12.0 * np.linalg.inv(H0 + np.diag(pb.q))
    st, trace, _ = run(pb, 0, expensive=1, Hinv=Hinv, valid=1)
    assert st["done"] and st["fail"] == 0 and st["tot_rejects"] > 0
    seen = 0
    for a, b in zip(trace, trace[1:]):
        if b["action"] == 0:
            assert nr.SHRINK_LO * a["alpha"] <= b["alpha"] <= nr.SHRINK_HI * a["alpha"]
            assert b["need_solve"] == 0 and np.array_equal(b["beta"], a["beta"])
            seen += 1
    assert seen == st["tot_rejects"]


def test_stored_pairs_satisfy_the_secant_equation():
    pb = Logistic(rho=0.05)
    _, _, H0 = pb.data(np.zeros(pb.D))
    Hinv = np.linalg.inv(H0 * 3.0 + np.diag(pb.q))
    _, trace, _ = run(pb, 0, expensive=1, Hinv=Hinv, valid=1, xtol=1e-6)
    checked = 0
    for st in trace:
        if st["stored_slot"] >= 0:
            sl = st["stored_slot"]
            assert sl == (st["bfgs_count"] - 1) % nr.BFGS_M
            s, y = st["bfgs_S"][sl], st["bfgs_Y"][sl]
            assert st["bfgs_rho"][sl] == 1.0 / float(np.sum(s * y))
            # the quasi-Newton matrix maps the newest y to its s: two_loop(y) = -s
            d, _ = cr.two_loop(Hinv, y, st["bfgs_S"], st["bfgs_Y"], st["bfgs_rho"], st["bfgs_count"], 1.0)
            assert np.abs(d + s).max() <= 1e-9 * np.abs(s).max()
            checked += 1
    assert checked >= 3


def test_cg_stops_at_the_first_step_that_meets_the_forcing_rule():
    pb = Logistic(rho=0.01)
    st, _, cg_log = run(pb, 2)
    assert st["done"] and st["fail"] == 0 and cg_log
    for rrs, iters in cg_log:
        assert iters == len(rrs)
        for rr, thr in rrs[:-1]:
            assert rr > thr
        rr, thr = rrs[-1]
        assert rr <= thr or iters == nr.CG_MAX_STEPS


def test_speculative_slot_defers_the_rebuild():
    pb = Logistic()
    _, plain, _ = run(pb, 0)
    due = next(i for i, st in enumerate(plain) if st["emit"] and not st["done"])   # the slot after this one rebuilds
    assert plain[due + 1]["hess_builds"] == plain[due]["hess_builds"] + 1
    st, trace, _ = run(pb, 0, spec=lambda s: 1 if s == due + 1 else 0)
    assert st["done"] and st["fail"] == 0
    # enqueued speculatively, that slot takes a chord step and keeps emit; the next regular slot rebuilds
    assert trace[due + 1]["hess_builds"] == trace[due]["hess_builds"] and trace[due + 1]["emit"] == 1
    assert trace[due + 1]["newton_steps"] == trace[due]["newton_steps"] + 1
    assert trace[due + 2]["hess_builds"] == trace[due]["hess_builds"] + 1


def test_reduce_partials_order():
    r = np.random.default_rng(3)
    parts = r.normal(size=(19, 5)) * 10.0 ** r.integers(-8, 8, (19, 5))
    for nct in (0, 1, 7, 8, 9, 19):
        got = nr.reduce_partials(parts, nct)
        for k in range(5):
            grp = [0.0] * 8
            for t in range(nct):
                grp[t % 8] += parts[t, k]
            a = 0.0
            for g in grp:
                a += g
            assert got[k] == a
    p32 = parts.astype(np.float32)
    assert np.array_equal(nr.reduce_partials(p32, 19, fp32=True), nr.reduce_partials(p32.astype(np.float64), 19))


def test_branch_names_are_known():
    pb = Logistic()
    seen = set()
    for policy in (0, 1, 2):
        for st in run(pb, policy)[1]:
            seen |= st["branch"]
    assert seen and seen <= set(nr.BRANCHES), seen - set(nr.BRANCHES)
