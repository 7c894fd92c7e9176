"""GPU tests (-m gpu) of the device-side Newton state machine (csrc/newton.cu) against its fp64 replica (newton_reference.py),
through the test hook mlease_internal_newton_stage (not part of the C ABI), which injects an x-update state into every problem of
an ADMM batch and runs the solver's own launchers once:

- the branch table on dyadic data (small integers times powers of two: every block reduction is exact whatever its order), every
  output compared with the replica bit for bit (up to the sign of a zero and the payload of a NaN) -- all of Ctrl, the trial point, the stored secant pair, g_acc, the first-loop q (qf on
  wide batches), the direction and the CG vectors; each test collects the branches its cases took in the replica and asserts the
  list it is responsible for;
- batches whose neighbouring problems take different branches in one launch, with done problems whose bytes must not change;
- generic (random) states within fp64 bounds, discrete outcomes equal wherever the deciding quantity is not within 1e-12 of its
  threshold, and run-to-run bit equality;
- the hook's refusals."""
import itertools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import newton_reference as nr  # noqa: E402

pytestmark = pytest.mark.gpu
M = nr.BFGS_M
SEEN, RAN = set(), set()   # branches the replica took over the whole file, and the test groups that contributed


@pytest.fixture(scope="module")
def mb():
    import mlease_b200
    return mlease_b200


def _sentinel(shape, dtype):
    return np.frombuffer(b"\xff" * (int(np.prod(shape)) * np.dtype(dtype).itemsize), dtype).reshape(shape).copy()


def _same(a, b):
    """Bit for bit, up to the sign of a zero and the payload of a NaN (a kernel may store -0 or its own NaN where numpy has +0 / another)."""
    a = np.ascontiguousarray(a)
    b = np.ascontiguousarray(b, a.dtype)
    u = np.uint64 if a.dtype.itemsize == 8 else np.uint32
    return bool(((a.view(u) == b.view(u)) | ((a == 0) & (b == 0)) | (np.isnan(a) & np.isnan(b))).all())


def _bytes_equal(a, b):
    return np.ascontiguousarray(a).tobytes() == np.ascontiguousarray(b).tobytes()


class _Sess:
    """A begun ADMM session of P partitions x L lambdas: kind "dense", "csr" (Gram path) or "mf" (matrix-free, policy 2)."""

    def __init__(self, mb, kind, D, P=1, L=1, policy=0):
        from mlease_b200 import _hooks
        import k1_reference as k1
        self.hook = _hooks.newton_stage
        r = np.random.default_rng(D + 7 * P + L)
        self.s = mb.AdmmSession(P, D, [1.0 + l for l in range(L)], hessian_policy=2 if kind == "mf" else policy, epsilon=0.0)
        self.s.__enter__()
        self.parts = []
        for p in range(P):
            if kind == "dense":
                X = r.normal(size=(64, D)).astype(np.float32)
                y = (r.random(64) < 0.5).astype(np.int32)
                self.s.add_partition_dense(p, X, y)
                self.parts.append(k1.Part.from_dense(X, y, np.ones(64), np.zeros(64)))
            else:
                n, nnz = 6000, min(3, D)
                ci = np.stack([np.sort(r.choice(D, nnz, replace=False)) for _ in range(n)]).astype(np.int32)
                rp, v, y = np.arange(n + 1, dtype=np.int64) * nnz, r.normal(size=n * nnz).astype(np.float32), (r.random(n) < 0.5).astype(np.int32)
                self.s.add_partition_csr(p, rp, ci.reshape(-1), v, y)
                self.parts.append(k1.Part.from_csr(rp, ci.reshape(-1), v, y, np.ones(n), np.zeros(n), D))
        self.s.begin()
        self.info = self.hook(self.s)["info"]
        self.nprob, self.Dt, self.ldx = self.info["nprob"], self.info["Dt"], self.info["ldx"]
        self.wide, self.mf = bool(self.info["ysym"]), bool(self.info["matrix_free"])
        assert self.nprob == P * L and self.Dt == D + 1

    def close(self):
        self.s.__exit__(None, None, None)

    def pack(self, states):
        """The hook's arrays for one state per problem (None: a done problem, every byte the sentinel)."""
        from mlease_b200._hooks import STAGE_CTRL
        n, Dt, ldx = self.nprob, self.Dt, self.ldx
        ctrl = np.zeros(n, STAGE_CTRL)
        vec = np.zeros((n, 12, ldx))
        ring = np.zeros((n, 2 * M * ldx + 2 * M))
        fvec = np.zeros((n, 3, ldx), np.float32)
        for b, st in enumerate(states):
            if st is None:
                vec[b], ring[b], fvec[b] = _sentinel(vec[b].shape, np.float64), _sentinel(ring[b].shape, np.float64), _sentinel(fvec[b].shape, np.float32)
                for k in nr.INT_FIELDS:
                    ctrl[b][k] = 7
                ctrl[b]["done"], ctrl[b]["k1_chunks"], ctrl[b]["bfgs_count"], ctrl[b]["hess_policy"] = 1, 0, 0, 2 if self.mf else 0
                ctrl[b]["cg_active"] = 0   # (as cg_begin leaves a done problem: the CG kernels look at nothing else)
                for k in nr.REAL_FIELDS:
                    ctrl[b][k] = -3.5
                continue
            for k in nr.INT_FIELDS:
                ctrl[b][k] = st[k]
            for k in nr.REAL_FIELDS:
                ctrl[b][k] = st[k]
            from mlease_b200._hooks import STAGE_VECS
            for i, k in enumerate(STAGE_VECS):
                if k in st:
                    vec[b, i, :len(st[k])] = st[k]   # (a state may carry whole ldx-long vectors: its padding then)
            rg = ring[b]
            S, Y = rg[:M * ldx].reshape(M, ldx), rg[M * ldx:2 * M * ldx].reshape(M, ldx)
            S[:, :st["bfgs_S"].shape[1]], Y[:, :st["bfgs_Y"].shape[1]] = st["bfgs_S"], st["bfgs_Y"]
            rg[2 * M * ldx:2 * M * ldx + M], rg[2 * M * ldx + M:] = st["bfgs_rho"], st["bfgs_alpha"]
            fvec[b, 0, :len(st["beta_tf"])] = st["beta_tf"]
            fvec[b, 1, :len(st["qf"])] = st.get("hv_vf", st["qf"])
            fvec[b, 2] = _sentinel(ldx, np.float32)   # tf: none of these stages writes it
        return ctrl, vec, ring, fvec

    def stage(self, states, stages, parts=None, spec=0, begin_args=None):
        """-> (inputs, outputs) of the hook; parts: per problem (gpart [nct, Dt], fpart [nct]) or None."""
        self.s.begin()
        ctrl, vec, ring, fvec = self.pack(states)
        gp = fp = None
        if parts is not None:
            cap = max([len(p[1]) for p in parts if p is not None] + [1])
            gp, fp = np.zeros((self.nprob, cap, self.ldx)), np.zeros((self.nprob, cap))
            for b, p in enumerate(parts):
                if p is not None and len(p[1]):
                    gp[b, :len(p[1]), :self.Dt], fp[b, :len(p[1])] = p[0], p[1]
        out = self.hook(self.s, stages, ctrl, vec, ring, fvec, gp, fp, spec=spec, begin_args=begin_args)
        return dict(ctrl=ctrl, vec=vec, ring=ring, fvec=fvec), out

    def compare(self, states, refs, inp, out, ints=nr.INT_FIELDS, reals=nr.REAL_FIELDS, tag=""):
        """Every output of every problem against the replica's state by bits; a done problem keeps its bytes."""
        from mlease_b200._hooks import STAGE_VECS
        Dt, ldx = self.Dt, self.ldx
        for b, (st, ref) in enumerate(zip(states, refs)):
            where = "%s problem %d %s" % (tag, b, sorted(ref["branch"]) if ref else "done")
            if st is None:
                for k in ("vec", "ring", "fvec"):
                    assert _bytes_equal(inp[k][b], out[k][b]), (where, k)
                for k in nr.INT_FIELDS + nr.REAL_FIELDS:
                    assert inp["ctrl"][b][k] == out["ctrl"][b][k], (where, k)
                for k in nr.TOTALS:
                    assert out["ctrl"][b][k] == 0, (where, k)   # (a fresh session: every cumulative counter starts at 0)
                continue
            c = out["ctrl"][b]
            for k in ints:
                assert int(c[k]) == int(ref[k]), (where, k, int(c[k]), int(ref[k]))
            for k in reals:
                assert _same(np.float64(c[k]), np.float64(ref[k])), (where, k, float(c[k]), float(ref[k]))
            for k in nr.TOTALS:
                assert int(c[k]) == ref[k], (where, k)
            for i, k in enumerate(STAGE_VECS[:12 if self.mf else 7]):
                if k not in ref:
                    continue
                v = out["vec"][b, i]
                assert _same(v[:Dt], ref[k][:Dt]), (where, k, np.flatnonzero(~((v[:Dt] == ref[k][:Dt]) | np.isnan(v[:Dt])))[:5])
                assert not v[Dt:].any(), (where, k, "padding")
            rg = out["ring"][b]
            if not self.mf:
                assert _same(rg[:M * ldx].reshape(M, ldx)[:, :Dt], ref["bfgs_S"]), (where, "bfgs_S")
                assert _same(rg[M * ldx:2 * M * ldx].reshape(M, ldx)[:, :Dt], ref["bfgs_Y"]), (where, "bfgs_Y")
                assert not rg[:2 * M * ldx].reshape(2 * M, ldx)[:, Dt:].any(), (where, "ring padding")
            assert _same(rg[2 * M * ldx:2 * M * ldx + M], ref["bfgs_rho"]), (where, "bfgs_rho")
            assert _same(rg[2 * M * ldx + M:], ref["bfgs_alpha"]), (where, "bfgs_alpha")
            f = out["fvec"][b]
            assert _same(f[0, :Dt], ref["beta_tf"]) and not f[0, Dt:].any(), (where, "beta_tf")
            assert _same(f[1, :Dt], ref.get("hv_vf", ref["qf"])) and not f[1, Dt:].any(), (where, "qf / hv_vf")
            assert _bytes_equal(f[2], inp["fvec"][b, 2]), (where, "tf")


# ---------------------------------------------------------------------------------------------------------------------------------
# dyadic states


def _dy(r, n, ints=3, exps=(-2, 3)):
    return r.integers(-ints, ints + 1, n) * 2.0 ** r.integers(exps[0], exps[1], n)


def _base(r, Dt, wide=False, mf=False, count=0):
    """A dyadic state with `count` pairs in the ring: pair slot j lives on the coordinates k % BFGS_M == j (the pairs never feed
    each other, so every value of both loops stays a short dyadic sum); slots not in use hold the sentinel."""
    st = nr.new_state(Dt, wide=wide, matrix_free=mf)
    for k in ("beta", "m", "g_t", "g_acc", "dir"):
        st[k] = _dy(r, Dt)
    st["beta"] = st["beta"].astype(np.float32).astype(np.float64)
    st["q"] = 2.0 ** r.integers(-2, 3, Dt)
    st["beta_t"] = st["beta"] + _dy(r, Dt, 2, (-1, 2))
    st["beta_tf"] = st["beta_t"].astype(np.float32)
    st["qf"] = _sentinel(Dt, np.float32)
    st.update(hess_valid=1, evals=3, newton_steps=2, max_newton=50, gnorm=8.0, gnorm_prev=16.0, dirnorm=1.0, k1_chunks=0,
              hess_policy=2 if mf else 0, bfgs_count=0 if mf else count)
    if not mf:
        st["bfgs_S"], st["bfgs_Y"] = _sentinel((M, Dt), np.float64), _sentinel((M, Dt), np.float64)
        st["bfgs_rho"], st["bfgs_alpha"] = _sentinel(M, np.float64), _sentinel(M, np.float64)
        for j in range(min(count, M)):
            sl = (count - 1 - j) % M
            cls = (np.arange(Dt) % M) == sl
            st["bfgs_S"][sl] = np.where(cls, _dy(r, Dt, 2, (-1, 2)), 0.0)
            st["bfgs_Y"][sl] = np.where(cls, _dy(r, Dt, 2, (-1, 2)), 0.0)
            st["bfgs_rho"][sl] = 2.0 ** r.integers(-3, 2)
            st["bfgs_alpha"][sl] = _dy(r, 1)[0]
    return st


def _parts(r, Dt, nct):
    """nct rows of dyadic partials (exact in fp32) and losses."""
    return _dy(r, (nct, Dt), 3, (-1, 2)), np.abs(_dy(r, nct, 3, (-1, 2)))


def _reduced(st, parts, fp32):
    """The state as the decide kernel finds it after the fixed-order reduction of its partials."""
    s = dict(st)
    if parts is not None and not st["skip_eval"] and not st["done"]:
        s["g_t"] = nr.reduce_partials(parts[0], len(parts[1]), fp32) if len(parts[1]) else np.zeros(len(st["g_t"]))
    return s


def _grad(st, parts):
    """The full gradient at beta_t: reduced data term plus prior term."""
    return _reduced(st, parts, False)["g_t"] + st["q"] * (st["beta_t"] - st["m"])


def _line_search_cases(r, Dt, wide, mf, nct_list):
    """(name, state, parts) of the accept / shrink / stop branches of the decide kernel."""
    cases = []
    it = itertools.cycle(nct_list)

    def mk(name, count=0, **kw):
        st = _base(r, Dt, wide, mf, count)
        nct = next(it)
        parts = _parts(r, Dt, nct)
        st["k1_chunks"] = nct
        st["have_dir"] = 1
        # phi > 0 for the line-search cases: flip dir if needed
        probe = nr.decide(_reduced(st, parts, False), parts[1])["scalars"]
        if probe["phi"] < 0:
            st["dir"] = -st["dir"]
        elif probe["phi"] == 0:
            st["dir"][0] += 4.0 * (1 if probe["ginf"] == 0 else np.sign(_grad(st, parts)[0]) or 1)
        phi = abs(nr.decide(_reduced(st, parts, False), parts[1])["scalars"]["phi"])
        st.update(kw)
        cases.append((name, st, parts, phi))
        return st, phi

    st = _base(r, Dt, wide, mf)
    parts = _parts(r, Dt, next(it))
    st.update(have_dir=0, k1_chunks=len(parts[1]), evals=0, newton_steps=0)
    cases.append(("accept:no_dir", st, parts, 0))
    st, phi = mk("at_half")
    st["phi0"] = -2.0 * phi
    st, phi = mk("just_above")
    st["phi0"] = -np.nextafter(2.0 * phi, 0.0)
    st, phi = mk("unclamped")
    st["phi0"], st["alpha"] = -phi, 0.5
    st, phi = mk("clamp_lo")
    st["phi0"] = -phi * 2.0 ** -10
    st, phi = mk("clamp_hi")
    st["phi0"], st["alpha"] = -1.75 * phi, 0.25
    st, phi = mk("give_up", rejects=nr.MAX_REJECTS)
    st["phi0"] = -phi
    st, phi = mk("not_yet_give_up", rejects=nr.MAX_REJECTS - 1)
    st["phi0"] = -phi
    st, phi = mk("nan")
    st["phi0"] = -phi
    st["dir"][Dt // 2] = np.nan
    st, phi = mk("first_exact", warm_used=1, evals=0)
    st["phi0"] = -phi * 2.0 ** -10
    st, phi = mk("warm_but_second", warm_used=1, evals=1)
    st["phi0"] = -phi * 2.0 ** -10
    # skip_eval: no evaluation is counted and g_t is taken as it is, whatever the partial rows hold
    st = _base(r, Dt, wide, mf)
    parts = _parts(r, Dt, next(it))
    st.update(have_dir=0, skip_eval=1, evals=0, newton_steps=0, k1_chunks=len(parts[1]))
    cases.append(("skip_eval", st, parts, 0))
    # zero gradient: the data term cancels the prior term exactly
    st = _base(r, Dt, wide, mf)
    st.update(have_dir=0, skip_eval=1, k1_chunks=0)
    st["g_t"] = -(st["q"] * (st["beta_t"] - st["m"]))
    cases.append(("zero_gradient", st, None, 0))
    st, phi = mk("max_newton", newton_steps=4, max_newton=5)
    st["phi0"] = -4.0 * phi
    st, phi = mk("below_max_newton", newton_steps=3, max_newton=5)
    st["phi0"] = -4.0 * phi
    return cases


def _pair_cases(r, Dt, wide, nct_list):
    """Accepted steps with a secant pair on the coordinates of its ring slot: stored / refused, the ring slots, h0_scale."""
    cases = []
    it = itertools.cycle(nct_list)

    def mk(name, count, s_scale=1.0, **kw):
        st = _base(r, Dt, wide, False, count)
        parts = _parts(r, Dt, next(it))
        st.update(have_dir=1, k1_chunks=len(parts[1]), phi0=-1.0)
        cls = (np.arange(Dt) % M) == (count % M)
        if not cls.any():
            cls[0] = True
        g = _grad(st, parts)     # the full gradient at beta_t
        step = np.where(cls, np.where(st["beta_t"] == st["beta"], 1.0, st["beta_t"] - st["beta"]), 0.0) * s_scale
        st["beta_t"] = (st["beta"] + step).astype(np.float32).astype(np.float64)
        st["beta_tf"] = st["beta_t"].astype(np.float32)
        g = _grad(st, parts)
        # y = sign(s) |y| on the slot's coordinates (s.y > 0), none elsewhere
        st["g_acc"] = np.where(cls, g - np.sign(step) * (1.0 + np.abs(_dy(r, Dt, 2, (-1, 2)))), g)
        st["dir"] = -np.sign(g) * np.abs(st["dir"])                   # phi <= 0: accepted
        st.update(kw)
        cases.append((name, st, parts, 0))
        return st, cls, g

    for count in (0, M - 1, M, 2 * M + 1):
        mk("stored_count_%d" % count, count)
    st, cls, g = mk("sy_negative", 1)
    st["g_acc"] = 2.0 * g - st["g_acc"]   # y -> -y
    st, cls, g = mk("sy_zero", 2)
    st["g_acc"] = g.copy()
    mk("refused_rebuild", 3, emit=1)
    mk("refused_rebuild_spec_keeps", 3, emit=1, _spec_only=1)
    if Dt >= 2 * M:
        # s.y just under / over SY_REL sqrt(s.s y.y): two coordinates of the slot with s = (1, 1), y = (2^20, -2^20 + e)
        for name, over in (("sy_small", 0), ("sy_over", 1)):
            st, cls, g = mk(name, 4)
            k0, k1 = np.flatnonzero(cls)[:2]
            st["beta_t"] = st["beta"].copy()
            st["beta_t"][[k0, k1]] += 1.0
            st["beta_tf"] = st["beta_t"].astype(np.float32)
            parts = cases[-1][2]
            g = _grad(st, parts)
            st["dir"] = -np.sign(g) * np.abs(st["dir"])
            thr = nr.SY_REL * np.sqrt(2.0 * 2.0 * 2.0 ** 40)
            e = np.ceil(thr * 2.0 ** 30) * 2.0 ** -30 + (2.0 ** -30 if over else -2.0 ** -30)
            st["g_acc"] = g.copy()
            st["g_acc"][k0] -= 2.0 ** 20
            st["g_acc"][k1] -= -2.0 ** 20 + e
    # h0_scale (expensive rebuilds): tau = -(alpha phi0) / s.y clamped, then the product
    for name, t, h0, exp in (("tau_lo", 0.125, 1.0, 1), ("tau_hi", 8.0, 1.0, 1), ("tau_free", 1.0, 4.0, 1), ("h0_clamp_lo", 0.5, 0.25, 1),
                             ("h0_clamp_hi", 2.0, 16.0, 1), ("cheap", 8.0, 4.0, 0)):
        st, cls, g = mk("h0_" + name, 1, rebuild_is_expensive=exp, h0_scale=h0)
        sy = nr.decide(_reduced(st, cases[-1][2], False), cases[-1][2][1])["scalars"]["sy"]
        st["phi0"] = -sy * t
    return cases


def _run_cases(t, cases, spec=0, seen=None, tag=""):
    """The cases over the batch, nprob at a time, a done problem at a rotating position in each launch."""
    fused = bool(t.info["fused"])
    per = max(1, t.nprob - 1) if t.nprob > 1 else 1
    for i0 in range(0, len(cases), per):
        chunk = list(cases[i0:i0 + per])
        states, parts, names = [c[1] for c in chunk], [c[2] for c in chunk], [c[0] for c in chunk]
        if t.nprob > 1:
            hole = (i0 // per) % t.nprob
            for lst, fill in ((states, None), (parts, None), (names, "done")):
                lst.insert(min(hole, len(lst)), fill)
        while len(states) < t.nprob:
            states.append(None); parts.append(None); names.append("done")
        refs = [None if st is None else nr.decide(_reduced(st, p, fused), p[1] if p else [], spec) for st, p in zip(states, parts)]
        inp, out = t.stage(states, ["decide"], parts=parts if any(p is not None for p in parts) else None, spec=spec)
        t.compare(states, refs, inp, out, tag="%s spec=%d %s" % (tag, spec, names))
        if seen is not None:
            for ref in refs:
                if ref is not None:
                    seen |= ref["branch"]


SHAPES = [("dense", 1, 2, 2), ("dense", 36, 2, 3), ("csr", 255, 2, 2), ("csr", 256, 1, 3), ("csr", 999, 2, 2), ("csr", 2078, 1, 3),
          ("csr", 2301, 2, 2)]


def _nct_list(t):
    rows = t.info["part_rows"]
    return sorted({n for n in (1, 7, 8, 9, rows) if n <= rows})


@pytest.mark.parametrize("kind,D,P,L", SHAPES)
def test_decide_branches_bit_for_bit(mb, kind, D, P, L):
    t = _Sess(mb, kind, D, P, L)
    try:
        Dt = t.Dt
        assert t.wide == (Dt > 2048)
        r = np.random.default_rng(100 + D)
        seen = set()
        cases = _line_search_cases(r, Dt, t.wide, False, _nct_list(t)) + _pair_cases(r, Dt, t.wide, _nct_list(t))
        for spec in (0, 1):
            _run_cases(t, [c for c in cases if spec or not c[1].get("_spec_only")], spec, seen, "%s D=%d" % (kind, D))
        want = {"accept:no_dir", "accept:curvature", "accept:first_exact", "reject:unclamped", "reject:clamp_lo", "reject:clamp_hi",
                "reject:nan", "reject:give_up", "eval:counted", "eval:skipped", "stop:zero_gradient", "stop:max_newton", "pair:stored",
                "pair:refused_sy_nonpositive", "pair:refused_rebuild", "h0:tau_lo", "h0:tau_hi", "h0:tau_free", "h0:clamp_lo",
                "h0:clamp_hi", "h0:cheap_unchanged", "need_hess", "emit:deferred", "spec:no_rebuild"}
        if Dt >= 2 * M:
            want.add("pair:refused_sy_small")
        assert want <= seen, sorted(want - seen)
        SEEN.update(seen)
        RAN.add(sys._getframe().f_code.co_name)
    finally:
        t.close()


def test_emit_table_bit_for_bit(mb):
    """policy x expensive x spec x emit x hess_valid x contraction x evals x steps on the factor, generated."""
    t = _Sess(mb, "csr", 36, 8, 4)
    try:
        r = np.random.default_rng(5)
        seen = set()
        for spec in (0, 1):
            cases = []
            for policy, exp, emit, valid, contr, evals, steps in itertools.product((0, 1, 2), (0, 1), (0, 1), (0, 1), (0.2, 0.3, 0.6), (1, 2),
                                                                                   (nr.STUCK_STEPS - 1, nr.STUCK_STEPS)):
                st = _base(r, t.Dt, False, False, count=0)   # (the new pair is dense here: alone in the ring, its loop stays exact)
                parts = _parts(r, t.Dt, 1 + len(cases) % t.info["part_rows"])
                st.update(have_dir=1, k1_chunks=len(parts[1]), hess_policy=policy, rebuild_is_expensive=exp, emit=emit, hess_valid=valid,
                          evals=evals - 1, build_step=3, newton_steps=3 + steps - 1)
                sc = nr.decide(_reduced(st, parts, False), parts[1])["scalars"]
                st["dir"] = st["dir"] if sc["phi"] <= 0 else -st["dir"]
                st["phi0"] = -1.0
                st["gnorm"] = sc["ginf"] / contr if sc["ginf"] > 0 else 1.0
                cases.append(("p%d e%d emit%d v%d c%.1f ev%d st%d" % (policy, exp, emit, valid, contr, evals, steps), st, parts, 0))
            _run_cases(t, cases, spec, seen, "emit table")
        want = {"emit:always", "emit:never", "emit:poor", "emit:stuck", "emit:invalid", "emit:deferred", "emit:none", "need_hess",
                "spec:no_rebuild", "pair:none_matrix_free", "pair:refused_rebuild", "pair:stored", "pair:refused_sy_nonpositive"}
        assert want - {"pair:refused_sy_nonpositive"} <= seen, sorted(want - seen)
        SEEN.update(seen)
        RAN.add(sys._getframe().f_code.co_name)
    finally:
        t.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# newton_solve_kernel (through newton_finish: the caller's r = H0^-1 q in dir) and newton_begin


def _solve_cases(r, Dt, wide, mf):
    cases = []

    def mk(name, count=0, **kw):
        st = _base(r, Dt, wide, mf, count)
        rr = np.abs(_dy(r, Dt, 2, (-1, 2))) + 0.25
        st["g_acc"] = np.where(st["g_acc"] == 0, 1.0, st["g_acc"])
        st["dir"] = np.sign(st["g_acc"]) * rr        # r . g > 0: a descent direction after the sign
        st.update(need_solve=1, have_dir=0, xtol=0.0, evals=2, newton_steps=1, stall=0, dirnorm=4.0, alpha=0.25, rejects=3, need_hess=1)
        st.update(kw)
        cases.append((name, st))
        return st

    mk("plain")
    for count in (1, M - 1, M, 2 * M + 1):
        if not mf:
            mk("pairs_%d" % count, count, h0_scale=1.0 if count == 1 else 2.0)
    mk("idle", need_solve=0)
    st = mk("fail_phi0")
    st["dir"] = -st["dir"]
    st = mk("fail_nan")
    st["dir"][Dt - 1] = np.nan
    mk("xtol_before_exact", xtol=2.0 ** 20, evals=0)
    mk("xtol_before_exact_late", xtol=2.0 ** 20, evals=0, newton_steps=3, dirnorm=2.0 ** -40)
    mk("xtol", xtol=2.0 ** 20, evals=1)
    st = mk("floor", xtol=2.0 ** 20, evals=1)
    st["beta"] = st["beta"] * 2.0 ** -12
    # the stall rule: |dir| <= STALL_TOL scale and no longer shrinking
    for name, kw in (("stall_counted", dict(stall=0)), ("stall_stop", dict(stall=1)), ("stall_too_early", dict(stall=1, newton_steps=1))):
        st = mk(name, newton_steps=kw.pop("newton_steps", 2), **kw)
        st["dir"] = st["dir"] * 2.0 ** -24
        st["beta"] = np.where(st["beta"] == 0, 1.0, st["beta"])
        st["dirnorm"] = 2.0 ** -24
    st = mk("stall_reset", stall=1, newton_steps=2)
    st["dir"] = st["dir"] * 2.0 ** -24
    st["dirnorm"] = 1.0
    for steps, exp, builds, policy in ((5, 0, 0, 0), (6, 0, 0, 0), (15, 1, 0, 0), (16, 1, 0, 0), (20, 0, 1, 0), (20, 0, 0, 1)):
        mk("refresh_%d_%d_%d_%d" % (steps, exp, builds, policy), xtol=2.0 ** 20, evals=1, newton_steps=steps, rebuild_is_expensive=exp,
           hess_builds=builds, hess_policy=2 if mf else policy)
    return cases


@pytest.mark.parametrize("kind,D,P,L", [("dense", 36, 2, 3), ("csr", 256, 1, 3), ("csr", 999, 2, 2), ("csr", 2301, 2, 2), ("mf", 300, 2, 2),
                                        ("mf", 2078, 1, 3)])
def test_solve_branches_bit_for_bit(mb, kind, D, P, L):
    t = _Sess(mb, kind, D, P, L)
    try:
        r = np.random.default_rng(200 + D)
        cases = _solve_cases(r, t.Dt, t.wide, t.mf)
        seen = set()
        per = t.nprob - 1
        for i0 in range(0, len(cases), per):
            chunk = cases[i0:i0 + per]
            states = [c[1] for c in chunk]
            states.insert((i0 // per) % t.nprob if len(states) == per else len(states), None)
            states += [None] * (t.nprob - len(states))
            refs = [None if st is None else nr.solve(st, st["dir"]) for st in states]
            inp, out = t.stage(states, ["finish"])
            t.compare(states, refs, inp, out, tag="solve %s" % [c[0] for c in chunk])
            for ref in refs:
                if ref is not None:
                    seen |= ref["branch"]
        want = {"solve:idle", "solve:fail_phi0", "solve:fail_nan", "solve:xtol", "solve:xtol_before_exact", "solve:stall_counted",
                "solve:stall_stop", "solve:stall_reset", "solve:floor"} | (set() if t.mf else {"solve:h0_scaled", "solve:refresh_next"})
        assert want <= seen, sorted(want - seen)
        SEEN.update(seen)
        RAN.add(sys._getframe().f_code.co_name)
    finally:
        t.close()


@pytest.mark.parametrize("kind,D", [("dense", 36), ("csr", 2301), ("mf", 300)])
def test_begin_bit_for_bit(mb, kind, D):
    t = _Sess(mb, kind, D, 2, 3)
    try:
        r = np.random.default_rng(300 + D)
        seen = set()
        policies = (2,) if t.mf else (0, 1, 2)
        for policy, invalidate, exp in itertools.product(policies, (0, 1), (0, 1)):
            states = []
            for b, (valid, refresh, skip, h0) in enumerate(((1, 0, 1, 3.0), (0, 0, 1, -1.0), (1, 1, 1, np.nan), (1, 0, 0, 0.0), (1, 0, 1, 0.5),
                                                                  (0, 1, 0, 2.0))):
                st = _base(r, t.Dt, t.wide, t.mf)
                st["beta"] = st["beta"] + 2.0 ** -30                     # off the float lattice
                full = np.zeros(t.ldx)
                full[:t.Dt] = st["beta"]
                full[t.Dt:] = 5.0                                        # [Dt, ldx) must be zeroed
                st["beta_padded"] = full
                st.update(hess_valid=valid, refresh_next=refresh, skip_eval=skip, h0_scale=h0, have_dir=1, need_solve=1, fail=2, stall=1,
                          rejects=2, hess_builds=1, warm_used=1, build_step=2, cg_active=1 if t.mf else 0, worst_ratio=0.5, f_acc=1.0)
                states.append(st)
            refs = [None if st is None else nr.begin(st, 2.0 ** -20, 17, policy, invalidate, exp) for st in states]
            self_states = []
            for st in states:
                if st is not None:
                    st = dict(st)
                    st["beta"] = st["beta_padded"]
                self_states.append(st)
            inp, out = t.stage(self_states, ["begin"], begin_args=[2.0 ** -20, 17, policy, invalidate, exp])
            t.compare(states, refs, inp, out, tag="begin p%d i%d e%d" % (policy, invalidate, exp))
            for ref in refs:
                if ref is not None:
                    seen |= ref["branch"]
        want = {"begin:no_emit", "begin:h0_repaired", "begin:skip_eval_kept"} | (set() if t.mf else {"begin:emit", "begin:skip_eval_cleared"})
        assert want <= seen, sorted(want - seen)
        SEEN.update(seen)
        RAN.add(sys._getframe().f_code.co_name)
    finally:
        t.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# the CG kernels of the matrix-free path


def _cg_state(r, Dt, wide):
    st = _base(r, Dt, wide, True)
    st.update(need_solve=1, cg_active=1, cg_iter=3)
    st["cg_diag"] = 2.0 ** r.integers(-2, 3, Dt) - st["q"]          # diag + q a power of two: z = r / m is exact
    st["cg_diag"] = np.where(st["cg_diag"] <= -st["q"], st["q"], st["cg_diag"])
    for k in ("cg_r", "cg_p", "cg_z", "cg_Hp"):
        st[k] = _dy(r, Dt)
    st["cg_p"] = np.where(st["cg_p"] == 0, 1.0, st["cg_p"])
    st["hv_vf"] = _sentinel(Dt, np.float32)
    st["cg_g2"] = 2.0 ** -40
    return st


def _cg_step_state(r, Dt, wide, kind):
    st = _cg_state(r, Dt, wide)
    st["cg_diag"] = 2.0 ** r.integers(-2, 3, Dt)
    st["cg_Hp"] = np.abs(st["cg_Hp"]) * np.sign(st["cg_p"])          # p . Hp > 0
    php = float(np.sum(st["cg_p"] * (st["cg_Hp"] + st["q"] * st["cg_p"])))
    pw = 2.0 ** np.floor(np.log2(php))
    # make p . H p a power of two: add the remainder to one coordinate's Hp through a unit p entry
    st["cg_p"][0], st["cg_Hp"][0] = 1.0, 0.0
    php = float(np.sum(st["cg_p"] * (st["cg_Hp"] + st["q"] * st["cg_p"])))
    pw = 2.0 ** np.ceil(np.log2(php))
    st["cg_Hp"][0] += pw - php
    st["cg_rz"] = pw * 0.25                                          # alpha = 1/4
    if kind == "curvature":
        st["cg_Hp"] = -st["cg_Hp"] - 2.0 * st["q"] * st["cg_p"]
    elif kind == "nan":
        st["cg_Hp"][Dt // 2] = np.nan
    elif kind == "cap":
        st["cg_iter"] = nr.CG_MAX_STEPS - 1
    elif kind in ("forcing_at", "forcing_above"):
        rr = nr.cg_step(st)["cg_margin"][0]
        g2 = rr / (nr.CG_ETA * nr.CG_ETA)
        while nr.CG_ETA * nr.CG_ETA * g2 < rr:
            g2 = np.nextafter(g2, np.inf)
        while nr.CG_ETA * nr.CG_ETA * np.nextafter(g2, 0.0) >= rr:
            g2 = np.nextafter(g2, 0.0)
        st["cg_g2"] = g2 if kind == "forcing_at" else np.nextafter(g2, 0.0)   # rr <= eta^2 g2 just holds / just fails
    elif kind == "idle":
        st["cg_active"] = 0
    return st


@pytest.mark.parametrize("D,P,L", [(36, 2, 3), (300, 2, 2), (2078, 1, 3)])
def test_cg_kernels_bit_for_bit(mb, D, P, L):
    t = _Sess(mb, "mf", D, P, L)
    try:
        assert t.mf
        r = np.random.default_rng(400 + D)
        seen = set()
        # cg_begin + cg_init: a column with neither diagonal nor prior is preconditioned by 1
        states = []
        for b in range(t.nprob - 1):
            st = _cg_state(r, t.Dt, t.wide)
            st.update(cg_active=0, need_solve=1 if b != 1 else 0, cg_iter=9)
            if b == 0:
                k = t.Dt // 2
                st["q"][k], st["cg_diag"][k] = 0.0, 0.0
            states.append(st)
        st = _cg_state(r, t.Dt, t.wide)     # a done problem: cg_begin clears its cg_active and cg_iter, nothing else changes
        st.update(done=1, need_solve=1, cg_active=1, cg_iter=9)
        states.insert(2, st)
        refs = [nr.cg_init(nr.cg_begin(st)) for st in states]
        inp, out = t.stage(states, ["cg_begin", "cg_init", "cg_poll"])
        t.compare(states, refs, inp, out, tag="cg_init")
        assert out["cg_any"] == 1
        for ref in refs:
            if ref is not None:
                seen |= ref["branch"]
        kinds = ["go", "curvature", "nan", "cap", "forcing_at", "forcing_above", "idle"]
        per = t.nprob - 1
        for i0 in range(0, len(kinds), per):
            chunk = kinds[i0:i0 + per]
            states = [_cg_step_state(r, t.Dt, t.wide, k) for k in chunk]
            states += [None] * (t.nprob - len(states))
            refs = [None if st is None else nr.cg_step(st) for st in states]
            inp, out = t.stage(states, ["cg_step", "cg_poll"])
            t.compare(states, refs, inp, out, tag="cg_step %s" % chunk)
            assert out["cg_any"] == int(any(ref is not None and ref["cg_active"] for ref in refs)), chunk
            for k, ref in zip(chunk, refs):
                seen |= ref["branch"]
                if k == "forcing_at":
                    assert "cg_step:forcing" in ref["branch"]
                if k == "forcing_above":
                    assert "cg_step:go" in ref["branch"]
        # the poll over a batch with exactly one problem still running, and with none
        for running in (1, 0):
            states = [_cg_step_state(r, t.Dt, t.wide, "idle") for _ in range(t.nprob)]
            if running:
                states[-1] = _cg_step_state(r, t.Dt, t.wide, "go")
            inp, out = t.stage(states, ["cg_step", "cg_poll"])
            assert out["cg_any"] == running
        want = {"cg_init:idle", "cg_init:unit_diagonal", "cg_step:idle", "cg_step:curvature", "cg_step:forcing", "cg_step:cap", "cg_step:go"}
        assert want <= seen, sorted(want - seen)
        SEEN.update(seen)
        RAN.add(sys._getframe().f_code.co_name)
    finally:
        t.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# slot audit of real x-updates (mlease_internal_xupdate_trace: the solver's own slot code, one slot at a time)


def _state_of(tr, e, b, Dt, ldx, wide, mf):
    """The replica state of problem b at trace entry e."""
    from mlease_b200._hooks import STAGE_VECS
    st = nr.new_state(Dt, wide=wide, matrix_free=mf)
    c = tr["ctrl"][e, b]
    for k in nr.INT_FIELDS + nr.TOTALS:
        st[k] = int(c[k])
    for k in nr.REAL_FIELDS:
        st[k] = float(c[k])
    for i, k in enumerate(STAGE_VECS[:12 if mf else 7]):
        st[k] = tr["vec"][e, b, i, :Dt].copy()
    rg = tr["ring"][e, b]
    st["bfgs_S"], st["bfgs_Y"] = rg[:M * ldx].reshape(M, ldx)[:, :Dt].copy(), rg[M * ldx:2 * M * ldx].reshape(M, ldx)[:, :Dt].copy()
    st["bfgs_rho"], st["bfgs_alpha"] = rg[2 * M * ldx:2 * M * ldx + M].copy(), rg[2 * M * ldx + M:].copy()
    st["beta_tf"] = tr["fvec"][e, b, 0, :Dt].copy()
    return st


def _close(a, b, scale=0.0, rel=1e-9):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return bool((np.abs(a - b) <= rel * (np.abs(b) + scale) + 1e-300).all())


def _audit(t, tr, seen):
    """Every slot transition of every problem against the gradient reference and the replica."""
    import k1_reference as k1
    Dt, ldx, L = t.Dt, t.ldx, t.nprob // len(t.parts)
    n = tr["nslots"]
    assert n >= 1
    for e in range(n):
        for b in range(t.nprob):
            where = "slot %d problem %d" % (e, b)
            c0, c1 = tr["ctrl"][e, b], tr["ctrl"][e + 1, b]
            if c0["done"]:
                # (cg_begin clears cg_active / cg_iter of a done problem; nothing else may change)
                for k in nr.INT_FIELDS + nr.REAL_FIELDS + nr.TOTALS:
                    if k not in ("cg_active", "cg_iter"):
                        assert c0[k] == c1[k] or (c0[k] != c0[k] and c1[k] != c1[k]), (where, "done", k)
                assert _bytes_equal(tr["vec"][e, b, 0], tr["vec"][e + 1, b, 0]), (where, "done: beta")
                continue
            st = _state_of(tr, e, b, Dt, ldx, t.wide, t.mf)
            part = t.parts[b // L]
            accepted = c1["tot_rejects"] == c0["tot_rejects"]
            g_dev = tr["vec"][e + 1, b, 5 if accepted else 4, :Dt]       # the full gradient the slot produced
            prior = st["q"] * (st["beta_t"] - st["m"])
            evaluated = c1["tot_evals"] > c0["tot_evals"]
            assert evaluated == (not st["skip_eval"]), where
            if evaluated:
                ref = k1.reference(part, st["beta_t"])
                A = np.bincount(part.colidx, np.abs(part.vals.astype(np.float64) * ref.r[part.rows]), Dt)
                A[-1] = np.abs(ref.r).sum()
                bound = 2e-5 * (A + A.mean())                           # the fp32 row dots of the K1 kernels, generously
                assert (np.abs(g_dev - (ref.g + prior)) <= bound).all(), (where, "gradient at float(beta_t)")
                st["g_t"] = g_dev - prior
            prior2 = float(np.sum(st["q"] * (st["beta_t"] - st["m"]) ** 2))
            st["k1_chunks"] = 1
            d = nr.decide(st, [float(c1["f_t"]) - 0.5 * prior2], int(tr["spec"][e]))
            seen |= d["branch"]
            if d["decide_margin"] and nr.near(*d["decide_margin"], rel=1e-6):
                continue
            assert bool(d["action"]) == bool(accepted), where
            assert _close(c1["alpha"] if not accepted else d["alpha"], d["alpha"]), (where, "alpha")
            for k in ("evals", "newton_steps", "warm_used", "skip_eval", "tot_evals", "tot_newton", "tot_rejects"):
                assert int(c1[k]) == int(d[k]), (where, k, int(c1[k]), int(d[k]))
            built = int(c1["hess_builds"] - c0["hess_builds"])
            assert built == int(d["need_hess"]) and int(c1["tot_hess"] - c0["tot_hess"]) == built, (where, "rebuild")
            if tr["spec"][e]:
                assert built == 0, (where, "a speculative slot never factorises")
            if built:
                assert tr["with_hess"][e] and not tr["spec"][e]
                d = nr.rebuilt(d)
                assert (c1["hess_valid"], c1["bfgs_count"], c1["h0_scale"], c1["build_step"]) == (1, 0, 1.0, d["build_step"]), (where, "after a rebuild")
            assert int(c1["emit"]) == int(d["emit"]) or d["done"], (where, "emit", sorted(d["branch"]))
            assert int(c1["bfgs_count"]) == int(d["bfgs_count"]), (where, "bfgs_count")
            if not t.mf:
                assert _close(c1["h0_scale"], d["h0_scale"]), (where, "h0_scale")
            if d["stored_slot"] >= 0:
                sl = d["stored_slot"]
                rg = tr["ring"][e + 1, b]
                gs = np.abs(g_dev).max()
                assert _bytes_equal(rg[:M * ldx].reshape(M, ldx)[sl, :Dt], d["bfgs_S"][sl]), (where, "stored s")
                assert _close(rg[M * ldx:2 * M * ldx].reshape(M, ldx)[sl, :Dt], d["bfgs_Y"][sl], gs), (where, "stored y")
                assert _close(rg[2 * M * ldx + sl], d["bfgs_rho"][sl], rel=1e-6), (where, "rho")
            if not accepted:
                got = tr["fvec"][e + 1, b, 0, :Dt]
                assert (np.abs(got - d["beta_tf"]) <= np.spacing(np.abs(d["beta_tf"]))).all(), (where, "shrunk trial point")
                assert (c1["done"], c1["fail"]) == (d["done"], d["fail"]), where
                continue
            assert _bytes_equal(tr["vec"][e + 1, b, 0, :Dt] if c1["done"] == 0 else st["beta_t"], st["beta_t"]), (where, "beta = accepted point")
            if d["done"] or not d["need_solve"]:
                assert (c1["done"], c1["fail"]) == (d["done"], d["fail"]), where
                continue
            # the stop rules and the next trial point on the direction the device formed
            dirv = tr["vec"][e + 1, b, 6, :Dt]
            d2 = dict(d, bfgs_count=0, h0_scale=1.0)
            r = nr.solve(d2, -dirv)
            seen |= r["branch"]
            assert _close(c1["phi0"], r["phi0"], float(np.abs(dirv * d["g_acc"]).sum()), 1e-10) and c1["dirnorm"] == r["dirnorm"], (where, "phi0 / dirnorm")
            if any(nr.near(*m_, rel=1e-9) for m_ in r["solve_margins"]):
                continue
            for k in ("done", "fail", "stall", "refresh_next", "have_dir", "rejects"):
                assert int(c1[k]) == int(r[k]), (where, k, sorted(r["branch"]))
            assert _bytes_equal(tr["fvec"][e + 1, b, 0, :Dt], r["beta_tf"]), (where, "next trial point")
            if r["fin"] == 1:
                assert _bytes_equal(tr["vec"][e + 1, b, 0, :Dt], r["beta"]), (where, "final step in double")
            if t.mf and c1["cg_iter"] < nr.CG_MAX_STEPS:
                ref = k1.reference(part, st["beta_t"])
                dd = part.w.astype(np.float64) * ref.p * ref.q
                xv = np.bincount(part.rows, part.vals.astype(np.float64) * dirv[part.colidx], part.n) + dirv[-1]
                Hd = np.bincount(part.colidx, part.vals.astype(np.float64) * (dd * xv)[part.rows], Dt)
                Hd[-1] = (dd * xv).sum()
                res = Hd + st["q"] * dirv + d["g_acc"]
                assert np.linalg.norm(res) <= nr.CG_ETA * np.linalg.norm(d["g_acc"]) * (1 + 1e-3), (where, "CG forcing rule", int(c1["cg_iter"]))
    last = tr["ctrl"][n]
    assert (last["done"] == 1).all() and (last["fail"] == 0).all(), "the x-update did not finish"


AUDIT = [("dense", 100, 2, 1), ("csr", 1000, 2, 3), ("csr", 2301, 1, 1), ("mf", 300, 2, 1)]


@pytest.mark.parametrize("kind,D,P,L", AUDIT)
@pytest.mark.parametrize("warm", [0, 3])
def test_slot_audit_of_real_xupdates(mb, kind, D, P, L, warm):
    """Cold and after `warm` ADMM iterations (fused batches then start from the estimated gradient: skip_eval), under the
    session's policy without and with speculative slots, and rebuilding at every step."""
    from mlease_b200 import _hooks
    seen = set()
    runs = [(2, ())] if kind == "mf" else [(0, ()), (0, tuple(range(1, 60))), (1, ())]
    for policy, spec in runs:
        t = _Sess(mb, kind, D, P, L, policy=policy)
        try:
            for _ in range(warm):
                t.s.iterate()
            tr = _hooks.xupdate_trace(t.s, policy=policy, invalidate=int(warm == 0), spec=spec)
            _audit(t, tr, seen)
            if spec:
                assert tr["spec"].any() or tr["nslots"] < 3, "no slot ran speculatively"
                # a rebuild a speculative slot deferred happens in the next regular slot
                for e in range(tr["nslots"] - 1):
                    for b in range(t.nprob):
                        c0, c1, c2 = tr["ctrl"][e, b], tr["ctrl"][e + 1, b], tr["ctrl"][e + 2, b]
                        if tr["spec"][e] and c0["emit"] and not c0["done"] and c1["newton_steps"] > c0["newton_steps"] and not c1["done"]:
                            assert c1["emit"] == 1 and c1["hess_builds"] == c0["hess_builds"], (e, b, "deferred")
                            if not tr["spec"][e + 1] and c2["newton_steps"] > c1["newton_steps"]:
                                assert tr["with_hess"][e + 1] and c2["hess_builds"] == c1["hess_builds"] + 1, (e, b, "the deferred rebuild")
            if not spec and policy != 0 and (L == 1 or warm):
                # the same slot sequence as the solver's own loop: the same bits as iterate() on an identical session
                u = _Sess(mb, kind, D, P, L, policy=policy)
                try:
                    for _ in range(warm + 1):
                        u.s.iterate()
                    for b in range(t.nprob):
                        assert _bytes_equal(tr["vec"][tr["nslots"], b, 0, :t.Dt], u.s.x(b // L, b % L)), ("x of problem", b)
                finally:
                    u.close()
        finally:
            t.close()
    if warm and kind == "csr" and D == 1000:
        # the consensus kernel handed the fused batch its estimated start gradient; the first exact evaluation is taken unconditionally
        assert {"eval:skipped", "accept:first_exact"} <= seen, sorted(seen)


def test_trace_refusals(mb):
    from mlease_b200 import _hooks
    t = _Sess(mb, "csr", 36, 2, 2, policy=1)
    try:
        for kw in (dict(policy=1, spec=(1,)), dict(policy=0, spec=(0,)), dict(policy=2), dict(policy=3), dict(policy=0, max_slots=0)):
            with pytest.raises(mb.MleaseError) as e:
                _hooks.xupdate_trace(t.s, **kw)
            assert e.value.code == 1, kw
        t.s.begin()
        for _ in range(2):
            t.s.iterate()
        assert np.isfinite(t.s.z(0)).all()
    finally:
        t.close()



# ---------------------------------------------------------------------------------------------------------------------------------
# generic data


def _generic(r, Dt, wide, count):
    st = nr.new_state(Dt, wide=wide)
    for k in ("beta", "m", "g_t", "g_acc", "dir"):
        st[k] = r.normal(size=Dt)
    st["beta"] = st["beta"].astype(np.float32).astype(np.float64)
    st["q"] = r.uniform(0.5, 2.0, Dt)
    st["beta_t"] = (st["beta"] + 0.3 * st["dir"]).astype(np.float32).astype(np.float64)
    st["beta_tf"] = st["beta_t"].astype(np.float32)
    st["bfgs_S"], st["bfgs_Y"] = r.normal(size=(M, Dt)), r.normal(size=(M, Dt))
    st["bfgs_Y"] = st["bfgs_S"] * r.uniform(0.5, 2.0, (M, Dt))
    st["bfgs_rho"] = 1.0 / np.sum(st["bfgs_S"] * st["bfgs_Y"], axis=1)
    st.update(have_dir=1, hess_valid=1, evals=3, newton_steps=2, gnorm=1.0, gnorm_prev=2.0, bfgs_count=count, alpha=0.3,
              rebuild_is_expensive=int(wide), h0_scale=1.5 if wide else 1.0, dirnorm=1.0)
    return st


@pytest.mark.parametrize("kind,D", [("dense", 36), ("csr", 999), ("csr", 2301)])
def test_generic_states_within_fp64_bounds(mb, kind, D):
    t = _Sess(mb, kind, D, 2, 3)
    try:
        r = np.random.default_rng(500 + D)
        Dt = t.Dt
        tol = 64 * Dt * 2.0 ** -53
        nct = min(9, t.info["part_rows"])
        states, parts = [], []
        for b in range(t.nprob):
            st = _generic(r, Dt, t.wide, (0, 2, M, 2 * M + 1, 3, 1)[b % 6])
            p = (r.normal(size=(nct, Dt)).astype(np.float32).astype(np.float64), r.uniform(0, 1, nct))
            st["k1_chunks"] = nct
            g = nr.decide(_reduced(st, p, False), p[1])
            # phi0 per problem: far on the accept side, far on the reject side, alternating
            st["phi0"] = -abs(g["scalars"]["phi"]) * (8.0 if b % 2 == 0 else 0.25) - 1e-3
            states.append(st)
            parts.append(p)
        outs = []
        for rep in range(2):
            inp, out = t.stage(states, ["decide", "finish"], parts=parts)
            outs.append(out)
        for k in ("vec", "ring", "fvec"):
            assert _bytes_equal(outs[0][k], outs[1][k]), "run to run: " + k
        assert outs[0]["ctrl"].tobytes() == outs[1]["ctrl"].tobytes()
        out = outs[0]
        for b, (st, p) in enumerate(zip(states, parts)):
            red = _reduced(st, p, bool(t.info["fused"]))
            # the fixed-order reduction is comparable by bits on any data: decide with emit = 0 leaves it in g_t only after the
            # prior term, so compare the accepted gradient / the first loop below within the bound instead
            d = nr.decide(red, p[1])
            assert not (d["decide_margin"] and nr.near(*d["decide_margin"])), (b, "the case was built away from its threshold")
            ref = nr.solve(d, d["dir"]) if d["need_solve"] else d
            c = out["ctrl"][b]
            for k in ("done", "need_solve", "have_dir", "newton_steps", "evals", "rejects", "bfgs_count", "emit", "need_hess", "fail"):
                assert int(c[k]) == int(ref[k]), (b, k)
            scale = float(np.abs(st["g_t"]).sum() + np.abs(st["q"] * (st["beta_t"] - st["m"])).sum()) * float(np.abs(st["dir"]).max() + 1)
            for k in ("alpha", "f_t", "gnorm", "h0_scale", "worst_ratio"):
                assert abs(c[k] - ref[k]) <= tol * max(abs(ref[k]), 1.0) * 8, (b, k, c[k], ref[k])
            assert abs(c["phi0"] - ref["phi0"]) <= tol * scale * 64, (b, "phi0")
            gs = float(np.abs(d["g_acc"]).max()) * (1.0 + float(np.abs(st["bfgs_S"]).max() * np.abs(st["bfgs_Y"]).max() * np.abs(st["bfgs_rho"]).max()) * Dt) ** 2
            assert (np.abs(out["vec"][b, 4, :Dt] - ref["g_t"]) <= tol * gs * 64).all(), (b, "g_t (the first-loop q, or the rejected gradient)")
            if d["stored_slot"] >= 0:
                sl = d["stored_slot"]
                assert abs(out["ring"][b][2 * M * t.ldx + sl] - d["bfgs_rho"][sl]) <= tol * 64 * abs(d["bfgs_rho"][sl]), (b, "rho")
                assert _bytes_equal(out["ring"][b][:M * t.ldx].reshape(M, t.ldx)[sl, :Dt], d["bfgs_S"][sl]), (b, "stored s")
            for i, k in ((0, "beta"), (1, "beta_t"), (5, "g_acc")):
                v = out["vec"][b, i, :Dt]
                bound = tol * (np.abs(ref[k]) + 1.0) if k != "beta_t" else 2.0 ** -23 * (np.abs(ref[k]) + 2.0 ** -100)
                assert (np.abs(v - ref[k]) <= bound).all(), (b, k)
    finally:
        t.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# refusals


def test_every_branch_of_the_replica_was_taken():
    """The union over the file (each test above asserts its own list): every branch the replica names, but decide:done -- done
    problems are injected as sentinels and checked by their bytes, not through the replica."""
    groups = {"test_decide_branches_bit_for_bit", "test_emit_table_bit_for_bit", "test_solve_branches_bit_for_bit", "test_begin_bit_for_bit",
              "test_cg_kernels_bit_for_bit"}
    if not groups <= RAN:
        pytest.skip("only part of the file ran")
    missing = set(nr.BRANCHES) - {"decide:done"} - SEEN
    assert not missing, sorted(missing)


def test_partial_reduction_bit_for_bit_on_order_sensitive_data(mb):
    """Random partials over ten orders of magnitude: with no prior (q = 0) and no direction the accepted gradient is the fixed-order
    sum itself, comparable by bits on any data."""
    for kind, D in (("dense", 36), ("csr", 999), ("csr", 2301)):
        t = _Sess(mb, kind, D, 2, 2)
        try:
            r = np.random.default_rng(600 + D)
            rows = t.info["part_rows"]
            states, parts = [], []
            for b in range(t.nprob):
                nct = (rows, min(9, rows), min(8, rows), min(7, rows))[b % 4]
                st = _base(r, t.Dt, t.wide, False)
                st["q"] = np.zeros(t.Dt)
                st.update(have_dir=0, evals=0, newton_steps=0, k1_chunks=nct)
                g = (r.normal(size=(nct, t.Dt)) * 10.0 ** r.integers(-5, 6, (nct, t.Dt))).astype(np.float32).astype(np.float64)
                states.append(st)
                parts.append((g, r.uniform(0, 1, nct)))
            inp, out = t.stage(states, ["decide"], parts=parts)
            for b in range(t.nprob):
                want = nr.reduce_partials(parts[b][0], len(parts[b][1]), bool(t.info["fused"]))
                assert _bytes_equal(out["vec"][b, 5, :t.Dt], want), (kind, D, b, "g_acc")
                assert _bytes_equal(out["vec"][b, 4, :t.Dt], want), (kind, D, b, "first-loop q with no pairs")
        finally:
            t.close()


def test_newton_solve_on_a_real_factor(mb):
    """newton_solve (the GEMV on the explicit inverse, then newton_solve_kernel) after a factorisation: the direction against the
    replica on the device's own Hinv; refused before any factorisation."""
    from mlease_b200 import _hooks
    t = _Sess(mb, "csr", 199, 2, 2)
    try:
        r = np.random.default_rng(77)
        Dt = t.Dt
        states = [_generic(r, Dt, False, (0, 2, M, 2 * M + 1)[b]) for b in range(t.nprob)]
        for st in states:
            st.update(have_dir=0, skip_eval=1, k1_chunks=0)
        with pytest.raises(mb.MleaseError) as e:
            t.stage(states, ["decide", "solve"])
        assert e.value.code == 1
        H = np.zeros((t.nprob, Dt, Dt))
        for b in range(t.nprob):
            A = r.normal(size=(Dt, 2 * Dt))
            H[b] = A @ A.T / (2 * Dt) + np.eye(Dt)
        t.s.begin()
        fac = _hooks.batch_factor(t.s, np.ones(t.nprob, np.int32), H=H)
        inp, out = t.stage(states, ["decide", "solve"])
        for b, st in enumerate(states):
            d = nr.decide(st, [])
            ref = nr.solve(d, fac["Hinv"][b][:Dt, :Dt] @ d["g_t"])
            got = out["vec"][b, 6, :Dt]
            scale = np.abs(fac["Hinv"][b][:Dt, :Dt]) @ np.abs(d["g_t"]) + np.abs(ref["dir"])
            assert (np.abs(got - ref["dir"]) <= 1e-9 * (scale + scale.max())).all(), (b, "dir")
            assert abs(out["ctrl"][b]["phi0"] - ref["phi0"]) <= 1e-9 * float(np.abs(ref["dir"] * d["g_acc"]).sum()), (b, "phi0")
            assert (np.abs(out["fvec"][b, 0, :Dt] - ref["beta_tf"]) <= np.spacing(np.abs(ref["beta_tf"]))).all(), (b, "trial point")
            assert int(out["ctrl"][b]["have_dir"]) == 1 and int(out["ctrl"][b]["done"]) == int(ref["done"])
    finally:
        t.close()


def test_hook_refusals(mb):
    from mlease_b200 import _hooks

    def refused(t, states, stages, **kw):
        with pytest.raises(mb.MleaseError) as e:
            t.stage(states, stages, **kw)
        assert e.value.code == 1, e.value       # MLEASE_ERR_INVALID

    for kind in ("csr", "mf"):
        t = _Sess(mb, kind, 36, 2, 2)
        try:
            r = np.random.default_rng(9)
            ok = [_base(r, t.Dt, False, t.mf) for _ in range(t.nprob)]

            def bad(**kw):
                states = [dict(s) for s in ok]
                states[1].update(kw)
                return states

            rows = t.info["part_rows"]
            big = (np.zeros((rows + 1, t.Dt)), np.zeros(rows + 1))
            refused(t, bad(k1_chunks=rows + 1), ["decide"], parts=[big] * t.nprob)
            refused(t, bad(k1_chunks=1), ["decide"])                       # no partials passed
            refused(t, bad(k1_chunks=-1), ["decide"])
            refused(t, bad(bfgs_count=-1), ["decide"])
            refused(t, bad(hess_policy=3), ["decide"])
            refused(t, ok, ["solve", "finish"])
            refused(t, ok, ["begin"])                                      # no arguments
            refused(t, ok, ["begin"], begin_args=[1e-8, 10, 5, 0, 0])
            refused(t, ok, ["decide"], spec=2)
            if t.mf:
                refused(t, ok, ["solve"])                                  # no factor to multiply
                refused(t, bad(hess_policy=0), ["decide"])                 # a pair would go to a ring that does not exist
                refused(t, ok, ["begin"], begin_args=[1e-8, 10, 0, 0, 0])
            else:
                for st in ("cg_begin", "cg_init", "cg_step", "cg_poll"):
                    refused(t, ok, [st])
            # nothing was launched on the refused states: the session still fits
            t.s.begin()
            for _ in range(3):
                t.s.iterate()
            z = t.s.z(0)
            assert np.isfinite(z).all() and np.abs(z).max() > 0
            fresh = _Sess(mb, kind, 36, 2, 2)
            try:
                for _ in range(3):
                    fresh.s.iterate()
                assert _bytes_equal(z, fresh.s.z(0))
            finally:
                fresh.close()
        finally:
            t.close()
